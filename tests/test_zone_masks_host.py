"""Zone masks at their limits on the CPU (tests/zone_cases.py): 32 zones up to 3840x2160, zones on the frame border,
single-pixel-wide and diagonal zones, centroid-key ties and the masks the library refuses.

  * the raster claim of filter/mask.py -- "the closed box meets the zone polygon" equals "the box covers a pixel of
    the zone's filled-contour raster" -- on every family, for the rasters `zone_rasters` builds;
  * a numpy restatement of apply_filters (csrc/kernels_post.cu: summed-area counts, then the predicate order) against
    oracle/filters.py's predicate chain on the same rows, so that the GPU tests compare with a pinned CPU side."""
import math

import cv2
import numpy as np
import pytest

from oracle.filters import AreaOracle, Det, MaskOracle, rect_intersects_polygon
from tests import zone_cases as zc
from watsor_b200.config.coco import COCO_CLASSES
from watsor_b200.filter.mask import find_contours, mask_tables, zone_rasters

NEG_INF = float('-inf')


@pytest.fixture(scope='module', params=sorted(zc.FAMILIES))
def family(request):
    mask = zc.FAMILIES[request.param]()
    return request.param, mask


def sat_of(raster):
    return np.pad(raster.astype(np.int64).cumsum(0).cumsum(1), ((1, 0), (1, 0)))


def covered(sat, boxes, width, height):
    """per box: does the box, clipped to the frame, cover a raster pixel (what apply_filters asks the table)"""
    b = np.asarray(boxes, np.int64).reshape(-1, 4)
    xa, xb = np.minimum(b[:, 0], b[:, 2]), np.maximum(b[:, 0], b[:, 2])
    ya, yb = np.minimum(b[:, 1], b[:, 3]), np.maximum(b[:, 1], b[:, 3])
    xa, ya = np.maximum(xa, 0), np.maximum(ya, 0)
    xb, yb = np.minimum(xb, width - 1), np.minimum(yb, height - 1)
    ok = (xa <= xb) & (ya <= yb)
    xa, xb, ya, yb = (np.where(ok, v, 0) for v in (xa, xb, ya, yb))
    cnt = sat[yb + 1, xb + 1] - sat[ya, xb + 1] - sat[yb + 1, xa] + sat[ya, xa]
    return ok & (cnt > 0)


# ------------------------------------------------------------------------------------------------- the masks
def test_family_zone_counts():
    assert {k: len(zc.zones_of(f())) for k, f in zc.FAMILIES.items()} == {
        'grid32-640x480': 32, 'grid32-1920x1080': 32, 'grid32-3840x2160': 32, 'border': 9, 'thin': 8,
        'diagonal-join': 1, 'ties': 7}


def test_library_and_oracle_number_zones_alike(family):
    name, mask = family
    ours = find_contours(np.ascontiguousarray(mask[..., 3]))
    theirs = zc.zones_of(mask)
    assert len(ours) == len(theirs)
    assert all(np.array_equal(a, b) for a, b in zip(ours, theirs)), name


def test_diagonal_pixel_joins_two_blocks_into_one_zone():
    """findContours follows 8-connected foreground: blocks that share only a corner pixel make one zone, whose ring
    passes the shared corner twice"""
    (c,) = zc.zones_of(zc.diagonal_join_mask())
    assert cv2.boundingRect(c) == (10, 10, 20, 20)
    assert cv2.moments(c)['m00'] == 162.0
    pts = [tuple(p) for p in c[:, 0].tolist()]
    assert pts.count((19, 19)) + pts.count((20, 20)) >= 2


def test_centroid_key_ties_keep_find_contours_order():
    mask = zc.tie_mask()
    _, thresh = cv2.threshold(255 - mask[..., 3], 0, 255, cv2.THRESH_BINARY_INV)
    raw = cv2.findContours(thresh, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)[-2]

    def key(c):
        m = cv2.moments(c)
        cx, cy = int(m['m10'] / m['m00']), int(m['m01'] / m['m00'])
        return cx * cx + cy * cy

    sorted_ = zc.zones_of(mask)
    keys = [key(c) for c in sorted_]
    assert keys == sorted(keys) and len(set(keys)) == 4          # three tied pairs and the zone on the diagonal
    raw_index = [next(i for i, r in enumerate(raw) if np.array_equal(r, c)) for c in sorted_]
    for k in set(keys):
        tied = [raw_index[i] for i in range(len(keys)) if keys[i] == k]
        assert tied == sorted(tied)                               # the stable sort keeps findContours' order


def test_over_limit_and_degenerate_masks_are_refused_on_the_host(tmp_path):
    from watsor_b200.filter.mask import MaskFilter
    from watsor_b200.output.effects import contour_bits
    mask = zc.over_limit_mask()
    assert len(zc.zones_of(mask)) == 33
    path = zc.write_mask(tmp_path, 'z33', mask)
    cfg = {'width': 640, 'height': 480, 'mask': path, 'detect': []}
    with pytest.raises(AssertionError, match='has more than 32 zones'):
        MaskFilter(cfg)
    with pytest.raises(AssertionError, match='at most 32 zones'):
        contour_bits(mask[..., 3])
    MaskOracle(cfg)                     # the reference itself takes any number of zones
    # a zone of 1 or 2 pixels has fewer than 3 contour points and zero area: the reference's centroid key divides
    # by m00 before shapely could refuse the ring, and the library fails the same way
    for n in (1, 2):
        tiny = zc.tiny_zone_mask(n_pixels=n)
        assert sorted(len(c) for c in cv2.findContours(
            cv2.threshold(255 - tiny[..., 3], 0, 255, cv2.THRESH_BINARY_INV)[1], cv2.RETR_EXTERNAL,
            cv2.CHAIN_APPROX_SIMPLE)[-2]) == [n, 4]
        path = zc.write_mask(tmp_path, 'tiny%d' % n, tiny)
        cfg = {'width': 40, 'height': 30, 'mask': path, 'detect': []}
        with pytest.raises(ZeroDivisionError):
            MaskOracle(cfg)
        with pytest.raises(ZeroDivisionError):
            MaskFilter(cfg)


# ------------------------------------------------------------------------------------------------- raster claim
def test_raster_claim_on_every_family(family):
    """bbox `intersects` zone polygon (mask.py:54)  <=>  the bbox covers a pixel of the raster zone_rasters draws,
    for every zone of the family: edge boxes on all its vertices, random boxes around it and the frame edge boxes"""
    name, mask = family
    h, w = mask.shape[:2]
    contours = zc.zones_of(mask)
    rng = np.random.default_rng(len(name))
    frame_boxes = zc.frame_edge_boxes(w, h)
    for z, c in enumerate(contours):
        raster = zone_rasters([c], w, h)[0]
        bx, by, bw, bh = cv2.boundingRect(c)
        boxes = zc.zone_edge_boxes([c], max_vertices=48) + frame_boxes
        n_random = max(0, 2000 - len(boxes))
        x = rng.integers(bx - 6, bx + bw + 6, (n_random, 2))
        y = rng.integers(by - 6, by + bh + 6, (n_random, 2))
        small = rng.integers(0, 4, (n_random, 2))
        x[::2, 1] = x[::2, 0] + small[::2, 0]
        y[::2, 1] = y[::2, 0] + small[::2, 1]
        boxes += [(int(a), int(b), int(c_), int(d)) for (a, c_), (b, d) in zip(x, y)]
        got = covered(sat_of(raster), boxes, w, h)
        poly = c[:, 0]
        for box, g in zip(boxes, got):
            assert bool(g) == rect_intersects_polygon(*box, poly), (name, z + 1, box)


# ------------------------------------------------------------------------------------------------- restatement
def restated_apply_filters(table, rasters, rows, check_label=True):
    """numpy restatement of apply_filters (csrc/kernels_post.cu) for caller rows: -> (verdicts, zones lists).
    A -inf confidence threshold is no confidence predicate (the stand-alone AreaFilter / MaskFilter tables)."""
    n_zones, h, w = rasters.shape
    boxes = [box for _, _, box in rows]
    hits = np.stack([covered(sat_of(rasters[p]), boxes, w, h) for p in range(n_zones)], axis=1)
    by_label = {label: (c, a, z) for label, c, a, z in table if label != -1}
    default = next(((c, a, z) for label, c, a, z in table if label == -1), None)
    verdicts, zones = [], []
    for r, (label, conf, (x0, y0, x1, y1)) in enumerate(rows):
        v, zl = 0, []
        verdicts.append(v)
        zones.append([0] * 10)
        if check_label:
            if not label > 0:
                continue
            v = 1
        entry = by_label.get(label) if 0 <= label < 128 else None
        entry = entry if entry is not None else default
        verdicts[-1] = v
        if entry is None:
            continue
        c, a, allowed = entry
        if c != NEG_INF and not conf >= c:
            continue
        v |= 2
        verdicts[-1] = v
        if not abs((x1 - x0 + 1) * (y1 - y0 + 1)) >= a:
            continue
        v |= 4
        verdicts[-1] = v
        zl = [p + 1 for p in range(n_zones) if (not allowed or p + 1 in allowed) and hits[r, p]][:10]
        zones[-1] = zl + [0] * (10 - len(zl))
        if not zl:
            continue
        verdicts[-1] = v | 8 | 16
    return verdicts, zones


def camera_table(n_zones, width, height, default=True):
    """a camera table that names zone 1, zone 31 and zone 32 (when the mask has them), labels 0, 90 and 127, and the
    default row"""
    last = n_zones
    mid = min(31, n_zones)
    area = lambda pct: pct / 100 * width * height
    t = [(1, 0.5, area(0.01), [1]), (2, 0.5, area(1), [mid, last]), (45, 0.25, 0.0, None), (90, 0.5, area(5), [last]),
         (127, 0.0, 0.0, sorted({1, mid, last})), (0, 0.125, 0.0, [min(2, last)]), (89, 0.5, area(150), None)]
    if default:
        t.append((-1, 0.3, area(0.5), sorted({1, mid, last})))
    return t


@pytest.mark.parametrize('check_label', [True, False], ids=['label-check', 'no-label-check'])
@pytest.mark.parametrize('default', [True, False], ids=['default-row', 'no-default'])
def test_restated_apply_filters_equals_oracle_chain(family, check_label, default, tmp_path):
    name, mask = family
    h, w = mask.shape[:2]
    path = zc.write_mask(tmp_path, name, mask)
    rasters = zone_rasters(zc.zones_of(mask), w, h)
    table = camera_table(rasters.shape[0], w, h, default)
    rows = zc.edge_rows(mask, np.random.default_rng(3), max_vertices=4, thresholds=(0.5, 0.25, 0.125, 0.3))
    got_v, got_z = restated_apply_filters(table, rasters, rows, check_label)
    dets = zc.to_dets(rows)
    want_v = zc.chain_verdicts(dets, zc.table_oracles(path, w, h, table), check_label)
    assert got_v == want_v, name
    assert got_z == [d.zones for d in dets], name
    assert any(z[9] for z in got_z) == (rasters.shape[0] > 10)    # full zones[] lists occur on the 32-zone grids


def test_restated_stand_alone_area_and_mask_tables_equal_their_oracles(tmp_path):
    """AreaFilter / MaskFilter tables carry a -inf confidence: no confidence predicate, so NaN confidences pass as in
    area.py / mask.py, and extreme int32 corners are sized in exact integers"""
    mask = zc.grid_mask(640, 480)
    path = zc.write_mask(tmp_path, 'grid', mask)
    cfg = {'width': 640, 'height': 480, 'mask': path,
           'detect': [{COCO_CLASSES[1]: {'area': 1, 'zones': [1, 32]}}, {COCO_CLASSES[90]: {'area': 50, 'zones': []}}]}
    rasters, zones_by_label = mask_tables(cfg)
    rows = zc.edge_rows(mask, np.random.default_rng(5), max_vertices=4)
    assert any(math.isnan(c) for _, c, _ in rows)
    dets = zc.to_dets(rows)
    area_table = [(1, NEG_INF, 0.01 * 640 * 480, None), (90, NEG_INF, 0.5 * 640 * 480, None)]
    v, _ = restated_apply_filters(area_table, rasters, rows, check_label=False)
    assert [bool(x & 4) for x in v] == [AreaOracle(cfg)(d) for d in dets]
    mask_table = [(-1, NEG_INF, 0.0, None)] + [(k, NEG_INF, 0.0, z) for k, z in zones_by_label.items()]
    v, zones = restated_apply_filters(mask_table, rasters, rows, check_label=False)
    oracle = MaskOracle(cfg)
    assert [bool(x & 8) for x in v] == [oracle(d) for d in dets]
    assert zones == [d.zones for d in dets]
    big = [Det(1, float('nan'), (zc.I32_MIN, 0, zc.I32_MAX, 0))]
    assert AreaOracle(cfg)(big[0])
    v, _ = restated_apply_filters(area_table, rasters, [(1, float('nan'), (zc.I32_MIN, 0, zc.I32_MAX, 0))], False)
    assert v[0] & 6 == 6
