"""Zone masks and filter predicates at their limits in every kernel that applies them (apply_filters in k_filter_rows,
k_merge_filter and k_window_merge; the zone outlines of k_fx_render), against oracle/filters.py and oracle/effects.py.
Every comparison is exact: verdict bits, zones[] contents and order, output bytes.  The masks and rows are those of
tests/zone_cases.py: 32 zones up to 3840x2160, border, thin, diagonal and tied zones; boxes on every zone corner and
next to it, covering the frame, outside it, with unordered corners and with extreme int32 corners; labels around 0,
90 and 128; confidences on a threshold and NaN."""
import ctypes

import numpy as np
import pytest

from oracle import effects as oracle_fx
from oracle.filters import AreaOracle, ConfidenceOracle, Det, MaskOracle, TrackOracle
from tests import zone_cases as zc
from watsor_b200 import _lib
from watsor_b200.config.coco import COCO_CLASSES
from watsor_b200.stream.share import Detection

pytestmark = pytest.mark.gpu
NAN = float('nan')


def detect_config(n_zones, width, height, path):
    """every COCO label, with confidences, areas and zone lists that vary with the label; the lists name zones 1, 10,
    11, 31 and 32 where the mask has them"""
    last, mid = n_zones, min(31, n_zones)
    lists = [[], [1, mid, last], [last], sorted({min(10, last), min(11, last)})]
    detect = [{COCO_CLASSES[k]: {'confidence': [0, 50, 25, 12.5][k % 4], 'area': [0, 0.01, 1, 0][k % 4],
                                 'zones': lists[(k // 4) % 4]}} for k in range(1, 91)]
    detect[88] = {COCO_CLASSES[89]: {'confidence': 50, 'area': 150, 'zones': []}}    # an area no box reaches
    return {'width': width, 'height': height, 'mask': path, 'detect': detect}


@pytest.fixture(scope='module')
def families(tmp_path_factory):
    d = tmp_path_factory.mktemp('zone_masks')
    out = {}
    for name, build in zc.FAMILIES.items():
        mask = build()
        out[name] = (mask, zc.write_mask(d, name, mask))
    return out


def copy_row(src):
    d = Detection()
    ctypes.memmove(ctypes.addressof(d), ctypes.addressof(src), ctypes.sizeof(Detection))
    return d


# ------------------------------------------------------------------------------------------------- stand-alone filters
@pytest.mark.parametrize('name', sorted(zc.FAMILIES))
def test_stand_alone_filters_equal_their_oracles(families, name):
    from watsor_b200.filter.area import AreaFilter
    from watsor_b200.filter.confidence import ConfidenceFilter
    from watsor_b200.filter.mask import MaskFilter
    mask, path = families[name]
    h, w = mask.shape[:2]
    cfg = detect_config(len(zc.zones_of(mask)), w, h, path)
    rows = zc.edge_rows(mask, np.random.default_rng(11), n_random=100, max_vertices=3,
                        thresholds=(0.5, 0.25, 0.125), limit=1500)
    arr = zc.to_detections(rows)
    pairs = [(ConfidenceFilter(cfg), ConfidenceOracle(cfg)), (AreaFilter(cfg), AreaOracle(cfg)),
             (MaskFilter(cfg), MaskOracle(cfg))]
    full = 0
    for f, oracle in pairs:
        for r, (label, conf, box) in enumerate(rows):
            d, o = copy_row(arr[r]), Det(label, conf, box)
            want = oracle(o)
            assert f(d) == want and list(d.zones) == o.zones, (type(f).__name__, label, conf, box, o.zones)
            full += o.zones[9] > 0
    assert (full > 0) == (len(zc.zones_of(mask)) > 10)


def test_extreme_corners_and_nan_confidences_in_stand_alone_filters(families):
    """area.py sizes a box in Python integers: a span of 2^32 or 3e9 px is that many pixels, not an int32 wrap; and
    area.py / mask.py never read the confidence, so a NaN confidence passes them (ConfidenceFilter rejects it)"""
    from watsor_b200.filter.area import AreaFilter
    from watsor_b200.filter.confidence import ConfidenceFilter
    from watsor_b200.filter.mask import MaskFilter
    _, path = families['grid32-640x480']
    cfg = {'width': 640, 'height': 480, 'mask': path,
           'detect': [{'person': {'confidence': 50, 'area': 50, 'zones': []}}]}
    area, conf, mask = AreaFilter(cfg), ConfidenceFilter(cfg), MaskFilter(cfg)
    lo, hi = zc.I32_MIN, zc.I32_MAX
    cases = [((lo, 0, hi, 0), True), ((hi, 0, lo, 0), True), ((lo, lo, hi, hi), True), ((-1500000000, 5, 1500000000, 5),
             True), ((0, -1500000000, 0, 1500000000), True), ((lo, 0, lo, 0), False), ((lo, 100, lo + 5, 200), False)]
    for box, big in cases:
        for c in (0.9, NAN):
            d = Detection(label=1, confidence=c)
            d.bounding_box.x_min, d.bounding_box.y_min, d.bounding_box.x_max, d.bounding_box.y_max = box
            o = Det(1, c, box)
            assert AreaOracle(cfg)(o) == big
            assert area(copy_row(d)) == big, (box, c)
            assert conf(copy_row(d)) == (c == 0.9)
            m = copy_row(d)
            assert mask(m) == MaskOracle(cfg)(o) and list(m.zones) == o.zones, (box, c)
    d = Detection(label=1, confidence=NAN)
    d.bounding_box.x_min, d.bounding_box.y_min, d.bounding_box.x_max, d.bounding_box.y_max = 0, 0, 639, 479
    assert area(copy_row(d)) and mask(copy_row(d)) and not conf(copy_row(d))


def test_track_filter_sieve_on_32_zones(families):
    """TrackFilter([Confidence, Area, Mask]) + sieve_frame against the oracle's track.py / sieve.py, with objects
    that meet more than 10 zones"""
    from watsor_b200.filter.area import AreaFilter
    from watsor_b200.filter.confidence import ConfidenceFilter
    from watsor_b200.filter.mask import MaskFilter
    from watsor_b200.filter.sieve import sieve_frame
    from watsor_b200.filter.track import TrackFilter
    mask, path = families['grid32-640x480']
    cfg = detect_config(32, 640, 480, path)
    ours = TrackFilter([ConfidenceFilter(cfg), AreaFilter(cfg), MaskFilter(cfg)], sensitivity=2, history=3)
    oracle = TrackOracle([ConfidenceOracle(cfg), AreaOracle(cfg), MaskOracle(cfg)], sensitivity=2, history=3)
    rng = np.random.default_rng(9)
    objects = [(0, 0, 639, 479, 1), (10, 10, 600, 300, 5), (300, 200, 639, 479, 6), (0, 240, 639, 250, 9),
               (100, 50, 130, 80, 13), (5, 5, 620, 470, 2)]
    edge = zc.edge_rows(mask, rng, n_random=0, max_vertices=2)
    for frame in range(5):
        picks = rng.choice(len(edge), 100 - len(objects), replace=False)
        rows_l = [(lab, 0.9, (x0 + int(rng.integers(-3, 4)), y0, x1, y1 + int(rng.integers(-3, 4))))
                  for x0, y0, x1, y1, lab in objects]
        rows_l += [edge[i] for i in picks]
        rows = zc.to_detections(rows_l)
        dets = zc.to_dets(rows_l)
        sus = sieve_frame(rows, [ours])
        want, want_sus = oracle(dets)
        assert sus == want_sus
        got = [(rows[r].label, rows[r].confidence, rows[r].bounding_box.x_min, rows[r].bounding_box.y_min,
                rows[r].bounding_box.x_max, rows[r].bounding_box.y_max, list(rows[r].zones)) for r in range(100)]
        exp = [(d.label, d.confidence, d.x_min, d.y_min, d.x_max, d.y_max, d.zones) for d in want]
        assert got[:len(exp)] == exp, frame
        assert all(g == (0, 0.0, 0, 0, 0, 0, [0] * 10) for g in got[len(exp):])
        assert frame < 1 or any(z[9] for z in (e[6] for e in exp))


# ------------------------------------------------------------------------------------------------- camera tables
GRIDS = ('grid32-640x480', 'grid32-1920x1080', 'grid32-3840x2160')
VARIANTS = [(True, True), (True, False), (False, True), (False, False)]     # (default row, label check)


def camera_table(n_zones, width, height, default):
    """names zones 1, 31 and 32, labels 0, 90 and 127, a label no box is large enough for, and the default row"""
    area = lambda pct: pct / 100 * width * height
    t = [(1, 0.5, area(0.01), [1]), (2, 0.5, area(1), [31, n_zones]), (45, 0.25, 0.0, None),
         (90, 0.5, area(5), [n_zones]), (127, 0.0, 0.0, [1, 31, n_zones]), (0, 0.125, 0.0, [2]),
         (89, 0.5, area(150), None)]
    if default:
        t.append((-1, 0.3, area(0.5), [1, 31, n_zones]))
    return t


@pytest.fixture(scope='module')
def table_engine(families):
    """one camera per grid and table variant, each configured once: 12 cameras, 4 of them 3840x2160 (32 summed-area
    tables of 33 MB each)"""
    from watsor_b200.engine import Engine
    from watsor_b200.filter._gpu import _null_model_blob
    from watsor_b200.filter.mask import zone_rasters
    with Engine(_null_model_blob(), device=0, max_batch=1) as e:
        cams = {}
        for g, name in enumerate(GRIDS):
            mask, path = families[name]
            h, w = mask.shape[:2]
            rasters = zone_rasters(zc.zones_of(mask), w, h)
            for v, (default, check) in enumerate(VARIANTS):
                table = camera_table(32, w, h, default)
                cam = 4 * g + v
                e.set_camera(cam, w, h, rasters, table, flags=0 if check else _lib.WB_CAM_NO_LABEL_CHECK)
                cams[(name, default, check)] = (cam, table)
            del rasters
        yield e, cams


@pytest.mark.parametrize('default,check', VARIANTS, ids=['default-check', 'default-nocheck', 'check', 'nocheck'])
@pytest.mark.parametrize('name', GRIDS)
def test_camera_tables_through_filter_rows(table_engine, families, name, default, check):
    e, cams = table_engine
    cam, table = cams[(name, default, check)]
    mask, path = families[name]
    h, w = mask.shape[:2]
    rows = zc.edge_rows(mask, np.random.default_rng(len(name)), n_random=300, max_vertices=6,
                        thresholds=(0.5, 0.25, 0.125, 0.3))
    arr = zc.to_detections(rows)
    verd = []
    for base in range(0, len(rows), 100):              # wb_filter_rows takes up to 100 rows per batch image
        chunk = (Detection * min(100, len(rows) - base)).from_address(ctypes.addressof(arr[base]))
        verd += [int(v) for v in e.filter_rows(cam, chunk)]
    dets = zc.to_dets(rows)
    want = zc.chain_verdicts(dets, zc.table_oracles(path, w, h, table), check)
    bad = [(rows[r], verd[r], want[r]) for r in range(len(rows)) if verd[r] != want[r]]
    assert not bad, bad[:5]
    assert [list(d.zones) for d in arr] == [d.zones for d in dets]
    assert any(d.zones[9] for d in dets)
    assert any(d.zones[0] == 32 or 32 in d.zones for d in dets)


def test_set_camera_refuses_33_zones():
    from watsor_b200.filter._gpu import filter_engine
    rasters = np.zeros((33, 48, 64), np.uint8)
    with pytest.raises(_lib.WatsorB200Error, match='at most 32 zones'):
        filter_engine().set_camera(250, 64, 48, rasters, [(-1, 0.0, 0.0, None)])


# ------------------------------------------------------------------------------------------------- fused detector path
def test_fused_detector_path_on_32_zones(coco_model, families):
    """k_merge_filter with WB_F_FUSE_FILTERS: heads with enc = 0 decode to the anchors themselves, the largest of which
    meet more than 10 zones; the reference is apply_predicates on the same engine's rows without the flag"""
    from watsor_b200.detection.b200 import camera_tables
    from watsor_b200.engine import Engine
    mask, path = families['grid32-640x480']
    cfg = detect_config(32, 640, 480, path)
    rasters, table = camera_tables(cfg, 640, 480)
    rng = np.random.default_rng(4)
    with Engine(coco_model.to_blob(), device=0, max_batch=2) as e:
        e.set_camera(0, 640, 480, rasters, table)
        N, C = e.num_anchors, e.num_classes
        enc = np.zeros((2, N, 4), np.float32)
        logits = np.full((2, N, C + 1), -12.0, np.float32)
        for f in range(2):
            picks = np.concatenate([np.arange(N - 120, N), rng.choice(N - 120, 120, replace=False)])
            for k, a in enumerate(picks):
                logits[f, a, 1 + (k * 7 + f) % C] = rng.uniform(-3.0, 6.0)
        rows_u, verd_u, *_ = e.postprocess(enc, logits, [0, 0], flags=0)
        rows_f, verd_f, *_ = e.postprocess(enc, logits, [0, 0], flags=_lib.WB_F_FUSE_FILTERS)
    oracles = [ConfidenceOracle(cfg), AreaOracle(cfg), MaskOracle(cfg)]
    full = 0
    for f in range(2):
        assert all(list(r.zones) == [0] * 10 for r in rows_u[f])
        dets = [Det(r.label, r.confidence, (r.bounding_box.x_min, r.bounding_box.y_min, r.bounding_box.x_max,
                                            r.bounding_box.y_max)) for r in rows_u[f]]
        assert sum(d.label > 0 for d in dets) > 50
        want = zc.chain_verdicts(dets, oracles, True)
        assert [int(v) for v in verd_f[f]] == want
        assert [int(v) for v in verd_u[f]] == want
        for ru, rf, d in zip(rows_u[f], rows_f[f], dets):
            assert (rf.label, rf.confidence, rf.bounding_box.x_min, rf.bounding_box.y_min, rf.bounding_box.x_max,
                    rf.bounding_box.y_max) == (ru.label, ru.confidence, ru.bounding_box.x_min, ru.bounding_box.y_min,
                                               ru.bounding_box.x_max, ru.bounding_box.y_max)
            assert list(rf.zones) == d.zones
            full += d.zones[9] > 0
    assert full > 0


# ------------------------------------------------------------------------------------------------- windowed path
def test_windowed_path_on_32_zones(tmp_path):
    """k_window_merge: a camera with three detection windows and 32 zones, as tall blobs 20 px apart; the merged rows'
    verdicts and zones equal the oracle's on those rows.  The model's boxes are small, so full zones[] lists are left to
    the fused path and the camera-table tests, which run the same apply_filters."""
    from tests import workload
    from tests.artist import artist_frame
    from tests.test_gpu_windows import assert_rows, expected, run
    from watsor_b200.detection.b200 import B200ObjectDetector
    path = zc.write_mask(tmp_path, 'stripes', zc.grid_mask(640, 480, 32, cols=32))
    cfg = detect_config(32, 640, 480, path)
    wins = [(0, 0, 640, 480), (0, 0, 320, 240), (320, 240, 320, 240)]
    with B200ObjectDetector(None, device=0, max_batch=16, precision=2,
                            model_blob=workload.v2_coco_model().to_blob()) as det:
        for c in (0, 1):
            det.configure_camera(c, 640, 480, dict(cfg, windows=[list(w) for w in wins]))
        frames = [artist_frame(640, 480, c, 3) for c in (0, 1)]
        want = expected(det, frames, [wins, wins], [0.5, 0.5], [cfg, cfg])
        rows, verd = run(det, frames, [0, 1], fuse_filters=True)
        assert_rows(rows, verd, want, True)
    assert any(v & _lib.WB_V_PASS for _, _, vs in want for v in vs)


# ------------------------------------------------------------------------------------------------- zone outlines
@pytest.mark.parametrize('size', [(640, 480), (1920, 1080)])
def test_zone_outlines_of_32_zones(families, size):
    from tests.fx_cases import random_rows
    from watsor_b200.output.effects import WB_FX_BLEND, WB_FX_CONTOURS, WB_FX_DRAW, EffectsEngine, contour_bits
    w, h = size
    mask, _ = families['grid32-%dx%d' % size]
    alpha = np.ascontiguousarray(mask[..., 3])
    rng = np.random.default_rng(w)
    lists = [[10, 11, 31, 32], list(range(1, 11)), list(range(23, 33)), [32], [31, 1], [11, 10, 9, 8, 7, 6, 5, 4, 3, 2]]
    with EffectsEngine(0) as engine:
        cam = engine.add_camera(w, h, alpha, contour_bits(alpha))
        for trial in range(2):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            rows = random_rows(rng, w, h, 30, n_zones=32)
            for k, zones in enumerate(lists):
                d = rows[90 + k]
                d.label, d.confidence = [1, 5, 90, 150, 2, 44][k], 0.75
                x0, y0 = int(rng.integers(0, w // 2)), int(rng.integers(0, h // 2))
                d.bounding_box.x_min, d.bounding_box.y_min = x0, y0
                d.bounding_box.x_max, d.bounding_box.y_max = x0 + int(rng.integers(1, w // 2)), y0 + int(
                    rng.integers(1, h // 2))
                for j in range(10):
                    d.zones[j] = zones[j] if j < len(zones) else 0
            out = np.zeros_like(img)
            engine.render([img], [out], [cam], [rows], WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS)
            ref = oracle_fx.effect_chain(img, rows, alpha)
            assert np.array_equal(ref, out), (size, trial, int((ref != out).sum()))
