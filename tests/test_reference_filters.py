"""The oracle's predicates against the reference's OWN filter classes, imported from the read-only tree and run here
(SURVEY.md 8c: "outputs of the reference itself run here").  ConfidenceFilter and AreaFilter are pure Python and run
as they are.  MaskFilter needs shapely, which is not installed: it is imported with a stand-in `shapely.geometry`
whose `Polygon.intersects` is the oracle's exact integer geometry, so this pins the reference's control flow --
alpha threshold, contour extraction and ordering, per-class zone lists, the order and cap of `zones[]` writes --
but not GEOS itself (that gap is stated in DESIGN.md).  CPU only; without an upstream checkout the upstream results
come from tests/golden/reference/ (tests/reference_golden.py)."""
import hashlib
import os
import sys
import types
from tempfile import NamedTemporaryFile

import numpy as np
import pytest

from oracle.filters import AreaOracle, ConfidenceOracle, Det, MaskOracle, rect_intersects_polygon
from tests.conftest import PORCH_CONFIG

from tests.conftest import REF_DIR as REF  # noqa: E402
from tests.reference_golden import upstream  # noqa: E402


class _StandInPolygon:
    """shapely.geometry.Polygon as far as mask.py uses it (mask.py:26,45-54)."""

    def __init__(self, points):
        self.points = np.asarray(points, dtype=np.int64).reshape(-1, 2)
        if len(self.points) < 3:
            raise ValueError('A linearring requires at least 4 coordinates.')

    def intersects(self, other):
        # self is the detection's box (4 corners, mask.py:45-48), other a zone polygon
        xs, ys = self.points[:, 0], self.points[:, 1]
        return bool(rect_intersects_polygon(int(xs[0]), int(ys[0]), int(xs[2]), int(ys[2]), other.points))


class ref_classes:
    """The reference's filter classes (MaskFilter with the stand-in shapely) for the duration of a `with` block."""

    def __enter__(self):
        self.saved = {k: sys.modules.get(k) for k in ('shapely', 'shapely.geometry')}
        shapely = types.ModuleType('shapely')
        geometry = types.ModuleType('shapely.geometry')
        geometry.Polygon = _StandInPolygon
        shapely.geometry = geometry
        sys.modules['shapely'], sys.modules['shapely.geometry'] = shapely, geometry
        sys.path.insert(0, REF)
        from watsor.filter.area import AreaFilter
        from watsor.filter.confidence import ConfidenceFilter
        from watsor.filter.mask import MaskFilter
        from watsor.stream.share import BoundingBox, Detection
        return types.SimpleNamespace(AreaFilter=AreaFilter, ConfidenceFilter=ConfidenceFilter, MaskFilter=MaskFilter,
                                     BoundingBox=BoundingBox, Detection=Detection)

    def __exit__(self, *exc):
        sys.path.remove(REF)
        for k, v in self.saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def random_dets(rng, w, h, n):
    out = []
    for r in range(n):
        x0, x1 = (int(v) for v in rng.integers(-5, w + 5, 2))
        y0, y1 = (int(v) for v in rng.integers(-5, h + 5, 2))
        if r % 3:
            x0, x1, y0, y1 = min(x0, x1), max(x0, x1), min(y0, y1), max(y0, y1)
        if r % 7 == 0:
            x1, y1 = x0, y0
        label = int(rng.integers(0, 6))
        conf = [0.5, 0.25, 0.75, float(np.float32(rng.random())), float(rng.random())][r % 5]
        out.append(Det(label, conf, (x0, y0, x1, y1)))
    return out


def ref_det(ref, d):
    return ref.Detection(label=d.label, confidence=d.confidence,
                         bounding_box=ref.BoundingBox(d.x_min, d.y_min, d.x_max, d.y_max))


def mask_token(got, zones):
    """'<0|1>:<zone>.<zone>...': a verdict and the zones[] list without its trailing zero padding."""
    z = list(zones)
    while z and z[-1] == 0:
        z.pop()
    return '%d:%s' % (int(bool(got)), '.'.join(str(v) for v in z))


def rows_digest(tokens):
    return hashlib.sha256(' '.join(tokens).encode()).hexdigest()


def mask_results(ref, cfg, dets):
    """Digest of the reference MaskFilter's verdict and zones[] for every detection."""
    rm = ref.MaskFilter(cfg)
    out = []
    for d in dets:
        rd = ref_det(ref, d)
        out.append(mask_token(rm(rd), rd.zones))
    return rows_digest(out)


def oracle_results(om, dets):
    tokens = []
    for od in dets:
        got = om(od)                                            # writes od.zones
        tokens.append(mask_token(got, od.zones))
    return tokens


@pytest.mark.parametrize('seed', range(4))
def test_confidence_and_area_oracles_equal_the_reference_classes(seed):
    rng = np.random.default_rng(seed)
    w, h = int(rng.integers(40, 2000)), int(rng.integers(40, 1200))
    cfg = {'width': w, 'height': h,
           'detect': [{'person': {'confidence': int(rng.integers(0, 101)), 'area': int(rng.integers(0, 101))}},
                      {'car': {'confidence': 50, 'area': 10}},
                      {'bicycle': {'confidence': 25, 'area': 0}},
                      {'motorcycle': {'confidence': 75, 'area': 100}}]}
    oc, oa = ConfidenceOracle(cfg), AreaOracle(cfg)
    dets = random_dets(rng, w, h, 1500)
    # the full-frame box is exactly 100 % (area.py:18, :24-26)
    full = Det(4, 0.75, (0, 0, w - 1, h - 1))

    def theirs():
        with ref_classes() as ref:
            rc, ra = ref.ConfidenceFilter(cfg), ref.AreaFilter(cfg)
            # two bits per detection (confidence verdict, area verdict) as a hex string
            bits = ''.join('%d%d' % (bool(rc(rd)), bool(ra(rd))) for rd in (ref_det(ref, d) for d in dets + [full]))
            return '%d:%x' % (len(bits), int('1' + bits, 2))
    n, packed = upstream('filters', 'confidence_area_%d' % seed, theirs).split(':')
    bits = bin(int(packed, 16))[3:]
    assert int(n) == len(bits) == 2 * (len(dets) + 1)
    ref = [(bits[i] == '1', bits[i + 1] == '1') for i in range(0, len(bits), 2)]
    for od, (c, a) in zip(dets, ref):
        assert c == oc(od) and a == oa(od), od.key()
    assert ref[-1] == (True, True) and oa(full) is True and oc(full) is True


def _random_alpha(rng, w, h):
    import cv2
    alpha = np.full((h, w), 216, np.uint8)
    for _ in range(int(rng.integers(1, 7))):
        x, y = int(rng.integers(0, w - 8)), int(rng.integers(0, h - 8))
        a, b = int(rng.integers(4, max(5, w // 3))), int(rng.integers(4, max(5, h // 3)))
        if rng.random() < 0.5:
            cv2.rectangle(alpha, (x, y), (min(w - 1, x + a), min(h - 1, y + b)), 255, -1)
        else:
            cv2.ellipse(alpha, (x + a // 2, y + b // 2), (a // 2 + 2, b // 2 + 2), 0, 0, 360, 255, -1)
    if rng.random() < 0.5:                                      # a hole: RETR_EXTERNAL ignores it
        cv2.circle(alpha, (w // 2, h // 2), min(w, h) // 10, 200, -1)
    return alpha


@pytest.mark.parametrize('seed', range(8))
def test_mask_oracle_equals_reference_control_flow(seed):
    import cv2
    rng = np.random.default_rng(50 + seed)
    w, h = int(rng.integers(60, 260)), int(rng.integers(60, 200))
    rgba = np.zeros((h, w, 4), np.uint8)
    rgba[..., 3] = _random_alpha(rng, w, h)
    tmp = NamedTemporaryFile(suffix='.png', delete=False)
    key = 'mask_%d' % seed
    try:
        cv2.imwrite(tmp.name, rgba)
        base = {'width': w, 'height': h, 'mask': tmp.name, 'detect': [{'person': {'zones': []}}]}
        try:
            n_zones = len(MaskOracle(base).polygons)
        except (AssertionError, ZeroDivisionError):
            def rejects():
                with ref_classes() as ref:
                    try:
                        ref.MaskFilter(base)
                    except (ValueError, ZeroDivisionError) as e:
                        return 'raises ' + type(e).__name__
                    return 'accepted'
            assert upstream('filters', key, rejects).startswith('raises ')   # the reference rejects the same masks
            return
        zones_b = sorted(int(z) for z in rng.choice(np.arange(1, n_zones + 1), size=int(rng.integers(1, n_zones + 1)),
                                                    replace=False))
        cfg = {'width': w, 'height': h, 'mask': tmp.name,
               'detect': [{'person': {'zones': []}}, {'bicycle': {'zones': zones_b}}, {'car': {'zones': [n_zones]}}]}
        om = MaskOracle(cfg)
        with pytest.raises(AssertionError):
            MaskOracle({**cfg, 'detect': [{'person': {'zones': [n_zones + 1]}}]})
        dets = random_dets(rng, w, h, 600)

        def theirs():
            with ref_classes() as ref:
                try:
                    ref.MaskFilter({**cfg, 'detect': [{'person': {'zones': [n_zones + 1]}}]})
                    bad_zone = 'accepted'
                except AssertionError:
                    bad_zone = 'raises AssertionError'
                return {'bad_zone': bad_zone, 'rows': mask_results(ref, cfg, dets)}
        ref = upstream('filters', key, theirs)
    finally:
        tmp.close()
        os.unlink(tmp.name)
    assert ref['bad_zone'] == 'raises AssertionError'
    assert rows_digest(oracle_results(om, dets)) == ref['rows']


def test_porch_mask_reference_control_flow():
    om = MaskOracle(PORCH_CONFIG)
    dets = random_dets(np.random.default_rng(3), 640, 480, 3000)

    def theirs():
        with ref_classes() as ref:
            return mask_results(ref, PORCH_CONFIG, dets)
    want = upstream('filters', 'porch', theirs)
    tokens = oracle_results(om, dets)
    assert rows_digest(tokens) == want
    hits = sum(t.startswith('1:') for t in tokens)
    assert 300 < hits < 2900
