"""The write loop of the reference detector (watsor/detection/tensorflow_cpu.py:74-92) run here, as it is, against
the oracle's `to_detections` (SURVEY.md 8a row a2).  TensorFlow is not installed, so the class is imported with an
empty stand-in `tensorflow` module and instantiated without `__init__`; only `detect()` runs, with the arrays a
`sess.run` would return supplied by the test.  Two readings of `int(np.float32 * int)`:
  * legacy promotion (numpy 1.23, the reference's pin, docker/Dockerfile.base:33): the product is a float64, i.e.
    exact -- reproduced on any numpy by handing the loop float64 copies of the float32 boxes;
  * NEP 50 (numpy >= 2): the product is rounded to float32 first; it differs from the exact reading only where that
    rounding lands on an integer -- counted here, and every such case is checked to be exactly that.
CPU only; without an upstream checkout the upstream rows come from tests/golden/reference/ as a digest (plus the
cells where the NEP 50 reading differs from the exact one), see tests/reference_golden.py."""
import hashlib
import json
import sys
import types

import numpy as np
import pytest

from oracle.ssd_graph import to_detections

from tests.conftest import REF_DIR as REF  # noqa: E402
from tests.reference_golden import upstream  # noqa: E402


def reference_classes():
    saved = sys.modules.get('tensorflow')
    sys.modules['tensorflow'] = types.ModuleType('tensorflow')
    sys.path.insert(0, REF)
    try:
        from watsor.detection.tensorflow_cpu import TensorFlowObjectDetector
        from watsor.stream.share import Detection
        return types.SimpleNamespace(Detector=TensorFlowObjectDetector, Detection=Detection)
    finally:
        sys.path.remove(REF)
        if saved is None:
            sys.modules.pop('tensorflow', None)
        else:
            sys.modules['tensorflow'] = saved


def plain(rows):
    return [[int(r[0]), float(r[1]), int(r[2]), int(r[3]), int(r[4]), int(r[5])] for r in rows]


def digest(rows):
    return hashlib.sha256(json.dumps(plain(rows)).encode()).hexdigest()[:16]


def run_reference_loop(boxes, classes, scores, shape, n_rows=100):
    ref = reference_classes()
    det = object.__new__(ref.Detector)
    setattr(det, '_TensorFlowObjectDetector__detect_fn', lambda image: (boxes, classes, scores))
    rows = (ref.Detection * n_rows)()
    ms = det.detect(shape, None, rows)
    assert ms >= 0.0
    return [(r.label, r.confidence, r.bounding_box.x_min, r.bounding_box.y_min, r.bounding_box.x_max,
             r.bounding_box.y_max) for r in rows]


def random_outputs(rng, n=100):
    boxes = rng.random((n, 4)).astype(np.float32)
    boxes[::7] = np.float32(1.0)                               # clipped to the window edge
    boxes[1::7] = np.float32(0.0)
    boxes[2::11, 2:] = np.nextafter(np.float32(1.0), np.float32(0.0))
    k = int(rng.integers(0, n))
    boxes[k:] = 0.0                                             # PadOrClipBoxList padding
    scores = np.sort(rng.random(n).astype(np.float32))[::-1].copy()
    scores[k:] = 0.0
    classes = rng.integers(1, 4, n).astype(np.float32)
    classes[k:] = 1.0                                           # padded rows: 0 + 1
    return boxes, classes, scores


@pytest.mark.parametrize('shape', [(480, 640, 3), (240, 320, 3), (1080, 1920, 3), (2, 2, 3), (1, 1, 3)])
def test_oracle_equals_reference_loop_under_legacy_promotion(shape):
    rng = np.random.default_rng(shape[0])
    for i in range(40):
        boxes, classes, scores = random_outputs(rng)
        want = upstream('detect_loop', 'legacy %r %d' % (shape, i),
                        lambda: digest(run_reference_loop(boxes.astype(np.float64), classes, scores, shape)))
        assert digest(to_detections(boxes, classes, scores, shape)) == want


def test_short_outputs_leave_the_remaining_rows_untouched():
    rng = np.random.default_rng(1)
    boxes, classes, scores = random_outputs(rng, 7)
    want = upstream('detect_loop', 'short',
                    lambda: digest(run_reference_loop(boxes.astype(np.float64), classes, scores, (480, 640, 3))))
    # share.py:47-50: the rows beyond the outputs keep their zeros
    assert digest(list(to_detections(boxes, classes, scores, (480, 640, 3))) + [(0, 0.0, 0, 0, 0, 0)] * 93) == want


def nep50_rows(i, boxes, classes, scores, shape):
    """The reference loop's rows on float32 boxes: stored as the cells that differ from the exact reading + a digest."""
    exact = plain(to_detections(boxes, classes, scores, shape))

    def theirs():
        rows = plain(run_reference_loop(boxes, classes, scores, shape))
        diff = [[d, c, rows[d][c]] for d in range(len(rows)) for c in range(6) if rows[d][c] != exact[d][c]]
        return {'digest': digest(rows), 'diff': diff}
    ref = upstream('detect_loop', 'nep50 %d' % i, theirs)
    rows = [list(r) for r in exact]
    for d, c, v in ref['diff']:
        rows[d][c] = v
    assert digest(rows) == ref['digest']
    return rows


def test_nep50_reading_differs_only_on_float32_rounding_to_an_integer():
    if int(np.__version__.split('.')[0]) < 2:
        pytest.skip('NEP 50 promotion needs numpy >= 2')
    rng = np.random.default_rng(7)
    shape = (1080, 1920, 3)
    differing = total = 0
    for i in range(200):
        boxes, classes, scores = random_outputs(rng)
        new = nep50_rows(i, boxes, classes, scores, shape)
        exact = plain(to_detections(boxes, classes, scores, shape))
        for d, (a, b) in enumerate(zip(new, exact)):
            assert a[:2] == b[:2]
            for j, (va, vb) in enumerate(zip(a[2:], b[2:])):
                total += 1
                if va != vb:
                    differing += 1
                    col = (1, 0, 3, 2)[j]                       # x_min,y_min,x_max,y_max <- boxes[:, 1,0,3,2]
                    mx = (shape[1] - 1) if j % 2 == 0 else (shape[0] - 1)
                    p32 = np.float32(boxes[d][col]) * np.float32(mx)
                    assert va == vb + 1 and float(p32) == float(va), (d, j, boxes[d][col])
    assert differing < total * 1e-3
