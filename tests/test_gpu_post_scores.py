"""k_nms scores its own class from the heads' logits, decodes the boxes it visits and hands the kept boxes' corners to
k_merge_filter.  These cases compare the post stage with the oracle's on 90-class heads built to reach the edges of
that code: classes without a candidate, a class whose candidates all share one score (the chunk holds every key),
scores below 2^-27 (histogram bin 0), exact score ties between anchors, a class that keeps max_per_class boxes, a
64-frame batch, and a windowed batch."""
import numpy as np
import pytest

from tests import workload
from tests.artist import artist_frame
from tests.gpu_util import new_rows, rows_bytes, rows_to_tuples
from tests.test_gpu_stages import check_post
from tests.window_merge import merge_windows, valid_rows
from watsor_b200.engine import PRECISION_TF32X3, Engine

pytestmark = pytest.mark.gpu
C1 = 91  # 90 classes + background


@pytest.fixture(scope='module')
def v2_model():
    return workload.v2_coco_model()


@pytest.fixture(scope='module')
def v2_oracle(v2_model):
    from oracle.ssd_model import SsdModelOracle
    return SsdModelOracle(v2_model)


@pytest.fixture(scope='module')
def v2_engine(v2_model):
    with Engine(v2_model.to_blob(), device=0, max_batch=64, precision=PRECISION_TF32X3) as e:
        e.set_camera(0, 640, 480)
        yield e


def heads(seed, n, enc_scale=0.8):
    rng = np.random.default_rng(seed)
    enc = (rng.standard_normal((n, 4)) * enc_scale).astype(np.float32)
    lg = (rng.standard_normal((n, C1)) * 1.5 - 3.0).astype(np.float32)
    return rng, enc, lg


def assert_post(engine, oracle, enc, lg, want_num=None):
    num, mism = check_post(engine, oracle, enc, lg)
    assert not mism, mism[:3]
    if want_num is not None:
        assert num == want_num
    return num


def test_classes_without_candidates(v2_engine, v2_oracle):
    """two thirds of the classes have no score above 1e-8 (sigmoid(-40) ~ 4e-18); one class has a single candidate"""
    n = v2_oracle.num_anchors
    rng, enc, lg = heads(1, n)
    lg[:, 1:61] = -40.0
    lg[:, 61] = -40.0
    lg[123, 61] = 2.0
    assert_post(v2_engine, v2_oracle, enc, lg, 100)
    lg[:, 1:] = -40.0                      # no candidate anywhere: 100 padding rows
    lg[7, 30] = 0.5
    enc[7] = 0.0                           # the anchor box itself: a positive clipped area
    assert_post(v2_engine, v2_oracle, enc, lg, 1)


def test_every_score_equal(v2_engine, v2_oracle):
    """all 1917 keys of a class in one histogram bin: the first chunk is the whole class, sorted by anchor alone"""
    n = v2_oracle.num_anchors
    rng, enc, lg = heads(2, n)
    lg[:, 1:] = 0.75
    assert_post(v2_engine, v2_oracle, enc, lg, 100)
    lg[:, 1:] = -4.0                       # the same with most classes cut by the frame-wide early exit
    lg[:, 17] = 1.25
    assert_post(v2_engine, v2_oracle, enc, lg, 100)


def test_scores_below_two_to_minus_27():
    """threshold 1e-12: candidates with scores under 2^-27 share histogram bin 0 with nothing above them"""
    from oracle.ssd_model import SsdModelOracle
    from watsor_b200.model import synthetic_ssd_mobilenet_v2
    model = synthetic_ssd_mobilenet_v2(num_classes=90, seed=0, score_thr=1e-12)
    oracle = SsdModelOracle(model)
    n = oracle.num_anchors
    rng, enc, lg = heads(3, n)
    lg[:, 1:] = (-25.0 + rng.standard_normal((n, 90)) * 1.5).astype(np.float32)   # sigmoid ~ 1e-11 .. 1e-10
    lg[:50, 3] = (-18.0 + rng.standard_normal(50)).astype(np.float32)             # a few above 2^-27
    lg[:, 9] = -40.0                                                              # below the threshold
    with Engine(model.to_blob(), device=0, max_batch=2, precision=PRECISION_TF32X3) as e:
        e.set_camera(0, 640, 480)
        assert_post(e, oracle, enc, lg, 100)


@pytest.mark.parametrize('quantum', [0.25, 1.0])
def test_equal_scores_on_different_anchors(v2_engine, v2_oracle, quantum):
    """quantised logits: thousands of exact ties, broken by the lower anchor index"""
    n = v2_oracle.num_anchors
    rng, enc, lg = heads(4, n, enc_scale=1.2)
    lg = (np.round(lg / quantum) * quantum).astype(np.float32)
    assert_post(v2_engine, v2_oracle, enc, lg, 100)


def test_class_keeps_max_per_class(v2_engine, v2_oracle):
    """small boxes on the ~500 anchor centres (boxes on one centre suppress each other, on different centres never),
    all inside the window: class 5 (highest scores) keeps 100 and fills the frame's 100 rows"""
    n = v2_oracle.num_anchors
    rng, enc, lg = heads(5, n)
    enc[:, :2] = 0.0
    enc[:, 2:] = -12.0
    lg[:, 5] = (6.0 + rng.random(n)).astype(np.float32)
    _, _, _, _, classes, _ = v2_engine.postprocess(enc[None], lg[None], [0])
    assert np.all(classes[0] == 5.0)
    assert_post(v2_engine, v2_oracle, enc, lg, 100)


def test_batch_of_64_frames(v2_engine, v2_oracle):
    """max_batch 64 at 90 classes: 5760 NMS blocks, each frame checked against the oracle"""
    n = v2_oracle.num_anchors
    rng = np.random.default_rng(6)
    enc = (rng.standard_normal((64, n, 4)) * 0.8).astype(np.float32)
    lg = (rng.standard_normal((64, n, C1)) * 1.5 - 3.0).astype(np.float32)
    lg[::7, :, 1:40] = -40.0
    from oracle.ssd_graph import to_detections
    rows, _, boxes, scores, classes, num = v2_engine.postprocess(enc, lg, [0] * 64)
    for f in range(64):
        b, s, cl, k = v2_oracle.postprocess(enc[f], lg[f])
        assert num[f] == k and np.array_equal(classes[f], cl), f
        assert np.allclose(boxes[f], b, rtol=0, atol=3e-7) and np.allclose(scores[f], s, rtol=0, atol=2e-7), f
        want = to_detections(b, cl, s, (480, 640, 3))
        got = rows_to_tuples(rows[f])
        assert all(g[0] == w[0] and g[2:] == w[2:] and abs(g[1] - w[1]) <= 2e-7 for g, w in zip(got, want)), f


def test_windowed_batch(v2_model):
    """a frame cut into three windows: the windows' rows (camera -1, valid-row counts for the merge) equal those of
    the same crops detected as frames of their own in a batch of the same size, and the merge equals
    tests/window_merge.py on them"""
    from watsor_b200.detection.b200 import B200ObjectDetector
    wins = [(0, 0, 640, 480), (600, 0, 640, 480), (300, 240, 640, 480)]
    frame = artist_frame(1240, 720, 0, 3)
    with B200ObjectDetector(None, device=0, max_batch=4, precision=PRECISION_TF32X3,
                            model_blob=v2_model.to_blob()) as det:
        det.configure_camera(0, 1240, 720, None)
        det.configure_camera(1, 640, 480, None)
        crops = [np.ascontiguousarray(frame[y:y + h, x:x + w]) for x, y, w, h in wins]
        crop_rows = new_rows(3)
        det.detect_batch(crops, [1, 1, 1], crop_rows, fuse_filters=False)
        det.engine.set_camera_windows(0, wins, 0.5)
        rows = new_rows(1)
        det.detect_batch([frame], [0], rows, fuse_filters=False)
        want = merge_windows([valid_rows(r) for r in crop_rows], [(x, y) for x, y, _, _ in wins], 0.5)
        assert rows_to_tuples(rows[0]) == want
        again = new_rows(1)
        det.detect_batch([frame], [0], again, fuse_filters=False)
        assert rows_bytes(again[0]) == rows_bytes(rows[0])
