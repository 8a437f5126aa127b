"""Detection windows on the GPU (wb_set_camera_windows, k_window_merge).  Every check is exact:

  * a window's rows are the existing path's rows for the frame cropped to the window, run as a camera of the window's
    size in a batch of the same model-image count (results depend on it, DESIGN.md 5), shifted by the window's origin;
  * the merge equals tests/window_merge.py on those rows, and the verdicts and zones equal oracle/filters.py on the
    merged rows;
  * a camera whose only window is the whole frame gives exactly the rows of the camera without windows.
"""
import numpy as np
import pytest

from oracle.filters import AreaOracle, ConfidenceOracle, Det, MaskOracle, apply_predicates
from tests import workload
from tests.artist import artist_frame
from tests.conftest import PORCH_CONFIG, load_golden_frame
from tests.gpu_util import new_rows, rows_bytes, rows_to_tuples, zones_of
from tests.window_merge import merge_windows, valid_rows
from tests.yuv_emulation import cv2_rgb, from_rgb, random_frame
from watsor_b200 import _lib
from watsor_b200.detection.b200 import B200ObjectDetector
from watsor_b200.windows import grid_windows

pytestmark = pytest.mark.gpu
MAX_BATCH = 16
CROP_CAM = 200          # cameras 200.. hold the crops of the oracle batches


@pytest.fixture(scope='module', params=[2, 0], ids=['fp32-3xtf32', 'fp32-cuda-cores'])
def v2det(request):
    """the 90-class v2 model at threshold 1e-8: 100 live rows per window, sensitive to every input bit"""
    with B200ObjectDetector(None, device=0, max_batch=MAX_BATCH, precision=request.param,
                            model_blob=workload.v2_coco_model().to_blob()) as d:
        yield d


def run(det, frames, cams, fuse_filters=False, **kw):
    rows = new_rows(len(frames))
    verd = np.zeros((len(frames), 100), np.uint32)
    det.detect_batch(frames, cams, rows, [verd[i] for i in range(len(frames))], fuse_filters=fuse_filters, **kw)
    return rows, verd


def crop_rows(det, frames, windows):
    """valid rows of every window (windows[i]: those of frame i) from ONE batch of host-cropped frames, in the windowed
    batch's order, each crop a camera of its own size without filters"""
    crops, cams, size_cam = [], [], {}
    for frame, wins in zip(frames, windows):
        for x, y, w, h in wins:
            if (w, h) not in size_cam:
                size_cam[(w, h)] = CROP_CAM + len(size_cam)
                det.configure_camera(size_cam[(w, h)], w, h, None)
            crops.append(np.ascontiguousarray(frame[y:y + h, x:x + w]))
            cams.append(size_cam[(w, h)])
    assert len(crops) <= det.max_batch
    rows, _ = run(det, crops, cams)
    out, k = [], 0
    for wins in windows:
        out.append([valid_rows(rows[k + i]) for i in range(len(wins))])
        k += len(wins)
    return out


def expected(det, frames, windows, thresholds, configs):
    """merged rows, zones and verdicts of every frame: tests/window_merge.py, then oracle/filters.py"""
    want = []
    for win_rows, wins, thr, cfg in zip(crop_rows(det, frames, windows), windows, thresholds, configs):
        merged = merge_windows(win_rows, [(x, y) for x, y, _, _ in wins], thr)
        dets = [Det(r[0], r[1], r[2:]) for r in merged]
        if cfg is None:                         # a camera without filters: only track.py's `label > 0`
            verd = [1 if d.label > 0 else 0 for d in dets]
        else:
            _, v = apply_predicates(dets, [ConfidenceOracle(cfg), AreaOracle(cfg), MaskOracle(cfg)])
            verd = [x | (_lib.WB_V_PASS if x == 15 else 0) for x in v]
        want.append((merged, [d.zones for d in dets], verd))
    return want


def assert_rows(rows, verd, want, fuse_filters):
    for i, (merged, zones, v) in enumerate(want):
        assert rows_to_tuples(rows[i]) == merged, i
        assert zones_of(rows[i]) == (zones if fuse_filters else [[0] * 10] * 100), i
        assert list(verd[i]) == v, i


def set_windows(det, cams, windows, thr):
    for cam, wins in zip(cams, windows):
        det.engine.set_camera_windows(cam, wins, thr)


@pytest.mark.parametrize('fuse', [True, False], ids=['fused-filters', 'unfused'])
def test_full_frame_window_is_identity(v2det, fuse):
    """configs[2]: 8 masked 640x480 cameras; the single window (0, 0, W, H) changes no byte and adds one launch"""
    cams = list(range(8))
    for c in cams:
        v2det.configure_camera(c, 640, 480, workload.camera_config(c))
    frames = [artist_frame(640, 480, c, c % 3) for c in cams]
    want = run(v2det, frames, cams, fuse)
    launches = v2det.engine.last_launch_count()
    for c in cams:
        v2det.engine.set_camera_windows(c, [(0, 0, 640, 480)])
    got = run(v2det, frames, cams, fuse)
    assert [rows_bytes(r) for r in got[0]] == [rows_bytes(r) for r in want[0]]
    assert np.array_equal(got[1], want[1])
    assert v2det.engine.last_launch_count() == launches + 1
    for c in cams:
        v2det.engine.set_camera_windows(c, [])
    again = run(v2det, frames, cams, fuse)
    assert [rows_bytes(r) for r in again[0]] == [rows_bytes(r) for r in want[0]]
    assert v2det.engine.last_launch_count() == launches


def test_window_rows_1080p_grid(v2det):
    wins = grid_windows(1920, 1080, 2, 2)
    frames = [artist_frame(1920, 1080, c, 2) for c in (0, 1)]
    for c in (0, 1):
        v2det.configure_camera(c, 1920, 1080, None)
    set_windows(v2det, (0, 1), [wins, wins], 1.0)
    rows, verd = run(v2det, frames, [0, 1])
    assert_rows(rows, verd, expected(v2det, frames, [wins, wins], [1.0, 1.0], [None, None]), False)


def test_window_rows_odd_windows_mixed_batch_submit_and_device_frames(v2det):
    torch = pytest.importorskip('torch')
    odd = [(0, 0, 640, 480), (13, 7, 301, 233), (300, 201, 339, 279), (611, 451, 29, 29)]
    grid = grid_windows(1920, 1080, 2, 2)
    v2det.configure_camera(0, 640, 480, None)
    v2det.configure_camera(1, 640, 480, None)            # no windows: one full-frame window in this batch
    v2det.configure_camera(2, 1920, 1080, None)
    set_windows(v2det, (0, 2), [odd, grid], 1.0)
    frames = [artist_frame(640, 480, 3, 1), load_golden_frame('artist_640x480_c0_f1'), artist_frame(1920, 1080, 5, 0)]
    cams = [0, 1, 2]
    windows = [odd, [(0, 0, 640, 480)], grid]               # 4 + 1 + 5 model images
    want = expected(v2det, frames, windows, [1.0, 0.5, 1.0], [None] * 3)
    rows, verd = run(v2det, frames, cams)
    assert_rows(rows, verd, want, False)
    v2det.submit(3, frames, cams, fuse_filters=False)
    rows = new_rows(3)
    verd = np.zeros((3, 100), np.uint32)
    v2det.collect(3, rows, [verd[i] for i in range(3)])
    assert_rows(rows, verd, want, False)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    torch.cuda.synchronize()
    rows, verd = run(v2det, [t.data_ptr() for t in dev], cams, frames_on_device=True)
    assert_rows(rows, verd, want, False)
    assert all(np.array_equal(t.cpu().numpy(), f) for t, f in zip(dev, frames))   # inputs untouched


def test_merge_with_masks_and_fused_filters(v2det):
    """default threshold 0.5 on masked 640x480 cameras: rows, zones and verdicts"""
    cams = [0, 1, 2]
    configs = [workload.camera_config(c) for c in cams]
    windows = [grid_windows(640, 480, 2, 2), grid_windows(640, 480, 3, 1, full_frame=False),
               [(0, 0, 640, 480), (100, 50, 320, 240)]]
    for c, cfg, wins in zip(cams, configs, windows):
        v2det.configure_camera(c, 640, 480, dict(cfg, windows=[list(w) for w in wins]))
    frames = [artist_frame(640, 480, c, 4) for c in cams]
    want = expected(v2det, frames, windows, [0.5] * 3, configs)
    rows, verd = run(v2det, frames, cams, fuse_filters=True)
    assert_rows(rows, verd, want, True)


def test_merge_real_weights_shapes_cut_by_window_borders(shapes_model):
    with B200ObjectDetector(None, device=0, max_batch=MAX_BATCH, precision=2, model_blob=shapes_model.to_blob()) as det:
        wins = grid_windows(640, 480, 2, 2, overlap=0.2)
        names = ('artist_640x480_c0_f0', 'artist_640x480_c0_f1', 'artist_640x480_c3_f7')
        for c, name in enumerate(names[:2]):
            det.configure_camera(c, 640, 480, dict(PORCH_CONFIG, windows=wins, window_merge_threshold=0.5))
        frames = [load_golden_frame(n) for n in names[:2]]
        want = expected(det, frames, [wins, wins], [0.5, 0.5], [PORCH_CONFIG] * 2)
        rows, verd = run(det, frames, [0, 1], fuse_filters=True)
        assert_rows(rows, verd, want, True)
        # without the merge the same shapes would be reported once per window that sees them
        assert sum(len(r) for r in crop_rows(det, frames, [wins, wins])[0]) > sum(r[1] > 0 for r in want[0][0])


@pytest.mark.parametrize('fmt', ['yuv420p', 'nv12'])
def test_yuv420_windows_equal_rgb_path(v2det, fmt):
    rng = np.random.default_rng(11)
    wins = [(0, 0, 640, 480), (12, 8, 300, 226), (320, 240, 320, 240), (2, 402, 78, 78)]
    for c in (0, 1):
        v2det.configure_camera(c, 640, 480, workload.camera_config(c))
        v2det.engine.set_camera_windows(c, wins)
    frames = [from_rgb(artist_frame(640, 480, 7, 0), fmt), random_frame(rng, 640, 480)]
    before = [f.copy() for f in frames]
    got = run(v2det, frames, [0, 1], True, pixel_format=fmt)
    want = run(v2det, [cv2_rgb(f, fmt) for f in frames], [0, 1], True)
    assert [rows_bytes(r) for r in got[0]] == [rows_bytes(r) for r in want[0]]
    assert np.array_equal(got[1], want[1])
    assert all(np.array_equal(a, b) for a, b in zip(before, frames))


def test_errors_leave_the_slot_usable(v2det):
    engine = v2det.engine
    v2det.configure_camera(0, 640, 480, None)
    wins = grid_windows(640, 480, 4, 2)                       # 9 windows: two frames need 18 > 16 model images
    engine.set_camera_windows(0, wins)
    frame = artist_frame(640, 480, 2, 2)
    with pytest.raises(_lib.WatsorB200Error, match='max_batch'):
        run(v2det, [frame, frame], [0, 0])
    good = run(v2det, [frame], [0])
    # an odd window in a 4:2:0 batch: Python refuses it, and so does the library (a raw address skips Python's check)
    engine.set_camera_windows(0, [(0, 0, 640, 480), (1, 0, 100, 100)])
    yuv = from_rgb(frame, 'nv12')
    with pytest.raises(ValueError, match='even window origin'):
        run(v2det, [yuv], [0], pixel_format='nv12')
    n, fp, cams, op, vp = engine._io([yuv.ctypes.data], [0], new_rows(1), None)
    with pytest.raises(_lib.WatsorB200Error, match='cam_id 0 window 1'):
        _lib.check(engine.lib.wb_detect(engine._ctx, n, fp, cams, _lib.WB_F_NV12, op, vp, None))
    # a window outside the frame
    with pytest.raises(ValueError, match='not inside'):
        engine.set_camera_windows(0, [(600, 0, 41, 10)])
    xywh = (_lib.c_int32 * 4)(600, 0, 41, 10)
    with pytest.raises(_lib.WatsorB200Error, match='not inside'):
        _lib.check(engine.lib.wb_set_camera_windows(engine._ctx, 0, 1, xywh, 0.5))
    with pytest.raises(_lib.WatsorB200Error, match=r'\[0, 1\]'):
        _lib.check(engine.lib.wb_set_camera_windows(engine._ctx, 0, 0, None, 1.5))
    engine.set_camera_windows(0, wins)
    again = run(v2det, [frame], [0])
    assert rows_bytes(again[0][0]) == rows_bytes(good[0][0]) and np.array_equal(again[1], good[1])
