"""4:2:0 frames (yuv420p, NV12) through detection and the effects pass.  The kernels convert them as cv2.cvtColor
does, so every result must equal, byte for byte, the RGB24 path on cvtColor of the same frame."""
import numpy as np
import pytest

from tests import workload
from tests.artist import artist_frame
from tests.conftest import PORCH_CONFIG, load_golden_frame
from tests.fx_cases import random_rows
from tests.gpu_util import new_rows, rows_bytes
from tests.yuv_emulation import all_triples, cv2_rgb, from_rgb, random_frame
from watsor_b200 import _lib
from watsor_b200.detection.b200 import B200ObjectDetector

pytestmark = pytest.mark.gpu
FORMATS = ['yuv420p', 'nv12']
SIZES = [(100, 100), (320, 240), (640, 480), (1920, 1080), (302, 226), (150, 100)]


@pytest.fixture(scope='module')
def fx():
    from watsor_b200.output.effects import EffectsEngine
    with EffectsEngine(0) as e:
        yield e


@pytest.fixture(scope='module', params=[2, 0], ids=['fp32-3xtf32', 'fp32-cuda-cores'])
def v2det(request):
    """the 90-class v2 model at threshold 1e-8: 100 live rows per frame, sensitive to every input bit"""
    with B200ObjectDetector(None, device=0, max_batch=8, precision=request.param,
                            model_blob=workload.v2_coco_model().to_blob()) as d:
        yield d


def run(det, frames, cams, pixel_format='rgb24', fuse_filters=False, **kw):
    rows = new_rows(len(frames))
    verd = np.zeros((len(frames), 100), np.uint32)
    det.detect_batch(frames, cams, rows, [verd[i] for i in range(len(frames))], fuse_filters=fuse_filters,
                     pixel_format=pixel_format, **kw)
    return [rows_bytes(r) for r in rows], verd


def assert_same_as_rgb(det, yuv_frames, cams, fmt, **kw):
    before = [f.copy() for f in yuv_frames]
    got = run(det, yuv_frames, cams, fmt, **kw)
    want = run(det, [cv2_rgb(f, fmt) for f in yuv_frames], cams, **kw)
    assert got[0] == want[0], fmt
    assert np.array_equal(got[1], want[1]), fmt
    assert all(np.array_equal(a, b) for a, b in zip(before, yuv_frames))   # inputs untouched


@pytest.mark.parametrize('fmt', FORMATS)
def test_exhaustive_conversion_equals_cvtcolor(fx, fmt):
    """every (Y, U, V) triple through k_fx_render without effects: the device routine itself"""
    cam = fx.add_camera(4096, 4096)
    frame = all_triples(fmt)
    out = np.zeros((4096, 4096, 3), np.uint8)
    fx.render([frame], [out], [cam], [new_rows()[0]], 0, pixel_format=fmt)
    assert np.array_equal(out, cv2_rgb(frame, fmt))


@pytest.mark.parametrize('fmt', FORMATS)
def test_detection_rows_equal_rgb_path(v2det, fmt):
    rng = np.random.default_rng(3)
    golden = {(640, 480): 'artist_640x480_c3_f7', (320, 240): 'artist_320x240_c2_f5', (100, 100): 'artist_100x100_c1_f0'}
    for k, (w, h) in enumerate(SIZES):
        cam = 20 + k
        v2det.configure_camera(cam, w, h, None)
        rgb = load_golden_frame(golden[(w, h)]) if (w, h) in golden else artist_frame(w, h, k, 1)
        assert_same_as_rgb(v2det, [from_rgb(rgb, fmt), random_frame(rng, w, h)], [cam, cam], fmt)


@pytest.mark.parametrize('fmt', FORMATS)
def test_masked_batch_with_fused_filters_submit_and_device_frames(v2det, fmt):
    torch = pytest.importorskip('torch')
    for c in range(8):
        v2det.configure_camera(c, 640, 480, workload.camera_config(c))
    rng = np.random.default_rng(8)
    frames = [from_rgb(artist_frame(640, 480, c, c % 3), fmt) if c % 2 == 0 else random_frame(rng, 640, 480)
              for c in range(8)]
    cams = list(range(8))
    assert_same_as_rgb(v2det, frames, cams, fmt, fuse_filters=True)
    want = run(v2det, frames, cams, fmt, fuse_filters=True)
    # asynchronous form
    v2det.submit(1, frames, cams, fuse_filters=True, pixel_format=fmt)
    rows = new_rows(8)
    verd = np.zeros((8, 100), np.uint32)
    v2det.collect(1, rows, [verd[i] for i in range(8)])
    assert [rows_bytes(r) for r in rows] == want[0] and np.array_equal(verd, want[1])
    # frames resident on the device (a GPU decoder's output)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    torch.cuda.synchronize()
    got = run(v2det, [t.data_ptr() for t in dev], cams, fmt, fuse_filters=True, frames_on_device=True)
    assert got[0] == want[0] and np.array_equal(got[1], want[1])
    # an RGB batch on the same slot and graph afterwards still reads RGB
    assert run(v2det, [cv2_rgb(f, fmt) for f in frames], cams, fuse_filters=True)[0] == want[0]


def test_real_weights_model(shapes_model):
    with B200ObjectDetector(None, device=0, max_batch=4, precision=2, model_blob=shapes_model.to_blob()) as det:
        det.configure_camera(0, 640, 480, PORCH_CONFIG)
        frames = [load_golden_frame(n) for n in ('artist_640x480_c0_f0', 'artist_640x480_c0_f1', 'artist_640x480_c3_f7')]
        for fmt in FORMATS:
            assert_same_as_rgb(det, [from_rgb(f, fmt) for f in frames], [0] * 3, fmt, fuse_filters=True)


def test_effects_equal_rgb_path(fx):
    from oracle import effects as oracle_fx
    from watsor_b200.filter.mask import get_alpha_channel
    from watsor_b200.output.effects import WB_FX_BLEND, WB_FX_CONTOURS, WB_FX_DRAW, contour_bits
    alpha, _ = get_alpha_channel(PORCH_CONFIG['mask'], 640, 480)
    cam = fx.add_camera(640, 480, alpha, contour_bits(alpha))
    rng = np.random.default_rng(4)
    rows = random_rows(rng, 640, 480, 12, n_zones=2)
    for fmt in FORMATS:
        for frame in (from_rgb(load_golden_frame('artist_640x480_c0_f0'), fmt), random_frame(rng, 640, 480)):
            rgb = cv2_rgb(frame, fmt)
            for flags in (WB_FX_BLEND, WB_FX_DRAW, WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS):
                got, want = np.zeros_like(rgb), np.zeros_like(rgb)
                fx.render([frame], [got], [cam], [rows], flags, pixel_format=fmt)
                fx.render([rgb], [want], [cam], [rows], flags)
                assert np.array_equal(got, want), (fmt, flags)
            assert np.array_equal(got, oracle_fx.effect_chain(rgb, rows, alpha))


def test_errors(v2det, fx):
    from watsor_b200.output.effects import WB_FX_NV12, WB_FX_YUV420P
    engine = v2det.engine
    v2det.configure_camera(40, 302, 100, None)
    v2det.configure_camera(41, 301, 100, None)
    v2det.configure_camera(42, 302, 101, None)
    frame = random_frame(np.random.default_rng(0), 302, 100)
    for cam in (41, 42):
        with pytest.raises(ValueError, match='even width and height'):
            v2det.detect_batch([frame], [cam], new_rows(1), pixel_format='nv12')
        # the library's own check (a raw address bypasses the Python one)
        with pytest.raises(_lib.WatsorB200Error, match='even width and height'):
            engine.detect([frame.ctypes.data], [cam], new_rows(1), flags=_lib.WB_F_YUV420P)
    with pytest.raises(_lib.WatsorB200Error, match='mutually exclusive'):
        engine.detect([frame.ctypes.data], [40], new_rows(1), flags=_lib.WB_F_YUV420P | _lib.WB_F_NV12)
    with pytest.raises(ValueError, match='shape'):
        v2det.detect_batch([cv2_rgb(frame, 'nv12')], [40], new_rows(1), pixel_format='nv12')
    with pytest.raises(ValueError, match='shape'):
        v2det.detect_batch([frame], [40], new_rows(1))
    assert_same_as_rgb(v2det, [frame], [40], 'nv12')                       # the context is still usable
    # effects
    cam = fx.add_camera(302, 100)
    odd = fx.add_camera(301, 100)
    rows = new_rows()[0]
    out = np.zeros((100, 302, 3), np.uint8)
    with pytest.raises(_lib.WatsorB200Error, match='in place'):
        fx.render([frame], [frame], [cam], [rows], 0, pixel_format='yuv420p')
    with pytest.raises(_lib.WatsorB200Error, match='mutually exclusive'):
        fx.render([frame.ctypes.data], [out.ctypes.data], [cam], [rows], WB_FX_YUV420P | WB_FX_NV12)
    with pytest.raises(_lib.WatsorB200Error, match='even width and height'):
        fx.render([frame.ctypes.data], [out.ctypes.data], [odd], [rows], WB_FX_NV12)
    with pytest.raises(ValueError, match='shape'):
        fx.render([cv2_rgb(frame, 'nv12')], [out], [cam], [rows], 0, pixel_format='nv12')
    fx.render([frame], [out], [cam], [rows], 0, pixel_format='nv12')
    assert np.array_equal(out, cv2_rgb(frame, 'nv12'))
