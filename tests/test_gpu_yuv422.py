"""Packed 4:2:2 frames (YUYV, UYVY) through detection and the effects pass.  The kernels convert them as cv2.cvtColor
does, so every result must equal, byte for byte, the RGB24 path on cvtColor of the same frame."""
import os

import numpy as np
import pytest

from oracle import effects as oracle_fx
from tests import workload
from tests import yuv_emulation as yuv420
from tests.artist import artist_frame
from tests.conftest import PORCH_CONFIG, load_golden_frame
from tests.fx_cases import random_alpha, random_rows
from tests.gpu_util import new_rows, rows_bytes
from tests.test_gpu_frame_path import _stem_model
from tests.yuv422_emulation import FORMATS, all_triples, cv2_rgb, from_rgb, random_frame
from watsor_b200 import _lib
from watsor_b200.detection.b200 import B200ObjectDetector
from watsor_b200.engine import Engine
from watsor_b200.windows import grid_windows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def fx():
    from watsor_b200.output.effects import EffectsEngine
    with EffectsEngine(0) as e:
        yield e


@pytest.fixture(scope='module', params=[2, 0, 4], ids=['tf32x3', 'fp32', 'fp16'])
def v2det(request):
    """the 90-class v2 model at threshold 1e-8: 100 live rows per frame, sensitive to every input bit"""
    with B200ObjectDetector(None, device=0, max_batch=8, precision=request.param,
                            model_blob=workload.v2_coco_model().to_blob()) as d:
        yield d


def to_device(frames, offset=0):
    """device copies of the frames, `offset` bytes past the start of a fresh allocation (which is 256-byte aligned)"""
    import torch
    bufs = []
    for f in frames:
        b = torch.zeros(f.size + 16, dtype=torch.uint8, device='cuda')
        b[offset:offset + f.size].copy_(torch.from_numpy(np.ascontiguousarray(f).reshape(-1)))
        bufs.append(b)
    torch.cuda.synchronize()
    return bufs, [b.data_ptr() + offset for b in bufs]


def run(det, frames, cams, pixel_format='rgb24', fuse_filters=False, **kw):
    rows = new_rows(len(frames))
    verd = np.zeros((len(frames), 100), np.uint32)
    det.detect_batch(frames, cams, rows, [verd[i] for i in range(len(frames))], fuse_filters=fuse_filters,
                     pixel_format=pixel_format, **kw)
    return [rows_bytes(r) for r in rows], verd


def submit_collect(det, slot, frames, cams, **kw):
    det.submit(slot, frames, cams, **kw)
    rows = new_rows(len(frames))
    verd = np.zeros((len(frames), 100), np.uint32)
    det.collect(slot, rows, [verd[i] for i in range(len(frames))])
    return [rows_bytes(r) for r in rows], verd


def same(got, want):
    return got[0] == want[0] and np.array_equal(got[1], want[1])


# ------------------------------------------------------------------------------- the device routine, exhaustively
@pytest.mark.parametrize('side', [0, 1], ids=['left', 'right'])
@pytest.mark.parametrize('fmt', FORMATS)
def test_exhaustive_conversion_equals_cvtcolor(fx, fmt, side):
    """every (Y, U, V) triple on the left or right pixel of a pair, through k_fx_render without effects"""
    frame = all_triples(fmt, side)
    h, w = frame.shape[:2]
    cam = fx.add_camera(w, h)
    out = np.zeros((h, w, 3), np.uint8)
    fx.render([frame], [out], [cam], [new_rows()[0]], 0, pixel_format=fmt)
    assert np.array_equal(out, cv2_rgb(frame, fmt))


# ------------------------------------------------------------------------------------------- the stem on frames
STEM_SIZES = [(2, 1), (2, 2), (300, 300), (600, 600), (640, 479), (1920, 1080), (3840, 2160)]
MIXED = [(640, 479), (2, 1), (3840, 2160), (300, 300)]


@pytest.mark.parametrize('precision', [2, 1], ids=['tf32x3', 'bf16'])
@pytest.mark.parametrize('stem', ['3x3s2_c32_300', '7x7s2_c24_300'], ids=['k_stem_3x3s2_c32', 'k_stem'])
def test_stem_on_frames_equals_rgb_path(stem, precision):
    """wb_backbone_frames stopped after the stem: 4:2:2 frames from the host and from 4-byte-aligned (not 16-byte)
    device addresses give the activation of the RGB24 frames cvtColor makes, bit for bit"""
    m = _stem_model(stem)
    L = m.layers[0]
    shape = (L.out_h, L.out_w, L.out_c)
    rng = np.random.default_rng(12)
    with Engine(m.to_blob(), device=0, max_batch=len(MIXED), precision=precision) as e:
        for sizes in [[s] for s in STEM_SIZES] + [MIXED]:
            cams = list(range(len(sizes)))
            for c, (w, h) in zip(cams, sizes):
                e.set_camera(c, w, h)
            for fmt in FORMATS:
                frames = [random_frame(rng, w, h, fmt) for w, h in sizes]
                want = e.backbone_frames([cv2_rgb(f, fmt) for f in frames], cams, stop_layer=0, layer_shape=shape)[2]
                assert np.abs(want).max() > 0
                got = e.backbone_frames(frames, cams, stop_layer=0, layer_shape=shape, pixel_format=fmt)[2]
                assert e.last_launch_count() == 1
                assert np.array_equal(got, want), (stem, fmt, sizes, 'host')
                bufs, ptrs = to_device(frames, offset=4)
                got = e.backbone_frames(ptrs, cams, stop_layer=0, layer_shape=shape, pixel_format=fmt,
                                        frames_on_device=True)[2]
                assert np.array_equal(got, want), (stem, fmt, sizes, 'device')


# ------------------------------------------------------------------------------------------------- detection
@pytest.mark.parametrize('fmt', FORMATS)
def test_configs2_rows_equal_rgb_path(v2det, fmt):
    """BASELINE configs[2]: 8 cameras of 640x480, a mask each, fused filters; detect_batch and submit/collect from
    host and device frames"""
    for c in range(8):
        v2det.configure_camera(c, 640, 480, workload.camera_config(c))
    rng = np.random.default_rng(8)
    frames = [from_rgb(artist_frame(640, 480, c, c % 3), fmt) if c % 2 == 0 else random_frame(rng, 640, 480, fmt)
              for c in range(8)]
    cams = list(range(8))
    before = [f.copy() for f in frames]
    want = run(v2det, [cv2_rgb(f, fmt) for f in frames], cams, fuse_filters=True)
    assert same(run(v2det, frames, cams, fmt, fuse_filters=True), want)
    assert all(np.array_equal(a, b) for a, b in zip(before, frames))          # inputs untouched
    assert same(submit_collect(v2det, 1, frames, cams, fuse_filters=True, pixel_format=fmt), want)
    for offset in (0, 4):
        bufs, ptrs = to_device(frames, offset)
        assert same(run(v2det, ptrs, cams, fmt, fuse_filters=True, frames_on_device=True), want), offset
        assert same(submit_collect(v2det, 2, ptrs, cams, fuse_filters=True, frames_on_device=True, pixel_format=fmt),
                    want), offset


def test_real_weights_model(shapes_model):
    with B200ObjectDetector(None, device=0, max_batch=4, precision=2, model_blob=shapes_model.to_blob()) as det:
        det.configure_camera(0, 640, 480, PORCH_CONFIG)
        rgb = [load_golden_frame(n) for n in ('artist_640x480_c0_f0', 'artist_640x480_c0_f1', 'artist_640x480_c3_f7')]
        for fmt in FORMATS:
            frames = [from_rgb(f, fmt) for f in rgb]
            want = run(det, [cv2_rgb(f, fmt) for f in frames], [0] * 3, fuse_filters=True)
            assert same(run(det, frames, [0] * 3, fmt, fuse_filters=True), want), fmt


WINDOWS = {
    'grid_2x2': grid_windows(1920, 1080, 2, 2),
    # odd y origins and heights, windows touching the right and the bottom border
    'odd_y_borders': [(0, 1, 960, 539), (960, 541, 960, 539), (2, 3, 1918, 1077), (1280, 0, 640, 1080),
                      (0, 1079, 1920, 1)],
}


@pytest.mark.parametrize('layout', list(WINDOWS))
def test_windows_equal_rgb_path(v2det, layout):
    cam = 30
    v2det.configure_camera(cam, 1920, 1080, workload.camera_config(0, 1920, 1080))
    v2det.engine.set_camera_windows(cam, WINDOWS[layout])
    rng = np.random.default_rng(9)
    for fmt in FORMATS:
        frames = [from_rgb(artist_frame(1920, 1080, 2, 1), fmt), random_frame(rng, 1920, 1080, fmt)]
        for f in frames:
            want = run(v2det, [cv2_rgb(f, fmt)], [cam], fuse_filters=True)
            assert same(run(v2det, [f], [cam], fmt, fuse_filters=True), want), (layout, fmt)
            bufs, ptrs = to_device([f], offset=4)
            assert same(run(v2det, ptrs, [cam], fmt, fuse_filters=True, frames_on_device=True), want), (layout, fmt)
    v2det.engine.set_camera_windows(cam, [])


def test_graph_replay_across_formats():
    """one engine and one graph key for batches in every format: each result equals an engine without graphs"""
    blob = workload.v2_coco_model().to_blob()
    os.environ['WB_NO_GRAPH'] = '1'
    try:
        plain = B200ObjectDetector(None, device=0, max_batch=2, precision=2, model_blob=blob)
    finally:
        os.environ.pop('WB_NO_GRAPH', None)
    sizes = [(640, 480), (1280, 720)]
    rng = np.random.default_rng(10)
    with plain, B200ObjectDetector(None, device=0, max_batch=2, precision=2, model_blob=blob) as det:
        for d in (det, plain):
            for cam, (w, h) in enumerate(sizes):
                d.configure_camera(cam, w, h, workload.camera_config(cam, w, h))
        for rnd in range(2):
            for fmt in ('rgb24', 'yuyv422', 'yuv420p', 'uyvy422', 'nv12'):
                if fmt == 'rgb24':
                    frames = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in sizes]
                elif fmt in FORMATS:
                    frames = [random_frame(rng, w, h, fmt) for w, h in sizes]
                else:
                    frames = [yuv420.random_frame(rng, w, h) for w, h in sizes]
                bufs, ptrs = to_device(frames) if rnd else (None, frames)
                kw = dict(fuse_filters=True, pixel_format=fmt, frames_on_device=bool(rnd))
                want = run(plain, ptrs, [0, 1], **kw)
                assert same(run(det, ptrs, [0, 1], **kw), want), (rnd, fmt)
                assert same(submit_collect(det, 3, ptrs, [0, 1], **kw), want), (rnd, fmt, 'slot 3')


# ----------------------------------------------------------------------------------------------------- effects
def test_effects_equal_rgb_path(fx):
    """blend, draw, contours and all three fused, from 4:2:2 input to every output format, host and device, on a
    batch of sizes with widths = 2 mod 4 (a last thread with one macropixel)"""
    import torch

    from watsor_b200.output.effects import WB_FX_BLEND, WB_FX_CONTOURS, WB_FX_DRAW, WB_FX_ON_DEVICE, contour_bits
    rng = np.random.default_rng(11)
    sizes = [(642, 480), (98, 50), (1920, 1080), (640, 480)]
    cams, rows, alphas = [], [], []
    for i, (w, h) in enumerate(sizes):
        alpha = random_alpha(rng, w, h, 2) if i % 2 == 0 else None
        cams.append(fx.add_camera(w, h, alpha, None if alpha is None else contour_bits(alpha)))
        alphas.append(alpha)
        rows.append(random_rows(rng, w, h, 8, n_zones=2 if alpha is not None else 0))
    shapes = {'rgb24': lambda w, h: (h, w, 3), 'yuv420p': lambda w, h: (h * 3 // 2, w)}
    shapes['nv12'] = shapes['yuv420p']
    all_flags = {'blend': WB_FX_BLEND, 'draw': WB_FX_DRAW, 'contours': WB_FX_DRAW | WB_FX_CONTOURS,
                 'fused': WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS}
    for fmt in FORMATS:
        frames = [from_rgb(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), fmt) if k % 2 else
                  random_frame(rng, w, h, fmt) for k, (w, h) in enumerate(sizes)]
        rgb = [cv2_rgb(f, fmt) for f in frames]
        d_in, p_in = to_device(frames, offset=2)
        for name, flags in all_flags.items():
            for out_fmt, shape in shapes.items():
                want = [np.zeros(shape(w, h), np.uint8) for w, h in sizes]
                fx.render(rgb, want, cams, rows, flags, output_format=out_fmt)
                if out_fmt == 'rgb24' and name == 'fused':
                    for k in range(len(sizes)):
                        assert np.array_equal(want[k], oracle_fx.effect_chain(rgb[k], rows[k], alphas[k])), sizes[k]
                got = [np.zeros_like(x) for x in want]
                fx.render(frames, got, cams, rows, flags, pixel_format=fmt, output_format=out_fmt)
                for k in range(len(sizes)):
                    assert np.array_equal(got[k], want[k]), (fmt, name, out_fmt, sizes[k], 'host')
                d_out = [torch.zeros(x.shape, dtype=torch.uint8, device='cuda') for x in want]
                torch.cuda.synchronize()
                fx.render(p_in, [t.data_ptr() for t in d_out], cams, rows, flags | WB_FX_ON_DEVICE,
                          pixel_format=fmt, output_format=out_fmt)
                for k in range(len(sizes)):
                    assert np.array_equal(d_out[k].cpu().numpy(), want[k]), (fmt, name, out_fmt, sizes[k], 'device')


# ------------------------------------------------------------------------------------------------------ errors
def test_errors(v2det, fx):
    from watsor_b200.output.effects import WB_FX_NV12, WB_FX_UYVY422, WB_FX_YUYV422
    engine = v2det.engine
    rng = np.random.default_rng(0)
    v2det.configure_camera(40, 302, 101, None)          # an odd height is fine for 4:2:2
    v2det.configure_camera(41, 301, 100, None)
    frame = random_frame(rng, 302, 101, 'yuyv422')
    raw = [frame.ctypes.data]
    for flags, names in ((_lib.WB_F_YUYV422 | _lib.WB_F_UYVY422, 'WB_F_YUYV422 and WB_F_UYVY422'),
                         (_lib.WB_F_NV12 | _lib.WB_F_YUYV422, 'WB_F_NV12 and WB_F_YUYV422'),
                         (_lib.WB_F_YUV420P | _lib.WB_F_NV12 | _lib.WB_F_UYVY422,
                          'WB_F_YUV420P, WB_F_NV12 and WB_F_UYVY422')):
        with pytest.raises(_lib.WatsorB200Error, match=names + ' are mutually exclusive'):
            engine.detect(raw, [40], new_rows(1), flags=flags)
    # odd width: the Python check, then the library's own (a raw address bypasses the Python one)
    with pytest.raises(ValueError, match='even width'):
        v2det.detect_batch([np.zeros((100, 301, 2), np.uint8)], [41], new_rows(1), pixel_format='uyvy422')
    with pytest.raises(_lib.WatsorB200Error, match='4:2:2 frames need an even width'):
        engine.detect(raw, [41], new_rows(1), flags=_lib.WB_F_YUYV422)
    # odd window x or width (windows that RGB24 frames may have)
    v2det.configure_camera(42, 640, 480, None)
    f42 = random_frame(rng, 640, 480, 'uyvy422')
    for wins in ([(0, 0, 640, 480), (1, 0, 320, 240)], [(0, 1, 321, 240)]):
        engine.set_camera_windows(42, wins)
        with pytest.raises(ValueError, match='even window x and width'):
            v2det.detect_batch([f42], [42], new_rows(1), pixel_format='uyvy422')
        with pytest.raises(_lib.WatsorB200Error, match='4:2:2 frames need an even window x and width'):
            engine.detect([f42.ctypes.data], [42], new_rows(1), flags=_lib.WB_F_UYVY422)
    engine.set_camera_windows(42, [])
    # wrong shapes
    for bad in (cv2_rgb(frame, 'yuyv422'), frame.reshape(101, 604), frame[:100]):
        with pytest.raises(ValueError, match='shape'):
            v2det.detect_batch([np.ascontiguousarray(bad)], [40], new_rows(1), pixel_format='yuyv422')
    with pytest.raises(ValueError, match='shape'):
        v2det.detect_batch([frame], [40], new_rows(1))                     # a 4:2:2 frame passed as RGB24
    # the context is still usable
    assert same(run(v2det, [frame], [40], 'yuyv422'), run(v2det, [cv2_rgb(frame, 'yuyv422')], [40]))
    # effects
    cam = fx.add_camera(302, 101)
    odd = fx.add_camera(301, 100)
    rows = new_rows()[0]
    out = np.zeros((101, 302, 3), np.uint8)
    with pytest.raises(_lib.WatsorB200Error, match='in place'):
        fx.render([frame], [frame], [cam], [rows], 0, pixel_format='yuyv422')
    with pytest.raises(_lib.WatsorB200Error, match='WB_FX_YUYV422 and WB_FX_UYVY422 are mutually exclusive'):
        fx.render(raw, [out.ctypes.data], [cam], [rows], WB_FX_YUYV422 | WB_FX_UYVY422)
    with pytest.raises(_lib.WatsorB200Error, match='WB_FX_NV12 and WB_FX_UYVY422 are mutually exclusive'):
        fx.render(raw, [out.ctypes.data], [cam], [rows], WB_FX_NV12 | WB_FX_UYVY422)
    with pytest.raises(_lib.WatsorB200Error, match='4:2:2 frames need an even width'):
        fx.render(raw, [out.ctypes.data], [odd], [rows], WB_FX_YUYV422)
    with pytest.raises(ValueError, match='even width'):
        fx.render([np.zeros((100, 301, 2), np.uint8)], [np.zeros((100, 301, 3), np.uint8)], [odd], [rows], 0,
                  pixel_format='yuyv422')
    with pytest.raises(ValueError, match='even width and height'):                 # 4:2:0 output of an odd height
        fx.render([frame], [np.zeros((151, 302), np.uint8)], [cam], [rows], 0, pixel_format='yuyv422',
                  output_format='nv12')
    with pytest.raises(ValueError, match='output_format must be one of'):          # 4:2:2 is an input format only
        fx.render([cv2_rgb(frame, 'yuyv422')], [frame], [cam], [rows], 0, output_format='yuyv422')
    with pytest.raises(ValueError, match='shape'):
        fx.render([cv2_rgb(frame, 'yuyv422')], [out], [cam], [rows], 0, pixel_format='yuyv422')
    fx.render([frame], [out], [cam], [rows], 0, pixel_format='yuyv422')
    assert np.array_equal(out, cv2_rgb(frame, 'yuyv422'))
