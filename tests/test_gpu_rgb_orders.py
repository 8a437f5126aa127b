"""BGR24, RGBA and BGRA frames through detection and the effects pass, and BGR24 output of the effects pass.  The
kernels read them as the RGB24 frame cv2.cvtColor makes, so every result must equal, byte for byte, the RGB24 path on
cvtColor of the same frame (effects output: cvtColor of the RGB24 call's output)."""
import os
import types

import numpy as np
import pytest

from oracle import effects as oracle_fx
from tests import workload
from tests import yuv_emulation as yuv420
from tests.artist import artist_frame
from tests.conftest import PORCH_CONFIG, load_golden_frame
from tests.fx_cases import random_alpha, random_rows
from tests.gpu_util import new_rows, rows_bytes
from tests.rgb_orders import FORMATS, LAYOUT, cv2_bgr, cv2_rgb, from_rgb, random_frame
from tests.test_gpu_frame_path import _stem_model
from tests.yuv_out_emulation import to_yuv420
from watsor_b200 import _lib
from watsor_b200.detection.b200 import B200ObjectDetector
from watsor_b200.engine import Engine

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


def frame_of(rng, w, h, fmt):
    """random bytes, or a picture the detector finds objects in"""
    if (w + h) % 2:
        return random_frame(rng, w, h, fmt)
    return from_rgb(artist_frame(w, h, w % 4, h % 3), fmt, rng)


# ------------------------------------------------------------------------------------------- the stem on frames
STEM_SIZES = [(1, 1), (2, 1), (3, 2), (300, 300), (601, 599), (640, 479), (1921, 1080), (3840, 2160)]
MIXED = [(641, 479), (1, 1), (3840, 2160), (299, 301)]


@pytest.mark.parametrize('precision', [2, 1], ids=['tf32x3', 'bf16'])
@pytest.mark.parametrize('stem', ['3x3s2_c32_300', '7x7s2_c24_300'], ids=['k_stem_3x3s2_c32', 'k_stem'])
def test_stem_on_frames_equals_rgb_path(stem, precision):
    """wb_backbone_frames stopped after the stem: BGR24 / RGBA / BGRA frames from the host and from device addresses
    at offsets 0 and 1 (word loads and the byte fallback) give the activation of the RGB24 frames cvtColor makes, bit
    for bit"""
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
                for offset in (0, 1):
                    bufs, ptrs = to_device(frames, offset=offset)
                    got = e.backbone_frames(ptrs, cams, stop_layer=0, layer_shape=shape, pixel_format=fmt,
                                            frames_on_device=True)[2]
                    assert np.array_equal(got, want), (stem, fmt, sizes, 'device', offset)


# ------------------------------------------------------------------------------------------------- detection
@pytest.mark.parametrize('fmt', FORMATS)
def test_configs2_rows_equal_rgb_path(v2det, fmt):
    """BASELINE configs[2]: 8 cameras of 640x480, a mask each, fused filters; detect_batch and submit/collect from
    host and device frames"""
    for c in range(8):
        v2det.configure_camera(c, 640, 480, workload.camera_config(c))
    rng = np.random.default_rng(8)
    frames = [from_rgb(artist_frame(640, 480, c, c % 3), fmt, rng) if c % 2 == 0 else random_frame(rng, 640, 480, fmt)
              for c in range(8)]
    cams = list(range(8))
    before = [f.copy() for f in frames]
    want = run(v2det, [cv2_rgb(f, fmt) for f in frames], cams, fuse_filters=True)
    assert same(run(v2det, frames, cams, fmt, fuse_filters=True), want)
    assert all(np.array_equal(a, b) for a, b in zip(before, frames))          # inputs untouched
    assert same(submit_collect(v2det, 1, frames, cams, fuse_filters=True, pixel_format=fmt), want)
    for offset in (0, 1):
        bufs, ptrs = to_device(frames, offset)
        assert same(run(v2det, ptrs, cams, fmt, fuse_filters=True, frames_on_device=True), want), offset
        assert same(submit_collect(v2det, 2, ptrs, cams, fuse_filters=True, frames_on_device=True, pixel_format=fmt),
                    want), offset


def test_real_weights_model(shapes_model):
    with B200ObjectDetector(None, device=0, max_batch=4, precision=2, model_blob=shapes_model.to_blob()) as det:
        det.configure_camera(0, 640, 480, PORCH_CONFIG)
        rgb = [load_golden_frame(n) for n in ('artist_640x480_c0_f0', 'artist_640x480_c0_f1', 'artist_640x480_c3_f7')]
        want = run(det, rgb, [0] * 3, fuse_filters=True)
        for fmt in FORMATS:
            frames = [from_rgb(f, fmt, np.random.default_rng(5)) for f in rgb]
            assert same(run(det, frames, [0] * 3, fmt, fuse_filters=True), want), fmt


# odd x origins and widths, windows touching the right and the bottom border
ODD_WINDOWS = [(0, 0, 1920, 1080), (1, 0, 961, 539), (959, 541, 961, 539), (3, 3, 1917, 1077), (1919, 0, 1, 1080),
               (0, 1079, 1920, 1), (641, 201, 637, 479)]


def test_windows_at_odd_x_equal_rgb_path(v2det):
    cam = 30
    v2det.configure_camera(cam, 1920, 1080, workload.camera_config(0, 1920, 1080))
    v2det.engine.set_camera_windows(cam, ODD_WINDOWS)
    rng = np.random.default_rng(9)
    try:
        for fmt in FORMATS:
            frames = [from_rgb(artist_frame(1920, 1080, 2, 1), fmt, rng), random_frame(rng, 1920, 1080, fmt)]
            for f in frames:
                want = run(v2det, [cv2_rgb(f, fmt)], [cam], fuse_filters=True)
                assert same(run(v2det, [f], [cam], fmt, fuse_filters=True), want), fmt
                for offset in (0, 1):
                    bufs, ptrs = to_device([f], offset=offset)
                    assert same(run(v2det, ptrs, [cam], fmt, fuse_filters=True, frames_on_device=True), want), \
                        (fmt, offset)
    finally:
        v2det.engine.set_camera_windows(cam, [])


def test_graph_replay_across_formats():
    """one engine and one graph key for batches in every byte order and a YUV layout between them: each result equals
    an engine without graphs"""
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
            for fmt in ('rgb24', 'bgra', 'nv12', 'bgr24', 'rgba'):
                cams = [0, 1]
                if fmt == 'nv12':
                    frames = [yuv420.random_frame(rng, w, h) for w, h in sizes]
                else:
                    frames = [frame_of(rng, w, h, fmt) for w, h in sizes]
                bufs, ptrs = to_device(frames, offset=rnd) if rnd else (None, frames)
                kw = dict(fuse_filters=True, pixel_format=fmt, frames_on_device=bool(rnd))
                want = run(plain, ptrs, cams, **kw)
                assert same(run(det, ptrs, cams, **kw), want), (rnd, fmt)
                assert same(submit_collect(det, 3, ptrs, cams, **kw), want), (rnd, fmt, 'slot 3')
                if fmt != 'nv12':
                    assert same(want, run(plain, [cv2_rgb(f, fmt) for f in frames], cams, fuse_filters=True)), fmt


# ----------------------------------------------------------------------------------------------------- effects
OUT_SHAPES = {'rgb24': lambda w, h: (h, w, 3), 'bgr24': lambda w, h: (h, w, 3),
              'yuv420p': lambda w, h: (h * 3 // 2, w), 'nv12': lambda w, h: (h * 3 // 2, w)}


def expected(rgb_out, out_fmt):
    """the output in out_fmt as cv2.cvtColor makes it from the RGB24 call's output"""
    if out_fmt == 'rgb24':
        return rgb_out
    if out_fmt == 'bgr24':
        return cv2_bgr(rgb_out)
    return to_yuv420(rgb_out, out_fmt)


def _cameras(fx, rng, sizes):
    from watsor_b200.output.effects import contour_bits
    cams, rows = [], []
    for i, (w, h) in enumerate(sizes):
        alpha = random_alpha(rng, w, h, 2) if i % 2 == 0 else None
        cams.append(fx.add_camera(w, h, alpha, None if alpha is None else contour_bits(alpha)))
        rows.append(random_rows(rng, w, h, 8, n_zones=2 if alpha is not None else 0))
    return cams, rows


def test_effects_equal_rgb_path(fx):
    """blend, draw, contours and all three fused, from every input layout to every output layout, host and device
    (unaligned buffers); RGB outputs on a batch with widths = 0, 1, 2 and 3 mod 4, 4:2:0 outputs (even sizes only) on
    one with widths = 0 and 2 mod 4"""
    import torch

    from watsor_b200.output.effects import WB_FX_BLEND, WB_FX_CONTOURS, WB_FX_DRAW, WB_FX_ON_DEVICE
    rng = np.random.default_rng(11)
    batches = {'rgb': [(641, 480), (98, 50), (1919, 1080), (640, 480), (303, 61)],
               'yuv': [(642, 480), (98, 50), (1920, 1080), (640, 480)]}
    setups = {k: _cameras(fx, rng, sizes) for k, sizes in batches.items()}
    all_flags = {'copy': 0, 'blend': WB_FX_BLEND, 'draw': WB_FX_DRAW, 'contours': WB_FX_DRAW | WB_FX_CONTOURS,
                 'fused': WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS}
    in_formats = ('rgb24', 'bgr24', 'rgba', 'bgra', 'yuv420p', 'nv12')
    for batch, sizes in batches.items():
        cams, rows = setups[batch]
        for fmt in in_formats:
            if fmt in LAYOUT:
                frames = [frame_of(rng, w, h, fmt) for w, h in sizes]
                rgb = [cv2_rgb(f, fmt) for f in frames]
            elif batch == 'yuv':
                frames = [yuv420.random_frame(rng, w, h) for w, h in sizes]
                rgb = [yuv420.cv2_rgb(f, fmt) for f in frames]
            else:
                continue
            out_formats = ('rgb24', 'bgr24') if batch == 'rgb' else ('bgr24', 'yuv420p', 'nv12')
            if fmt not in FORMATS and batch == 'yuv':
                out_formats = ('bgr24',)                     # the new output from the existing input layouts
            d_in, p_in = to_device(frames, offset=1)
            for name, flags in all_flags.items():
                ref = [np.zeros((h, w, 3), np.uint8) for w, h in sizes]
                fx.render(rgb, ref, cams, rows, flags)
                for out_fmt in out_formats:
                    want = [expected(r, out_fmt) for r in ref]
                    got = [np.zeros(OUT_SHAPES[out_fmt](w, h), np.uint8) for w, h in sizes]
                    fx.render(frames, got, cams, rows, flags, pixel_format=fmt, output_format=out_fmt)
                    for k in range(len(sizes)):
                        assert np.array_equal(got[k], want[k]), (fmt, name, out_fmt, sizes[k], 'host')
                    d_out = [torch.zeros(x.size + 16, dtype=torch.uint8, device='cuda') for x in want]
                    torch.cuda.synchronize()
                    fx.render(p_in, [t.data_ptr() + 3 for t in d_out], cams, rows, flags | WB_FX_ON_DEVICE,
                              pixel_format=fmt, output_format=out_fmt)
                    for k in range(len(sizes)):
                        dev = d_out[k][3:3 + want[k].size].cpu().numpy().reshape(want[k].shape)
                        assert np.array_equal(dev, want[k]), (fmt, name, out_fmt, sizes[k], 'device')


def test_effects_in_place_rgb24_bgr24(fx):
    """bgr24 -> rgb24, rgb24 -> bgr24 and bgr24 -> bgr24 with images_out = images_in, host and device (aligned and
    not): the frame becomes the out-of-place result"""
    import torch

    from watsor_b200.output.effects import WB_FX_BLEND, WB_FX_DRAW, WB_FX_ON_DEVICE
    rng = np.random.default_rng(13)
    sizes = [(641, 480), (98, 50), (1280, 720)]
    cams, rows = _cameras(fx, rng, sizes)
    flags = WB_FX_BLEND | WB_FX_DRAW
    for fmt, out_fmt in (('bgr24', 'rgb24'), ('rgb24', 'bgr24'), ('bgr24', 'bgr24')):
        frames = [frame_of(rng, w, h, fmt) for w, h in sizes]
        want = [np.zeros((h, w, 3), np.uint8) for w, h in sizes]
        fx.render(frames, want, cams, rows, flags, pixel_format=fmt, output_format=out_fmt)
        host = [f.copy() for f in frames]
        fx.render(host, host, cams, rows, flags, pixel_format=fmt, output_format=out_fmt)
        for k in range(len(sizes)):
            assert np.array_equal(host[k], want[k]), (fmt, out_fmt, sizes[k], 'host')
        for offset in (0, 1):
            bufs, ptrs = to_device(frames, offset)
            fx.render(ptrs, ptrs, cams, rows, flags | WB_FX_ON_DEVICE, pixel_format=fmt, output_format=out_fmt)
            torch.cuda.synchronize()
            for k, f in enumerate(frames):
                dev = bufs[k][offset:offset + f.size].cpu().numpy().reshape(f.shape)
                assert np.array_equal(dev, want[k]), (fmt, out_fmt, sizes[k], 'device', offset)


def test_fused_effects_bgr24_output(fx):
    """FusedEffects(output_format='bgr24'): the reference's effect chain, then COLOR_RGB2BGR, for cv2.imencode; any
    width, since BGR24 has no chroma"""
    from watsor_b200.filter.mask import get_alpha_channel
    from watsor_b200.output.effects import FusedEffects
    rng = np.random.default_rng(14)
    img = load_golden_frame('artist_640x480_c3_f7')
    no_mask = {k: v for k, v in PORCH_CONFIG.items() if k != 'mask'}
    for cfg in (PORCH_CONFIG, dict(no_mask, width=639)):              # blend + contours; copy + draw at an odd width
        w = cfg['width']
        alpha = get_alpha_channel(cfg['mask'], w, 480)[0] if 'mask' in cfg else None
        effects = FusedEffects(cfg, engine=fx, output_format='bgr24')
        rows = random_rows(rng, w, 480, 12, n_zones=2 if alpha is not None else 0)
        frame = np.ascontiguousarray(img[:, :w])
        out = np.zeros((480, w, 3), np.uint8)
        header = types.SimpleNamespace(detections=rows)
        effects.apply(frame, out, frame.shape, header, header)
        assert np.array_equal(out, cv2_bgr(oracle_fx.effect_chain(frame, rows, alpha))), w


# ------------------------------------------------------------------------------------------------------ errors
def test_errors(v2det, fx):
    from watsor_b200.output.effects import (WB_FX_BGR24, WB_FX_BGRA, WB_FX_NV12, WB_FX_OUT_BGR24, WB_FX_OUT_NV12,
                                            WB_FX_OUT_YUV420P, WB_FX_RGBA)
    engine = v2det.engine
    rng = np.random.default_rng(0)
    v2det.configure_camera(40, 301, 101, None)
    frame = random_frame(rng, 301, 101, 'rgba')
    raw = [frame.ctypes.data]
    for flags, names in ((_lib.WB_F_RGBA | _lib.WB_F_BGRA, 'WB_F_RGBA and WB_F_BGRA'),
                         (_lib.WB_F_BGR24 | _lib.WB_F_NV12, 'WB_F_NV12 and WB_F_BGR24'),
                         (_lib.WB_F_YUYV422 | _lib.WB_F_BGR24 | _lib.WB_F_RGBA, 'WB_F_YUYV422, WB_F_BGR24 and WB_F_RGBA')):
        with pytest.raises(_lib.WatsorB200Error, match=names + ' are mutually exclusive'):
            engine.detect(raw, [40], new_rows(1), flags=flags)
    # wrong shapes: (H, W, 3) given as rgba, (H, W, 4) as bgr24 or rgb24, another size
    for bad, fmt in ((cv2_rgb(frame, 'rgba'), 'rgba'), (cv2_rgb(frame, 'rgba'), 'bgra'), (frame, 'bgr24'),
                     (frame, 'rgb24'), (frame[:100], 'rgba'), (frame.reshape(101, 301 * 4), 'bgra')):
        with pytest.raises(ValueError, match='shape'):
            v2det.detect_batch([np.ascontiguousarray(bad)], [40], new_rows(1), pixel_format=fmt)
    with pytest.raises(ValueError, match='pixel_format must be one of'):
        v2det.detect_batch([frame], [40], new_rows(1), pixel_format='argb')
    # the context is still usable
    assert same(run(v2det, [frame], [40], 'rgba'), run(v2det, [cv2_rgb(frame, 'rgba')], [40]))
    # effects
    cam = fx.add_camera(301, 101)
    even = fx.add_camera(302, 100)
    rows = new_rows()[0]
    out = np.zeros((101, 301, 3), np.uint8)
    with pytest.raises(_lib.WatsorB200Error, match='WB_FX_RGBA and WB_FX_BGRA are mutually exclusive'):
        fx.render(raw, [out.ctypes.data], [cam], [rows], WB_FX_RGBA | WB_FX_BGRA)
    with pytest.raises(_lib.WatsorB200Error, match='WB_FX_NV12 and WB_FX_BGR24 are mutually exclusive'):
        fx.render(raw, [out.ctypes.data], [cam], [rows], WB_FX_NV12 | WB_FX_BGR24)
    with pytest.raises(_lib.WatsorB200Error, match='WB_FX_OUT_NV12 and WB_FX_OUT_BGR24 are mutually exclusive'):
        fx.render(raw, [out.ctypes.data], [cam], [rows], WB_FX_OUT_NV12 | WB_FX_OUT_BGR24)
    with pytest.raises(_lib.WatsorB200Error,
                       match='WB_FX_OUT_YUV420P, WB_FX_OUT_NV12 and WB_FX_OUT_BGR24 are mutually exclusive'):
        fx.render(raw, [out.ctypes.data], [cam], [rows], WB_FX_OUT_YUV420P | WB_FX_OUT_NV12 | WB_FX_OUT_BGR24)
    # in place across pixel sizes, and with a YUV side; the message names both formats
    img = random_frame(rng, 302, 100, 'bgra')
    for flags, names in ((WB_FX_BGRA, 'bgra input, rgb24 output'), (WB_FX_RGBA | WB_FX_OUT_BGR24, 'rgba input, bgr24 output'),
                         (WB_FX_BGR24 | WB_FX_OUT_NV12, 'bgr24 input, nv12 output'),
                         (WB_FX_NV12 | WB_FX_OUT_BGR24, 'nv12 input, bgr24 output')):
        with pytest.raises(_lib.WatsorB200Error, match='cannot be rendered in place.*cam_id %d, %s' % (even, names)):
            fx.render([img.ctypes.data], [img.ctypes.data], [even], [rows], flags)
    with pytest.raises(_lib.WatsorB200Error, match='in place'):
        fx.render([img], [img], [even], [rows], 0, pixel_format='bgra')
    with pytest.raises(ValueError, match='output_format must be one of'):          # RGBA is an input format only
        fx.render([cv2_rgb(frame, 'rgba')], [frame], [cam], [rows], 0, output_format='rgba')
    with pytest.raises(ValueError, match='shape'):
        fx.render([cv2_rgb(frame, 'rgba')], [out], [cam], [rows], 0, pixel_format='bgra')
    with pytest.raises(ValueError, match='shape'):
        fx.render([frame], [frame], [cam], [rows], 0, pixel_format='rgba', output_format='bgr24')
    fx.render([frame], [out], [cam], [rows], 0, pixel_format='rgba', output_format='bgr24')
    assert np.array_equal(out, cv2_bgr(cv2_rgb(frame, 'rgba')))
