"""The effects pass writing 4:2:0 output (WB_FX_OUT_YUV420P / WB_FX_OUT_NV12) for an encoder.  The kernel converts the
frame it rendered as cv2.cvtColor(COLOR_RGB2YUV_I420) does, so every output must equal, byte for byte, that conversion
of the same call's RGB24 output and of the reference's effect chain (oracle/effects.py)."""
import types

import numpy as np
import pytest

from oracle import effects as oracle_fx
from tests.conftest import PORCH_CONFIG, load_golden_frame
from tests.fx_cases import random_alpha, random_rows
from tests.gpu_util import new_rows
from tests.yuv_emulation import cv2_rgb, from_rgb, i420_to_nv12
from tests.yuv_out_emulation import to_yuv420, top_left_frames
from watsor_b200 import _lib

pytestmark = pytest.mark.gpu
IN_FORMATS = ['rgb24', 'yuv420p', 'nv12']
OUT_FORMATS = ['yuv420p', 'nv12']


@pytest.fixture(scope='module')
def fx():
    from watsor_b200.output.effects import EffectsEngine
    with EffectsEngine(0) as e:
        yield e


def effect_flags():
    from watsor_b200.output.effects import WB_FX_BLEND, WB_FX_CONTOURS, WB_FX_DRAW
    return WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS


def frame_in(rgb, fmt):
    """the camera frame in `fmt`, and the RGB24 frame the effects see"""
    if fmt == 'rgb24':
        return rgb, rgb
    frame = from_rgb(rgb, fmt)
    return frame, cv2_rgb(frame, fmt)


def out_like(fmt, w, h):
    return np.zeros((h, w, 3) if fmt == 'rgb24' else (h * 3 // 2, w), np.uint8)


@pytest.fixture(scope='module')
def every_triple():
    """16 frames of 2048 x 2048 holding every (R, G, B) triple as a 2x2 block's top-left pixel, and their I420
    restatement (made once: NV12 is the same bytes interleaved)"""
    frames = top_left_frames(np.random.default_rng(5))
    return frames, [to_yuv420(f, 'yuv420p') for f in frames]


@pytest.mark.parametrize('out_fmt', OUT_FORMATS)
def test_exhaustive_conversion(fx, every_triple, out_fmt):
    """every (R, G, B) triple as a 2x2 block's top-left pixel, through k_fx_render without effects"""
    frames, i420 = every_triple
    side = frames[0].shape[0]
    cam = fx.add_camera(side, side)
    outs = [out_like(out_fmt, side, side) for _ in frames]
    fx.render(frames, outs, [cam] * len(frames), [new_rows()[0]] * len(frames), 0, output_format=out_fmt)
    for k, (want, out) in enumerate(zip(i420, outs)):
        if out_fmt == 'nv12':
            want = i420_to_nv12(want, side, side)
        assert np.array_equal(out, want), (k, int((out != want).sum()))


def test_effects_equal_cvtcolor_of_rgb_output(fx):
    import torch

    from watsor_b200.filter.mask import get_alpha_channel
    from watsor_b200.output.effects import WB_FX_ON_DEVICE, contour_bits
    w, h = 640, 480
    alpha, _ = get_alpha_channel(PORCH_CONFIG['mask'], w, h)
    cam = fx.add_camera(w, h, alpha, contour_bits(alpha))
    rng = np.random.default_rng(6)
    rows = random_rows(rng, w, h, 12, n_zones=2)
    flags = effect_flags()
    for rgb0 in (load_golden_frame('artist_640x480_c0_f0'), rng.integers(0, 256, (h, w, 3), dtype=np.uint8)):
        for in_fmt in IN_FORMATS:
            frame, rgb = frame_in(rgb0, in_fmt)
            rgb_out = out_like('rgb24', w, h)
            fx.render([frame], [rgb_out], [cam], [rows], flags, pixel_format=in_fmt)
            assert np.array_equal(rgb_out, oracle_fx.effect_chain(rgb, rows, alpha)), in_fmt
            for out_fmt in OUT_FORMATS:
                want = from_rgb(rgb_out, out_fmt)
                got = out_like(out_fmt, w, h)
                fx.render([frame], [got], [cam], [rows], flags, pixel_format=in_fmt, output_format=out_fmt)
                assert np.array_equal(got, want), (in_fmt, out_fmt)
                # the same call on device pointers
                d_in = torch.from_numpy(frame).cuda()
                d_out = torch.zeros(got.shape, dtype=torch.uint8, device='cuda')
                torch.cuda.synchronize()
                fx.render([d_in.data_ptr()], [d_out.data_ptr()], [cam], [rows], flags | WB_FX_ON_DEVICE,
                          pixel_format=in_fmt, output_format=out_fmt)
                assert np.array_equal(d_out.cpu().numpy(), want), (in_fmt, out_fmt, 'device')


@pytest.mark.parametrize('out_fmt', OUT_FORMATS)
def test_batch_of_sizes_and_unaligned_device_outputs(fx, out_fmt):
    """widths = 2 mod 4 (a last thread with one chroma sample) and output pointers 1 and 2 bytes past alignment
    (byte and pair stores)"""
    import torch

    from watsor_b200.output.effects import WB_FX_ON_DEVICE, contour_bits
    rng = np.random.default_rng(7)
    sizes = [(642, 480), (98, 50), (1920, 1080), (640, 480)]
    cams, imgs, rows, alphas = [], [], [], []
    for i, (w, h) in enumerate(sizes):
        alpha = random_alpha(rng, w, h, 2) if i % 2 == 0 else None
        cams.append(fx.add_camera(w, h, alpha, None if alpha is None else contour_bits(alpha)))
        alphas.append(alpha)
        imgs.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        rows.append(random_rows(rng, w, h, 8, n_zones=2 if alpha is not None else 0))
    flags = effect_flags()
    rgb_outs = [np.zeros_like(i) for i in imgs]
    fx.render(imgs, rgb_outs, cams, rows, flags)
    for k in range(len(sizes)):
        assert np.array_equal(rgb_outs[k], oracle_fx.effect_chain(imgs[k], rows[k], alphas[k])), sizes[k]
    wants = [from_rgb(o, out_fmt) for o in rgb_outs]
    outs = [out_like(out_fmt, w, h) for w, h in sizes]
    fx.render(imgs, outs, cams, rows, flags, output_format=out_fmt)
    for k in range(len(sizes)):
        assert np.array_equal(outs[k], wants[k]), (sizes[k], 'host')
    d_in = [torch.from_numpy(i).cuda() for i in imgs]
    for off in (0, 1, 2):
        bufs = [torch.full((o.size + 4,), 7, dtype=torch.uint8, device='cuda') for o in outs]
        torch.cuda.synchronize()
        fx.render([t.data_ptr() for t in d_in], [b.data_ptr() + off for b in bufs], cams, rows, flags | WB_FX_ON_DEVICE,
                  output_format=out_fmt)
        for k, b in enumerate(bufs):
            got = b.cpu().numpy()
            assert np.array_equal(got[off:off + wants[k].size].reshape(wants[k].shape), wants[k]), (sizes[k], off)
            assert (got[:off] == 7).all() and (got[off + wants[k].size:] == 7).all(), (sizes[k], off, 'outside')


@pytest.mark.parametrize('out_fmt', OUT_FORMATS)
def test_fused_effects_output_format(fx, out_fmt):
    from watsor_b200.filter.mask import get_alpha_channel
    from watsor_b200.output.effects import FusedEffects
    w, h = 640, 480
    alpha, _ = get_alpha_channel(PORCH_CONFIG['mask'], w, h)
    effects = FusedEffects(PORCH_CONFIG, engine=fx, output_format=out_fmt)
    rng = np.random.default_rng(8)
    rows = random_rows(rng, w, h, 12, n_zones=2)
    img = load_golden_frame('artist_640x480_c3_f7')
    out = out_like(out_fmt, w, h)
    header = types.SimpleNamespace(detections=rows)
    effects.apply(img, out, img.shape, header, header)
    want = from_rgb(oracle_fx.effect_chain(img, rows, alpha), out_fmt)
    assert np.array_equal(out, want)
    with pytest.raises(ValueError, match='even width and height'):
        FusedEffects(dict(PORCH_CONFIG, width=641), engine=fx, output_format=out_fmt)


def test_errors(fx):
    from watsor_b200.output.effects import WB_FX_OUT_NV12, WB_FX_OUT_YUV420P
    cam = fx.add_camera(302, 100)
    odd_w, odd_h = fx.add_camera(301, 100), fx.add_camera(302, 101)
    rows = new_rows()[0]
    img = np.random.default_rng(9).integers(0, 256, (100, 302, 3), dtype=np.uint8)
    out = out_like('nv12', 302, 100)
    with pytest.raises(_lib.WatsorB200Error, match='WB_FX_OUT_YUV420P and WB_FX_OUT_NV12 are mutually exclusive'):
        fx.render([img.ctypes.data], [out.ctypes.data], [cam], [rows], WB_FX_OUT_YUV420P | WB_FX_OUT_NV12)
    for odd, (w, h) in ((odd_w, (301, 100)), (odd_h, (302, 101))):
        odd_img = np.zeros((h, w, 3), np.uint8)
        with pytest.raises(_lib.WatsorB200Error, match='cam_id %d is %dx%d: 4:2:0 frames need an even' % (odd, w, h)):
            fx.render([odd_img.ctypes.data], [out.ctypes.data], [odd], [rows], WB_FX_OUT_NV12)
        with pytest.raises(ValueError, match='even width and height'):
            fx.render([odd_img], [out], [odd], [rows], 0, output_format='yuv420p')
    with pytest.raises(_lib.WatsorB200Error, match=r'4:2:0 output cannot be rendered in place.*cam_id %d' % cam):
        fx.render([img.ctypes.data], [img.ctypes.data], [cam], [rows], WB_FX_OUT_YUV420P)
    with pytest.raises(ValueError, match='shape'):
        fx.render([img], [np.zeros_like(img)], [cam], [rows], 0, output_format='nv12')
    with pytest.raises(ValueError, match='output_format|pixel_format must be one of'):
        fx.render([img], [out], [cam], [rows], 0, output_format='yuv422p')
    # the context is still usable
    fx.render([img], [out], [cam], [rows], 0, output_format='nv12')
    assert np.array_equal(out, to_yuv420(img, 'nv12'))
