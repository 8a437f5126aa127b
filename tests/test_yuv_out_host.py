"""The RGB24 -> 4:2:0 restatement of the effects pass's output (tests/yuv_out_emulation.py) against OpenCV, on every
(R, G, B) triple and on whole frames, and the frame shapes the Python side checks outputs against."""
import cv2
import numpy as np
import pytest

from tests.yuv_emulation import i420_to_nv12
from tests.yuv_out_emulation import N_TRIPLES, rgb_to_yuv, to_yuv420, top_left_frames, triple
from watsor_b200.engine import check_frames, frame_shape


def test_luma_equals_cvtcolor_on_every_triple():
    r, g, b = triple(np.arange(N_TRIPLES))
    rgb = np.stack([r, g, b], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
    want = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)[:4096]
    assert np.array_equal(rgb_to_yuv(r, g, b)[0].reshape(4096, 4096), want)


def test_every_triple_as_top_left_pixel_equals_cvtcolor():
    """U and V of a block come from its top-left pixel alone: the other three pixels are random"""
    rng = np.random.default_rng(1)
    for k, rgb in enumerate(top_left_frames(rng)):
        want = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
        got = to_yuv420(rgb, 'yuv420p')
        assert np.array_equal(got, want), (k, int((got != want).sum()))


@pytest.mark.parametrize('size', [(2, 2), (2, 44), (98, 50), (640, 480), (1920, 1080)])
def test_frames_equal_cvtcolor(size):
    w, h = size
    rng = np.random.default_rng(w * h)
    rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    rgb.reshape(-1, 3)[:4] = [(0, 0, 0), (255, 255, 255), (255, 0, 0), (0, 0, 255)][:min(4, w * h)]
    i420 = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
    assert np.array_equal(to_yuv420(rgb, 'yuv420p'), i420)
    nv12 = to_yuv420(rgb, 'nv12')
    assert np.array_equal(nv12, i420_to_nv12(i420, w, h))
    # NV12: the same luma, then (U, V) pairs
    q = (w // 2) * (h // 2)
    assert np.array_equal(nv12[:h], i420[:h])
    assert np.array_equal(nv12[h:].reshape(-1)[0::2], i420[h:].reshape(-1)[:q])
    assert np.array_equal(nv12[h:].reshape(-1)[1::2], i420[h:].reshape(-1)[q:])


@pytest.mark.parametrize('fmt', ['yuv420p', 'nv12'])
def test_output_frame_shapes(fmt):
    for w, h in ((98, 50), (642, 480), (1920, 1080)):
        out = np.zeros(frame_shape(fmt, w, h), np.uint8)
        assert out.nbytes == w * h * 3 // 2
        check_frames([out], [(w, h)], fmt)
        with pytest.raises(ValueError, match='shape'):
            check_frames([np.zeros((h, w, 3), np.uint8)], [(w, h)], fmt)
    with pytest.raises(ValueError, match='even width and height'):
        frame_shape(fmt, 97, 50)
