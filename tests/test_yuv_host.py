"""4:2:0 input, host side (no GPU): the conversion the kernels implement (tests/yuv_emulation.py) equals
cv2.cvtColor on every (Y, U, V) triple in both layouts, and the Python layer's frame checks."""
import numpy as np
import pytest

from tests.yuv_emulation import all_triples, cv2_rgb, from_rgb, i420_to_nv12, random_frame, to_rgb
from watsor_b200.engine import check_frames, frame_shape


@pytest.mark.parametrize('fmt', ['yuv420p', 'nv12'])
def test_all_triples_equal_cvtcolor(fmt):
    frame = all_triples(fmt)
    flat = all_triples('yuv420p').reshape(-1)
    y = flat[:4096 * 4096].reshape(4096, 4096)
    pair = flat[4096 * 4096:].reshape(2, -1).astype(np.int64)
    # the frame does hold each triple once
    blocks = y.reshape(2048, 2, 2048, 2).transpose(0, 2, 1, 3).reshape(-1, 4).astype(np.int64)
    keys = (((pair[0] << 8) | pair[1])[:, None] << 8) | blocks
    assert np.array_equal(np.sort(keys.reshape(-1)), np.arange(1 << 24))
    assert np.array_equal(to_rgb(frame, 4096, 4096, fmt), cv2_rgb(frame, fmt))


@pytest.mark.parametrize('fmt', ['yuv420p', 'nv12'])
@pytest.mark.parametrize('size', [(2, 2), (302, 226), (640, 480)])
def test_frames_equal_cvtcolor(fmt, size):
    w, h = size
    rng = np.random.default_rng(w)
    for frame in (random_frame(rng, w, h), from_rgb(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), fmt)):
        assert np.array_equal(to_rgb(frame, w, h, fmt), cv2_rgb(frame, fmt))


def test_nv12_interleaves_the_chroma():
    i420 = random_frame(np.random.default_rng(1), 8, 4)
    nv12 = i420_to_nv12(i420, 8, 4)
    flat = i420.reshape(-1)
    assert np.array_equal(nv12[:4], i420[:4])
    assert list(nv12[4:].reshape(-1)) == [b for uv in zip(flat[32:40], flat[40:48]) for b in uv]


def test_frame_shapes():
    assert frame_shape('rgb24', 640, 480) == (480, 640, 3)
    assert frame_shape('yuv420p', 640, 480) == (720, 640)
    assert frame_shape('nv12', 1920, 1080) == (1620, 1920)
    assert frame_shape('rgb24', 301, 101) == (101, 301, 3)
    for w, h in ((301, 100), (300, 101)):
        for fmt in ('yuv420p', 'nv12'):
            with pytest.raises(ValueError, match='even width and height'):
                frame_shape(fmt, w, h)
    with pytest.raises(ValueError, match='pixel_format must be one of'):
        frame_shape('bgr24', 640, 480)


def test_check_frames():
    sizes = [(640, 480), (320, 240)]
    ok = [np.zeros((720, 640), np.uint8), np.zeros((360, 320), np.uint8)]
    check_frames(ok, sizes, 'nv12')
    check_frames(ok, sizes, 'yuv420p')
    check_frames([np.zeros((480, 640, 3), np.uint8)], sizes[:1], 'rgb24')
    check_frames([0x7f0000000000, 0x7f0000100000], sizes, 'nv12')   # raw addresses: the caller's responsibility
    check_frames([np.zeros(3, np.uint8)], [None], 'nv12')           # unknown camera: the library reports it
    bad = [
        ([np.zeros((480, 640, 3), np.uint8)], 'nv12'),               # an RGB frame passed as 4:2:0
        ([np.zeros((720, 640), np.uint8)], 'rgb24'),                 # and the other way round
        ([np.zeros((480, 640), np.uint8)], 'yuv420p'),               # luma only
        ([np.zeros((720, 640), np.int16)], 'yuv420p'),               # not bytes
        ([np.zeros((720, 1280), np.uint8)[:, ::2]], 'nv12'),         # not contiguous
    ]
    for frames, fmt in bad:
        with pytest.raises(ValueError, match='frame 0'):
            check_frames(frames, sizes[:1], fmt)
    with pytest.raises(ValueError, match='even width and height'):
        check_frames([np.zeros((150, 301), np.uint8)], [(301, 100)], 'yuv420p')
    with pytest.raises(ValueError, match='pixel_format'):
        check_frames(ok, sizes, 'i420')
