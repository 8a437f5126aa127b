"""Packed 4:2:2 input (YUYV, UYVY), host side (no GPU): where the kernels find each pixel's Y, U and V, with the
conversion arithmetic, equals cv2.cvtColor on every (Y, U, V) triple in both layouts, and the Python layer's frame and
window checks."""
import numpy as np
import pytest

from tests import yuv_emulation as yuv420
from tests.yuv422_emulation import FORMATS, all_triples, cv2_rgb, from_i420, from_rgb, pack, random_frame, to_rgb
from watsor_b200.engine import PIXEL_FORMATS, check_frames, frame_shape
from watsor_b200.windows import check_windows, grid_windows


@pytest.mark.parametrize('side', [0, 1], ids=['left', 'right'])
@pytest.mark.parametrize('fmt', FORMATS)
def test_all_triples_equal_cvtcolor(fmt, side):
    frame = all_triples(fmt, side)
    # the frame does hold each triple once, on the chosen pixel of its pair
    other = all_triples('uyvy422' if fmt == 'yuyv422' else 'yuyv422', side)
    yuyv = frame if fmt == 'yuyv422' else other
    mp = yuyv.reshape(-1, 4).astype(np.int64)                              # Y0 U Y1 V
    keys = (mp[:, 2 * side] << 16) | (mp[:, 1] << 8) | mp[:, 3]
    assert np.array_equal(np.sort(keys), np.arange(1 << 24))
    assert np.array_equal(to_rgb(frame, fmt), cv2_rgb(frame, fmt))


def test_layouts_place_the_samples():
    Y = np.array([[10, 11, 12, 13]], np.uint8)
    U, V = np.array([[20, 21]], np.uint8), np.array([[30, 31]], np.uint8)
    assert list(pack(Y, U, V, 'yuyv422').reshape(-1)) == [10, 20, 11, 30, 12, 21, 13, 31]
    assert list(pack(Y, U, V, 'uyvy422').reshape(-1)) == [20, 10, 30, 11, 21, 12, 31, 13]


@pytest.mark.parametrize('fmt', FORMATS)
@pytest.mark.parametrize('size', [(2, 1), (2, 3), (302, 225), (640, 480)])
def test_frames_equal_cvtcolor(fmt, size):
    w, h = size
    rng = np.random.default_rng(w + h)
    for frame in (random_frame(rng, w, h, fmt), from_rgb(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), fmt)):
        assert np.array_equal(to_rgb(frame, fmt), cv2_rgb(frame, fmt))


@pytest.mark.parametrize('fmt', FORMATS)
def test_from_i420_keeps_the_pixels(fmt):
    i420 = yuv420.random_frame(np.random.default_rng(2), 64, 48)
    assert np.array_equal(cv2_rgb(from_i420(i420, fmt), fmt), yuv420.cv2_rgb(i420, 'yuv420p'))


def test_frame_shapes():
    for fmt in FORMATS:
        assert frame_shape(fmt, 640, 480) == (480, 640, 2)
        assert frame_shape(fmt, 1920, 1081) == (1081, 1920, 2)          # any height
        assert frame_shape(fmt, 2, 1) == (1, 2, 2)
        with pytest.raises(ValueError, match='even width'):
            frame_shape(fmt, 301, 100)
    with pytest.raises(ValueError, match='pixel_format must be one of') as e:
        frame_shape('yvyu422', 640, 480)
    for name in ('rgb24', 'yuv420p', 'nv12', 'yuyv422', 'uyvy422'):
        assert name in str(e.value)
    assert set(PIXEL_FORMATS) == {'rgb24', 'yuv420p', 'nv12', 'yuyv422', 'uyvy422'}


@pytest.mark.parametrize('fmt', FORMATS)
def test_check_frames(fmt):
    sizes = [(640, 480), (302, 225)]
    ok = [np.zeros((480, 640, 2), np.uint8), np.zeros((225, 302, 2), np.uint8)]
    check_frames(ok, sizes, fmt)
    check_frames([0x7f0000000000, 0x7f0000100000], sizes, fmt)   # raw addresses: the caller's responsibility
    check_frames([np.zeros(3, np.uint8)], [None], fmt)           # unknown camera: the library reports it
    bad = [
        np.zeros((480, 640, 3), np.uint8),                       # an RGB frame passed as 4:2:2
        np.zeros((720, 640), np.uint8),                          # a 4:2:0 frame
        np.zeros((480, 1280), np.uint8),                         # the right bytes, not (H, W, 2)
        np.zeros((480, 640, 2), np.int16),                       # not bytes
        np.zeros((480, 1280, 2), np.uint8)[:, ::2],              # not contiguous
        np.zeros((481, 640, 2), np.uint8),                       # another height
    ]
    for frame in bad:
        with pytest.raises(ValueError, match='frame 0'):
            check_frames([frame], sizes[:1], fmt)
    with pytest.raises(ValueError, match='even width'):
        check_frames([np.zeros((100, 301, 2), np.uint8)], [(301, 100)], fmt)
    # a 4:2:2 frame is not an RGB frame either
    with pytest.raises(ValueError, match='frame 0'):
        check_frames([ok[0]], sizes[:1], 'rgb24')
    with pytest.raises(ValueError, match='pixel_format'):
        check_frames(ok, sizes, 'yuyv')


@pytest.mark.parametrize('fmt', FORMATS)
def test_window_checks(fmt):
    w, h = 1920, 1080
    good = [(0, 0, w, h), (2, 1, 640, 359), (1280, 721, 640, 359), (0, 3, 2, 1)]   # odd y and height are fine
    assert check_windows(good, w, h, fmt) == good
    assert check_windows(grid_windows(w, h, 2, 2), w, h, fmt)
    assert check_windows(grid_windows(1918, 1081, 3, 3), 1918, 1081, fmt)
    for win in ((1, 0, 640, 360), (0, 0, 641, 360), (1919, 0, 1, 1)):
        with pytest.raises(ValueError, match='even window x and width'):
            check_windows([win], w, h, fmt)
        check_windows([win], w, h, 'rgb24')                     # the same windows are fine for RGB24
    with pytest.raises(ValueError, match='inside'):
        check_windows([(2, 0, 1920, 1080)], w, h, fmt)
