"""BGR24, RGBA and BGRA frames and BGR24 output, host side (no GPU): the byte permutations the kernels apply equal
cv2.cvtColor, the per-format table of the CUDA header is the one restated here, the Python layer's frame and window
checks take the new shapes, and its flag tables match the C header's."""
import os
import re

import numpy as np
import pytest

from tests.rgb_orders import FORMATS, LAYOUT, cv2_bgr, cv2_rgb, from_rgb, random_frame, to_bgr, to_rgb
from watsor_b200 import _lib
from watsor_b200.engine import FRAME_FORMATS, PIXEL_FORMATS, RGB_ORDERS, check_frames, frame_shape, layout_shape
from watsor_b200.output import effects
from watsor_b200.windows import check_windows, grid_windows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1, 1), (2, 1), (1, 3), (3, 2), (5, 7), (301, 225), (640, 480), (641, 479), (1919, 1081), (1920, 1080)]


def _read(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


@pytest.mark.parametrize('fmt', FORMATS)
@pytest.mark.parametrize('size', SIZES, ids=['%dx%d' % s for s in SIZES])
def test_permutations_equal_cvtcolor(fmt, size):
    w, h = size
    rng = np.random.default_rng(w * 7 + h)
    frame = random_frame(rng, w, h, fmt)
    assert np.array_equal(to_rgb(frame, fmt), cv2_rgb(frame, fmt))
    rgb = random_frame(rng, w, h, 'rgb24')
    assert np.array_equal(to_bgr(rgb), cv2_bgr(rgb))                         # the BGR24 output
    assert np.array_equal(to_rgb(from_rgb(rgb, fmt, rng), fmt), rgb)


def test_alpha_byte_is_not_read():
    rgb = np.random.default_rng(1).integers(0, 256, (7, 9, 3), dtype=np.uint8)
    for fmt in ('rgba', 'bgra'):
        a, b = from_rgb(rgb, fmt, np.random.default_rng(2)), from_rgb(rgb, fmt, np.random.default_rng(3))
        assert not np.array_equal(a, b)
        assert np.array_equal(cv2_rgb(a, fmt), cv2_rgb(b, fmt)) and np.array_equal(to_rgb(a, fmt), rgb)


def test_layout_table_is_the_headers():
    """rgb_layout of csrc/yuv420.cuh holds the same bytes per pixel and R, G, B offsets as LAYOUT"""
    src = _read('watsor_b200', 'csrc', 'yuv420.cuh')
    fmts = {int(v): k.lower() for k, v in re.findall(r'#define WB_FMT_(\w+) (\d+)', src)}
    assert [fmts[i] for i in sorted(fmts)] == ['rgb24', 'yuv420p', 'nv12', 'yuyv422', 'uyvy422', 'bgr24', 'rgba', 'bgra']
    body = re.search(r'RgbLayout rgb_layout\(int fmt\) \{(.*?)\n\}', src, re.S).group(1)
    table = {k.lower(): tuple(int(x) for x in v.split(','))
             for k, v in re.findall(r'fmt == WB_FMT_(\w+)\s*\?\s*RgbLayout\{([\d, ]+)\}', body)}
    table['rgb24'] = tuple(int(x) for x in re.search(r':\s*RgbLayout\{([\d, ]+)\};', body).group(1).split(','))
    assert table == LAYOUT
    names = re.search(r'names\[\] = \{(.*?)\};', src).group(1)
    assert re.findall(r'"(\w+)"', names) == [fmts[i] for i in sorted(fmts)]


def _header_flags():
    return {k: int(v) for k, v in re.findall(r'#define (WB_FX?_\w+) (\d+)u', _read('include', 'watsor_b200.h'))}


def test_flag_tables_match_the_header():
    flags = _header_flags()
    for name in ('WB_F_YUV420P', 'WB_F_NV12', 'WB_F_YUYV422', 'WB_F_UYVY422', 'WB_F_BGR24', 'WB_F_RGBA', 'WB_F_BGRA'):
        assert getattr(_lib, name) == flags[name], name
    assert (flags['WB_F_BGR24'], flags['WB_F_RGBA'], flags['WB_F_BGRA']) == (128, 256, 512)
    for fmt, flag in FRAME_FORMATS.items():
        assert flag == (0 if fmt == 'rgb24' else flags['WB_F_' + fmt.upper()]), fmt
    for fmt, flag in effects._FX_FORMATS.items():
        assert flag == (0 if fmt == 'rgb24' else flags['WB_FX_' + fmt.upper()]), fmt
    for fmt, flag in effects._FX_OUT_FORMATS.items():
        assert flag == (0 if fmt == 'rgb24' else flags['WB_FX_OUT_' + fmt.upper()]), fmt
    for name in ('WB_FX_BGR24', 'WB_FX_RGBA', 'WB_FX_BGRA', 'WB_FX_OUT_BGR24'):
        assert getattr(effects, name) == flags[name] and name in effects.__all__, name
    assert (flags['WB_FX_BGR24'], flags['WB_FX_RGBA'], flags['WB_FX_BGRA'], flags['WB_FX_OUT_BGR24']) == \
        (1024, 2048, 4096, 8192)
    # every flag bit of one call is distinct
    for prefix in ('WB_F_', 'WB_FX_'):
        bits = [v for k, v in flags.items() if k.startswith(prefix) and (prefix == 'WB_FX_' or not k.startswith('WB_FX_'))]
        assert all(b & (b - 1) == 0 for b in bits) and len(set(bits)) == len(bits), prefix


def test_library_tables_name_each_flag_by_its_format():
    """kFrameFormats (wb_api.cu) and the effects' in_formats / out_formats (kernels_fx.cu): flag, format, name"""
    for path, prefixes in ((('watsor_b200', 'csrc', 'wb_api.cu'), ('WB_F_',)),
                           (('watsor_b200', 'csrc', 'kernels_fx.cu'), ('WB_FX_', 'WB_FX_OUT_'))):
        entries = re.findall(r'\{(WB_FX?_\w+), WB_FMT_(\w+), "(\w+)"\}', _read(*path))
        for flag, fmt, name in entries:
            assert flag == name and any(flag == p + fmt for p in prefixes), (path, flag, fmt)
        got = {fmt.lower() for flag, fmt, _ in entries}
        assert {'bgr24', 'rgba', 'bgra'} <= got, path


def test_layout_shapes():
    for fmt, bpp in (('rgb24', 3), ('bgr24', 3), ('rgba', 4), ('bgra', 4)):
        for w, h in SIZES:
            assert layout_shape(fmt, w, h) == (h, w, bpp)                       # any size
    assert set(RGB_ORDERS) == set(FORMATS)
    assert set(FRAME_FORMATS) == set(PIXEL_FORMATS) | set(FORMATS)
    with pytest.raises(ValueError, match='pixel_format must be one of') as e:
        layout_shape('argb', 640, 480)
    for name in FRAME_FORMATS:
        assert name in str(e.value)
    # the RGB24 and YUV layouts: layout_shape is frame_shape, size rules included
    for fmt in PIXEL_FORMATS:
        for w, h in ((640, 480), (1920, 1080), (302, 101)):
            if fmt in ('yuv420p', 'nv12') and h % 2:
                with pytest.raises(ValueError, match='even width and height'):
                    layout_shape(fmt, w, h)
            else:
                assert layout_shape(fmt, w, h) == frame_shape(fmt, w, h)


def test_frame_shape_keeps_its_formats():
    """frame_shape takes the layouts of PIXEL_FORMATS only, as it always has; its refusal of another byte order
    points at layout_shape"""
    for fmt in FORMATS:
        with pytest.raises(ValueError, match='pixel_format must be one of .*layout_shape gives the shape of a ' + fmt):
            frame_shape(fmt, 640, 480)
    with pytest.raises(ValueError, match='pixel_format must be one of') as e:
        frame_shape('argb', 640, 480)
    assert 'layout_shape' not in str(e.value)


@pytest.mark.parametrize('fmt', FORMATS)
def test_check_frames(fmt):
    bpp = LAYOUT[fmt][0]
    sizes = [(640, 480), (301, 225)]
    ok = [np.zeros((480, 640, bpp), np.uint8), np.zeros((225, 301, bpp), np.uint8)]
    check_frames(ok, sizes, fmt)
    check_frames([0x7f0000000000, 0x7f0000100000], sizes, fmt)   # raw addresses: the caller's responsibility
    bad = [
        np.zeros((480, 640, 7 - bpp), np.uint8),                 # the other pixel size: (H, W, 3) given as rgba etc.
        np.zeros((480, 640, 2), np.uint8),                       # a 4:2:2 frame
        np.zeros((720, 640), np.uint8),                          # a 4:2:0 frame
        np.zeros((480, 640 * bpp), np.uint8),                    # the right bytes, not (H, W, bpp)
        np.zeros((480, 640, bpp), np.int16),                     # not bytes
        np.zeros((480, 1280, bpp), np.uint8)[:, ::2],            # not contiguous
        np.zeros((481, 640, bpp), np.uint8),                     # another height
    ]
    for frame in bad:
        with pytest.raises(ValueError, match='frame 0'):
            check_frames([frame], sizes[:1], fmt)
    if bpp == 4:                                                 # a 4-byte frame is not an RGB24 or BGR24 frame
        for other in ('rgb24', 'bgr24'):
            with pytest.raises(ValueError, match='frame 0'):
                check_frames([ok[0]], sizes[:1], other)


@pytest.mark.parametrize('fmt', FORMATS)
def test_window_checks(fmt):
    w, h = 1919, 1081
    odd = [(0, 0, w, h), (1, 0, 641, 360), (3, 5, 1, 1), (1918, 1080, 1, 1), (959, 1, 960, 1079)]
    assert check_windows(odd, w, h, fmt) == odd
    assert check_windows(grid_windows(w, h, 3, 3, align=1), w, h, fmt)
    with pytest.raises(ValueError, match='inside'):
        check_windows([(1, 0, 1919, 1081)], w, h, fmt)
    with pytest.raises(ValueError, match='empty'):
        check_windows([(1, 0, 0, 10)], w, h, fmt)

