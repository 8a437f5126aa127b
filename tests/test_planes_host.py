"""Host side of frames given as planes: the plane geometry (engine.layout_planes), the address and pitch the Python
layer takes from numpy views, CPU tensors and device pairs, the refusals it makes itself, and the C struct
wb_frame_planes against its ctypes mirror."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile
import types

import numpy as np
import pytest

from tests.conftest import ROOT
from watsor_b200 import _lib
from watsor_b200.engine import FRAME_FORMATS, Engine, layout_planes, layout_shape, plane_address


def test_layout_planes():
    assert layout_planes('rgb24', 641, 479) == ((479, 1923),)
    assert layout_planes('bgr24', 5, 3) == ((3, 15),)
    assert layout_planes('rgba', 641, 479) == ((479, 2564),)
    assert layout_planes('bgra', 1, 1) == ((1, 4),)
    assert layout_planes('yuyv422', 642, 479) == ((479, 1284),)
    assert layout_planes('uyvy422', 2, 1) == ((1, 4),)
    assert layout_planes('nv12', 1920, 1080) == ((1080, 1920), (540, 1920))
    assert layout_planes('yuv420p', 1920, 1080) == ((1080, 1920), (540, 960), (540, 960))
    assert layout_planes('yuv420p', 2, 2) == ((2, 2), (1, 1), (1, 1))
    # the planes of a packed frame fill its layout_shape exactly
    for fmt in FRAME_FORMATS:
        for w, h in ((640, 480), (1920, 1080), (2, 2), (642, 478)):
            assert sum(r * b for r, b in layout_planes(fmt, w, h)) == np.prod(layout_shape(fmt, w, h)), (fmt, w, h)
    with pytest.raises(ValueError, match='nv12 frames need an even width and height'):
        layout_planes('nv12', 641, 480)
    with pytest.raises(ValueError, match='yuyv422 frames need an even width'):
        layout_planes('yuyv422', 641, 480)
    with pytest.raises(ValueError, match='pixel_format must be one of'):
        layout_planes('p010', 640, 480)


def test_plane_address_of_numpy_views():
    big = np.zeros((1080, 1920, 3), np.uint8)
    crop = big[100:580, 33:673]                              # a 640x480 window of a 1920x1080 RGB24 frame
    assert plane_address(crop, 480, 1920, False, 'x') == (big.ctypes.data + 100 * 5760 + 33 * 3, 5760)
    assert plane_address(big, 1080, 5760, False, 'x') == (big.ctypes.data, 5760)
    # an AVFrame-style plane: linesize 704 for 640 luma bytes, the row padding outside the view
    buf = np.zeros(480 * 704, np.uint8)
    y = buf.reshape(480, 704)[:, :640]
    assert plane_address(y, 480, 640, False, 'x') == (buf.ctypes.data, 704)
    # NV12 chroma as (h/2, w/2, 2) pairs, one row
    uv = np.zeros((240, 320, 2), np.uint8)
    assert plane_address(uv, 240, 640, False, 'x') == (uv.ctypes.data, 640)
    one = big[7:8, :2]                                       # one row keeps its parent's pitch
    assert plane_address(one, 1, 6, False, 'x') == (big.ctypes.data + 7 * 5760, 5760)
    assert plane_address(np.zeros((1, 1), np.uint8)[:, :1], 1, 1, False, 'x')[1] == 1
    assert plane_address(big[:, :, :], None, None, False, 'x')[1] == 5760


def test_plane_address_of_tensors_and_pairs():
    torch = pytest.importorskip('torch')
    t = torch.zeros((1080, 2048), dtype=torch.uint8)
    view = t[10:490, 64:704]
    assert plane_address(view, 480, 640, False, 'x') == (t.data_ptr() + 10 * 2048 + 64, 2048)
    assert plane_address(t.view(1080, 512, 4)[:, :480], 1080, 1920, False, 'x') == (t.data_ptr(), 2048)
    assert plane_address((0x7f0000001000, 4096), 480, 640, True, 'x') == (0x7f0000001000, 4096)
    with pytest.raises(ValueError, match='x: a CPU tensor, but frames_on_device is True'):
        plane_address(view, 480, 640, True, 'x')
    with pytest.raises(ValueError, match='uint8'):
        plane_address(t.float()[:480, :640], 480, 640, False, 'x')


def test_plane_address_refusals():
    big = np.zeros((480, 704), np.uint8)
    cases = [
        (big[:, ::2], 480, 352, False, 'the bytes of a row must be dense'),
        (big.T, 704, 480, False, 'the bytes of a row must be dense'),
        (big[:, :640], 240, 640, False, '240 rows of 640 bytes expected, not 480 rows of 640 bytes'),
        (big[:, :641], 480, 640, False, '480 rows of 640 bytes expected, not 480 rows of 641 bytes'),
        (big[::-1, :640], 480, 640, False, 'the row pitch -704 is below the row bytes 640'),
        (big.view(np.uint16), 480, 704, False, 'uint8'),
        (big, 480, 704, True, 'a numpy array is host memory, but frames_on_device is set'),
        ((big.ctypes.data, 704), 480, 704, False, r'an \(address, pitch\) pair is a device plane'),
        ((1, 2, 3), 480, 704, True, r'a device plane is an \(address, pitch\) pair, not 3 values'),
        ([big], 480, 704, False, 'a plane is a uint8 numpy array or torch tensor, not list'),
    ]
    for plane, rows, row_bytes, dev, msg in cases:
        with pytest.raises(ValueError, match='frame 3 plane 1: .*' + msg):
            plane_address(plane, rows, row_bytes, dev, 'frame 3 plane 1')


def _engine(cameras):
    return types.SimpleNamespace(cameras=cameras)


def test_frame_planes_of_a_batch():
    """tuples of planes go through as given; a packed frame of the same batch becomes its planes at packed offsets"""
    packed = np.zeros((720, 640), np.uint8)                   # nv12 640x480
    buf = np.zeros(480 * 704 + 240 * 1024, np.uint8)
    y = buf[:480 * 704].reshape(480, 704)[:, :640]
    uv = buf[480 * 704:].reshape(240, 1024)[:, :640]
    arr = Engine._frame_planes(_engine({0: (640, 480), 1: (640, 480)}), [(y, uv), packed], [0, 1], 'nv12', False)
    assert ctypes.sizeof(arr) == 2 * 48
    assert list(arr[0].plane)[:2] == [buf.ctypes.data, buf.ctypes.data + 480 * 704]
    assert list(arr[0].pitch) == [704, 1024, 0] and arr[0].plane[2] is None
    assert list(arr[1].plane)[:2] == [packed.ctypes.data, packed.ctypes.data + 640 * 480]
    assert list(arr[1].pitch) == [640, 640, 0]
    # device pairs, and a device frame given by its address
    arr = Engine._frame_planes(_engine({5: (2, 2)}), [((4096, 64), (8192, 64), (12288, 64)), 65536], [5, 5],
                               'yuv420p', True)
    assert list(arr[0].plane) == [4096, 8192, 12288] and list(arr[0].pitch) == [64, 64, 64]
    assert list(arr[1].plane) == [65536, 65540, 65541] and list(arr[1].pitch) == [2, 1, 1]


def test_frame_planes_refusals():
    eng = _engine({0: (640, 480)})
    y = np.zeros((480, 640), np.uint8)
    with pytest.raises(ValueError, match='frame 1: a yuv420p frame has 3 planes, not 2'):
        Engine._frame_planes(eng, [(y, y[:240, :320], y[240:, 320:]), (y, y)], [0, 0], 'yuv420p', False)
    with pytest.raises(ValueError, match='frame 0: a rgba frame has 1 plane, not 2'):
        Engine._frame_planes(eng, [(y, y)], [0], 'rgba', False)
    with pytest.raises(ValueError, match=r'frame 0 \(nv12\) plane 1: 240 rows of 640 bytes expected'):
        Engine._frame_planes(eng, [(y, y)], [0], 'nv12', False)
    with pytest.raises(ValueError, match='frame 1: a numpy array is host memory, but frames_on_device is set'):
        Engine._frame_planes(eng, [((1, 640), (2, 640)), np.zeros((720, 640), np.uint8)], [0, 0], 'nv12', True)


def test_word_loads_need_aligned_pointer_and_pitch():
    """The RGBA / BGRA stems read a pixel as one 32-bit word only when every row starts word-aligned.  Row y starts at
    ptr + y * pitch, so that holds exactly when ptr and pitch are both multiples of 4 (for frames of two rows or more);
    a word-aligned ptr alone, the condition of packed frames (pitch 4w), would give misaligned loads on odd rows when
    pitch % 4 == 2."""
    def words(ptr, pitch):                                    # restates `aligned` in resized_pixel_load
        return ((ptr | pitch) & 3) == 0

    for ptr in range(8):
        for pitch in range(8, 24):
            rows_aligned = all((ptr + y * pitch) % 4 == 0 for y in range(4))
            assert words(ptr, pitch) == rows_aligned, (ptr, pitch)
    assert not words(256, 4 * 641 + 2) and (256 + 1 * (4 * 641 + 2)) % 4 == 2
    src = open(os.path.join(ROOT, 'watsor_b200', 'csrc', 'kernels_pre.cu')).read()
    assert re.search(r'aligned = \(\(reinterpret_cast<uintptr_t>\(fd\.ptr\) \| \(uintptr_t\)fd\.pitch\) & 3\) == 0',
                     src)


def test_frame_planes_struct_matches_header():
    cc = shutil.which('cc') or shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler')
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "watsor_b200.h"
int main(void) {
  wb_frame_planes p;
  printf("%zu %zu %zu %zu %zu\n", sizeof(wb_frame_planes), offsetof(wb_frame_planes, plane),
         offsetof(wb_frame_planes, pitch), sizeof(p.plane[0]), sizeof(p.pitch[0]));
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, 'planes.c'), os.path.join(tmp, 'planes')
        with open(src, 'w') as f:
            f.write(prog)
        subprocess.check_call([cc, '-std=c99', '-I', os.path.join(ROOT, 'include'), src, '-o', exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    P = _lib.FramePlanes
    assert got == [ctypes.sizeof(P), P.plane.offset, P.pitch.offset, ctypes.sizeof(ctypes.c_void_p),
                   ctypes.sizeof(ctypes.c_int64)]
    assert got == [48, 0, 24, 8, 8]
