"""Frames given as planes with row pitches (wb_detect_planes / wb_submit_planes): decoder surfaces, ffmpeg frames and
views of larger frames.  Device planes are read in place and host planes are packed as they are uploaded; either way
the kernels must read the bytes of the packed copy of the frame, so every result must equal, byte for byte, wb_detect
on that packed copy (rows and verdicts, fused filters and zone masks on)."""
import os

import numpy as np
import pytest

from tests import workload
from tests import yuv422_emulation as yuv422
from tests import yuv_emulation as yuv420
from tests.artist import artist_frame
from tests.gpu_util import new_rows, rows_bytes
from tests.rgb_orders import LAYOUT, from_rgb
from watsor_b200 import _lib
from watsor_b200.detection.b200 import B200ObjectDetector
from watsor_b200.engine import FRAME_FORMATS, layout_planes, layout_shape

pytestmark = pytest.mark.gpu

FORMATS = tuple(FRAME_FORMATS)                     # all eight
# camera sizes per format: the configs, the full-HD surface, the smallest frame, odd sizes where the format allows them
SIZES = {fmt: [(640, 480), (1920, 1080), (2, 2), (641, 479)] for fmt in LAYOUT}
SIZES.update({fmt: [(640, 480), (1920, 1080), (2, 2), (642, 479)] for fmt in yuv422.FORMATS})
SIZES.update({fmt: [(640, 480), (1920, 1080), (2, 2), (318, 238)] for fmt in ('yuv420p', 'nv12')})
# how each plane's rows are laid out: 'contiguous' = views of the packed frame (one copy per host frame); the others
# put every plane in a buffer of its own, rows `pitch` bytes apart
PITCHES = ('contiguous', 'packed', '+1', '+3', '64', '512')


def pitch_of(kind, row_bytes):
    if kind in ('contiguous', 'packed'):
        return row_bytes
    if kind.startswith('+'):
        return row_bytes + int(kind[1:])
    a = int(kind)
    return -(-row_bytes // a) * a


def packed_frame(rng, fmt, w, h):
    """a picture the detector finds objects in for the camera sizes, random bytes for the others"""
    if w < 64 or (w + h) % 2:
        return rng.integers(0, 256, layout_shape(fmt, w, h), dtype=np.uint8)
    rgb = artist_frame(w, h, w % 5, h % 3)
    if fmt in LAYOUT:
        return from_rgb(rgb, fmt, rng)
    if fmt in yuv422.FORMATS:
        return yuv422.from_rgb(rgb, fmt)
    return yuv420.from_rgb(rgb, fmt)


def plane_views(packed, fmt, w, h):
    """the planes of a packed frame, as (rows, row bytes) views of it"""
    flat, out, off = packed.reshape(-1), [], 0
    for rows, row_bytes in layout_planes(fmt, w, h):
        out.append(flat[off:off + rows * row_bytes].reshape(rows, row_bytes))
        off += rows * row_bytes
    return out


def padded(plane, pitch, rng, offset=0):
    """a buffer of random bytes holding the plane's rows `pitch` bytes apart from `offset` on, and the view of them"""
    rows, row_bytes = plane.shape
    buf = rng.integers(0, 256, offset + rows * pitch + 64, dtype=np.uint8)
    view = buf[offset:offset + rows * pitch].reshape(rows, pitch)[:, :row_bytes]
    view[...] = plane
    return buf, view


class Planes:
    """a frame as planes in host or device memory; keeps every buffer alive"""

    def __init__(self, packed, fmt, w, h, kind, rng, device, offset=0, pairs=None):
        import torch
        views = plane_views(packed, fmt, w, h)
        self.keep = [packed]
        if kind == 'contiguous' and not device:
            self.frame = tuple(views)
            return
        planes = []
        for k, v in enumerate(views):
            pitch = pitch_of(kind, v.shape[1])
            if kind == 'contiguous':                   # device: the packed frame in one allocation
                pitch = v.shape[1]
            buf, view = padded(v, pitch, rng, offset)
            if not device:
                planes.append(view)
                self.keep.append(buf)
                continue
            t = torch.from_numpy(buf).cuda()
            self.keep.append(t)
            if pairs if pairs is not None else (k + len(kind)) % 2 == 0:
                planes.append((t.data_ptr() + offset, pitch))
            else:
                planes.append(t[offset:offset + v.shape[0] * pitch].view(v.shape[0], pitch)[:, :v.shape[1]])
        if kind == 'contiguous':
            t = torch.from_numpy(np.ascontiguousarray(packed).reshape(-1)).cuda()
            self.keep.append(t)
            planes, off = [], 0
            for v in views:
                planes.append((t.data_ptr() + off, v.shape[1]))
                off += v.size
        self.frame = tuple(planes)
        torch.cuda.synchronize()


def run(det, frames, cams, fmt, **kw):
    rows = new_rows(len(frames))
    verd = np.zeros((len(frames), 100), np.uint32)
    det.detect_batch(frames, cams, rows, [verd[i] for i in range(len(frames))], fuse_filters=True,
                     pixel_format=fmt, **kw)
    return [rows_bytes(r) for r in rows], verd


def submit_collect(det, slot, frames, cams, fmt, **kw):
    det.submit(slot, frames, cams, fuse_filters=True, pixel_format=fmt, **kw)
    rows = new_rows(len(frames))
    verd = np.zeros((len(frames), 100), np.uint32)
    det.collect(slot, rows, [verd[i] for i in range(len(frames))])
    return [rows_bytes(r) for r in rows], verd


def same(got, want):
    return got[0] == want[0] and np.array_equal(got[1], want[1])


def configure(det, sizes, first=0):
    cams = []
    for i, (w, h) in enumerate(sizes):
        det.configure_camera(first + i, w, h, workload.camera_config(first + i, w, h, mask=w >= 64 and h >= 64))
        cams.append(first + i)
    return cams


def detector(precision, blob=None, max_batch=8):
    return B200ObjectDetector(None, device=0, max_batch=max_batch, precision=precision,
                              model_blob=blob or workload.v2_coco_model().to_blob())


@pytest.fixture(scope='module')
def det():
    """the 90-class v2 model at threshold 1e-8: 100 live rows per frame, sensitive to every input bit"""
    with detector(2) as d:
        yield d


# ------------------------------------------------------------------------------------------ 1: every layout
@pytest.mark.parametrize('fmt', FORMATS)
def test_planes_equal_packed(det, fmt):
    """host and device planes at every pitch, on a batch mixing four camera sizes (each frame with its own pitch)"""
    rng = np.random.default_rng(FORMATS.index(fmt))
    sizes = SIZES[fmt]
    cams = configure(det, sizes)
    packed = [packed_frame(rng, fmt, w, h) for w, h in sizes]
    want = run(det, packed, cams, fmt)
    for device in (False, True):
        for kind in PITCHES:
            frames = [Planes(p, fmt, w, h, kind, rng, device) for p, (w, h) in zip(packed, sizes)]
            got = run(det, [f.frame for f in frames], cams, fmt, frames_on_device=device)
            assert same(got, want), (fmt, kind, 'device' if device else 'host')


# ------------------------------------------------------------------------------- 2: planes in any order
def test_separate_chroma_allocations(det):
    """yuv420p with U and V in allocations of their own, V below U in memory; NV12 with its chroma in an allocation
    of its own whose pitch differs from the luma pitch; host and device"""
    import torch
    rng = np.random.default_rng(20)
    sizes = [(640, 480), (1920, 1080)]
    cams = configure(det, sizes)
    for fmt in ('yuv420p', 'nv12'):
        packed = [packed_frame(rng, fmt, w, h) for w, h in sizes]
        want = run(det, packed, cams, fmt)
        for device in (False, True):
            frames, keep = [], []
            for p, (w, h) in zip(packed, sizes):
                views = plane_views(p, fmt, w, h)
                pitches = [w + 64] + ([w // 2 + 32] * 2 if fmt == 'yuv420p' else [w + 512])   # chroma != luma pitch
                host = [padded(v, pitch, rng) for v, pitch in zip(views, pitches)]
                bufs = [buf for buf, _ in host]
                if not device:
                    if fmt == 'yuv420p':                # V's buffer below U's
                        lo, hi = sorted(bufs[1:], key=lambda x: x.ctypes.data)
                        lo[...], hi[...] = bufs[2].copy(), bufs[1].copy()
                        bufs = [bufs[0], hi, lo]
                    keep += bufs
                    layout = layout_planes(fmt, w, h)
                    frames.append(tuple(buf[:rows * pitch].reshape(rows, pitch)[:, :row_bytes]
                                        for buf, pitch, (rows, row_bytes) in zip(bufs, pitches, layout)))
                    continue
                dev = [torch.from_numpy(buf).cuda() for buf in bufs]
                if fmt == 'yuv420p':
                    lo, hi = sorted(dev[1:], key=lambda t: t.data_ptr())
                    lo.copy_(torch.from_numpy(bufs[2]))
                    hi.copy_(torch.from_numpy(bufs[1]))
                    dev = [dev[0], hi, lo]
                keep += dev
                frames.append(tuple((t.data_ptr(), pitch) for t, pitch in zip(dev, pitches)))
            if fmt == 'yuv420p':
                assert all(f[2][0] < f[1][0] if device else f[2].ctypes.data < f[1].ctypes.data for f in frames)
            torch.cuda.synchronize()
            assert same(run(det, frames, cams, fmt, frames_on_device=device), want), (fmt, device)


# ---------------------------------------------------------------------- 3: 4-byte pixels at unaligned pitches
def test_rgba_device_pitches(det):
    """RGBA / BGRA read in place with pitch % 4 = 2 from a word-aligned pointer, and the other (pointer, pitch)
    alignments: the 32-bit loads are taken only where every row is word-aligned"""
    rng = np.random.default_rng(30)
    sizes = [(640, 480), (641, 479), (1920, 1080)]
    cams = configure(det, sizes)
    for fmt in ('rgba', 'bgra'):
        packed = [packed_frame(rng, fmt, w, h) for w, h in sizes]
        want = run(det, packed, cams, fmt)
        for kind, offset in (('+2', 0), ('+6', 0), ('+4', 0), ('+4', 1), ('+2', 2), ('+1', 3), ('64', 0)):
            frames = [Planes(p, fmt, w, h, kind, rng, True, offset=offset) for p, (w, h) in zip(packed, sizes)]
            assert same(run(det, [f.frame for f in frames], cams, fmt, frames_on_device=True), want), (fmt, kind,
                                                                                                       offset)


# -------------------------------------------------------------------------------- 4: padding is never read
def test_padding_is_not_read(det):
    rng = np.random.default_rng(40)
    sizes = [(640, 480), (641, 479)]
    for fmt in FORMATS:
        sz = [(w + (w % 2 and fmt not in LAYOUT), h + (h % 2 and fmt in ('yuv420p', 'nv12'))) for w, h in sizes]
        cams = configure(det, sz)
        packed = [packed_frame(rng, fmt, w, h) for w, h in sz]
        want = run(det, packed, cams, fmt)
        for device in (False, True):
            for seed in (1, 2):                         # the same rows, other random bytes between them
                pad_rng = np.random.default_rng(seed)
                frames = [Planes(p, fmt, w, h, '512', pad_rng, device) for p, (w, h) in zip(packed, sz)]
                assert same(run(det, [f.frame for f in frames], cams, fmt, frames_on_device=device), want), \
                    (fmt, device, seed)


# ------------------------------------------------------------------------------------------ 5: windows
ODD_WINDOWS = [(0, 0, 1920, 1080), (1, 0, 961, 539), (959, 541, 961, 539), (3, 3, 1917, 1077), (1919, 0, 1, 1080),
               (641, 201, 637, 479)]
WINDOWS = {'420': [(0, 0, 1920, 1080), (2, 0, 960, 540), (958, 540, 962, 540), (640, 200, 640, 480)],
           '422': [(0, 0, 1920, 1080), (2, 1, 960, 539), (958, 541, 962, 539), (1918, 0, 2, 1080)]}


def test_windows_on_pitched_device_frames(det):
    """a windowed 1920x1080 camera next to cameras without windows, each frame with its own pitch"""
    rng = np.random.default_rng(50)
    try:
        for fmt in FORMATS:
            wins = WINDOWS['420'] if fmt in ('yuv420p', 'nv12') else WINDOWS['422'] if fmt in yuv422.FORMATS \
                else ODD_WINDOWS
            sizes = [(1920, 1080), (640, 480), SIZES[fmt][3]]
            cams = configure(det, sizes)
            det.engine.set_camera_windows(cams[0], wins)
            packed = [packed_frame(rng, fmt, w, h) for w, h in sizes]
            want = run(det, packed, cams, fmt)
            frames = [Planes(p, fmt, w, h, kind, rng, True)
                      for p, (w, h), kind in zip(packed, sizes, ('+3', '512', '+1'))]
            assert same(run(det, [f.frame for f in frames], cams, fmt, frames_on_device=True), want), fmt
            frames = [Planes(p, fmt, w, h, kind, rng, False)
                      for p, (w, h), kind in zip(packed, sizes, ('64', '+1', '+3'))]
            assert same(run(det, [f.frame for f in frames], cams, fmt), want), (fmt, 'host')
    finally:
        det.engine.set_camera_windows(0, [])


# -------------------------------------------------------------------------------------- 6: graph replay
def test_graph_replay_alternating_packed_and_planes():
    """one engine, one graph key: packed and planes batches with new pointers, pitches and slots each call equal an
    engine without graphs"""
    import torch
    blob = workload.v2_coco_model().to_blob()
    os.environ['WB_NO_GRAPH'] = '1'
    try:
        plain = detector(2, blob, max_batch=2)
    finally:
        os.environ.pop('WB_NO_GRAPH', None)
    sizes = [(640, 480), (1280, 720)]
    rng = np.random.default_rng(60)
    with plain, detector(2, blob, max_batch=2) as d:
        for x in (d, plain):
            configure(x, sizes)
        cams = [0, 1]
        for rnd in range(2):
            for fmt in ('nv12', 'rgba'):
                packed = [packed_frame(rng, fmt, w, h) for w, h in sizes]
                calls = [('packed', False, packed)]
                for device, kind in ((True, '+1'), (False, '64'), (True, '512'), (True, '+2')):
                    frames = [Planes(p, fmt, w, h, kind, rng, device, offset=rnd) for p, (w, h) in zip(packed, sizes)]
                    calls.append((kind, device, frames))
                dev = [torch.from_numpy(p.reshape(-1).copy()).cuda() for p in packed]
                torch.cuda.synchronize()
                calls.append(('packed device', True, [t.data_ptr() for t in dev]))
                want = run(plain, packed, cams, fmt)
                for slot, (name, device, frames) in enumerate(calls):
                    fr = [f.frame if hasattr(f, 'frame') else f for f in frames]
                    assert same(run(plain, fr, cams, fmt, frames_on_device=device), want), (rnd, fmt, name, 'plain')
                    assert same(run(d, fr, cams, fmt, frames_on_device=device), want), (rnd, fmt, name)
                    assert same(submit_collect(d, 1 + slot % 5, fr, cams, fmt, frames_on_device=device), want), \
                        (rnd, fmt, name, 'slot')


# --------------------------------------------------------------------------------- 7: every stem storage type
@pytest.mark.parametrize('precision', [0, 2, 1, 4], ids=['fp32', 'tf32x3', 'bf16', 'fp16'])
def test_precisions(precision):
    rng = np.random.default_rng(70 + precision)
    with detector(precision) as d:
        for fmt in ('rgb24', 'rgba', 'bgr24', 'nv12', 'yuv420p', 'yuyv422'):
            sizes = [(640, 480), (1920, 1080), SIZES[fmt][3]]
            cams = configure(d, sizes)
            packed = [packed_frame(rng, fmt, w, h) for w, h in sizes]
            want = run(d, packed, cams, fmt)
            for device, kind in ((True, '+2'), (True, '512'), (False, '+3')):
                frames = [Planes(p, fmt, w, h, kind, rng, device) for p, (w, h) in zip(packed, sizes)]
                assert same(run(d, [f.frame for f in frames], cams, fmt, frames_on_device=device), want), (fmt, kind)


def test_inception_generic_stem():
    """SSD-Inception-v2's 7x7 stem runs the generic k_stem"""
    from watsor_b200.model import synthetic_ssd_inception_v2
    blob = synthetic_ssd_inception_v2(num_classes=90, seed=0, score_thr=1e-8).to_blob()
    rng = np.random.default_rng(71)
    sizes = [(1920, 1080), (1920, 1080)]
    with detector(2, blob, max_batch=2) as d:
        cams = configure(d, sizes)
        for fmt, device, kind in (('nv12', True, '512'), ('rgba', True, '+2'), ('yuv420p', False, '64'),
                                  ('uyvy422', True, '+1')):
            packed = [packed_frame(rng, fmt, w, h) for w, h in sizes]
            want = run(d, packed, cams, fmt)
            frames = [Planes(p, fmt, w, h, kind, rng, device) for p, (w, h) in zip(packed, sizes)]
            assert same(run(d, [f.frame for f in frames], cams, fmt, frames_on_device=device), want), fmt


# ------------------------------------------------------------------------------------------- 8: refusals
def test_refusals_leave_the_slot_free(det):
    """each malformed batch is refused with a message naming the frame, the format and the value; the slot then
    takes a valid batch"""
    import ctypes

    import torch
    engine = det.engine
    rng = np.random.default_rng(80)
    sizes = [(640, 480), (64, 1), (642, 480), (641, 479)]
    cams = configure(det, sizes)
    big = torch.zeros(4 << 20, dtype=torch.uint8, device='cuda')     # holds every plane read below
    host = np.zeros(4 << 20, np.uint8)
    torch.cuda.synchronize()
    fmt_flag = {fmt: flag for fmt, flag in FRAME_FORMATS.items()}

    def submit(fmt, cam, planes, pitches, device=True, slot=3):
        arr = (_lib.FramePlanes * 1)()
        for k, (p, pitch) in enumerate(zip(planes, pitches)):
            arr[0].plane[k], arr[0].pitch[k] = p, pitch
        flags = fmt_flag[fmt] | _lib.WB_F_FUSE_FILTERS | (_lib.WB_F_FRAMES_ON_DEVICE if device else 0)
        return engine.lib.wb_submit_planes(engine._ctx, slot, 1, arr, (ctypes.c_int32 * 1)(cam), flags)

    d0, h0 = big.data_ptr(), host.ctypes.data
    cases = [
        ('nv12', 0, [d0, d0 + 640 * 480, d0 + 2 * 640 * 480], [640, 640, 640], True,
         r'frame 0 \(nv12\): nv12 has 2 planes, but plane\[2\] is given'),
        ('rgb24', 0, [d0, d0], [1920, 1920], True, r'frame 0 \(rgb24\): rgb24 has 1 plane, but plane\[1\] is given'),
        ('yuv420p', 0, [h0, None, h0 + 640 * 480], [640, 320, 320], False, r'frame 0 \(yuv420p\): plane\[1\] is NULL'),
        ('rgb24', 0, [d0], [1919], True,
         r"frame 0 \(rgb24\): pitch\[0\] = 1919 is below the plane's row bytes \(1920\)"),
        ('nv12', 0, [d0, d0 + 640 * 480], [640, 639], True,
         r"frame 0 \(nv12\): pitch\[1\] = 639 is below the plane's row bytes \(640\)"),
        ('rgba', 1, [d0], [1 << 31], True, r'frame 0 \(rgba\): pitch\[0\] = 2147483648 is 2\^31 or more'),
        ('yuyv422', 1, [d0], [-128], True, r"frame 0 \(yuyv422\): pitch\[0\] = -128 is below the plane's row bytes"),
        ('yuv420p', 0, [d0, d0 + 640 * 480, d0 + 700 * 480], [640, 320, 336], True,
         r'frame 0 \(yuv420p\): the U and V planes need the same pitch, not pitch\[1\] = 320 and pitch\[2\] = 336'),
        ('nv12', 3, [d0, d0 + 641 * 479], [641, 641], True,
         r'frame 0 \(nv12\): cam_id 3 is 641x479: 4:2:0 frames need an even width and height'),
        ('uyvy422', 3, [d0], [1282], True,
         r'frame 0 \(uyvy422\): cam_id 3 is 641x479: 4:2:2 frames need an even width'),
    ]
    for fmt, cam, planes, pitches, device, msg in cases:
        assert submit(fmt, cam, planes, pitches, device) != 0, msg
        with pytest.raises(_lib.WatsorB200Error, match=msg):
            _lib.check(1)
    det.engine.set_camera_windows(cams[2], [(0, 0, 642, 480), (1, 2, 320, 240)])
    try:
        assert submit('nv12', 2, [d0, d0 + 642 * 480], [642, 642]) != 0
        with pytest.raises(_lib.WatsorB200Error, match=r'frame 0 \(nv12\): cam_id 2 window 1 \(1, 2, 320, 240\): '
                                                       r'4:2:0 frames need an even window origin'):
            _lib.check(1)
    finally:
        det.engine.set_camera_windows(cams[2], [])
    # the Python layer refuses what it can see before the library does
    frame = packed_frame(rng, 'nv12', 640, 480)
    y, uv = plane_views(frame, 'nv12', 640, 480)
    with pytest.raises(ValueError, match='frame 0: a nv12 frame has 2 planes, not 1'):
        det.submit(3, [(y,)], [0], pixel_format='nv12')
    with pytest.raises(ValueError, match='frame 0 \\(nv12\\) plane 1: 240 rows of 640 bytes expected'):
        det.submit(3, [(y, y)], [0], pixel_format='nv12')
    with pytest.raises(ValueError, match='numpy array is host memory'):
        det.submit(3, [(y, uv)], [0], pixel_format='nv12', frames_on_device=True)
    # slot 3 is free and takes a valid batch: the same rows as the packed frame
    want = run(det, [frame], [0], 'nv12')
    planes = Planes(frame, 'nv12', 640, 480, '+3', rng, True)
    assert same(submit_collect(det, 3, [planes.frame], [0], 'nv12', frames_on_device=True), want)
    assert same(submit_collect(det, 3, [(y, uv)], [0], 'nv12'), want)
