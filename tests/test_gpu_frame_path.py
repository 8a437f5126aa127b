"""The detection path as it runs, from camera frames (`wb_backbone_frames`), against the stage-level path and float64.

The product path never takes a pre-processed input: its stem samples the u8 frame itself (the `pre == nullptr` branch
of `k_stem_3x3s2_c32` and `k_stem`, 4:2:0 loads and window addressing included), and the batch replays as a CUDA
graph.  Three groups of checks:

  (a) the stem on frames, one tiny one-stem model per stem kernel: bit-identical to the stem on `preprocess()` of the
      same RGB images (the frame, its cv2.cvtColor conversion, or the host crop of a window) in a batch of the same
      image count, and within the float64 bound of tests/layer_reference.py computed on `oracle.preprocess` -- which
      does not rely on the stage path being right.  One launch per call, of the kernel the shape selects;
  (b) whole networks: the heads of the graph-replayed product path are bit-identical to the stage path's, and the rows
      and verdicts of `detect` byte-identical to `postprocess` of those heads.  Slot 0 first runs other frames, so a
      head row that no kernel writes would keep their values;
  (c) one engine replays its graphs over batches that share a graph key and differ in everything the key leaves out
      (contents, camera sizes, pixel format, host / device frames, window layout, slot): heads bit-identical to the
      stage path, rows and verdicts byte-identical to an engine that runs without graphs.

Every comparison in (b) and (c) is exact: both sides run the same kernels with the same plan."""
import os

import numpy as np
import pytest

from tests import layer_reference as R
from tests import workload
from tests.artist import artist_frame
from tests.conftest import PORCH_CONFIG, load_golden_frame
from tests.gpu_util import new_rows, rows_bytes
from tests.test_gpu_layer_kernels import _kernels, build, record
from tests.test_gpu_layer_kernels import report  # noqa: F401  (the largest error / bound per family)
from tests.yuv_emulation import cv2_rgb, random_frame
from watsor_b200 import _lib
from watsor_b200.detection.b200 import B200ObjectDetector
from watsor_b200.engine import Engine
from watsor_b200.model import synthetic_ssd_inception_v2

pytestmark = pytest.mark.gpu
FUSE = _lib.WB_F_FUSE_FILTERS
PRE_MUL, PRE_SUB = float(np.float32(2.0 / 255.0)), 1.0     # the SSD graphs' normalisation to [-1, 1]


# ------------------------------------------------------------------------------------------------ (a) stem on frames
STEMS = {
    '3x3s2_c32_300': ('stem', 300, 300, 3, 2, 32),
    '3x3s2_c32_299x301': ('stem', 299, 301, 3, 2, 32),        # pad_t = pad_l = 1 (0 at 300)
    '7x7s2_c24_300': ('stem', 300, 300, 7, 2, 24),
    '3x3s1_c16_300': ('stem', 300, 300, 3, 1, 16),
    '1x1_c16_300': ('stem', 300, 300, 1, 1, 16),
}
# (width, height) per camera: degenerate, thin, odd, around and at the identity scale (lo = hi, lerp = 0), the exact 2x
# upscale, camera sizes
RGB_SIZES = [(1, 1), (2, 2), (7, 900), (900, 7), (53, 37), (299, 301), (300, 300), (301, 299), (150, 150), (640, 480),
             (1920, 1080), (3840, 2160)]
EVEN_SIZES = [(2, 2), (150, 150), (300, 300), (640, 480), (1920, 1080), (3840, 2160)]
MIXED_RGB = [(53, 37), (1920, 1080), (2, 2), (301, 299)]           # one batch, each image its own scale
MIXED_EVEN = [(2, 2), (640, 480), (150, 150), (1920, 1080)]
# detection windows: odd origins, windows touching the right and bottom borders, the whole frame; a camera without
# windows is one full-frame window of the batch
RGB_WINDOWS = {0: ((1920, 1080), [(13, 7, 301, 233), (1619, 847, 301, 233), (0, 0, 1920, 1080), (1917, 1, 3, 1079)]),
               1: ((53, 37), [(1, 3, 52, 34), (0, 0, 53, 37)]),
               2: ((640, 480), [])}
YUV_WINDOWS = {3: ((640, 480), [(0, 0, 640, 480), (12, 8, 300, 226), (340, 254, 300, 226)]),
               4: ((1920, 1080), [(2, 4, 640, 360), (1280, 720, 640, 360)])}
GROUPS = ['rgb', 'yuv420p', 'nv12', 'windows']
MAX_IMAGES = 8


def _frame(rng, fmt, w, h):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8) if fmt == 'rgb24' else random_frame(rng, w, h)


def _batch(rng, fmt, cams):
    """cams: {cam: ((w, h), windows)} -> (fmt, cams, frames, RGB model images in the batch's order)"""
    frames, images = [], []
    for (w, h), wins in cams.values():
        f = _frame(rng, fmt, w, h)
        rgb = f if fmt == 'rgb24' else cv2_rgb(f, fmt)
        frames.append(f)
        images += [np.ascontiguousarray(rgb[y:y + wh, x:x + ww]) for x, y, ww, wh in (wins or [(0, 0, w, h)])]
    return fmt, cams, frames, images


@pytest.fixture(scope='module')
def batches():
    """the batches of every group, shared by all stems and precisions (so is their float64 reference)"""
    rng = np.random.default_rng(2024)

    def sized(sizes, cam0):
        return {cam0 + i: (s, []) for i, s in enumerate(sizes)}

    out = {'rgb': [_batch(rng, 'rgb24', sized([s], 10 + k)) for k, s in enumerate(RGB_SIZES)] +
           [_batch(rng, 'rgb24', sized(MIXED_RGB, 30))]}
    for fmt in ('yuv420p', 'nv12'):
        out[fmt] = [_batch(rng, fmt, sized([s], 40 + k)) for k, s in enumerate(EVEN_SIZES)] + \
                   [_batch(rng, fmt, sized(MIXED_EVEN, 50))]
    out['windows'] = [_batch(rng, 'rgb24', RGB_WINDOWS), _batch(rng, 'yuv420p', YUV_WINDOWS),
                      _batch(rng, 'nv12', YUV_WINDOWS)]
    return out


REFS = {}           # (stem, group, batch) -> float64 (z·s, P, y) of the stem on oracle.preprocess of the batch's images


def _stem_model(name):
    m, li, _, _ = build(STEMS[name], seed=len(name))
    assert li == 0
    m.pre_mul, m.pre_sub = PRE_MUL, PRE_SUB
    return m


def _stem_reference(m, images):
    from oracle.ssd_model import SsdModelOracle
    L = m.layers[0]
    a = np.stack([SsdModelOracle(m).preprocess(img) for img in images]).astype(np.float64)
    wt = np.asarray(m.tensors[L.w_tensor], np.float64).reshape(L.kh * L.kw * 3, L.n_pad)[:, :L.out_c]
    wt = wt.reshape(L.kh, L.kw, 3, L.out_c)
    sc = np.asarray(m.tensors[L.scale_tensor], np.float64)[:L.out_c]
    of = np.asarray(m.tensors[L.offset_tensor], np.float64)[:L.out_c]
    z, P = R.conv2d(a, wt, L.stride), R.conv2d(np.abs(a), np.abs(wt), L.stride)
    return z * sc, P, R.affine(z, sc, of, L.act), sc, of


def _to_device(frames):
    import torch
    dev = [torch.from_numpy(f).cuda() for f in frames]
    torch.cuda.synchronize()
    return dev


def _configure(e, cams):
    for cam, ((w, h), wins) in cams.items():
        e.set_camera(cam, w, h)
        if wins:
            e.set_camera_windows(cam, wins)


@pytest.mark.parametrize('group', GROUPS)
@pytest.mark.parametrize('precision', [0, 2, 1], ids=lambda p: R.PRECISIONS[p].name)
@pytest.mark.parametrize('stem', list(STEMS))
def test_stem_on_frames(batches, stem, precision, group):
    import torch
    from torch.profiler import ProfilerActivity, profile
    m = _stem_model(stem)
    L = m.layers[0]
    shape = (L.out_h, L.out_w, L.out_c)
    plan = R.plan(L, 1, precision, torch.cuda.get_device_properties(0).multi_processor_count)
    with Engine(m.to_blob(), device=0, max_batch=MAX_IMAGES, precision=precision) as e:
        runs = []
        for fmt, cams, frames, images in batches[group]:
            _configure(e, cams)
            runs += [(fmt, cams, frames, images, False, frames), (fmt, cams, frames, images, True, _to_device(frames))]

        def frame_calls():
            out = []
            for fmt, cams, _, images, on_dev, src in runs:
                ptrs = [t.data_ptr() for t in src] if on_dev else src
                _, _, y, n_img = e.backbone_frames(ptrs, list(cams), stop_layer=0, layer_shape=shape, pixel_format=fmt,
                                                   frames_on_device=on_dev)
                assert n_img == len(images)
                assert e.last_launch_count() == 1
                out.append(y)
            torch.cuda.synchronize()
            return out

        # now and then a profiler session misses device activity (the library's own count says one launch per call):
        # trace again then
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                got = frame_calls()
            kernels = [k for k, _ in _kernels(prof)]
            if len(kernels) == len(runs):
                break
        assert len(kernels) == len(runs), kernels
        assert all(R.kernel_name_pattern(plan, precision) in k for k in kernels), (plan['kernel'], kernels)

        for b, (fmt, cams, frames, images) in enumerate(batches[group]):
            # (1) the stage path on the same RGB images, as one batch of the same image count
            want = e.backbone(e.preprocess(images), stop_layer=0, layer_shape=shape)[2]
            for on_dev in (False, True):
                y = got[2 * b + on_dev]
                assert np.array_equal(y, want), (fmt, list(cams.values()), 'device' if on_dev else 'host')
            # (2) float64 on oracle.preprocess
            key = (stem, group, b)
            if key not in REFS:
                REFS[key] = _stem_reference(m, images)
            zs, P, yr, sc, of = REFS[key]
            bound = R.chain_bound(P, zs, yr, sc, of, L.kh * L.kw * 3, precision)
            err = np.abs(got[2 * b] - yr)
            ratio = record('frames:' + plan['kernel'], precision, err, bound)
            assert np.all(err <= bound), (fmt, list(cams.values()), ratio)
            assert np.abs(yr).max() > 0


# ---------------------------------------------------------------------------------- (b) frames -> heads -> rows
def _shapes(request):
    m = request.getfixturevalue('shapes_model')
    cams = {0: (640, 480, PORCH_CONFIG), 1: (640, 480, PORCH_CONFIG), 2: (320, 240, None)}
    frames = [load_golden_frame(n) for n in ('artist_640x480_c0_f0', 'artist_640x480_c3_f7', 'artist_320x240_c0_f0')]
    stale = [artist_frame(640, 480, 5, 1), artist_frame(640, 480, 6, 2), artist_frame(320, 240, 7, 3)]
    return m, cams, frames, stale


def _v2_configs2(request):
    cams = {c: (640, 480, workload.camera_config(c)) for c in range(8)}
    frames = [artist_frame(640, 480, c, c % 3) for c in range(8)]
    rng = np.random.default_rng(8)
    stale = [rng.integers(0, 256, (480, 640, 3), dtype=np.uint8) for _ in range(8)]
    return workload.v2_coco_model(), cams, frames, stale


def _inception(request):
    cams = {0: (1920, 1080, None), 1: (1920, 1080, None)}
    frames = [artist_frame(1920, 1080, 3, 0), artist_frame(1920, 1080, 4, 1)]
    stale = [artist_frame(1920, 1080, 8, 2), artist_frame(1920, 1080, 9, 3)]
    return synthetic_ssd_inception_v2(num_classes=90, seed=0, score_thr=1e-8), cams, frames, stale


NETWORKS = {'shapes_v1': _shapes, 'v2_configs2': _v2_configs2, 'inception_1080p': _inception}


def _detect(det, frames, cams, **kw):
    rows = new_rows(len(frames))
    verd = np.zeros((len(frames), 100), np.uint32)
    det.detect_batch(frames, cams, rows, [verd[i] for i in range(len(frames))], fuse_filters=True, **kw)
    return [rows_bytes(r) for r in rows], verd


@pytest.mark.parametrize('precision', [0, 1, 2, 3], ids=lambda p: R.PRECISIONS[p].name)
@pytest.mark.parametrize('net', list(NETWORKS))
def test_network_frames_equal_stage_path(request, net, precision):
    m, cams, frames, stale = NETWORKS[net](request)
    ids = list(cams)
    with B200ObjectDetector(None, device=0, max_batch=len(frames), precision=precision, model_blob=m.to_blob()) as det:
        e = det.engine
        for cam, (w, h, cfg) in cams.items():
            det.configure_camera(cam, w, h, cfg)
        _detect(det, stale, ids)                                   # slot 0's head buffers now hold other frames' rows
        enc, lg, _, n_img = e.backbone_frames(frames, ids, flags=FUSE)
        assert n_img == len(frames)
        s_enc, s_lg, _ = e.backbone(e.preprocess(frames))
        assert np.array_equal(enc, s_enc) and np.array_equal(lg, s_lg)
        rows, verd = _detect(det, frames, ids)
        p_rows, p_verd = e.postprocess(enc, lg, ids, FUSE)[:2]
        assert rows == [rows_bytes(r) for r in p_rows]
        assert np.array_equal(verd, p_verd)
        assert any(int(v) & _lib.WB_V_LABEL for v in verd.ravel())


# ---------------------------------------------------------------------------- (c) graph replay depends on its key
def _even(v):
    return v - v % 2


def _layout(kind, size, odd):
    """windows of cameras A and B: 'l1' = A 3 windows, B none; 'l2' = 2 each (4 model images either way); odd
    origins for RGB24 batches, even ones for 4:2:0"""
    w, h = size
    half, quarter = (_even(w // 2), _even(h // 2)), (_even(w // 4) + odd, _even(h // 4) + odd)
    if kind == 'l1':
        return [(0, 0, w, h), (2 - odd, 2 - odd) + half, (w - half[0] - odd, h - half[1]) + half], []
    if kind == 'l2':
        return [(0, 0, w, h), quarter + half], [(odd, odd) + half, (w - half[0] - odd, 0) + half]
    return [], []


# (size of A, size of B, pixel format, device frames, window layout for the windowed sequence)
SEQUENCE = [((640, 480), (640, 480), 'rgb24', False, 'l1'),
            ((640, 480), (640, 480), 'rgb24', False, 'l1'),          # other contents
            ((640, 480), (1280, 720), 'rgb24', False, 'l1'),         # a mixed-size batch
            ((640, 480), (1280, 720), 'nv12', False, 'l1'),
            ((640, 480), (1280, 720), 'yuv420p', False, 'l2'),
            ((640, 480), (1280, 720), 'yuv420p', True, 'l2'),
            ((640, 480), (1280, 720), 'rgb24', True, 'l2'),
            ((320, 240), (1920, 1080), 'rgb24', False, 'l1'),
            ((320, 240), (1920, 1080), 'nv12', True, 'l2'),
            ((640, 480), (640, 480), 'rgb24', False, 'l2'),
            ((640, 480), (640, 480), 'yuv420p', False, 'l1')]


@pytest.mark.parametrize('windowed', [False, True], ids=['frames', 'windows'])
@pytest.mark.parametrize('precision', [2, 1], ids=lambda p: R.PRECISIONS[p].name)
def test_graph_replay_depends_only_on_its_key(precision, windowed):
    blob = workload.v2_coco_model().to_blob()
    os.environ['WB_NO_GRAPH'] = '1'
    try:
        plain = B200ObjectDetector(None, device=0, max_batch=4, precision=precision, model_blob=blob)
    finally:
        os.environ.pop('WB_NO_GRAPH', None)
    rng = np.random.default_rng(5)
    with plain, B200ObjectDetector(None, device=0, max_batch=4, precision=precision, model_blob=blob) as det:
        e = det.engine
        for i, (size_a, size_b, fmt, on_dev, layout) in enumerate(SEQUENCE):
            kind, odd = layout if windowed else None, int(fmt == 'rgb24')
            wins = _layout(kind, size_a, odd)[0], _layout(kind, size_b, odd)[1]
            for d in (det, plain):
                for cam, size, wl in ((0, size_a, wins[0]), (1, size_b, wins[1])):
                    d.configure_camera(cam, *size, workload.camera_config(cam, *size))
                    if wl:
                        d.engine.set_camera_windows(cam, wl)
            _, _, frames, images = _batch(rng, fmt, {0: (size_a, wins[0]), 1: (size_b, wins[1])})
            dev = _to_device(frames) if on_dev else None
            src = [t.data_ptr() for t in dev] if on_dev else frames
            kw = dict(pixel_format=fmt, frames_on_device=on_dev)
            what = (i, size_a, size_b, fmt, 'device' if on_dev else 'host', wins)
            # slot 0: the graph that backbone_frames and detect share (same key)
            enc, lg, _, n_img = e.backbone_frames(src, [0, 1], flags=FUSE, **kw)
            assert n_img == len(images) == (4 if windowed else 2), what
            s_enc, s_lg, _ = e.backbone(e.preprocess(images))
            assert np.array_equal(enc, s_enc) and np.array_equal(lg, s_lg), what
            want = _detect(plain, src, [0, 1], **kw)
            got = _detect(det, src, [0, 1], **kw)
            assert got[0] == want[0] and np.array_equal(got[1], want[1]), what
            # slots 1..5, each with its own graph, replayed with this batch
            slot = 1 + i % 5
            det.submit(slot, src, [0, 1], fuse_filters=True, **kw)
            rows = new_rows(2)
            verd = np.zeros((2, 100), np.uint32)
            det.collect(slot, rows, [verd[0], verd[1]])
            assert [rows_bytes(r) for r in rows] == want[0] and np.array_equal(verd, want[1]), what + (slot,)
