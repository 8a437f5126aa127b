#!/usr/bin/env python
"""Detection on frames given as planes (wb_detect_planes) against packing them first and calling the packed API.

    python tools/bench_planes.py --steps 200 --warmup 20 --rounds 5

Workloads (tests/workload.py): BASELINE configs[2] (8 cameras of 640x480, SSD-MobileNet-v2 with 90 classes at score
threshold 1e-8, a mask per camera, fused filters) and 2 cameras of 1920x1080 with the same model.  Two comparisons per
workload, each pair of arms run alternately within every round:
  nv12_device   NVDEC-style NV12 surfaces in device memory: one allocation per frame, rows 512-byte aligned, the chroma
                plane after the luma height rounded up to 16 rows.
                  in_place  the surfaces' planes passed as (address, pitch) pairs and read by the kernels in place
                  memcpy2d  cudaMemcpy2DAsync of each plane into a packed buffer, then the packed API on it
  yuv420p_host  ffmpeg-style yuv420p frames in pageable host memory: Y, U and V in three separate buffers with
                linesizes rounded up to 64 bytes.
                  planes    the three planes passed as views; the library packs them as it uploads them (one
                            cudaMemcpy2DAsync per plane)
                  numpy     the planes copied into one packed numpy frame, then the packed API on it
Per arm and round:
  device_fps  frames / s over the batch's device time: the library's CUDA-event time of the call (which covers its
              host-to-device copies), plus, for memcpy2d, CUDA-event time of the packing copies
  e2e_fps     frames / s of synchronous calls, wall clock, packing included
The figures are medians over rounds, with the spread.  The script checks that every arm computes the rows and verdicts
of the packed frames.  One JSON line per workload and comparison, with the card's name, power limit and maximum SM
clock read in the same run."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import workload  # noqa: E402
from tests.artist import artist_frame  # noqa: E402
from tests.gpu_util import new_rows, rows_bytes  # noqa: E402
from tests.yuv_emulation import from_rgb  # noqa: E402
from watsor_b200.detection.b200 import B200ObjectDetector  # noqa: E402

CUDA_MEMCPY_DEVICE_TO_DEVICE = 3


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True, check=True).stdout
    name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(',')]
    return {'gpu': name, 'power_limit': power, 'sm_max_clock': clock}


def cudart():
    """the CUDA runtime torch has loaded (for cudaMemcpy2DAsync)"""
    lib = ctypes.CDLL('libcudart.so.12')
    lib.cudaMemcpy2DAsync.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                      ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
    return lib


def align(v, a):
    return -(-v // a) * a


def timed(args, frames, arms, res, last, snapshot):
    """one round: the arms one after the other, each warmed up, then `steps` calls for the device time and `steps`
    for the wall clock"""
    for name, call in arms.items():
        for s in range(args.warmup):
            call(s)
        ms = [call(s) for s in range(args.steps)]
        res[name]['device_fps'].append(frames * 1000.0 / float(np.mean(ms)))
        t0 = time.perf_counter()
        for s in range(args.steps):
            call(s)
        res[name]['e2e_fps'].append(frames * args.steps / (time.perf_counter() - t0))
        last[name] = snapshot()


def run_workload(det, w, h, cams, args, torch, rt):
    for c in range(cams):
        det.configure_camera(c, w, h, workload.camera_config(c, w, h))
    ids = list(range(cams))
    ring = 4
    rgb = [artist_frame(w, h, c, r) for r in range(ring) for c in range(cams)]
    nv12 = [from_rgb(f, 'nv12') for f in rgb]
    i420 = [from_rgb(f, 'yuv420p') for f in rgb]
    rows = new_rows(cams)
    verd = np.zeros((cams, 100), np.uint32)
    vptr = [verd[i] for i in range(cams)]

    def snapshot():
        return [rows_bytes(r) for r in rows], verd.copy()

    def detect(frames, fmt, on_device):
        return det.detect_batch(frames, ids, rows, vptr, fuse_filters=True, frames_on_device=on_device,
                                pixel_format=fmt)

    # ---- NV12 surfaces on the device
    pitch, luma_rows = align(w, 512), align(h, 16)
    surfaces = []
    for f in nv12:
        s = torch.zeros(pitch * (luma_rows + h // 2), dtype=torch.uint8, device='cuda')
        y = s[:h * pitch].view(h, pitch)
        uv = s[luma_rows * pitch:(luma_rows + h // 2) * pitch].view(h // 2, pitch)
        y[:, :w].copy_(torch.from_numpy(f[:h]))
        uv[:, :w].copy_(torch.from_numpy(f[h:]))
        surfaces.append(s)
    staging = [torch.empty(w * h * 3 // 2, dtype=torch.uint8, device='cuda') for _ in range(cams)]
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def in_place(step):
        k = (step % ring) * cams
        planes = [((s.data_ptr(), pitch), (s.data_ptr() + luma_rows * pitch, pitch)) for s in surfaces[k:k + cams]]
        return detect(planes, 'nv12', True)

    def memcpy2d(step):
        k = (step % ring) * cams
        stream = torch.cuda.current_stream().cuda_stream
        ev0.record()
        for s, dst in zip(surfaces[k:k + cams], staging):
            for src_row, dst_off, rows_ in ((0, 0, h), (luma_rows, w * h, h // 2)):
                rc = rt.cudaMemcpy2DAsync(dst.data_ptr() + dst_off, w, s.data_ptr() + src_row * pitch, pitch, w, rows_,
                                          CUDA_MEMCPY_DEVICE_TO_DEVICE, stream)
                assert rc == 0, rc
        ev1.record()
        det.engine.stream_fence(stream, 0)               # the slot waits for the copies
        ms = detect([t.data_ptr() for t in staging], 'nv12', True)
        ev1.synchronize()
        return ms + ev0.elapsed_time(ev1)

    # ---- yuv420p frames in three pageable buffers each
    linesize = [align(w, 64), align(w // 2, 64), align(w // 2, 64)]
    av = []
    for f in i420:
        flat, planes, off = f.reshape(-1), [], 0
        for k, (rows_, rb) in enumerate(((h, w), (h // 2, w // 2), (h // 2, w // 2))):
            buf = np.zeros(rows_ * linesize[k], np.uint8)
            view = buf.reshape(rows_, linesize[k])[:, :rb]
            view[...] = flat[off:off + rows_ * rb].reshape(rows_, rb)
            off += rows_ * rb
            planes.append(view)
        av.append(tuple(planes))
    packed_host = [np.empty((h * 3 // 2, w), np.uint8) for _ in range(cams)]

    def planes_arm(step):
        k = (step % ring) * cams
        return detect(av[k:k + cams], 'yuv420p', False)

    def numpy_arm(step):
        k = (step % ring) * cams
        for (y, u, v), dst in zip(av[k:k + cams], packed_host):
            flat = dst.reshape(-1)
            flat[:w * h].reshape(h, w)[...] = y
            flat[w * h:w * h * 5 // 4].reshape(h // 2, w // 2)[...] = u
            flat[w * h * 5 // 4:].reshape(h // 2, w // 2)[...] = v
        return detect(packed_host, 'yuv420p', False)

    lines = []
    for comparison, fmt, arms in (('nv12_device', 'nv12', {'in_place': in_place, 'memcpy2d': memcpy2d}),
                                  ('yuv420p_host', 'yuv420p', {'planes': planes_arm, 'numpy': numpy_arm})):
        res = {a: {'device_fps': [], 'e2e_fps': []} for a in arms}
        last = {}
        for _ in range(args.rounds):
            timed(args, cams, arms, res, last, snapshot)
        # the last step used ring slot (steps - 1) % ring; compare against the packed frames of that slot
        k = ((args.steps - 1) % ring) * cams
        src = nv12 if fmt == 'nv12' else i420
        detect(src[k:k + cams], fmt, False)
        want = snapshot()
        same = all(last[a][0] == want[0] and np.array_equal(last[a][1], want[1]) for a in arms)
        line = {'workload': 'configs[2]' if (w, h, cams) == (640, 480, 8) else '1080p', 'comparison': comparison,
                'cameras': cams, 'frame': '%dx%d' % (w, h), 'steps': args.steps, 'rounds': args.rounds,
                'rows_equal_packed': bool(same)}
        if fmt == 'nv12':
            line['surface'] = {'pitch': pitch, 'chroma_row': luma_rows}
        else:
            line['linesize'] = linesize
        for a in arms:
            line[a] = {m: round(float(np.median(v)), 1) for m, v in res[a].items()}
            line[a]['spread'] = {m: [round(min(v), 1), round(max(v), 1)] for m, v in res[a].items()}
        lines.append((line, same))
    return lines


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--precision', type=int, default=2, help='2 = fp32 via 3xTF32 wgmma (bench.py\'s default)')
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    rt = cudart()
    info = card()
    ok = True
    with B200ObjectDetector(None, device=0, max_batch=8, precision=args.precision,
                            model_blob=workload.v2_coco_model().to_blob()) as det:
        for w, h, cams in ((640, 480, 8), (1920, 1080, 2)):
            for line, same in run_workload(det, w, h, cams, args, torch, rt):
                line.update(info)
                print(json.dumps(line), flush=True)
                ok = ok and same
    return 0 if ok else 1


if __name__ == '__main__':
    sys.exit(main())
