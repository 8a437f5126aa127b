#!/usr/bin/env python
"""Detection throughput by input pixel format: rgb24 against the 4:2:0 layouts decoders emit (yuv420p, NV12) and the
packed 4:2:2 layouts of webcams and capture cards (yuyv422, uyvy422).

    python tools/bench_yuv.py --steps 200 --warmup 20 --rounds 5

Workloads (tests/workload.py): BASELINE configs[2] (8 cameras of 640x480, SSD-MobileNet-v2 with 90 classes at score
threshold 1e-8, a mask per camera, fused filters) and 2 cameras of 1920x1080 with the same model.  The RGB frames are
cv2.cvtColor of the 4:2:0 ones and the 4:2:2 frames repeat each 4:2:0 chroma row for its two luma rows, so every format
computes the same rows, and the script checks that the last step's rows and verdicts are identical across the
formats.  Per format and round:
  device_fps  frames / s from the library's device time (CUDA events) with the frames resident on the GPU
  e2e_fps     frames / s of synchronous detect_batch calls from pinned host frames (H2D + kernels + D2H), wall clock
The formats run alternately within each round; the figures are the medians over rounds.  One JSON line per
workload, with the card's name, power limit and maximum SM clock."""
import argparse
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
from tests.yuv422_emulation import from_i420  # noqa: E402
from tests.yuv_emulation import cv2_rgb, from_rgb  # noqa: E402
from watsor_b200.detection.b200 import B200ObjectDetector  # noqa: E402

FORMATS = ('rgb24', 'yuv420p', 'nv12', 'yuyv422', 'uyvy422')


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True, check=True).stdout
    name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(',')]
    return {'gpu': name, 'power_limit': power, 'sm_max_clock': clock}


def frames_for(w, h, cams, ring):
    """ring x cams frames per format: 4:2:0 made from Artist frames, RGB = cvtColor of the yuv420p ones, 4:2:2 with
    the yuv420p ones' pixels"""
    out = {f: [] for f in FORMATS}
    for r in range(ring):
        for c in range(cams):
            rgb = artist_frame(w, h, c, r)
            i420 = from_rgb(rgb, 'yuv420p')
            out['yuv420p'].append(i420)
            out['nv12'].append(from_rgb(rgb, 'nv12'))
            out['rgb24'].append(np.ascontiguousarray(cv2_rgb(i420, 'yuv420p')))
            for f in ('yuyv422', 'uyvy422'):
                out[f].append(from_i420(i420, f))
    return out


def run_workload(det, name, w, h, cams, args, torch):
    for c in range(cams):
        det.configure_camera(c, w, h, workload.camera_config(c, w, h))
    ids = list(range(cams))
    ring = 4
    host = frames_for(w, h, cams, ring)
    pinned = {f: [torch.from_numpy(a).pin_memory() for a in host[f]] for f in FORMATS}
    dev = {f: [torch.from_numpy(a).cuda() for a in host[f]] for f in FORMATS}
    torch.cuda.synchronize()
    rows = new_rows(cams)
    verd = np.zeros((cams, 100), np.uint32)
    vptr = [verd[i] for i in range(cams)]

    def batch(f, step, src):
        k = (step % ring) * cams
        on_dev = src is dev
        ptrs = [t.data_ptr() for t in src[f][k:k + cams]]
        return det.detect_batch(ptrs, ids, rows, vptr, fuse_filters=True, frames_on_device=on_dev, pixel_format=f)

    res = {f: {'device_fps': [], 'e2e_fps': []} for f in FORMATS}
    last = {}
    for _ in range(args.rounds):
        for f in FORMATS:
            for s in range(args.warmup):
                batch(f, s, dev)
                batch(f, s, pinned)
            ms = [batch(f, s, dev) for s in range(args.steps)]
            res[f]['device_fps'].append(cams * 1000.0 / float(np.mean(ms)))
            t0 = time.perf_counter()
            for s in range(args.steps):
                batch(f, s, pinned)
            res[f]['e2e_fps'].append(cams * args.steps / (time.perf_counter() - t0))
            last[f] = ([rows_bytes(r) for r in rows], verd.copy())
    same = all(last[f][0] == last['rgb24'][0] and np.array_equal(last[f][1], last['rgb24'][1]) for f in FORMATS)
    line = {'workload': name, 'cameras': cams, 'frame': '%dx%d' % (w, h), 'steps': args.steps, 'rounds': args.rounds,
            'rows_identical_across_formats': same,
            'frame_bytes': {'rgb24': w * h * 3, 'yuv420p': w * h * 3 // 2, 'nv12': w * h * 3 // 2}}
    for f in FORMATS:
        line[f] = {k: round(float(np.median(v)), 1) for k, v in res[f].items()}
        line[f]['spread'] = {k: [round(min(v), 1), round(max(v), 1)] for k, v in res[f].items()}
    return line, same


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--precision', type=int, default=2, help='2 = fp32 via 3xTF32 wgmma (bench.py\'s default)')
    args = ap.parse_args()
    import torch
    info = card()
    ok = True
    with B200ObjectDetector(None, device=0, max_batch=8, precision=args.precision,
                            model_blob=workload.v2_coco_model().to_blob()) as det:
        for name, w, h, cams in (('configs[2]', 640, 480, 8), ('1080p', 1920, 1080, 2)):
            line, same = run_workload(det, name, w, h, cams, args, torch)
            line.update(info)
            print(json.dumps(line), flush=True)
            ok = ok and same
    return 0 if ok else 1


if __name__ == '__main__':
    sys.exit(main())
