#!/usr/bin/env python
"""Detection throughput with detection windows (wb_set_camera_windows) on high-resolution cameras.

    python tools/bench_windows.py --steps 100 --warmup 10 --rounds 3

Workload: 8 cameras of 1920x1080 (Artist frames), SSD-MobileNet-v2 with 90 classes at score threshold 1e-8 and a mask
per camera (tests/workload.py), fused filters, fp32 via 3xTF32 wgmma.  Window layouts (watsor_b200.windows.grid_windows):
  none      the whole frame only (today's path, 8 model images per batch)
  full+2x2  the whole frame and a 2x2 grid (40 model images)
  full+3x2  the whole frame and a 3x2 grid (56 model images)
Per layout, the medians over rounds of
  device_fps  frames / s from the library's device time (CUDA events) with the frames resident on the GPU
  e2e_fps     frames / s of synchronous detect_batch calls from pinned host frames (H2D + kernels + D2H), wall clock
  images_per_s = device_fps x model images per frame
  merge_us    mean device time of one k_window_merge launch (torch.profiler, CUDA activities, a separate pass)
The layouts run alternately within each round.  One JSON line per layout, with the card's name, power limit and
maximum SM clock read in the same run."""
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
from tests.gpu_util import new_rows  # noqa: E402
from watsor_b200.detection.b200 import B200ObjectDetector  # noqa: E402
from watsor_b200.windows import grid_windows  # noqa: E402

W, H, CAMS = 1920, 1080, 8
LAYOUTS = (('none', None), ('full+2x2', (2, 2)), ('full+3x2', (3, 2)))


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True, check=True).stdout
    name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(',')]
    return {'gpu': name, 'power_limit': power, 'sm_max_clock': clock}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    import torch
    info = card()
    ring = 2
    host = [artist_frame(W, H, c, r) for r in range(ring) for c in range(CAMS)]
    pinned = [torch.from_numpy(a).pin_memory() for a in host]
    dev = [torch.from_numpy(a).cuda() for a in host]
    torch.cuda.synchronize()
    ids = list(range(CAMS))
    rows = new_rows(CAMS)
    verd = np.zeros((CAMS, 100), np.uint32)
    vptr = [verd[i] for i in range(CAMS)]
    windows = {name: (grid_windows(W, H, *grid) if grid else []) for name, grid in LAYOUTS}
    max_images = CAMS * max(max(len(w) for w in windows.values()), 1)
    with B200ObjectDetector(None, device=0, max_batch=max_images, precision=2,
                            model_blob=workload.v2_coco_model().to_blob()) as det:
        for c in ids:
            det.configure_camera(c, W, H, workload.camera_config(c, W, H))

        def use(name):
            for c in ids:
                det.engine.set_camera_windows(c, windows[name])

        def batch(step, src):
            k = (step % ring) * CAMS
            ptrs = [t.data_ptr() for t in src[k:k + CAMS]]
            return det.detect_batch(ptrs, ids, rows, vptr, fuse_filters=True, frames_on_device=src is dev)

        res = {name: {'device_fps': [], 'e2e_fps': []} for name, _ in LAYOUTS}
        launches = {}
        for _ in range(args.rounds):
            for name, _ in LAYOUTS:
                use(name)
                for s in range(args.warmup):
                    batch(s, dev)
                    batch(s, pinned)
                ms = [batch(s, dev) for s in range(args.steps)]
                launches[name] = det.engine.last_launch_count()
                res[name]['device_fps'].append(CAMS * 1000.0 / float(np.mean(ms)))
                t0 = time.perf_counter()
                for s in range(args.steps):
                    batch(s, pinned)
                res[name]['e2e_fps'].append(CAMS * args.steps / (time.perf_counter() - t0))
        merge_us = {}
        from torch.profiler import ProfilerActivity, profile
        for name, grid in LAYOUTS:
            if not grid:
                continue
            use(name)
            batch(0, dev)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for s in range(20):
                    batch(s, dev)
                torch.cuda.synchronize()
            times = [e.device_time for e in prof.events() if 'k_window_merge' in e.name]
            merge_us[name] = round(float(np.mean(times)), 2) if times else None
    for name, _ in LAYOUTS:
        per_frame = max(len(windows[name]), 1)
        line = {'layout': name, 'cameras': CAMS, 'frame': '%dx%d' % (W, H), 'model_images_per_frame': per_frame,
                'steps': args.steps, 'rounds': args.rounds, 'launches': launches[name]}
        line.update({k: round(float(np.median(v)), 1) for k, v in res[name].items()})
        line['images_per_s'] = round(line['device_fps'] * per_frame, 1)
        line['spread'] = {k: [round(min(v), 1), round(max(v), 1)] for k, v in res[name].items()}
        line['merge_us'] = merge_us.get(name)
        line.update(info)
        print(json.dumps(line), flush=True)
    return 0


if __name__ == '__main__':
    sys.exit(main())
