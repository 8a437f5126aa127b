#!/usr/bin/env python
"""Device time of the post stage (per-class NMS, top-100 merge, predicates) inside the graphed detection step.

    python tools/bench_post.py --steps 1000 --warmup 50 --profile-steps 200

Workload: BASELINE configs[2] (tests/workload.py): 8 cameras of 640x480, SSD-MobileNet-v2 with 90 classes at score
threshold 1e-8 (every anchor is a candidate in every class), a mask per camera, fused filters, frames resident on the
GPU, six batches in flight through submit / collect as bench.py runs them.  Two runs in one process:
  timing    the step loop with the profiler off: ms_per_step from CUDA events around the loop
  profile   the same loop under torch.profiler (CUDA activities): device time per kernel, summed over the steps of
            the profiled window and divided by their number.  `post` lists the post-stage kernels, `all_kernels_us`
            is the sum over every kernel of the step (the SM-time the step asks for; with several batches in flight
            kernels overlap, so it exceeds ms_per_step), and `post_share` is the post kernels' part of it.
One JSON line, with the card's name, power limit and maximum SM clock, and the median SM clock during the timing run."""
import argparse
import json
import os
import subprocess
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import workload  # noqa: E402
from tests.artist import artist_frame  # noqa: E402
from tools.bench_yuv import card  # noqa: E402
from watsor_b200.detection.b200 import B200ObjectDetector  # noqa: E402
from watsor_b200.engine import PRECISIONS  # noqa: E402

MODES = {m: PRECISIONS[m] for m in ('fp32', 'bf16', 'fp16', 'tf32x3')}
CAMS, W, H, RING, SLOTS = 8, 640, 480, 8, 6
POST_KERNELS = ('k_decode_scores', 'k_nms', 'k_merge_filter')


class SmClock:
    """nvidia-smi's SM clock every 100 ms while the timing loop runs."""

    def __init__(self):
        self.samples, self.proc = [], None

    def __enter__(self):
        self.proc = subprocess.Popen(['nvidia-smi', '-i', '0', '--query-gpu=clocks.sm', '--format=csv,noheader,nounits',
                                      '-lms', '100'], stdout=subprocess.PIPE, text=True)
        self.thread = threading.Thread(target=self._read, daemon=True)
        self.thread.start()
        return self

    def _read(self):
        for line in self.proc.stdout:
            if line.strip().isdigit():
                self.samples.append(int(line))

    def __exit__(self, *exc):
        self.proc.terminate()
        self.proc.wait()
        self.thread.join(timeout=2)

    def median(self):
        return float(np.median(self.samples)) if self.samples else None


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--profile-steps', type=int, default=200)
    ap.add_argument('--precision', default='tf32x3', choices=sorted(MODES))
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from watsor_b200.stream.share import Detection
    line = {'workload': 'configs[2]', 'cameras': CAMS, 'frame': '%dx%d' % (W, H), 'precision': args.precision,
            'batches_in_flight': SLOTS}
    line.update(card())
    model = workload.v2_coco_model()
    det = B200ObjectDetector(None, device=0, max_batch=CAMS, precision=MODES[args.precision],
                             model_blob=model.to_blob())
    ids = list(range(CAMS))
    for c in ids:
        det.configure_camera(c, W, H, workload.camera_config(c, W, H))
    dev = [torch.from_numpy(artist_frame(W, H, c, r)).cuda() for r in range(RING) for c in range(CAMS)]
    rows = [[(Detection * 100)() for _ in range(CAMS)] for _ in range(SLOTS)]
    verd = [[np.zeros(100, np.uint32) for _ in range(CAMS)] for _ in range(SLOTS)]
    torch.cuda.synchronize()

    def steps(n):
        for i in range(n):
            s = i % SLOTS
            if i >= SLOTS:
                det.collect(s, rows[s], verd[s])
            k = (i % RING) * CAMS
            det.submit(s, [t.data_ptr() for t in dev[k:k + CAMS]], ids, fuse_filters=True, frames_on_device=True)
        for i in range(max(0, n - SLOTS), n):
            det.collect(i % SLOTS, rows[i % SLOTS], verd[i % SLOTS])

    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    steps(args.warmup)
    line['launches_per_step'] = det.engine.last_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with SmClock() as clk:
        torch.cuda.synchronize()
        e0.record(stream)
        det.engine.stream_fence(stream.cuda_stream, 0)
        steps(args.steps)
        det.engine.stream_fence(stream.cuda_stream, 1)
        e1.record(stream)
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    line.update({'steps': args.steps, 'ms_per_step': round(ms, 4), 'value': round(CAMS * 1e3 / ms, 1),
                 'sm_clock_median_mhz': clk.median()})

    steps(args.warmup)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        steps(args.profile_steps)
        torch.cuda.synchronize()
    per_kernel = {}
    for ev in prof.events():
        if ev.device_type.name != 'CUDA' or ev.device_time <= 0:
            continue
        k = per_kernel.setdefault(ev.name, [0, 0.0])
        k[0] += 1
        k[1] += ev.device_time  # us
    n = args.profile_steps
    total = sum(t for name, (_, t) in per_kernel.items() if not name.startswith('Memset') and 'Memcpy' not in name)
    post = {name: {'calls_per_step': round(cnt / n, 2), 'us_per_step': round(t / n, 2)}
            for name, (cnt, t) in per_kernel.items() if any(name.startswith(p) for p in POST_KERNELS)}
    post_us = sum(v['us_per_step'] for v in post.values())
    line.update({'profile_steps': n, 'post': post, 'post_us_per_step': round(post_us, 2),
                 'all_kernels_us_per_step': round(total / n, 2),
                 'post_share': round(post_us / (total / n), 4) if total else None,
                 'top_kernels': sorted(([name[:60], round(t / n, 2)] for name, (_, t) in per_kernel.items()),
                                       key=lambda x: -x[1])[:12]})
    det.engine.close()
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
