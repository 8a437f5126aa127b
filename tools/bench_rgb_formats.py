#!/usr/bin/env python
"""Detection and effects-pass throughput by packed RGB byte order: rgb24 against OpenCV's bgr24 and the 4-byte rgba /
bgra of GPU pipelines, and the effects pass's bgr24 output (for cv2.imencode) against its other outputs.

    python tools/bench_rgb_formats.py --steps 200 --warmup 20 --rounds 5

Detection workloads (tests/workload.py): BASELINE configs[2] (8 cameras of 640x480, SSD-MobileNet-v2 with 90 classes at
score threshold 1e-8, a mask per camera, fused filters) and 2 cameras of 1920x1080 with the same model.  The frames of
every order hold the pixels of the same Artist frames, so every order computes the same rows; the script checks that
the last step's rows and verdicts are identical across the orders.  Per order and round:
  device_fps  frames / s from the library's device time (CUDA events) with the frames resident on the GPU
  e2e_fps     frames / s of synchronous detect_batch calls from pinned host frames (H2D + kernels + D2H), wall clock
Effects workload: bench.py's effects record (8 masked cameras of 640x480, 8 labelled detections per frame,
BlendEffect + DrawEffectWithContours as one wb_fx_render per tick) from every input order to every output layout
(rgb24, bgr24, yuv420p, nv12), device_fps and e2e_fps as above; the script checks each output against cv2.cvtColor of
the RGB24 call's output.  Orders and pairs run alternately within each round; the figures are the medians over rounds.
One JSON line per workload, with the card's name, power limit and maximum SM clock."""
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
from tests.fx_cases import random_rows  # noqa: E402
from tests.gpu_util import new_rows, rows_bytes  # noqa: E402
from tests.rgb_orders import cv2_bgr, from_rgb  # noqa: E402
from tests.yuv_out_emulation import to_yuv420  # noqa: E402
from watsor_b200.detection.b200 import B200ObjectDetector  # noqa: E402
from watsor_b200.engine import layout_shape  # noqa: E402

DETECT_FORMATS = ('rgb24', 'bgr24', 'rgba', 'bgra')
FX_IN = ('rgb24', 'bgr24', 'rgba', 'bgra')
FX_OUT = ('rgb24', 'bgr24', 'yuv420p', 'nv12')


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True, check=True).stdout
    name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(',')]
    return {'gpu': name, 'power_limit': power, 'sm_max_clock': clock}


def summary(res):
    out = {k: round(float(np.median(v)), 1) for k, v in res.items()}
    out['spread'] = {k: [round(min(v), 1), round(max(v), 1)] for k, v in res.items()}
    return out


def run_detection(det, name, w, h, cams, args, torch):
    for c in range(cams):
        det.configure_camera(c, w, h, workload.camera_config(c, w, h))
    ids = list(range(cams))
    ring = 4
    rng = np.random.default_rng(1)
    host = {f: [] for f in DETECT_FORMATS}
    for r in range(ring):
        for c in range(cams):
            rgb = artist_frame(w, h, c, r)
            for f in DETECT_FORMATS:
                host[f].append(from_rgb(rgb, f, rng))
    pinned = {f: [torch.from_numpy(a).pin_memory() for a in host[f]] for f in DETECT_FORMATS}
    dev = {f: [torch.from_numpy(a).cuda() for a in host[f]] for f in DETECT_FORMATS}
    torch.cuda.synchronize()
    rows = new_rows(cams)
    verd = np.zeros((cams, 100), np.uint32)
    vptr = [verd[i] for i in range(cams)]

    def batch(f, step, src):
        k = (step % ring) * cams
        ptrs = [t.data_ptr() for t in src[f][k:k + cams]]
        return det.detect_batch(ptrs, ids, rows, vptr, fuse_filters=True, frames_on_device=src is dev, pixel_format=f)

    res = {f: {'device_fps': [], 'e2e_fps': []} for f in DETECT_FORMATS}
    last = {}
    for _ in range(args.rounds):
        for f in DETECT_FORMATS:
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
    same = all(last[f][0] == last['rgb24'][0] and np.array_equal(last[f][1], last['rgb24'][1]) for f in DETECT_FORMATS)
    line = {'workload': name, 'cameras': cams, 'frame': '%dx%d' % (w, h), 'steps': args.steps, 'rounds': args.rounds,
            'rows_identical_across_formats': same,
            'frame_bytes': {f: host[f][0].nbytes for f in DETECT_FORMATS}}
    for f in DETECT_FORMATS:
        line[f] = summary(res[f])
    return line, same


def run_effects(args, torch):
    from watsor_b200.filter.mask import get_alpha_channel
    from watsor_b200.output.effects import (WB_FX_BLEND, WB_FX_CONTOURS, WB_FX_DRAW, WB_FX_ON_DEVICE, EffectsEngine,
                                            contour_bits)
    n, w, h = 8, 640, 480
    rng = np.random.default_rng(3)
    eng = EffectsEngine(0)
    cams, rows, frames = [], [], {f: [] for f in FX_IN}
    for c in range(n):
        alpha, _ = get_alpha_channel(workload.camera_config(c)['mask'], w, h)
        cams.append(eng.add_camera(w, h, alpha, contour_bits(alpha)))
        rows.append(random_rows(rng, w, h, 8, n_zones=1))
        rgb = artist_frame(w, h, c, 0)
        for f in FX_IN:
            frames[f].append(from_rgb(rgb, f, rng))
    flags = WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS
    combos = [(i, o) for i in FX_IN for o in FX_OUT]
    d_in = {f: [torch.from_numpy(a).cuda() for a in frames[f]] for f in FX_IN}
    d_out = {f: [torch.empty(layout_shape(f, w, h), dtype=torch.uint8, device='cuda') for _ in range(n)]
             for f in FX_OUT}
    h_in = {f: [torch.from_numpy(a).pin_memory().numpy() for a in frames[f]] for f in FX_IN}
    h_out = {f: [torch.empty(layout_shape(f, w, h), dtype=torch.uint8).pin_memory().numpy() for _ in range(n)]
             for f in FX_OUT}
    torch.cuda.synchronize()
    ref = [np.zeros((h, w, 3), np.uint8) for _ in range(n)]
    eng.render(frames['rgb24'], ref, cams, rows, flags)
    want = {'rgb24': ref, 'bgr24': [cv2_bgr(r) for r in ref], 'yuv420p': [to_yuv420(r, 'yuv420p') for r in ref],
            'nv12': [to_yuv420(r, 'nv12') for r in ref]}

    def on_device(i, o):
        return eng.render([t.data_ptr() for t in d_in[i]], [t.data_ptr() for t in d_out[o]], cams, rows,
                          flags | WB_FX_ON_DEVICE, pixel_format=i, output_format=o)

    def from_host(i, o):
        return eng.render(h_in[i], h_out[o], cams, rows, flags, pixel_format=i, output_format=o)

    res = {c: {'device_fps': [], 'e2e_fps': []} for c in combos}
    same = True
    for _ in range(args.rounds):
        for i, o in combos:
            for _ in range(args.warmup):
                on_device(i, o)
                from_host(i, o)
            ms = [on_device(i, o) for _ in range(args.steps)]
            res[(i, o)]['device_fps'].append(n * 1000.0 / float(np.median(ms)))
            t0 = time.perf_counter()
            for _ in range(args.steps):
                from_host(i, o)
            res[(i, o)]['e2e_fps'].append(n * args.steps / (time.perf_counter() - t0))
            same = same and all(np.array_equal(h_out[o][k], want[o][k]) for k in range(n))
            same = same and all(np.array_equal(d_out[o][k].cpu().numpy(), want[o][k]) for k in range(n))
    eng.close()
    line = {'workload': 'bench.py effects record, %d masked cameras of %dx%d, 8 labels per frame' % (n, w, h),
            'chain': 'BlendEffect + DrawEffectWithContours, one wb_fx_render per tick', 'steps': args.steps,
            'rounds': args.rounds, 'outputs_equal_cvtcolor_of_rgb24_output': same}
    for i, o in combos:
        line['%s->%s' % (i, o)] = summary(res[(i, o)])
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
            line, same = run_detection(det, name, w, h, cams, args, torch)
            line.update(info)
            print(json.dumps(line), flush=True)
            ok = ok and same
    line, same = run_effects(args, torch)
    line.update(info)
    print(json.dumps(line), flush=True)
    return 0 if ok and same else 1


if __name__ == '__main__':
    sys.exit(main())
