#!/usr/bin/env python
"""Effects-pass throughput by input and output pixel format: RGB24 output against the 4:2:0 layouts an encoder takes.

    python tools/bench_fx_formats.py --steps 200 --warmup 20 --rounds 5

Workload: bench.py's effects record -- 8 masked cameras of 640x480 (tests/workload.py), 8 labelled detections per
frame, BlendEffect + DrawEffectWithContours as one wb_fx_render per tick -- with the input in rgb24, NV12, YUYV or UYVY
and the output in rgb24, yuv420p or NV12.  The RGB input frames are cv2.cvtColor of the NV12 ones and the 4:2:2 ones
repeat each 4:2:0 chroma row for its two luma rows, so every combination renders the same pixels.  Per combination and round:
  device_fps  frames / s from the library's device time (CUDA events, kernels only) with device pointers
  e2e_fps     frames / s of synchronous wb_fx_render calls from pinned host frames to pinned host frames
              (H2D + kernels + D2H), wall clock
The combinations run alternately within each round; the figures are the medians over rounds.  The script checks that
every 4:2:0 output equals cv2.cvtColor(COLOR_RGB2YUV_I420) (NV12: the same bytes interleaved) of the RGB24 output of
the same input, and prints one JSON line with the card's name, power limit and maximum SM clock."""
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
from tests.yuv422_emulation import from_i420  # noqa: E402
from tests.yuv_emulation import cv2_rgb, from_rgb  # noqa: E402
from watsor_b200.engine import frame_shape  # noqa: E402
from watsor_b200.filter.mask import get_alpha_channel  # noqa: E402
from watsor_b200.output.effects import (WB_FX_BLEND, WB_FX_CONTOURS, WB_FX_DRAW, WB_FX_ON_DEVICE,  # noqa: E402
                                        EffectsEngine, contour_bits)

IN_FORMATS = ('rgb24', 'nv12', 'yuyv422', 'uyvy422')
OUT_FORMATS = ('rgb24', 'yuv420p', 'nv12')
CAMS, W, H = 8, 640, 480


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True, check=True).stdout
    name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(',')]
    return {'gpu': name, 'power_limit': power, 'sm_max_clock': clock}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    import torch
    info = card()
    rng = np.random.default_rng(3)
    eng = EffectsEngine(0)
    cams, rows, frames = [], [], {f: [] for f in IN_FORMATS}
    for c in range(CAMS):
        alpha, _ = get_alpha_channel(workload.camera_config(c)['mask'], W, H)
        cams.append(eng.add_camera(W, H, alpha, contour_bits(alpha)))
        rows.append(random_rows(rng, W, H, 8, n_zones=1))
        i420 = from_rgb(artist_frame(W, H, c, 0), 'yuv420p')
        nv12 = from_rgb(artist_frame(W, H, c, 0), 'nv12')
        frames['nv12'].append(nv12)
        for f in ('yuyv422', 'uyvy422'):
            frames[f].append(from_i420(i420, f))
        frames['rgb24'].append(np.ascontiguousarray(cv2_rgb(nv12, 'nv12')))
    flags = WB_FX_BLEND | WB_FX_DRAW | WB_FX_CONTOURS
    combos = [(i, o) for i in IN_FORMATS for o in OUT_FORMATS]
    d_in = {f: [torch.from_numpy(a).cuda() for a in frames[f]] for f in IN_FORMATS}
    d_out = {f: [torch.empty(frame_shape(f, W, H), dtype=torch.uint8, device='cuda') for _ in range(CAMS)]
             for f in OUT_FORMATS}
    h_in = {f: [torch.from_numpy(a).pin_memory().numpy() for a in frames[f]] for f in IN_FORMATS}
    h_out = {f: [torch.empty(frame_shape(f, W, H), dtype=torch.uint8).pin_memory().numpy() for _ in range(CAMS)]
             for f in OUT_FORMATS}
    torch.cuda.synchronize()

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
            res[(i, o)]['device_fps'].append(CAMS * 1000.0 / float(np.median(ms)))
            t0 = time.perf_counter()
            for _ in range(args.steps):
                from_host(i, o)
            res[(i, o)]['e2e_fps'].append(CAMS * args.steps / (time.perf_counter() - t0))
            # the host outputs of the last call, against cvtColor of this input's RGB24 output
            if o == 'rgb24':
                rgb_out = [a.copy() for a in h_out['rgb24']]
            else:
                same = same and all(np.array_equal(h_out[o][k], from_rgb(rgb_out[k], o)) for k in range(CAMS))
                same = same and all(np.array_equal(d_out[o][k].cpu().numpy(), h_out[o][k]) for k in range(CAMS))
    eng.close()
    line = {'workload': 'bench.py effects record, %d masked cameras of %dx%d, 8 labels per frame' % (CAMS, W, H),
            'chain': 'BlendEffect + DrawEffectWithContours, one wb_fx_render per tick', 'steps': args.steps,
            'rounds': args.rounds, 'outputs_equal_cvtcolor_of_rgb24_output': same}
    for i, o in combos:
        key = '%s->%s' % (i, o)
        line[key] = {k: round(float(np.median(v)), 1) for k, v in res[(i, o)].items()}
        line[key]['spread'] = {k: [round(min(v), 1), round(max(v), 1)] for k, v in res[(i, o)].items()}
        line[key]['in_bytes_per_frame'] = frames[i][0].nbytes
        line[key]['out_bytes_per_frame'] = int(np.prod(frame_shape(o, W, H)))
    line.update(info)
    print(json.dumps(line), flush=True)
    assert same, '4:2:0 output differs from cv2.cvtColor of the RGB24 output'
    return 0


if __name__ == '__main__':
    sys.exit(main())
