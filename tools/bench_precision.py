#!/usr/bin/env python
"""Detection throughput and accuracy by precision mode: bf16 and fp16 (the 16-bit tensor-core modes) against tf32x3
(the fp32-faithful default).

    python tools/bench_precision.py --steps 200 --warmup 20 --rounds 5

Workload: BASELINE configs[2] (tests/workload.py): 8 cameras of 640x480, SSD-MobileNet-v2 with 90 classes at score
threshold 1e-8, a mask per camera, fused filters.  One detector per mode lives in the process; the modes run
alternately within each round, and the figures are the medians over rounds.  Per mode:
  device_fps        frames / s from the library's device time (CUDA events), frames resident on the GPU
  e2e_fps           frames / s of synchronous detect_batch calls from pinned host frames (H2D + kernels + D2H)
  launches          kernel launches per step (the 16-bit modes run the same plan, so they must be equal)
  layer_err         max |GPU - fp32 oracle| / max(1, max |oracle|) per backbone layer (the measure of
                    tests/test_gpu_v2.py::test_v2_layer_by_layer), over two frames: worst and median layer; 16-bit
                    modes only
  rows_equal_tf32x3 the share of rows whose label and integer box equal tf32x3's on the same frames
One JSON line, with the card's name, power limit and maximum SM clock."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import workload  # noqa: E402
from tests.artist import artist_frame  # noqa: E402
from tests.gpu_util import new_rows, rows_to_tuples  # noqa: E402
from tools.bench_yuv import card  # noqa: E402
from watsor_b200.detection.b200 import B200ObjectDetector  # noqa: E402
from watsor_b200.engine import PRECISIONS  # noqa: E402
from watsor_b200.model import OP_HEAD  # noqa: E402

MODES = {m: PRECISIONS[m] for m in ('bf16', 'fp16', 'tf32x3')}
CAMS, W, H, RING = 8, 640, 480, 4


def layer_error(det, model, oracle, frames):
    err = {}
    for img in frames:
        pre = oracle.preprocess(img)
        _, _, memo = oracle.raw_heads(pre, return_memo=True)
        for li, layer in enumerate(model.layers):
            if layer.op == OP_HEAD:
                continue
            want = oracle.feature(memo, li)
            got = det.engine.backbone(pre[None], stop_layer=li, layer_shape=want.shape)[2][0]
            e = float(np.abs(got - want).max()) / max(1.0, float(np.abs(want).max()))
            err[li] = max(err.get(li, 0.0), e)
    return {'worst': float('%.3g' % max(err.values())), 'median': float('%.3g' % np.median(list(err.values())))}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    import torch
    from oracle.ssd_model import SsdModelOracle
    info = card()
    model = workload.v2_coco_model()
    blob = model.to_blob()
    host = [artist_frame(W, H, c, r) for r in range(RING) for c in range(CAMS)]
    pinned = [torch.from_numpy(a).pin_memory() for a in host]
    dev = [torch.from_numpy(a).cuda() for a in host]
    torch.cuda.synchronize()
    ids = list(range(CAMS))
    dets = {m: B200ObjectDetector(None, device=0, max_batch=CAMS, precision=p, model_blob=blob) for m, p in MODES.items()}
    for det in dets.values():
        for c in ids:
            det.configure_camera(c, W, H, workload.camera_config(c, W, H))
    rows = new_rows(CAMS)

    def batch(det, step, src):
        k = (step % RING) * CAMS
        return det.detect_batch([t.data_ptr() for t in src[k:k + CAMS]], ids, rows, fuse_filters=True,
                                frames_on_device=src is dev)

    res = {m: {'device_fps': [], 'e2e_fps': []} for m in MODES}
    launches = {}
    for _ in range(args.rounds):
        for m, det in dets.items():
            for s in range(args.warmup):
                batch(det, s, dev)
                batch(det, s, pinned)
            ms = [batch(det, s, dev) for s in range(args.steps)]
            launches[m] = det.engine.last_launch_count()
            res[m]['device_fps'].append(CAMS * 1000.0 / float(np.mean(ms)))
            t0 = time.perf_counter()
            for s in range(args.steps):
                batch(det, s, pinned)
            res[m]['e2e_fps'].append(CAMS * args.steps / (time.perf_counter() - t0))
    # accuracy: rows of every ring frame against tf32x3's, per-layer error against the fp32 oracle
    got = {}
    for m, det in dets.items():
        got[m] = []
        for r in range(RING):
            batch(det, r, dev)
            got[m] += [[t[:1] + t[2:] for t in rows_to_tuples(x)] for x in rows]
    oracle = SsdModelOracle(model)
    line = {'workload': 'configs[2]', 'cameras': CAMS, 'frame': '%dx%d' % (W, H), 'steps': args.steps,
            'rounds': args.rounds}
    for m, det in dets.items():
        line[m] = {k: round(float(np.median(v)), 1) for k, v in res[m].items()}
        line[m]['spread'] = {k: [round(min(v), 1), round(max(v), 1)] for k, v in res[m].items()}
        line[m]['launches'] = launches[m]
        pairs = [(a, b) for fa, fb in zip(got[m], got['tf32x3']) for a, b in zip(fa, fb)]
        line[m]['rows_equal_tf32x3'] = round(sum(a == b for a, b in pairs) / len(pairs), 4)
        if m != 'tf32x3':
            line[m]['layer_err'] = layer_error(det, model, oracle, host[:2])
    for det in dets.values():
        det.engine.close()
    line.update(info)
    print(json.dumps(line), flush=True)
    return 0 if launches['fp16'] == launches['bf16'] else 1


if __name__ == '__main__':
    sys.exit(main())
