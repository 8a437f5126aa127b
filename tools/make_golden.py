#!/usr/bin/env python
"""Generates tests/golden/* from an upstream watsor checkout (oracle/reference_build.py); outputs are committed.

Inputs follow the reference's own frame generator
(`watsor.test.detect_stream.Artist.draw_random_shapes`, detect_stream.py:42-70; restated in
tests/artist.py because the original passes floats to random.randrange, which Python 3.12
rejects) with `random.seed(1000*cam + frame)` (SURVEY.md 8d); expected outputs by the GraphDef-driven
oracle (oracle/ssd_graph.py) on the reference's vendored model
(watsor/test/model/cpu.pb).  NOT TensorFlow outputs: TensorFlow is not
installed, see oracle/__init__.py ("parity unpinned" at the TF boundary).
"""
import hashlib
import json
import os
import random
import sys

import numpy as np
from PIL import Image, ImageDraw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.reference_build import reference_dir  # noqa: E402

REF = reference_dir()
sys.path.insert(0, REF)

from tests.artist import draw_random_shapes  # noqa: E402  (restated recipe, see tests/artist.py)

from oracle.filters import AreaOracle, ConfidenceOracle, Det, MaskOracle, apply_predicates  # noqa: E402
from oracle.ssd_graph import SsdGraphOracle, to_detections  # noqa: E402

PB = os.path.join(REF, 'watsor/test/model/cpu.pb')
OUT = os.path.join(ROOT, 'tests', 'golden')
CASES = [(100, 100, 0, 0), (100, 100, 0, 1), (100, 100, 1, 0), (320, 240, 0, 0), (320, 240, 2, 5),
         (640, 480, 0, 0), (640, 480, 0, 1), (640, 480, 3, 7)]


def artist_frame(w, h, cam, frame):
    random.seed(1000 * cam + frame)
    with Image.new('RGB', (w, h)) as image:
        draw = ImageDraw.Draw(image)
        draw_random_shapes(image, draw)
        return np.array(image)


def f32hex(a):
    return np.ascontiguousarray(a, dtype='<f4').tobytes().hex()


def main():
    os.makedirs(os.path.join(OUT, 'frames'), exist_ok=True)
    o32 = SsdGraphOracle(PB, np.float32)
    o64 = SsdGraphOracle(PB, np.float64)
    porch = {'width': 640, 'height': 480, 'mask': os.path.join(REF, 'config/porch.png'),
             'detect': [{'person': {'confidence': 50, 'area': 1, 'zones': []}},      # label 1 = triangle
                        {'bicycle': {'confidence': 50, 'area': 1, 'zones': [2]}},    # label 2 = ellipse
                        {'car': {'confidence': 50, 'area': 10, 'zones': []}}]}       # label 3 = rectangle
    filters = [ConfidenceOracle(porch), AreaOracle(porch), MaskOracle(porch)]
    cases = []
    for (w, h, cam, frame) in CASES:
        img = artist_frame(w, h, cam, frame)
        name = 'artist_%dx%d_c%d_f%d' % (w, h, cam, frame)
        Image.fromarray(img).save(os.path.join(OUT, 'frames', name + '.png'))
        pre = o32.preprocess(img)
        enc, lg = o32.raw_heads(pre)
        b, s, cl, n = o32.postprocess(enc, lg)
        b64, s64, cl64, n64 = o64.postprocess(*o64.raw_heads(pre))
        rows = to_detections(b, cl, s, img.shape)
        case = {
            'name': name, 'width': w, 'height': h, 'cam': cam, 'frame': frame,
            'frame_md5': hashlib.md5(img.tobytes()).hexdigest(),
            'pre_md5': hashlib.md5(pre.tobytes()).hexdigest(),
            'enc_md5': hashlib.md5(enc.tobytes()).hexdigest(),
            'logits_md5': hashlib.md5(lg.tobytes()).hexdigest(),
            'num': int(n), 'boxes_f32': f32hex(b[:n]), 'scores_f32': f32hex(s[:n]),
            'classes': [int(x) for x in cl[:n]],
            'rows': [list(r) for r in rows[:n]],
            # float64 evaluation of the same graph: distance of each coordinate from an integer
            # boundary tells a test whether an int mismatch is a genuine rounding tie
            'num_f64': int(n64), 'boxes_f64': [[float(v) for v in bb] for bb in b64[:n64]],
        }
        if (w, h) == (640, 480):
            dets = [Det(r[0], r[1], (r[2], r[3], r[4], r[5])) for r in rows]
            _, verdicts = apply_predicates(dets, filters)
            case['porch_verdicts'] = verdicts[:n]
            case['porch_zones'] = [d.zones for d in dets[:n]]
        cases.append(case)
        print(name, n, rows[:n])
    meta = {
        'generator': 'tools/make_golden.py', 'model': 'watsor/test/model/cpu.pb (asmirnou/watsor @127f125)',
        'model_md5': hashlib.md5(open(PB, 'rb').read()).hexdigest(),
        'oracle': 'oracle/ssd_graph.py (numpy %s + torch-CPU %s fp32), NOT TensorFlow' % (
            np.__version__, __import__('torch').__version__),
        'porch_config': {k: v for k, v in porch.items() if k != 'mask'},
        'anchors_md5': hashlib.md5(o32.anchors.tobytes()).hexdigest(),
        'cases': cases,
    }
    with open(os.path.join(OUT, 'ssd_shapes_golden.json'), 'w') as f:
        json.dump(meta, f, indent=1)
    # the porch mask travels as a fixture too (config/porch.png is data, 640x480 RGBA)
    import shutil
    shutil.copy(os.path.join(REF, 'config/porch.png'), os.path.join(OUT, 'porch.png'))


if __name__ == '__main__':
    main()
