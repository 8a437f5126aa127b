#!/usr/bin/env python
"""Pin the oracle's conv arithmetic with an INDEPENDENT executor of the reference's own graph.

    python tools/make_golden_cvdnn.py            (needs an upstream checkout; writes tests/golden/cvdnn_heads.npz)

TensorFlow -- the sole owner of the conv arithmetic in the reference (watsor/detection/tensorflow_cpu.py:104-121)
-- cannot be installed here, and the reference's only model test asserts a detection count, not tensors
(watsor/test/test_detect.py:28-77).  OpenCV's dnn module *is* in the image and has its own importer and its own
CPU kernels for TensorFlow GraphDefs.  This script

  1. cuts the vendored frozen graph `watsor/test/model/cpu.pb` down to the sub-graph between
     `Preprocessor/sub` (replaced by a float32 Placeholder, 1x300x300x3) and the twelve head tensors
     `BoxPredictor_i/{BoxEncodingPredictor,ClassPredictor}/BiasAdd` -- Conv2D, DepthwiseConv2dNative,
     FusedBatchNormV3, Relu6, BiasAdd, Identity and Const nodes only, weights untouched;
  2. runs it with `cv2.dnn.readNetFromTensorflow(...).forward(...)` on pre-processed Artist frames;
  3. stores the twelve outputs (re-ordered NCHW -> NHWC and concatenated exactly as the graph's own
     Reshape + `concat` / `concat_1` nodes do) as golden vectors, labelled "OpenCV-dnn, not TensorFlow".

tests/test_oracle_cvdnn.py asserts `oracle.raw_heads(pre)` equals these vectors to 1e-4 (CPU suite, reads only
the committed .npz), and -- where an upstream checkout is present -- re-runs OpenCV live.  What this pins: 99 % of the
arithmetic (every convolution, batch norm, activation and bias of the backbone and heads; SAME padding, strides,
layout).  What it does NOT pin: the legacy ResizeBilinear, the anchor generator, box decoding, sigmoid,
NonMaxSuppressionV5 and the top-100 assembly -- those remain restated from the graph/TF kernel semantics
(oracle/ssd_graph.py) and are checked for bit-exactness GPU-vs-oracle only.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.reference_build import reference_pb  # noqa: E402

REF_PB = reference_pb()
OUT = os.path.join(ROOT, 'tests', 'golden', 'cvdnn_heads.npz')
CUT_INPUT = 'Preprocessor/sub'
FRAMES = [(100, 100, 1, 0), (320, 240, 2, 1), (640, 480, 3, 2)]     # (w, h, cam, frame) of tests/artist.py


def head_nodes(g):
    """The BiasAdd node behind every Reshape that feeds `concat` (boxes) / `concat_1` (classes)."""
    def bias_of(reshape):
        b = g.inputs(reshape)[0][0]
        assert g.node(b).op == 'BiasAdd', (reshape, g.node(b).op)
        return b
    boxes = [bias_of(i[0]) for i in g.inputs('concat')[:-1]]
    classes = [bias_of(i[0]) for i in g.inputs('concat_1')[:-1]]
    return boxes, classes


def dnn_layer_name(g_inputs, bias_node):
    """OpenCV's importer folds a BiasAdd into the convolution layer in front of it and keeps the Conv2D's name."""
    return g_inputs(bias_node)[0][0]


def cut_graph(pb_path):
    """-> (serialized GraphDef of the sub-graph, box head names, class head names, num_classes + 1)"""
    from tensorboard.compat.proto import graph_pb2, types_pb2

    from oracle.tf_graph import FrozenGraph
    g = FrozenGraph(pb_path)
    boxes, classes = head_nodes(g)
    keep, stack = set(), list(boxes + classes)
    while stack:
        name = stack.pop()
        if name in keep or name == CUT_INPUT:
            continue
        keep.add(name)
        stack.extend(i[0] for i in g.inputs(name))
    allowed = {'Conv2D', 'DepthwiseConv2dNative', 'FusedBatchNormV3', 'FusedBatchNorm', 'Relu6', 'BiasAdd', 'Identity',
               'Const'}
    ops = {g.node(n).op for n in keep}
    assert ops <= allowed, ops - allowed
    out = graph_pb2.GraphDef()
    ph = out.node.add()
    ph.name = CUT_INPUT
    ph.op = 'Placeholder'
    ph.attr['dtype'].type = types_pb2.DT_FLOAT
    for d in (1, 300, 300, 3):
        ph.attr['shape'].shape.dim.add().size = d
    for name in g.order:                       # original (topological) order
        if name not in keep:
            continue
        n = out.node.add()
        n.CopyFrom(g.node(name))
        del n.input[:]
        n.input.extend(i for i in g.node(name).input if not i.startswith('^'))
        if n.op == 'FusedBatchNormV3':
            # same inference arithmetic; OpenCV's importer knows the op under its V1 name
            n.op = 'FusedBatchNorm'
            if 'U' in n.attr:
                del n.attr['U']
    ncp1 = int(g.const(g.inputs(g.inputs(g.inputs('concat_1')[0][0])[1][0])[-1][0]))
    return (out.SerializeToString(), [dnn_layer_name(g.inputs, b) for b in boxes],
            [dnn_layer_name(g.inputs, c) for c in classes], ncp1)


def run_cvdnn(graph_bytes, boxes, classes, ncp1, pre_hwc, fusion=True):
    """pre-processed [300,300,3] f32 -> (box_encodings [N,4], class_logits [N,C+1]) by OpenCV's dnn module."""
    import cv2
    net = cv2.dnn.readNetFromTensorflow(np.frombuffer(graph_bytes, np.uint8))
    net.setPreferableBackend(cv2.dnn.DNN_BACKEND_OPENCV)
    net.setPreferableTarget(cv2.dnn.DNN_TARGET_CPU)
    net.enableFusion(fusion)      # True (OpenCV's default): BN/ReLU6 folded into the conv layers; False: layer by layer
    blob = np.ascontiguousarray(pre_hwc.transpose(2, 0, 1)[None].astype(np.float32))     # NCHW, as dnn expects
    net.setInput(blob)
    outs = net.forward(boxes + classes)
    enc = [o[0].transpose(1, 2, 0).reshape(-1, 4) for o in outs[:len(boxes)]]             # graph: Reshape [B,-1,1,4]
    lg = [o[0].transpose(1, 2, 0).reshape(-1, ncp1) for o in outs[len(boxes):]]           # graph: Reshape [B,-1,C+1]
    return np.concatenate(enc, 0), np.concatenate(lg, 0)


def main():
    import cv2

    from oracle.ssd_graph import SsdGraphOracle
    from tests.artist import artist_frame
    graph_bytes, boxes, classes, ncp1 = cut_graph(REF_PB)
    oracle = SsdGraphOracle(REF_PB)
    store = {'opencv_version': np.array(cv2.__version__), 'source': np.array('OpenCV-dnn, not TensorFlow')}
    for (w, h, cam, frame) in FRAMES:
        pre = oracle.preprocess(artist_frame(w, h, cam, frame))
        enc, lg = run_cvdnn(graph_bytes, boxes, classes, ncp1, pre)
        oenc, olg = oracle.raw_heads(pre)
        enc_nf, lg_nf = run_cvdnn(graph_bytes, boxes, classes, ncp1, pre, fusion=False)
        print('   unfused OpenCV run vs fused: %.3g %.3g' % (np.abs(enc_nf - enc).max(), np.abs(lg_nf - lg).max()))
        key = 'artist_%dx%d_c%d_f%d' % (w, h, cam, frame)
        store[key + '_enc'] = enc.astype(np.float32)
        store[key + '_logits'] = lg.astype(np.float32)
        print('%s: OpenCV-dnn vs oracle  max|d enc| %.3g  max|d logits| %.3g  (enc range %.2f, logit range %.2f)'
              % (key, np.abs(enc - oenc).max(), np.abs(lg - olg).max(), np.abs(oenc).max(), np.abs(olg).max()))
    np.savez_compressed(OUT, **store)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
