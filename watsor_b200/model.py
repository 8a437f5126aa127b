"""Model compiler: frozen TF Object-Detection SSD graph -> H100 layer program.

The reference loads `frozen_inference_graph.pb` / `cpu.pb` into a TF session
(watsor/detection/tensorflow_cpu.py:50-62) or a UFF/ONNX file into TensorRT
(watsor/engine.py:17-51).  Here the GraphDef is walked once, on the host, and turned
into a flat program of fused layers (conv + BatchNorm/bias + ReLU6) with a liveness-
planned activation arena; the result is serialised into a `.wb200` blob that
`wb_create()` (include/watsor_b200.h) uploads to HBM.

Blob layout (little endian), mirrored by watsor_b200/csrc/model_format.h:
    header (256 B) | layers[n_layers] (128 B each) | tensors[n_tensors] (16 B each) | float32 data
"""
import struct
from dataclasses import dataclass, field
from typing import List

import numpy as np

from .graphdef import GraphDef

MAGIC = b'WB200M01'
OP_STEM, OP_DW, OP_PW, OP_CONV, OP_ADD, OP_HEAD, OP_MAXPOOL, OP_AVGPOOL, OP_COPY = 1, 2, 3, 4, 5, 6, 7, 8, 9
OP_NAMES = {1: 'stem', 2: 'dw', 3: 'pw', 4: 'conv', 5: 'add', 6: 'head', 7: 'maxpool', 8: 'avgpool', 9: 'copy'}
ACT_NONE, ACT_RELU6 = 0, 1
HEADER_BYTES, LAYER_BYTES, TENSOR_BYTES = 256, 128, 16
N_ALIGN = 16          # weight matrices are padded to a multiple of 16 output channels
ARENA_ALIGN = 256     # per-frame activation offsets are multiples of 256 elements


def same_pad(in_size, k, s):
    """TensorFlow `SAME` padding: out = ceil(in/s); the odd pixel goes after."""
    out = -(-in_size // s)
    total = max((out - 1) * s + k - in_size, 0)
    return out, total // 2


@dataclass
class Layer:
    op: int
    act: int = ACT_NONE
    in_h: int = 0
    in_w: int = 0
    in_c: int = 0
    out_h: int = 0
    out_w: int = 0
    out_c: int = 0
    kh: int = 1
    kw: int = 1
    stride: int = 1
    pad_t: int = 0
    pad_l: int = 0
    in_off: int = 0          # arena offsets, elements per frame
    in2_off: int = 0
    out_off: int = 0
    w_tensor: int = -1       # [kh*kw*in_c, n_pad] row-major (dw: [kh*kw, c])
    scale_tensor: int = -1   # per output channel, n_pad
    offset_tensor: int = -1
    n_pad: int = 0
    anchors_per_loc: int = 0  # head only
    row_off: int = 0          # head only: first anchor row of this feature map
    n_box: int = 0            # head only: A*4 columns, then A*(C+1) class columns
    n_cls: int = 0
    name: str = ''
    # symbolic tensor ids used by the arena planner (not serialised)
    src: str = ''
    src2: str = ''
    dst: str = ''

    @property
    def macs(self):
        if self.op == OP_DW:
            return self.out_h * self.out_w * self.out_c * self.kh * self.kw
        if self.op in (OP_ADD, OP_MAXPOOL, OP_AVGPOOL, OP_COPY):
            return 0
        return self.out_h * self.out_w * self.out_c * self.kh * self.kw * self.in_c


@dataclass
class Model:
    input_h: int = 300
    input_w: int = 300
    num_classes: int = 0
    num_anchors: int = 0
    pre_mul: float = 0.0
    pre_sub: float = 0.0
    scale_y: float = 10.0
    scale_x: float = 10.0
    scale_h: float = 5.0
    scale_w: float = 5.0
    logit_scale: float = 1.0
    iou_thr: float = 0.6
    score_thr: float = 0.3
    max_per_class: int = 100
    max_total: int = 100
    class_offset: float = 1.0
    arena_elems: int = 0
    anchors_tensor: int = -1
    layers: List[Layer] = field(default_factory=list)
    tensors: List[np.ndarray] = field(default_factory=list)
    name: str = ''

    # ------------------------------------------------------------------ helpers
    def add_tensor(self, arr):
        self.tensors.append(np.ascontiguousarray(arr, dtype=np.float32))
        return len(self.tensors) - 1

    @property
    def anchors(self):
        return self.tensors[self.anchors_tensor].reshape(-1, 4)

    @property
    def macs_per_frame(self):
        return sum(l.macs for l in self.layers)

    def plan_arena(self):
        """Greedy first-fit activation planner: a tensor's slot is freed after its
        last reader, so the arena stays small enough for batches to live in L2."""
        last_use = {}
        for i, l in enumerate(self.layers):
            for t in (l.src, l.src2):
                if t:
                    last_use[t] = i
        # a depthwise layer may be fused into the following 1x1 conv, and into the residual `Add` of that conv's output
        # after it (csrc/kernels_fused.cu): the fused kernel reads the depthwise INPUT while it writes the 1x1 (or
        # Add) OUTPUT, so that input must outlive the kernel's last layer
        for i, l in enumerate(self.layers[:-1]):
            nxt = self.layers[i + 1]
            if l.op == OP_DW and nxt.op == OP_PW and nxt.src == l.dst and l.src:
                end_ = i + 1
                if i + 2 < len(self.layers) and self.layers[i + 2].op == OP_ADD and \
                        nxt.dst in (self.layers[i + 2].src, self.layers[i + 2].src2):
                    end_ = i + 2
                last_use[l.src] = max(last_use[l.src], end_)
        # a linear 1x1 projection followed by the residual `Add` of its output runs as one kernel (the shortcut is
        # added in the GEMM epilogue, csrc/wb_api.cu run_layers): that kernel reads the projection's INPUT while it
        # writes the Add's OUTPUT, so the input must outlive the Add layer
        for i, l in enumerate(self.layers[:-1]):
            nxt = self.layers[i + 1]
            if l.op == OP_PW and nxt.op == OP_ADD and l.dst in (nxt.src, nxt.src2) and l.src:
                last_use[l.src] = max(last_use[l.src], i + 1)
        size = {}
        for l in self.layers:
            if l.dst:
                size[l.dst] = -(-(l.out_h * l.out_w * l.out_c) // ARENA_ALIGN) * ARENA_ALIGN
        free = []            # (offset, size)
        top = 0
        where = {}

        def alloc(n):
            nonlocal top
            for k, (o, s) in enumerate(free):
                if s >= n:
                    if s == n:
                        free.pop(k)
                    else:
                        free[k] = (o + n, s - n)
                    return o
            o = top
            top += n
            return o

        def release(o, n):
            free.append((o, n))
            free.sort()
            merged = []
            for o2, s2 in free:
                if merged and merged[-1][0] + merged[-1][1] == o2:
                    merged[-1] = (merged[-1][0], merged[-1][1] + s2)
                else:
                    merged.append((o2, s2))
            free[:] = merged

        for i, l in enumerate(self.layers):
            if l.dst:
                if l.dst not in where:          # a concat tensor is written by several COPY layers: allocate it once
                    where[l.dst] = alloc(size[l.dst])
                l.out_off = where[l.dst]
            if l.src and l.src in where:
                l.in_off = where[l.src]
            if l.src2 and l.src2 in where:
                l.in2_off = where[l.src2]
            for t in [t for t, lu in last_use.items() if lu == i and t in where]:
                release(where[t], size[t])
        self.arena_elems = top

    # -------------------------------------------------------------- (de)serialise
    def to_blob(self):
        hdr = struct.pack(
            '<8sIIIIIIfffffffffIIfIIQ', MAGIC, len(self.layers), len(self.tensors), self.input_h,
            self.input_w, self.num_classes, self.num_anchors, self.pre_mul, self.pre_sub,
            self.scale_y, self.scale_x, self.scale_h, self.scale_w, self.logit_scale, self.iou_thr,
            self.score_thr, self.max_per_class, self.max_total, self.class_offset,
            self.anchors_tensor, 0, self.arena_elems)
        hdr = hdr.ljust(HEADER_BYTES, b'\0')
        out = [hdr]
        for l in self.layers:
            rec = struct.pack(
                '<IIIIIIIIIIIIIIIIiiiIIIII', l.op, l.act, l.in_h, l.in_w, l.in_c, l.out_h, l.out_w,
                l.out_c, l.kh, l.kw, l.stride, l.pad_t, l.pad_l, l.in_off, l.in2_off, l.out_off,
                l.w_tensor, l.scale_tensor, l.offset_tensor, l.n_pad, l.anchors_per_loc, l.row_off,
                l.n_box, l.n_cls)
            name = l.name.encode()[:LAYER_BYTES - len(rec) - 1]
            out.append((rec + name).ljust(LAYER_BYTES, b'\0'))
        off = 0
        for t in self.tensors:
            out.append(struct.pack('<QQ', off, t.size))
            off += -(-t.size // 64) * 64
        for t in self.tensors:
            pad = -(-t.size // 64) * 64 - t.size
            out.append(t.tobytes())
            if pad:
                out.append(b'\0' * (4 * pad))
        return b''.join(out)

    @staticmethod
    def from_blob(blob):
        m = Model()
        f = struct.unpack_from('<8sIIIIIIfffffffffIIfIIQ', blob, 0)
        assert f[0] == MAGIC, 'not a WB200 model blob'
        (n_layers, n_tensors, m.input_h, m.input_w, m.num_classes, m.num_anchors, m.pre_mul,
         m.pre_sub, m.scale_y, m.scale_x, m.scale_h, m.scale_w, m.logit_scale, m.iou_thr,
         m.score_thr, m.max_per_class, m.max_total, m.class_offset, m.anchors_tensor, _,
         m.arena_elems) = f[1:]
        pos = HEADER_BYTES
        for _ in range(n_layers):
            v = struct.unpack_from('<IIIIIIIIIIIIIIIIiiiIIIII', blob, pos)
            l = Layer(*v)
            name = blob[pos + 96:pos + LAYER_BYTES].split(b'\0')[0].decode()
            l.name = name
            m.layers.append(l)
            pos += LAYER_BYTES
        table = []
        for _ in range(n_tensors):
            table.append(struct.unpack_from('<QQ', blob, pos))
            pos += TENSOR_BYTES
        data = np.frombuffer(blob, dtype=np.float32, offset=pos)
        for off, cnt in table:
            m.tensors.append(data[off:off + cnt])
        return m

    def save(self, path):
        with open(path, 'wb') as f:
            f.write(self.to_blob())

    @staticmethod
    def load(path):
        with open(path, 'rb') as f:
            return Model.from_blob(f.read())


def _pad_cols(w, n_pad):
    if w.shape[-1] == n_pad:
        return w
    out = np.zeros(w.shape[:-1] + (n_pad,), np.float32)
    out[..., :w.shape[-1]] = w
    return out


def _pad_vec(v, n_pad, fill=0.0):
    out = np.full(n_pad, fill, np.float32)
    out[:v.size] = v
    return out


class _Emitter:
    """Shared by the GraphDef compiler and the synthetic-architecture builders."""

    def __init__(self, model):
        self.m = model
        self.shape = {}          # tensor id -> (h, w, c)

    def conv(self, name, src, dst, w_hwio, scale, offset, stride, act, depthwise=False):
        h, w_, c = self.shape[src]
        kh, kw = int(w_hwio.shape[0]), int(w_hwio.shape[1])
        oh, pt = same_pad(h, kh, stride)
        ow, pl = same_pad(w_, kw, stride)
        m = self.m
        if depthwise:
            assert w_hwio.shape[2] == c and w_hwio.shape[3] == 1
            oc = c
            n_pad = c
            wt = m.add_tensor(w_hwio.reshape(kh * kw, c))
            op = OP_DW
        else:
            assert w_hwio.shape[2] == c, (name, w_hwio.shape, c)
            oc = int(w_hwio.shape[3])
            n_pad = -(-oc // N_ALIGN) * N_ALIGN
            wt = m.add_tensor(_pad_cols(w_hwio.reshape(kh * kw * c, oc), n_pad))
            if src == 'image':
                op = OP_STEM
            elif kh == 1 and kw == 1 and stride == 1:
                op = OP_PW
            else:
                op = OP_CONV
        l = Layer(op=op, act=act, in_h=h, in_w=w_, in_c=c, out_h=oh, out_w=ow, out_c=oc, kh=kh,
                  kw=kw, stride=stride, pad_t=pt, pad_l=pl, w_tensor=wt,
                  scale_tensor=m.add_tensor(_pad_vec(scale, n_pad, 1.0)),
                  offset_tensor=m.add_tensor(_pad_vec(offset, n_pad, 0.0)), n_pad=n_pad,
                  name=name, src='' if src == 'image' else src, dst=dst)
        m.layers.append(l)
        self.shape[dst] = (oh, ow, oc)

    def add(self, name, a, b, dst):
        h, w_, c = self.shape[a]
        assert self.shape[b] == (h, w_, c)
        self.m.layers.append(Layer(op=OP_ADD, in_h=h, in_w=w_, in_c=c, out_h=h, out_w=w_, out_c=c,
                                   name=name, src=a, src2=b, dst=dst))
        self.shape[dst] = (h, w_, c)

    def pool(self, name, src, dst, k, stride, kind):
        """TF `MaxPool` / `AvgPool`, padding SAME (the average divides by the number of in-image taps)."""
        h, w_, c = self.shape[src]
        oh, pt = same_pad(h, k, stride)
        ow, pl = same_pad(w_, k, stride)
        self.m.layers.append(Layer(op=OP_MAXPOOL if kind == 'max' else OP_AVGPOOL, in_h=h, in_w=w_, in_c=c, out_h=oh,
                                   out_w=ow, out_c=c, kh=k, kw=k, stride=stride, pad_t=pt, pad_l=pl, name=name,
                                   src=src, dst=dst))
        self.shape[dst] = (oh, ow, c)

    def concat(self, name, srcs, dst):
        """`ConcatV2` along channels: one COPY layer per input writes its channel slice of `dst`
        (in_c = slice width, out_c = total width, row_off = first channel of the slice)."""
        h, w_, _ = self.shape[srcs[0]]
        total = sum(self.shape[s_][2] for s_ in srcs)
        off = 0
        for k, s_ in enumerate(srcs):
            assert self.shape[s_][:2] == (h, w_)
            c = self.shape[s_][2]
            self.m.layers.append(Layer(op=OP_COPY, in_h=h, in_w=w_, in_c=c, out_h=h, out_w=w_, out_c=total, row_off=off,
                                       name='%s/%d' % (name, k), src=s_, dst=dst))
            off += c
        self.shape[dst] = (h, w_, total)

    def head(self, name, src, w_box, b_box, w_cls, b_cls, row_off, num_classes_p1):
        """One GEMM per feature map: [box columns | class columns] (both 1x1 + bias)."""
        h, w_, c = self.shape[src]
        assert w_box.shape[:3] == (1, 1, c) and w_cls.shape[:3] == (1, 1, c), \
            'only kernel_size 1 box predictors are supported (convolutional_box_predictor)'
        n_box, n_cls = int(w_box.shape[3]), int(w_cls.shape[3])
        a = n_box // 4
        assert n_cls == a * num_classes_p1
        n = n_box + n_cls
        n_pad = -(-n // N_ALIGN) * N_ALIGN
        wcat = np.concatenate([w_box.reshape(c, n_box), w_cls.reshape(c, n_cls)], axis=1)
        m = self.m
        l = Layer(op=OP_HEAD, act=ACT_NONE, in_h=h, in_w=w_, in_c=c, out_h=h, out_w=w_, out_c=n,
                  w_tensor=m.add_tensor(_pad_cols(wcat, n_pad)),
                  scale_tensor=m.add_tensor(np.ones(n_pad, np.float32)),
                  offset_tensor=m.add_tensor(_pad_vec(np.concatenate([b_box, b_cls]), n_pad)),
                  n_pad=n_pad, anchors_per_loc=a, row_off=row_off, n_box=n_box, n_cls=n_cls,
                  name=name, src=src)
        m.layers.append(l)
        return h * w_ * a


def compile_frozen_graph(pb_path, name=None):
    """Walk a TF Object-Detection SSD GraphDef (MobileNet-style feature extractor:
    Conv2D / DepthwiseConv2dNative + FusedBatchNorm + Relu6, residual Add, 1x1 box
    predictors) and emit the layer program."""
    g = GraphDef(pb_path)
    m = Model(name=name or pb_path)
    em = _Emitter(m)

    rb = g.ops('ResizeBilinear')
    if len(rb) != 1:
        raise ValueError('expected exactly one ResizeBilinear (fixed_shape_resizer)')
    if g.attr(rb[0], 'align_corners', False) or g.attr(rb[0], 'half_pixel_centers', False):
        raise ValueError('only the legacy bilinear sampling of fixed_shape_resizer is supported')
    size = g.const(g.nodes[rb[0]].data_inputs()[1][0])
    m.input_h, m.input_w = int(size[0]), int(size[1])
    m.pre_mul = float(g.const('Preprocessor/mul/x'))
    m.pre_sub = float(g.const('Preprocessor/sub/y'))
    em.shape['image'] = (m.input_h, m.input_w, 3)

    def bn_affine(node):
        ins = g.nodes[node].data_inputs()
        gamma, beta, mean, var = (g.const(i[0]).astype(np.float32) for i in ins[1:5])
        eps = np.float32(g.attr(node, 'epsilon'))
        scale = (gamma * (np.float32(1) / np.sqrt(var + eps))).astype(np.float32)
        offset = (beta - mean * scale).astype(np.float32)
        return scale, offset

    done = {'Preprocessor/sub': 'image'}

    def emit(tensor):
        """Returns the tensor id holding `tensor`, emitting layers on demand."""
        if tensor in done:
            return done[tensor]
        node = tensor
        act = ACT_NONE
        n = g.nodes[node]
        if n.op == 'Relu6':
            act = ACT_RELU6
            node = n.data_inputs()[0][0]
            n = g.nodes[node]
        if n.op in ('Add', 'AddV2') and act == ACT_NONE:
            a = emit(n.data_inputs()[0][0])
            b = emit(n.data_inputs()[1][0])
            em.add(tensor, a, b, tensor)
            done[tensor] = tensor
            return tensor
        scale = offset = None
        if n.op in ('FusedBatchNorm', 'FusedBatchNormV3'):
            if g.attr(node, 'is_training', False):
                raise ValueError('training-mode batch norm in %s' % node)
            scale, offset = bn_affine(node)
            node = n.data_inputs()[0][0]
            n = g.nodes[node]
        elif n.op == 'BiasAdd':
            offset = g.const(n.data_inputs()[1][0]).astype(np.float32)
            node = n.data_inputs()[0][0]
            n = g.nodes[node]
        if n.op == 'Identity':
            r = emit(n.data_inputs()[0][0])
            done[tensor] = r
            return r
        if n.op not in ('Conv2D', 'DepthwiseConv2dNative'):
            raise NotImplementedError('unsupported op %s at %s' % (n.op, node))
        if g.attr(node, 'padding') != b'SAME' or g.attr(node, 'data_format', b'NHWC') != b'NHWC':
            raise NotImplementedError('only NHWC / SAME convolutions (%s)' % node)
        if g.attr(node, 'dilations', [1, 1, 1, 1]) not in ([], [1, 1, 1, 1]):
            raise NotImplementedError('dilated convolution (%s)' % node)
        strides = g.attr(node, 'strides')
        assert strides[1] == strides[2]
        src = emit(n.data_inputs()[0][0])
        w = g.const(n.data_inputs()[1][0]).astype(np.float32)
        oc = w.shape[2] if n.op == 'DepthwiseConv2dNative' else w.shape[3]
        if scale is None:
            scale = np.ones(oc, np.float32)
        if offset is None:
            offset = np.zeros(oc, np.float32)
        em.conv(tensor, src, tensor, w, scale, offset, int(strides[1]), act,
                depthwise=(n.op == 'DepthwiseConv2dNative'))
        done[tensor] = tensor
        return tensor

    box_heads = [i[0] for i in g.nodes['concat'].data_inputs()[:-1]]
    cls_heads = [i[0] for i in g.nodes['concat_1'].data_inputs()[:-1]]
    pack = g.nodes[cls_heads[0]].data_inputs()[1][0]
    num_classes_p1 = int(g.const(g.nodes[pack].data_inputs()[-1][0]))
    m.num_classes = num_classes_p1 - 1
    row = 0
    for k, (rb_, rc_) in enumerate(zip(box_heads, cls_heads)):
        def conv_of(reshape):
            bias = g.nodes[reshape].data_inputs()[0][0]
            assert g.nodes[bias].op == 'BiasAdd'
            conv = g.nodes[bias].data_inputs()[0][0]
            assert g.nodes[conv].op == 'Conv2D' and g.attr(conv, 'strides') == [1, 1, 1, 1]
            return (g.nodes[conv].data_inputs()[0][0],
                    g.const(g.nodes[conv].data_inputs()[1][0]).astype(np.float32),
                    g.const(g.nodes[bias].data_inputs()[1][0]).astype(np.float32))
        fb, wb, bb = conv_of(rb_)
        fc, wc, bc = conv_of(rc_)
        assert fb == fc
        src = emit(fb)
        row += em.head('BoxPredictor_%d' % k, src, wb, bb, wc, bc, row, num_classes_p1)

    anchors = g.fold('Concatenate/concat').astype(np.float32)
    assert anchors.shape == (row, 4), (anchors.shape, row)
    m.num_anchors = row
    m.anchors_tensor = m.add_tensor(anchors)

    d = 'Postprocessor/Decode/'
    m.scale_y = float(g.const(d + 'truediv/y'))
    m.scale_x = float(g.const(d + 'truediv_1/y'))
    m.scale_h = float(g.const(d + 'truediv_2/y'))
    m.scale_w = float(g.const(d + 'truediv_3/y'))
    m.logit_scale = float(g.const('Postprocessor/scale_logits/y'))
    nms = g.ops('NonMaxSuppressionV5')
    if not nms:
        old = g.ops('NonMaxSuppressionV4') + g.ops('NonMaxSuppressionV3') + g.ops('NonMaxSuppressionV2') + \
            g.ops('NonMaxSuppression')
        if old:
            # e.g. the 2018 model-zoo exports (ssd_mobilenet_v1_coco_2018_01_28): per class they run
            # FilterGreaterThan_k and ClipToWindow_k BEFORE NonMaxSuppressionV2/V3, i.e. IoU on clipped boxes and the
            # score threshold as a separate Greater node.  The CUDA post stage implements the newer export order
            # (NMS on unclipped boxes -> sort -> ClipToWindow -> prune -> top-k); compiling such a graph silently
            # would change detections for boxes that cross the image border.
            raise NotImplementedError(
                'this graph uses %s (an older TF Object-Detection export with clip-before-NMS); only the '
                'NonMaxSuppressionV5 post-processing topology is implemented' % g.nodes[old[0]].op)
        raise ValueError('no NonMaxSuppression node found')
    scope = nms[0].split('non_max_suppression')[0]
    per_class_pre = [n for n in g.order if n.startswith(scope) and
                     (n[len(scope):].startswith('ClipToWindow_') or n[len(scope):].startswith('FilterGreaterThan'))]
    if per_class_pre:
        raise NotImplementedError('per-class %s before the NMS node: clip/filter-before-NMS export order is not '
                                  'implemented' % per_class_pre[0][len(scope):].split('/')[0])
    if len(nms) != m.num_classes:
        raise NotImplementedError('expected one NonMaxSuppressionV5 per class (%d), found %d'
                                  % (m.num_classes, len(nms)))
    ins = g.nodes[nms[0]].data_inputs()
    if len(ins) < 6:
        raise ValueError('NonMaxSuppressionV5 with %d inputs' % len(ins))
    m.iou_thr = float(g.const(ins[3][0]))
    m.score_thr = float(g.const(ins[4][0]))
    if float(g.const(ins[5][0])) != 0.0:
        raise NotImplementedError('soft-NMS')
    m.max_per_class = int(g.const(scope + 'Minimum/x'))
    total = [n for n in g.order if n.startswith(scope) and n.endswith('/x') and
             g.nodes[n].op == 'Const' and '/Minimum_' in n]
    m.max_total = int(g.const(sorted(total, key=lambda s: int(s.split('Minimum_')[1].split('/')[0]))[-1]))
    m.class_offset = float(g.const('add/y'))
    m.plan_arena()
    return m


# ----------------------------------------------------------------- synthetic models
def ssd_anchors(feature_maps, min_scale=0.20000000298, max_scale=0.949999988079,
                aspect_ratios=(1.0, 2.0, 0.5, 3.0, 0.333299994469), reduce_lowest=True):
    """`ssd_anchor_generator` (watsor/test/model/prepare.py:113-124 config) restated:
    the same float32 operation order as the graph's MultipleGridAnchorGenerator, so
    it reproduces the folded graph constant bit for bit (tests/test_model.py)."""
    f32 = np.float32
    n = len(feature_maps)
    scales = [min_scale + (max_scale - min_scale) * i / (n - 1) for i in range(n)] + [1.0]
    out = []
    for k, (fh, fw) in enumerate(feature_maps):
        if k == 0 and reduce_lowest:
            sc = [0.1, scales[0], scales[0]]
            ar = [1.0, 2.0, 0.5]
        else:
            sc = [scales[k]] * len(aspect_ratios) + [float(np.sqrt(scales[k] * scales[k + 1]))]
            ar = list(aspect_ratios) + [1.0]
        sc = np.asarray(sc, f32)
        ratio_sqrt = np.sqrt(np.asarray(ar, f32))
        heights = (sc / ratio_sqrt) * f32(1.0)
        widths = (sc * ratio_sqrt) * f32(1.0)
        sy, sx = f32(1.0) / f32(fh), f32(1.0) / f32(fw)
        oy, ox = f32(0.5) * sy, f32(0.5) * sx
        yc = np.arange(fh).astype(f32) * sy + oy
        xc = np.arange(fw).astype(f32) * sx + ox
        a = len(sc)
        cy = np.broadcast_to(yc[:, None, None], (fh, fw, a))
        cx = np.broadcast_to(xc[None, :, None], (fh, fw, a))
        hh = np.broadcast_to(heights[None, None, :], (fh, fw, a))
        ww = np.broadcast_to(widths[None, None, :], (fh, fw, a))
        ymin = cy - f32(0.5) * hh
        xmin = cx - f32(0.5) * ww
        ymax = cy + f32(0.5) * hh
        xmax = cx + f32(0.5) * ww
        out.append(np.stack([ymin, xmin, ymax, xmax], -1).reshape(-1, 4).astype(f32))
    return np.concatenate(out, 0)


def synthetic_ssd_mobilenet_v1(num_classes=90, seed=0, score_thr=1e-8, input_size=300):
    """SSD-MobileNet-v1 architecture descriptor (TF-slim mobilenet_v1 + the SSD extra
    layers of ssd_mobilenet_v1_feature_extractor) with seeded synthetic weights.

    No COCO weights exist offline (README.md:446-451 are download links), so this is
    what the 90-class configs of BASELINE.json run on; it is checked GPU-vs-oracle only.
    Weights are He-initialised; the folded BatchNorm is identity-like (scale close to 1,
    small offset) so that activations keep a healthy range through ReLU6.
    """
    rng = np.random.default_rng(seed)
    m = Model(name='ssd_mobilenet_v1_synthetic_c%d' % num_classes, input_h=input_size,
              input_w=input_size, num_classes=num_classes, score_thr=score_thr, iou_thr=0.6,
              pre_mul=float(np.float32(2.0 / 255.0)), pre_sub=1.0)
    em = _Emitter(m)
    em.shape['image'] = (input_size, input_size, 3)

    def he(shape, fan_in):
        return (rng.standard_normal(shape) * np.sqrt(2.0 / fan_in)).astype(np.float32)

    def bn(c):
        return ((1.0 + 0.1 * rng.standard_normal(c)).astype(np.float32),
                (0.1 * rng.standard_normal(c)).astype(np.float32))

    cur = 'image'
    s, o = bn(32)
    em.conv('Conv2d_0', cur, 'c0', he((3, 3, 3, 32), 27), s, o, 2, ACT_RELU6)
    cur = 'c0'
    cfg = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1),
           (512, 1), (512, 1), (1024, 2), (1024, 1)]
    taps = {}
    c_in = 32
    for i, (c_out, stride) in enumerate(cfg, 1):
        s, o = bn(c_in)
        em.conv('Conv2d_%d_depthwise' % i, cur, 'dw%d' % i, he((3, 3, c_in, 1), 9) * 1.5, s, o,
                stride, ACT_RELU6, depthwise=True)
        s, o = bn(c_out)
        em.conv('Conv2d_%d_pointwise' % i, 'dw%d' % i, 'pw%d' % i, he((1, 1, c_in, c_out), c_in),
                s, o, 1, ACT_RELU6)
        cur = 'pw%d' % i
        c_in = c_out
        taps[i] = cur
    feats = [taps[11], taps[13]]
    for j, (mid, out_c) in enumerate([(256, 512), (128, 256), (128, 256), (64, 128)], 2):
        s, o = bn(mid)
        em.conv('Conv2d_13_pointwise_1_Conv2d_%d_1x1_%d' % (j, mid), cur, 'e%da' % j,
                he((1, 1, c_in, mid), c_in), s, o, 1, ACT_RELU6)
        s, o = bn(out_c)
        em.conv('Conv2d_13_pointwise_2_Conv2d_%d_3x3_s2_%d' % (j, out_c), 'e%da' % j, 'e%db' % j,
                he((3, 3, mid, out_c), 9 * mid), s, o, 2, ACT_RELU6)
        cur = 'e%db' % j
        c_in = out_c
        feats.append(cur)
    # heads are emitted right after... (program order is free: re-sort below)
    row = 0
    fmaps = []
    head_layers = []
    for k, f in enumerate(feats):
        h, w_, c = em.shape[f]
        a = 3 if k == 0 else 6
        fmaps.append((h, w_))
        n0 = len(m.layers)
        row += em.head('BoxPredictor_%d' % k, f, he((1, 1, c, a * 4), c) * 0.5,
                       (0.05 * rng.standard_normal(a * 4)).astype(np.float32),
                       he((1, 1, c, a * (num_classes + 1)), c),
                       (-2.0 + 0.5 * rng.standard_normal(a * (num_classes + 1))).astype(np.float32),
                       row, num_classes + 1)
        head_layers.append(m.layers.pop(n0))
    # place every head right after the layer that produces its feature map
    for hl in head_layers:
        idx = max(i for i, l in enumerate(m.layers) if l.dst == hl.src)
        m.layers.insert(idx + 1, hl)
    m.num_anchors = row
    m.anchors_tensor = m.add_tensor(ssd_anchors(fmaps))
    m.plan_arena()
    return m


def synthetic_ssd_mobilenet_v2(num_classes=90, seed=0, score_thr=1e-8, input_size=300, cls_gain=0.3, cls_bias=-4.5):
    """SSD-MobileNet-v2 architecture descriptor (TF-slim mobilenet_v2, depth multiplier 1.0, plus the
    SSD feature-map layout of ssd_mobilenet_v2_feature_extractor: taps `layer_15/expansion_output`
    19x19x576 and `layer_19` 10x10x1280, then four 1x1 -> 3x3/s2 extra pairs 512/256/256/128) with
    seeded synthetic weights.  BASELINE.json's 640x480 configs name this model; no weights for it
    exist offline, so it runs on He-initialised tensors and is checked GPU-vs-oracle only.

    Inverted residual block: 1x1 expand (x6, BN, ReLU6) -> 3x3 depthwise (stride s, BN, ReLU6) ->
    1x1 linear projection (BN), residual add when stride == 1 and channels match.

    `cls_gain` / `cls_bias` shape the class logits like a trained detector's: with plain He weights the logits
    of this random net have std 3.7 around -2, i.e. thousands of (anchor, class) scores saturate at 1.0 - 6e-8 and
    the top-100 list is a block of exact fp32 ties.  Gain 0.3 / bias -4.5 gives logits ~ N(-4.5, 1.2^2): almost
    every score is ~0.01 (they all still pass the 1e-8 threshold, so the per-class NMS sees all 1917 anchors in
    every class, as with the zoo models), and the tail reaches 0.4 .. 0.8 in a handful of classes.
    """
    rng = np.random.default_rng(seed)
    m = Model(name='ssd_mobilenet_v2_synthetic_c%d' % num_classes, input_h=input_size, input_w=input_size,
              num_classes=num_classes, score_thr=score_thr, iou_thr=0.6,
              pre_mul=float(np.float32(2.0 / 255.0)), pre_sub=1.0)
    em = _Emitter(m)
    em.shape['image'] = (input_size, input_size, 3)

    def he(shape, fan_in, gain=2.0):
        return (rng.standard_normal(shape) * np.sqrt(gain / fan_in)).astype(np.float32)

    def bn(c, spread=0.1):
        return ((1.0 + spread * rng.standard_normal(c)).astype(np.float32),
                (spread * rng.standard_normal(c)).astype(np.float32))

    s, o = bn(32)
    em.conv('Conv', 'image', 'conv0', he((3, 3, 3, 32), 27), s, o, 2, ACT_RELU6)
    cur, c_in = 'conv0', 32
    # expanded_conv (t = 1): depthwise + linear projection to 16
    s, o = bn(32)
    em.conv('expanded_conv/depthwise', cur, 'b0dw', he((3, 3, 32, 1), 9) * 1.5, s, o, 1, ACT_RELU6, depthwise=True)
    s, o = bn(16)
    em.conv('expanded_conv/project', 'b0dw', 'b0', he((1, 1, 32, 16), 32, 1.0), s, o, 1, ACT_NONE)
    cur, c_in = 'b0', 16
    tap15 = None
    idx = 1
    for (t, c, n, stride0) in [(6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]:
        for i in range(n):
            stride = stride0 if i == 0 else 1
            name = 'expanded_conv_%d' % idx
            ce = c_in * t
            s, o = bn(ce)
            em.conv(name + '/expand', cur, name + 'e', he((1, 1, c_in, ce), c_in), s, o, 1, ACT_RELU6)
            if idx == 13:
                tap15 = name + 'e'                     # layer_15/expansion_output
            s, o = bn(ce)
            em.conv(name + '/depthwise', name + 'e', name + 'd', he((3, 3, ce, 1), 9) * 1.5, s, o, stride,
                    ACT_RELU6, depthwise=True)
            s, o = bn(c)
            em.conv(name + '/project', name + 'd', name + 'p', he((1, 1, ce, c), ce, 1.0), s, o, 1, ACT_NONE)
            if stride == 1 and c_in == c:
                em.add(name + '/add', cur, name + 'p', name + 'a')
                cur = name + 'a'
            else:
                cur = name + 'p'
            c_in = c
            idx += 1
    s, o = bn(1280)
    em.conv('Conv_1', cur, 'conv1', he((1, 1, c_in, 1280), c_in), s, o, 1, ACT_RELU6)
    cur, c_in = 'conv1', 1280
    feats = [tap15, 'conv1']
    for j, (mid, out_c) in enumerate([(256, 512), (128, 256), (128, 256), (64, 128)], 2):
        s, o = bn(mid)
        em.conv('layer_19_1_Conv2d_%d_1x1_%d' % (j, mid), cur, 'x%da' % j, he((1, 1, c_in, mid), c_in), s, o, 1, ACT_RELU6)
        s, o = bn(out_c)
        em.conv('layer_19_2_Conv2d_%d_3x3_s2_%d' % (j, out_c), 'x%da' % j, 'x%db' % j, he((3, 3, mid, out_c), 9 * mid),
                s, o, 2, ACT_RELU6)
        cur, c_in = 'x%db' % j, out_c
        feats.append(cur)
    row, fmaps, head_layers = 0, [], []
    for k, f in enumerate(feats):
        h, w_, c = em.shape[f]
        a = 3 if k == 0 else 6
        fmaps.append((h, w_))
        n0 = len(m.layers)
        row += em.head('BoxPredictor_%d' % k, f, he((1, 1, c, a * 4), c) * 0.5,
                       (0.05 * rng.standard_normal(a * 4)).astype(np.float32),
                       he((1, 1, c, a * (num_classes + 1)), c) * np.float32(cls_gain),
                       (cls_bias + 0.5 * rng.standard_normal(a * (num_classes + 1))).astype(np.float32),
                       row, num_classes + 1)
        head_layers.append(m.layers.pop(n0))
    for hl in head_layers:
        at = max(i for i, l in enumerate(m.layers) if l.dst == hl.src)
        m.layers.insert(at + 1, hl)
    m.num_anchors = row
    m.anchors_tensor = m.add_tensor(ssd_anchors(fmaps))
    m.plan_arena()
    return m


def synthetic_ssd_inception_v2(num_classes=90, seed=0, score_thr=1e-8, input_size=300, cls_gain=0.3, cls_bias=-4.5):
    """SSD-Inception-v2 architecture descriptor (TF-slim inception_v2, depth multiplier 1.0, separable 7x7 stem;
    SSD feature maps `Mixed_4c` 19x19x576 and `Mixed_5c` 10x10x1024 plus four 1x1 -> 3x3/s2 extra pairs 512/256/256/128,
    as in ssd_inception_v2_feature_extractor) with seeded synthetic weights.  BASELINE.json configs[4] names this
    model (ref: README.md:446-451 lists it among the supported zoo models); no weights exist offline, so it is checked
    GPU-vs-oracle only.  Every conv is Conv2D + BatchNorm + ReLU6 (the extractor's conv_hyperparams in the zoo config).
    Inception module: [1x1] | [1x1 -> 3x3] | [1x1 -> 3x3 -> 3x3] | [3x3 pool -> 1x1], concatenated along channels;
    the stride-2 modules Mixed_4a / Mixed_5a have two conv branches and a max-pool branch."""
    rng = np.random.default_rng(seed)
    m = Model(name='ssd_inception_v2_synthetic_c%d' % num_classes, input_h=input_size, input_w=input_size,
              num_classes=num_classes, score_thr=score_thr, iou_thr=0.6, pre_mul=float(np.float32(2.0 / 255.0)), pre_sub=1.0)
    em = _Emitter(m)
    em.shape['image'] = (input_size, input_size, 3)

    def he(shape, fan_in, gain=2.0):
        return (rng.standard_normal(shape) * np.sqrt(gain / fan_in)).astype(np.float32)

    def bn(c, spread=0.1):
        return ((1.0 + spread * rng.standard_normal(c)).astype(np.float32),
                (spread * rng.standard_normal(c)).astype(np.float32))

    def conv(name, src, out_c, k=1, stride=1):
        c_in = em.shape[src][2]
        s_, o_ = bn(out_c)
        em.conv(name, src, name, he((k, k, c_in, out_c), k * k * c_in), s_, o_, stride, ACT_RELU6)
        return name

    # Conv2d_1a_7x7: separable_conv2d(depth_multiplier=8) = 7x7 depthwise 3 -> 24 (no BN / activation in between),
    # then 1x1 24 -> 64.  The depthwise part with a channel multiplier is a dense 7x7 conv with block-diagonal weights.
    wd = np.zeros((7, 7, 3, 24), np.float32)
    for c in range(3):
        wd[:, :, c, c * 8:(c + 1) * 8] = he((7, 7, 8), 49)
    em.conv('Conv2d_1a_7x7/depthwise', 'image', 'c1dw', wd, np.ones(24, np.float32), np.zeros(24, np.float32), 2, ACT_NONE)
    s_, o_ = bn(64)
    em.conv('Conv2d_1a_7x7/pointwise', 'c1dw', 'c1', he((1, 1, 24, 64), 24), s_, o_, 1, ACT_RELU6)
    em.pool('MaxPool_2a_3x3', 'c1', 'p2a', 3, 2, 'max')
    cur = conv('Conv2d_2b_1x1', 'p2a', 64)
    cur = conv('Conv2d_2c_3x3', cur, 192, 3)
    em.pool('MaxPool_3a_3x3', cur, 'p3a', 3, 2, 'max')
    cur = 'p3a'

    def mixed(name, src, b0, b1, b2, b3, pool='avg'):
        outs = [conv(name + '/b0_1x1', src, b0)]
        t = conv(name + '/b1_1x1', src, b1[0])
        outs.append(conv(name + '/b1_3x3', t, b1[1], 3))
        t = conv(name + '/b2_1x1', src, b2[0])
        t = conv(name + '/b2_3x3a', t, b2[1], 3)
        outs.append(conv(name + '/b2_3x3b', t, b2[2], 3))
        em.pool(name + '/b3_pool', src, name + '/b3p', 3, 1, pool)
        outs.append(conv(name + '/b3_1x1', name + '/b3p', b3))
        em.concat(name + '/concat', outs, name)
        return name

    def reduction(name, src, b0, b1):
        t = conv(name + '/b0_1x1', src, b0[0])
        o0 = conv(name + '/b0_3x3', t, b0[1], 3, 2)
        t = conv(name + '/b1_1x1', src, b1[0])
        t = conv(name + '/b1_3x3a', t, b1[1], 3)
        o1 = conv(name + '/b1_3x3b', t, b1[2], 3, 2)
        em.pool(name + '/b2_pool', src, name + '/b2p', 3, 2, 'max')
        em.concat(name + '/concat', [o0, o1, name + '/b2p'], name)
        return name

    cur = mixed('Mixed_3b', cur, 64, (64, 64), (64, 96, 96), 32)
    cur = mixed('Mixed_3c', cur, 64, (64, 96), (64, 96, 96), 64)
    cur = reduction('Mixed_4a', cur, (128, 160), (64, 96, 96))
    cur = mixed('Mixed_4b', cur, 224, (64, 96), (96, 128, 128), 128)
    cur = mixed('Mixed_4c', cur, 192, (96, 128), (96, 128, 128), 128)
    feat0 = cur
    cur = mixed('Mixed_4d', cur, 160, (128, 160), (128, 160, 160), 96)
    cur = mixed('Mixed_4e', cur, 96, (128, 192), (160, 192, 192), 96)
    cur = reduction('Mixed_5a', cur, (128, 192), (192, 256, 256))
    cur = mixed('Mixed_5b', cur, 352, (192, 320), (160, 224, 224), 128)
    cur = mixed('Mixed_5c', cur, 352, (192, 320), (192, 224, 224), 128, pool='max')
    feats = [feat0, cur]
    for j, (mid, out_c) in enumerate([(256, 512), (128, 256), (128, 256), (64, 128)], 2):
        t = conv('Mixed_5c_1_Conv2d_%d_1x1_%d' % (j, mid), cur, mid)
        cur = conv('Mixed_5c_2_Conv2d_%d_3x3_s2_%d' % (j, out_c), t, out_c, 3, 2)
        feats.append(cur)
    row, fmaps, head_layers = 0, [], []
    for k, f in enumerate(feats):
        h, w_, c = em.shape[f]
        a = 3 if k == 0 else 6
        fmaps.append((h, w_))
        n0 = len(m.layers)
        row += em.head('BoxPredictor_%d' % k, f, he((1, 1, c, a * 4), c) * 0.5,
                       (0.05 * rng.standard_normal(a * 4)).astype(np.float32),
                       he((1, 1, c, a * (num_classes + 1)), c) * np.float32(cls_gain),
                       (cls_bias + 0.5 * rng.standard_normal(a * (num_classes + 1))).astype(np.float32),
                       row, num_classes + 1)
        head_layers.append(m.layers.pop(n0))
    for hl in head_layers:
        at = max(i for i, l in enumerate(m.layers) if l.dst == hl.src)
        m.layers.insert(at + 1, hl)
    m.num_anchors = row
    m.anchors_tensor = m.add_tensor(ssd_anchors(fmaps))
    m.plan_arena()
    return m
