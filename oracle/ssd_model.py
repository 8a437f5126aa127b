"""Oracle driven by a compiled `.wb200` model blob instead of the GraphDef.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Same arithmetic as
oracle/ssd_graph.py (it inherits preprocess / decode / NMS / post-process from it); only
the source of the layer list and constants differs.  This is the form the GPU tests use
(they never read the GraphDef): tests/test_model.py checks, where the
GraphDef is available, that both forms agree bit for bit on the vendored model, so a
parity test against this class is a parity test against the GraphDef restatement.
Synthetic-weight architectures (90-class heads) exist only in this form.
"""
import numpy as np
import torch
import torch.nn.functional as F

from watsor_b200.model import (OP_ADD, OP_AVGPOOL, OP_CONV, OP_COPY, OP_DW, OP_HEAD, OP_MAXPOOL, OP_PW, OP_STEM,
                               Model)

from .ssd_graph import SsdGraphOracle


class SsdModelOracle(SsdGraphOracle):
    def __init__(self, model, dtype=np.float32, num_threads=None):
        if not isinstance(model, Model):
            model = Model.load(model)
        self.model = m = model
        self.dtype = np.dtype(dtype)
        self.tdtype = torch.float32 if self.dtype == np.float32 else torch.float64
        if num_threads:
            torch.set_num_threads(num_threads)
        f32 = np.float32
        self.in_h, self.in_w = m.input_h, m.input_w
        self.pre_mul, self.pre_sub = f32(m.pre_mul), f32(m.pre_sub)
        self.num_classes = m.num_classes
        self.num_classes_p1 = m.num_classes + 1
        self.anchors = np.array(m.anchors, dtype=f32)
        self.num_anchors = m.num_anchors
        self.scale_y, self.scale_x = f32(m.scale_y), f32(m.scale_x)
        self.scale_h, self.scale_w = f32(m.scale_h), f32(m.scale_w)
        self.logit_scale = f32(m.logit_scale)
        self.iou_thr, self.score_thr = f32(m.iou_thr), f32(m.score_thr)
        self.max_per_class, self.max_total = m.max_per_class, m.max_total
        self.class_offset = f32(m.class_offset)
        self._w = {}

    def _tt(self, idx):
        if idx not in self._w:
            self._w[idx] = torch.from_numpy(np.array(self.model.tensors[idx], dtype=self.dtype))
        return self._w[idx]

    def raw_heads(self, pre_hwc, return_memo=False):
        m = self.model
        x0 = torch.from_numpy(np.ascontiguousarray(pre_hwc.astype(self.dtype))).permute(2, 0, 1).unsqueeze(0)
        arena = {}
        memo = {}
        enc = torch.zeros((self.num_anchors, 4), dtype=self.tdtype)
        logits = torch.zeros((self.num_anchors, self.num_classes_p1), dtype=self.tdtype)
        with torch.no_grad():
            for li, l in enumerate(m.layers):
                x = x0 if l.op == OP_STEM else arena[l.in_off]
                if l.op == OP_ADD:
                    v = x + arena[l.in2_off]
                elif l.op in (OP_MAXPOOL, OP_AVGPOOL):
                    # TF MaxPool / AvgPool, padding SAME: the maximum ignores the padding, the average divides by the
                    # number of taps that fall inside the image
                    pb = max((l.out_h - 1) * l.stride + l.kh - l.in_h - l.pad_t, 0)
                    pr = max((l.out_w - 1) * l.stride + l.kw - l.in_w - l.pad_l, 0)
                    if l.op == OP_MAXPOOL:
                        xp = F.pad(x, (l.pad_l, pr, l.pad_t, pb), value=float('-inf'))
                        v = F.max_pool2d(xp, (l.kh, l.kw), stride=l.stride)
                    else:
                        xp = F.pad(x, (l.pad_l, pr, l.pad_t, pb))
                        ones = F.pad(torch.ones_like(x[:, :1]), (l.pad_l, pr, l.pad_t, pb))
                        num = F.avg_pool2d(xp, (l.kh, l.kw), stride=l.stride, divisor_override=1)
                        cnt = F.avg_pool2d(ones, (l.kh, l.kw), stride=l.stride, divisor_override=1)
                        v = num / cnt
                elif l.op == OP_COPY:
                    dst = arena.get(('cat', l.out_off))
                    if dst is None or dst.shape[1] != l.out_c:
                        dst = torch.zeros((1, l.out_c, l.out_h, l.out_w), dtype=self.tdtype)
                    dst = dst.clone()
                    dst[:, l.row_off:l.row_off + l.in_c] = x
                    arena[('cat', l.out_off)] = dst
                    v = dst
                else:
                    w = self._tt(l.w_tensor)
                    scale = self._tt(l.scale_tensor)[:l.out_c]
                    offset = self._tt(l.offset_tensor)[:l.out_c]
                    pb = max((l.out_h - 1) * l.stride + l.kh - l.in_h - l.pad_t, 0)
                    pr = max((l.out_w - 1) * l.stride + l.kw - l.in_w - l.pad_l, 0)
                    xp = F.pad(x, (l.pad_l, pr, l.pad_t, pb))
                    if l.op == OP_DW:
                        wt = w.reshape(l.kh, l.kw, l.out_c, 1).permute(2, 3, 0, 1).contiguous()
                        v = F.conv2d(xp, wt, stride=l.stride, groups=l.out_c)
                    else:
                        wt = w.reshape(l.kh, l.kw, l.in_c, l.n_pad)[..., :l.out_c]
                        wt = wt.permute(3, 2, 0, 1).contiguous()
                        v = F.conv2d(xp, wt, stride=l.stride)
                    v = v * scale.view(1, -1, 1, 1) + offset.view(1, -1, 1, 1)
                    if l.act == 1:
                        v = torch.clamp(v, 0.0, 6.0)
                if l.op == OP_HEAD:
                    t = v.permute(0, 2, 3, 1).reshape(l.out_h * l.out_w, l.out_c)
                    a = l.anchors_per_loc
                    rows = l.out_h * l.out_w * a
                    enc[l.row_off:l.row_off + rows] = t[:, :l.n_box].reshape(rows, 4)
                    logits[l.row_off:l.row_off + rows] = t[:, l.n_box:].reshape(rows, self.num_classes_p1)
                else:
                    arena[l.out_off] = v
                    memo[li] = v
        if return_memo:
            return enc.numpy(), logits.numpy(), memo
        return enc.numpy(), logits.numpy()

    def feature(self, memo, layer_index):
        return memo[layer_index][0].permute(1, 2, 0).contiguous().numpy()
