"""Arena plan of the fused depthwise -> 1x1 (-> residual Add) kernel (csrc/kernels_fused.cu), on the CPU.

The kernel reads the depthwise INPUT while it writes the 1x1 output, or the Add's output when the projection is
followed by a residual Add.  The executor (csrc/wb_api.cu fused_span) runs such a group unfused when those arena
ranges overlap, so plan_arena must keep the depthwise input alive through the group's last layer."""
import pytest

from tests import workload
from watsor_b200.model import OP_ADD, OP_DW, OP_PW, synthetic_ssd_mobilenet_v2


def _range(off, l, side):
    h, w, c = (l.in_h, l.in_w, l.in_c) if side == 'in' else (l.out_h, l.out_w, l.out_c)
    return off, off + h * w * c


def _overlap(a, b):
    return a[0] < b[1] and b[0] < a[1]


def fused_groups(m):
    """(dw, pw, add or None) for every group whose shapes the fused kernel takes (fused_dwpw_supported)."""
    out = []
    for i, d in enumerate(m.layers[:-1]):
        p = m.layers[i + 1]
        if not (d.op == OP_DW and p.op == OP_PW and p.src == d.dst and d.kh == 3 and d.kw == 3 and d.stride in (1, 2)):
            continue
        if d.out_c % 4 or -(-d.out_c // 32) >= 16 or p.n_pad > 64 or p.out_c % 4:
            continue
        a = m.layers[i + 2] if i + 2 < len(m.layers) else None
        if a is not None and not (a.op == OP_ADD and p.dst in (a.src, a.src2) and a.src != a.src2):
            a = None
        out.append((d, p, a))
    return out


@pytest.mark.parametrize('name', ['configs2_v2_coco', 'v2_3class_seed2'])
def test_fused_depthwise_input_outlives_the_group(name):
    m = workload.v2_coco_model() if name == 'configs2_v2_coco' else \
        synthetic_ssd_mobilenet_v2(num_classes=3, seed=2, score_thr=0.3)
    groups = fused_groups(m)
    # v2: the 150x150 block-0 pair and the nine pairs of blocks 1..9 (N <= 64), three of them with stride 2 and
    # six followed by a residual Add
    assert len(groups) == 10
    assert sum(d.stride == 2 for d, _, _ in groups) == 3
    assert sum(a is not None for _, _, a in groups) == 6
    for d, p, a in groups:
        src = _range(d.in_off, d, 'in')
        assert not _overlap(src, _range(p.out_off, p, 'out')), d.name
        if a is not None:
            assert not _overlap(src, _range(a.out_off, a, 'out')), d.name
