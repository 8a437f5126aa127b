"""Every backbone layer kernel against the float64 restatement of its operation (tests/layer_reference.py), one tiny
model per case, at the shapes where its dispatch changes.

A case's tested layer reads a signed, partly clamped input: a 3x3 stem with ReLU6 and random offsets, then a linear
1x1 "mixer".  The reference is computed from the GPU's own input (read back with `stop_layer`), so only the tested
kernel's error counts, and it is held to a per-element bound.  Each case also proves that it reached the branch it
names: `plan()` for the device's SM count, the launch count, and the kernel name (and, for the tensor-core GEMM, the
cluster split in grid.z) recorded by torch.profiler.  The tf32x3 cases with K >= 256 also run in tf32x1 and must
fail the tf32x3 bound there: the bar detects a lost correction term."""
import json
import os
import tempfile
from collections import namedtuple

import numpy as np
import pytest

from tests import layer_reference as R
from watsor_b200.model import ACT_NONE, ACT_RELU6, OP_HEAD, Model, _Emitter

pytestmark = pytest.mark.gpu

Case = namedtuple('Case', 'name family spec n precisions claim env prepare')


def case(name, family, spec, n, precisions, claim, env=(), prepare=None):
    """claim: plan() entries the tested layer must show, per precision ('all', or 0 / 1 / 'tf32' for 2 and 3; fp16
    runs bf16's plan and claims 1's).  prepare(m, L): rewrites the model's weights after build()."""
    return Case(name, family, spec, n, tuple(precisions), claim, tuple(env), prepare)


def claim_for(c, precision):
    key = {2: 'tf32', 3: 'tf32', 4: 1}.get(precision, precision)
    return c.claim.get(key, c.claim.get('all', {}))


TC = (2, 3, 1)
CASES = []
for n in (1, 2):
    CASES += [
        case('stem3x3s2_300_n%d' % n, 'stem', ('stem', 300, 300, 3, 2, 32), n, (0, 2, 1), {'all': {'kernel': 'k_stem_3x3s2_c32'}}),
        case('stem3x3s2_299x301_n%d' % n, 'stem', ('stem', 299, 301, 3, 2, 32), n, (0, 2, 1), {'all': {'kernel': 'k_stem_3x3s2_c32'}}),
        case('stem1x1_n%d' % n, 'stem', ('stem', 37, 41, 1, 1, 16), n, (0, 2, 1), {'all': {'kernel': 'k_stem'}}),
        case('stem7x7s2_n%d' % n, 'stem', ('stem', 75, 77, 7, 2, 24), n, (0, 2, 1), {'all': {'kernel': 'k_stem'}}),
        case('stem3x3s1_n%d' % n, 'stem', ('stem', 33, 31, 3, 1, 48), n, (0, 2, 1), {'all': {'kernel': 'k_stem'}}),
    ]
# heads: 90 classes, N = 285 (a = 3) / 570 (a = 6), not multiples of 4 -- ('head', hw, K, anchors per location)
for a, n1, n8 in ((3, 5, 5), (6, 5, 3)):
    CASES += [
        case('head_a%d_K1280_n1' % a, 'tc_head', ('head', 10, 1280, a), 1, TC,
             {'tf32': {'kernel': 'k_gemm_tc', 'splits': n1, 'bn': 128}, 1: {'splits': 2}}),
        case('head_a%d_K1280_n8' % a, 'tc_head', ('head', 10, 1280, a), 8, TC,
             {'tf32': {'kernel': 'k_gemm_tc', 'splits': n8}, 1: {'splits': 2}}),
        case('head_a%d_K96_n3' % a, 'tc_head', ('head', 5, 96, a), 3, TC, {'all': {'kernel': 'k_gemm_tc', 'splits': 1}}),
    ]
for n in (1, 2):
    CASES.append(case('heads2_rowoff_n%d' % n, 'tc_head', ('heads2', 5, 256), n, TC, {'all': {'kernel': 'k_gemm_tc'}}))
# implicit-GEMM convolutions -- ('gemm', hw, C_in, N, k, stride, act)
CASES += [
    case('conv3x3s2_10to5_256to512_n1', 'tc_conv', ('gemm', 10, 256, 512, 3, 2, ACT_RELU6), 1, TC,
         {'tf32': {'kernel': 'k_gemm_tc', 'splits': 8, 'rows_per_tile': 125}, 1: {'splits': 4}}),
    case('conv3x3s2_10to5_256to512_n8', 'tc_conv', ('gemm', 10, 256, 512, 3, 2, ACT_RELU6), 8, TC,
         {'tf32': {'kernel': 'k_gemm_tc', 'splits': 8}}),
    case('conv3x3s2_3to2_128_n1', 'tc_conv', ('gemm', 3, 128, 128, 3, 2, ACT_RELU6), 1, TC, {'all': {'kernel': 'k_gemm_tc'}}),
    case('conv3x3s2_3to2_128_n3', 'tc_conv', ('gemm', 3, 128, 128, 3, 2, ACT_RELU6), 3, TC, {'all': {'kernel': 'k_gemm_tc'}}),
    case('conv3x3s2_2to1_128_n1', 'tc_conv', ('gemm', 2, 128, 128, 3, 2, ACT_NONE), 1, TC,
         {'all': {'kernel': 'k_gemm_tc', 'rows_per_tile': 128}}),
    case('conv3x3s2_2to1_128_n8', 'tc_conv', ('gemm', 2, 128, 128, 3, 2, ACT_NONE), 8, TC, {'all': {'kernel': 'k_gemm_tc'}}),
    case('conv3x3s1_11_64to48_n1', 'tc_conv', ('gemm', 11, 64, 48, 3, 1, ACT_RELU6), 1, TC,
         {'all': {'kernel': 'k_gemm_tc', 'rows_per_tile': 121, 'bn': 64}}),
    case('conv3x3s1_11_64to48_n2', 'tc_conv', ('gemm', 11, 64, 48, 3, 1, ACT_RELU6), 2, TC, {'all': {'kernel': 'k_gemm_tc'}}),
    case('conv3x3s2_7to4_64_n1', 'tc_conv', ('gemm', 7, 64, 64, 3, 2, ACT_NONE), 1, TC, {'all': {'kernel': 'k_gemm_tc'}}),
    case('conv3x3s2_7to4_64_n5', 'tc_conv', ('gemm', 7, 64, 64, 3, 2, ACT_NONE), 5, TC,
         {'all': {'kernel': 'k_gemm_tc', 'rows_per_tile': 128}}),
    case('conv1x1s2_10to5_64_n1', 'tc_conv', ('gemm', 10, 64, 64, 1, 2, ACT_RELU6), 1, TC, {'all': {'kernel': 'k_gemm_tc'}}),
    case('conv1x1s2_10to5_64_n2', 'tc_conv', ('gemm', 10, 64, 64, 1, 2, ACT_RELU6), 2, TC, {'all': {'kernel': 'k_gemm_tc'}}),
    case('conv3x3s2_10to5_256to512_nosplit', 'tc_conv', ('gemm', 10, 256, 512, 3, 2, ACT_RELU6), 1, (2,),
         {'tf32': {'kernel': 'k_gemm_tc', 'splits': 1}}, env=('WB_NO_SPLITK',)),
    # 1x1 splits that no other case reaches with a profiler check (test_pointwise_gemm checks their arithmetic too)
    case('pw_K1024_N128_7_n1', 'tc_pw', ('gemm', 7, 1024, 128, 1, 1, ACT_RELU6), 1, TC, {'tf32': {'splits': 4}}),
    case('pw_K768_N96_19_n2', 'tc_pw', ('gemm', 19, 768, 96, 1, 1, ACT_NONE), 2, TC, {'tf32': {'splits': 3}}),
    # K = 1300: a bf16 row of 2600 bytes cannot be a tensor map, so bf16 runs it on CUDA cores
    case('pw_K1300_N48_10_n1', 'tc_pw', ('gemm', 10, 1300, 48, 1, 1, ACT_NONE), 1, TC,
         {'tf32': {'splits': 5, 'bn': 64}, 1: {'kernel': 'k_gemm_cc'}}),
    case('pw_K2048_N64_10_n1', 'tc_pw', ('gemm', 10, 2048, 64, 1, 1, ACT_NONE), 1, TC, {'tf32': {'splits': 8}}),
    case('pw_K1536_N32_10_n1', 'tc_pw', ('gemm', 10, 1536, 32, 1, 1, ACT_NONE), 1, TC, {'tf32': {'splits': 6, 'bn': 32}}),
    case('pw_K1792_N128_19_n1', 'tc_pw', ('gemm', 19, 1792, 128, 1, 1, ACT_NONE), 1, TC, {'tf32': {'splits': 7}}),
    # long K but enough tiles to fill the SMs: no split
    case('pw_K512_N64_38_n1', 'tc_pw', ('gemm', 38, 512, 64, 1, 1, ACT_RELU6), 1, TC, {'tf32': {'splits': 2}}),
    case('pw_K512_N64_38_n8', 'tc_pw', ('gemm', 38, 512, 64, 1, 1, ACT_RELU6), 8, TC, {'tf32': {'splits': 1}}),
]
# residual epilogue: stem -> mixer x -> linear 1x1 p -> Add(x, p), stopped at the Add -- ('pw_add', hw, C)
for hw, C, n in ((19, 64, 1), (19, 64, 3), (10, 512, 1)):
    sp = 'split' if C == 512 else 'nosplit'
    CASES += [
        case('pw_add_fused_%s_n%d' % (sp, n), 'residual', ('pw_add', hw, C), n, (2, 3),
             {'tf32': {'fused_add': True, 'splits': 2 if C == 512 else 1}}),
        case('pw_add_unfused_%s_n%d' % (sp, n), 'residual', ('pw_add', hw, C), n, (2, 3),
             {'tf32': {'fused_add': False}}, env=('WB_NO_FUSE_ADD',)),
        case('pw_add_fp32_%s_n%d' % (sp, n), 'residual', ('pw_add', hw, C), n, (0,), {0: {'kernel': 'k_gemm_cc'}}),
    ]
# CUDA-core GEMM: precision 0, and precision 2 where the tensor-core path does not take the layer
CASES += [
    case('cc_pw_big_K64_N256_75_n8', 'cc', ('gemm', 75, 64, 256, 1, 1, ACT_RELU6), 8, (0,), {0: {'tile': 128}}),
    case('cc_pw_K64_N256_75_n1', 'cc', ('gemm', 75, 64, 256, 1, 1, ACT_RELU6), 1, (0,), {0: {'tile': 64, 'splits': 1}}),
    case('cc_pw_small_K256_N64_100_n1', 'cc', ('gemm', 100, 256, 64, 1, 1, ACT_NONE), 1, (0,), {0: {'tile': 64, 'splits': 1}}),
    case('cc_pw_split_K512_N128_10_n1', 'cc', ('gemm', 10, 512, 128, 1, 1, ACT_RELU6), 1, (0,), {0: {'tile': 64, 'splits': 4}}),
    case('cc_pw_split_K512_N128_10_n2', 'cc', ('gemm', 10, 512, 128, 1, 1, ACT_RELU6), 2, (0,), {0: {'tile': 64}}),
    case('cc_head_split_n1', 'cc', ('head', 10, 1280, 6), 1, (0,), {0: {'tile': 64, 'splits': 10}}),
    case('cc_head_n2', 'cc', ('head', 5, 96, 3), 2, (0,), {0: {'tile': 64, 'splits': 1}}),
    case('cc_conv3x3s1_38_96to128_n1', 'cc', ('gemm', 38, 96, 128, 3, 1, ACT_RELU6), 1, (0, 2, 1), {'all': {'splits': 6}}),
    case('cc_conv3x3s1_38_96to128_n8', 'cc', ('gemm', 38, 96, 128, 3, 1, ACT_RELU6), 8, (0, 2), {'all': {'tile': 64, 'splits': 1}}),
    case('cc_conv3x3s2_75to38_n1', 'cc', ('gemm', 75, 64, 96, 3, 2, ACT_RELU6), 1, (0, 2), {'all': {'tile': 64}}),
    case('cc_conv3x3s2_75to38_n2', 'cc', ('gemm', 75, 64, 96, 3, 2, ACT_RELU6), 2, (0, 2, 1), {'all': {'tile': 64}}),
    case('cc_conv3x3_10_cin48_n1', 'cc', ('gemm', 10, 48, 64, 3, 1, ACT_NONE), 1, (2,), {'all': {'kernel': 'k_gemm_cc'}}),
    case('cc_conv3x3_10_cin48_n3', 'cc', ('gemm', 10, 48, 64, 3, 1, ACT_NONE), 3, (2, 0), {'all': {'kernel': 'k_gemm_cc'}}),
]
# depthwise 3x3 -- ('dw', hw, C, stride); out_w mod 4 = 3, 2, 1, 0, and maps narrower than one 4-pixel strip (the
# strip kernel's bounds-checked column loads and its stores that stop at out_w)
for hw, s in ((19, 1), (38, 1), (9, 1), (12, 1), (75, 2), (19, 2), (9, 2), (14, 2), (3, 2), (2, 2), (3, 1)):
    for n in (1, 3):
        name = ('dw_narrow_%d_s%d_n%d' if hw < 4 else 'dw_%d_s%d_n%d') % (hw, s, n)
        CASES.append(case(name, 'dw', ('dw', hw, 48 if hw % 2 else 32, s), n, (0, 1),
                          {'all': {'kernel': 'k_dw_strip', 'stride': s}}))
# pooling, bit-exact -- ('pool', hw, C, k, stride, kind)
for hw in (75, 38, 19, 10, 2):
    for s in (1, 2):
        for kind in ('max', 'avg'):
            CASES.append(case('%spool_%d_s%d' % (kind, hw, s), 'pool', ('pool', hw, 16, 3, s, kind), 2, (0, 1),
                              {'all': {'kernel': 'k_pool'}}))
# concat of 3 slices into 192 channels, and an Add of 300 elements per image (a multiple of 4, not of 1024)
for n in (1, 3):
    CASES += [case('concat_3_slices_n%d' % n, 'copy', ('concat', 10, (64, 96, 32)), n, (0, 1),
                   {'all': {'kernel': 'k_copy_channels'}}),
              case('add_5x5x12_n%d' % n, 'add', ('add', 5, 12), n, (0, 1), {'all': {'kernel': 'k_add'}})]


# ----------------------------------------------------------------------------------------------- model building
def build(spec, seed=0):
    """The case's model.  Returns (model, tested layer index, input layer indices, pre shape (h, w))."""
    rng = np.random.default_rng(seed)
    kind = spec[0]
    if kind == 'stem':
        _, h, w, k, s, oc = spec
    else:
        h = w = spec[1]
    m = Model(name='layer-test', input_h=h, input_w=w, num_classes=90, num_anchors=1)
    em = _Emitter(m)
    em.shape['image'] = (h, w, 3)

    def bn(c, spread=0.1):
        return ((1.0 + spread * rng.standard_normal(c)).astype(np.float32),
                (spread * rng.standard_normal(c)).astype(np.float32))

    def he(shape, fan_in):
        return (rng.standard_normal(shape) * np.sqrt(2.0 / fan_in)).astype(np.float32)

    if kind == 'stem':
        sc, of = bn(oc, 0.3)
        em.conv('stem', 'image', 'y', he((k, k, 3, oc), k * k * 3), sc, of, s, ACT_RELU6)
        return _finish(m), 0, [], (h, w)
    # stem with ReLU6 and offsets of +-1.5: 0 and 6 clamp a part of the values
    sc, of = bn(32)
    em.conv('stem', 'image', 's', he((3, 3, 3, 32), 27) * 3, sc, 1.5 * rng.standard_normal(32).astype(np.float32), 1,
            ACT_RELU6)

    def mixer(dst, c):
        em.conv('mix_' + dst, 's', dst, (rng.standard_normal((1, 1, 32, c)) / np.sqrt(32)).astype(np.float32),
                *bn(c), 1, ACT_NONE)
        return len(m.layers) - 1

    if kind == 'gemm':
        _, hw, cin, cout, k, s, act = spec
        x = mixer('x', cin)
        em.conv('tested', 'x', 'y', he((k, k, cin, cout), k * k * cin), *bn(cout), s, act)
        return _finish(m), len(m.layers) - 1, [x], (h, w)
    if kind in ('head', 'heads2'):
        hw, cin = spec[1], spec[2]
        x = mixer('x', cin)
        anchors = [spec[3]] if kind == 'head' else [3, 6]
        row = 0
        for i, a in enumerate(anchors):
            row += em.head('head%d' % i, 'x', he((1, 1, cin, a * 4), cin) * 0.5,
                           (0.05 * rng.standard_normal(a * 4)).astype(np.float32), he((1, 1, cin, a * 91), cin),
                           (-2.0 + 0.5 * rng.standard_normal(a * 91)).astype(np.float32), row, 91)
        m.num_anchors = row
        return _finish(m), len(m.layers) - 1, [x], (h, w)
    if kind == 'pw_add':
        _, hw, c = spec
        x = mixer('x', c)
        em.conv('project', 'x', 'p', he((1, 1, c, c), c) * 0.5, *bn(c), 1, ACT_NONE)
        em.add('add', 'x', 'p', 'y')
        return _finish(m), len(m.layers) - 1, [x], (h, w)
    if kind == 'dw':
        _, hw, c, s = spec
        x = mixer('x', c)
        em.conv('dw', 'x', 'y', he((3, 3, c, 1), 9) * 1.5, *bn(c), s, ACT_RELU6, depthwise=True)
        return _finish(m), len(m.layers) - 1, [x], (h, w)
    if kind == 'pool':
        _, hw, c, k, s, pk = spec
        x = mixer('x', c)
        em.pool('pool', 'x', 'y', k, s, pk)
        return _finish(m), len(m.layers) - 1, [x], (h, w)
    if kind == 'concat':
        _, hw, widths = spec
        ins = [mixer('x%d' % i, c) for i, c in enumerate(widths)]
        em.concat('concat', ['x%d' % i for i in range(len(widths))], 'y')
        return _finish(m), len(m.layers) - 1, ins, (h, w)
    if kind == 'add':
        _, hw, c = spec
        ins = [mixer('a', c), mixer('b', c)]
        em.add('add', 'a', 'b', 'y')
        return _finish(m), len(m.layers) - 1, ins, (h, w)
    raise ValueError(kind)


def _finish(m):
    m.anchors_tensor = m.add_tensor(np.zeros((m.num_anchors, 4), np.float32))
    m.plan_arena()
    return m


# ----------------------------------------------------------------------------------------------------- running
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(m, li, inputs, pre, precision, env):
    """Runs the model to the tested layer under torch.profiler.  Returns (inputs read back, output(s), launches,
    kernels in launch order as (name, grid))."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from watsor_b200.engine import Engine
    for k in env:
        os.environ[k] = '1'
    try:
        with Engine(m.to_blob(), device=0, max_batch=pre.shape[0], precision=precision) as e:
            xs = [e.backbone(pre, stop_layer=i, layer_shape=_shape(m.layers[i]))[2] for i in inputs]
            torch.cuda.synchronize()
            # a short profiler session now and then delivers a trace without any device activity: trace again then
            for _ in range(2):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    enc, lg, y = e.backbone(pre, stop_layer=li,
                                            layer_shape=None if m.layers[li].op == OP_HEAD else _shape(m.layers[li]))
                    torch.cuda.synchronize()
                kernels = _kernels(prof)
                if kernels:
                    break
            launches = e.last_launch_count()
    finally:
        for k in env:
            os.environ.pop(k, None)
    return xs, (enc, lg, y), launches, kernels


def _kernels(prof):
    """(name, grid) of the kernels in a profiler trace, in launch order."""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'trace.json')
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)['traceEvents']
    kernels = sorted((ev for ev in events if ev.get('cat') == 'kernel'), key=lambda ev: ev['ts'])
    return [(ev['name'], ev.get('args', {}).get('grid')) for ev in kernels]


def _shape(L):
    return (L.out_h, L.out_w, L.out_c)


WORST = {}          # (family, precision) -> largest error / bound


@pytest.fixture(scope='module', autouse=True)
def report():
    """At the end of each module that uses it (test_gpu_frame_path and test_gpu_fp16 import it), the largest error /
    bound its tests recorded."""
    yield
    if WORST:
        print('\nlargest error / bound per family and precision:')
        for (fam, p), r in sorted(WORST.items()):
            print('  %-18s %-7s %.3g' % (fam, R.PRECISIONS[p].name, r))
        WORST.clear()


def record(family, precision, err, bound):
    ratio = float(np.max(err / bound))
    key = (family, precision)
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    return ratio


def _weights(m, L, precision, tc):
    K = L.kh * L.kw * L.in_c
    w = np.asarray(m.tensors[L.w_tensor], np.float32).reshape(K, L.n_pad)[:, :L.out_c]
    if tc:
        w = R.PRECISIONS[precision].tc_round(w)     # the tensor-core weights are rounded once on the host
    return w.astype(np.float64).reshape(L.kh, L.kw, L.in_c, L.out_c)


PARAMS = [pytest.param(c, p, id='%s-%s' % (c.name, R.PRECISIONS[p].name)) for c in CASES for p in c.precisions]


@pytest.mark.parametrize('c,precision', PARAMS)
def test_layer_kernel(c, precision):
    check_layer(c, precision)


def check_layer(c, precision):
    """Case c in a `precision` engine: the branch it claims, and its arithmetic against float64 (module docstring)."""
    m, li, inputs, (h, w) = build(c.spec, seed=len(c.name))
    L = m.layers[li]
    if c.prepare:
        c.prepare(m, L)
    sms = _sms()
    pre = np.random.default_rng(c.n).standard_normal((c.n, h, w, 3)).astype(np.float32)
    xs, (enc, lg, y), launches, kernels = _run(m, li, inputs, pre, precision, c.env)

    # ---- the branch: plan(), launch count, kernel name (+ cluster split)
    pair = c.spec[0] == 'pw_add'              # linear 1x1 -> Add: one span, planned on the 1x1
    plans = []
    for i, Li in enumerate(m.layers[:li + 1]):
        if pair and i == li:
            continue
        plans.append(R.plan(Li, c.n, precision, sms, c.env, fuse_add_next=pair and i == li - 1))
    p = plans[-1]
    want = claim_for(c, precision)
    assert {k: p[k] for k in want} == want, (p, want)
    assert launches == sum(q['launches'] for q in plans), (launches, plans)
    names = [k for k, _ in kernels]
    assert len(names) == launches, names
    last = len(kernels) - 1
    if pair and not p.get('fused_add', False):
        assert 'k_add<' in names[last], names
        last -= 1
    if p['kernel'] == 'k_gemm_cc' and p['splits'] > 1:
        assert 'k_splitk_reduce<%s>' % R.PRECISIONS[precision].storage in names[last], names
        last -= 1
    tested = kernels[last]
    assert R.kernel_name_pattern(p, precision) in tested[0], (tested, p, names)
    if p['kernel'] == 'k_gemm_tc' and tested[1] is not None:
        assert tested[1][2] == p['splits'], (tested, p)

    # ---- the arithmetic
    kind = c.spec[0]
    f64 = [np.asarray(x, np.float64) for x in xs]
    if kind in ('pool', 'add', 'concat'):
        if kind == 'pool':
            want_y = R.pool_f32(xs[0], L.kh, L.stride, c.spec[5], precision)
        elif kind == 'add':
            want_y = R.add_f32(xs[0], xs[1], precision)
        else:
            cl = [m.layers[i] for i in range(li - 2, li + 1)]
            want_y = R.copy_channels_f32(xs, [q.row_off for q in cl], L.out_c, precision)
        assert np.array_equal(y, want_y)
        assert np.abs(y).max() > 0
        return
    sc = np.asarray(m.tensors[L.scale_tensor], np.float64)[:L.out_c]
    of = np.asarray(m.tensors[L.offset_tensor], np.float64)[:L.out_c]
    if kind == 'stem':
        a = pre.astype(np.float64)
        wt = _weights(m, L, precision, False)
        z, P = R.conv2d(a, wt, L.stride), R.conv2d(np.abs(a), np.abs(wt), L.stride)
        yr = R.affine(z, sc, of, L.act)
        bound = R.chain_bound(P, z * sc, yr, sc, of, L.kh * L.kw * 3, precision)
        err = np.abs(y - yr)
        record(c.family, precision, err, bound)
        assert np.all(err <= bound)
        return
    if kind == 'dw':
        wt = np.asarray(m.tensors[L.w_tensor], np.float64).reshape(3, 3, L.out_c)
        z, P = R.depthwise(f64[0], wt, L.stride), R.depthwise(np.abs(f64[0]), np.abs(wt), L.stride)
        yr = R.affine(z, sc, of, L.act)
        bound = R.chain_bound(P, z * sc, yr, sc, of, 9, precision)
        err = np.abs(y - yr)
        record(c.family, precision, err, bound)
        assert np.all(err <= bound)
        return
    G = m.layers[li - 1] if kind == 'pw_add' else L           # the GEMM layer
    gp = plans[-1]
    tc = gp['kernel'] == 'k_gemm_tc'
    wt = _weights(m, G, precision, tc)
    sc = np.asarray(m.tensors[G.scale_tensor], np.float64)[:G.out_c]
    of = np.asarray(m.tensors[G.offset_tensor], np.float64)[:G.out_c]
    z, P = R.conv2d(f64[0], wt, G.stride), R.conv2d(np.abs(f64[0]), np.abs(wt), G.stride)
    yr = R.affine(z, sc, of, G.act)
    K = G.kh * G.kw * G.in_c

    def bound_for(bp, q):
        """the bound of the layer's kernel in a `bp` engine (2: the tf32x3 bar)"""
        return R.dense_bound(P, z * sc, yr, sc, of, bp, k_blocks=q.get('k_blocks', 1), splits=q['splits'],
                             kb_per=q.get('kb_per'), K=K, tc=tc, head=G.op == OP_HEAD)

    if G.op == OP_HEAD:
        # every head of the model, scattered into the whole enc / logits arrays: a row written twice or not at all fails
        ref = [np.zeros(enc.shape), np.zeros(lg.shape)]
        bnd = {bp: [np.zeros(enc.shape), np.zeros(lg.shape)] for bp in {precision, 2 if tc else precision}}
        for hl in (q for q in m.layers if q.op == OP_HEAD):
            hw_t = _weights(m, hl, precision, tc)
            sc = np.asarray(m.tensors[hl.scale_tensor], np.float64)[:hl.out_c]
            of = np.asarray(m.tensors[hl.offset_tensor], np.float64)[:hl.out_c]
            z, P = R.conv2d(f64[0], hw_t, 1), R.conv2d(np.abs(f64[0]), np.abs(hw_t), 1)
            yr = R.affine(z, sc, of, hl.act)
            hq = R.plan(hl, c.n, precision, sms, c.env)
            R.head_scatter(yr, hl.anchors_per_loc, hl.n_box, hl.row_off, *ref)
            for bp, arrs in bnd.items():
                R.head_scatter(bound_for(bp, hq), hl.anchors_per_loc, hl.n_box, hl.row_off, *arrs)
        err = np.concatenate([np.abs(enc - ref[0]).ravel(), np.abs(lg - ref[1]).ravel()])
        yr = np.concatenate([r.ravel() for r in ref])
        bound, bound3 = (np.concatenate([b.ravel() for b in bnd[bp]]) for bp in (precision, 2 if tc else precision))
    else:
        err = np.abs(y - yr)
        bound = bound_for(precision, gp)
        bound3 = bound_for(2, gp) if tc else None
    if kind == 'pw_add':
        # Add(x, p): one more fp32 rounding, fused or not
        yr = yr + f64[0]
        err = np.abs(y - yr)
        bound, bound3 = (None if b is None else b + R.U * (np.abs(yr) + b) for b in (bound, bound3))
    ratio = record(c.family, precision, err, bound)
    assert np.all(err <= bound), (ratio, float(err.max()))
    assert np.abs(yr).max() > 0
    if precision == 3 and K >= 256:
        # the same kernel without the correction products must fail the tf32x3 bar
        assert np.max(err / bound3) > 1, 'the tf32x3 bound does not tell tf32x1 apart'
