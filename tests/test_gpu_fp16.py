"""The fp16 mode (precision 4) on the GPU: every backbone kernel that runs in bf16 runs again in fp16 against the float64
restatement of tests/layer_reference.py (fp16 storage, bounds and dispatch: tests/fp16_reference.py), the stem on
camera frames, the frame path's bit-identity with the stage path, saturation of overflowing activations at ±65504,
the refusal of weights beyond the fp16 range, and the whole-network error of fp16 against bf16's on the configs[2]
model."""
import numpy as np
import pytest

from tests import fp16_reference as F
from tests import layer_reference as R
from tests import test_gpu_frame_path as FP
from tests import test_gpu_layer_kernels as LK
from tests import workload
from tests.artist import artist_frame
from tests.test_gpu_frame_path import batches  # noqa: F401  (the frame batches fixture, shared with that module)
from watsor_b200._lib import WatsorB200Error
from watsor_b200.engine import PRECISION_BF16_TC, PRECISION_FP16_TC, Engine
from watsor_b200.model import ACT_NONE, ACT_RELU6, OP_HEAD, Model, _Emitter

pytestmark = pytest.mark.gpu
FP16 = PRECISION_FP16_TC
WORST = {}          # family -> largest error / bound


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    if WORST:
        print('\nfp16: largest error / bound per family:')
        for fam, r in sorted(WORST.items()):
            print('  %-18s %.3g' % (fam, r))


def _record(family, err, bound):
    ratio = float(np.max(err / bound))
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    return ratio


# --------------------------------------------------------------------------------------- (1) every kernel vs float64
# every case that runs in bf16, and a 1x1 whose weights are all fp16 subnormals (|w| < 2^-14): the bound has no
# absolute term for the product chain, so a tensor core that flushed subnormal operands would fail it
SUBNORMAL = LK.case('pw_subnormal_weights_K64_N64_10_n2', 'tc_pw', ('gemm', 10, 64, 64, 1, 1, ACT_NONE), 2, (FP16,),
                    {'all': {'kernel': 'k_gemm_tc', 'splits': 1}})
CASES = [c for c in LK.CASES if 1 in c.precisions] + [SUBNORMAL]


def _subnormal_weights(m, L, seed):
    """the tested 1x1's weights -> fp16 subnormals of both signs, scale 1, offset 0: y = z exactly"""
    rng = np.random.default_rng(seed)
    w = m.tensors[L.w_tensor]
    m.tensors[L.w_tensor] = (rng.choice([-1.0, 1.0], w.shape) * rng.uniform(2.0 ** -24, 2.0 ** -15, w.shape)).astype(np.float32)
    m.tensors[L.scale_tensor] = np.ones_like(m.tensors[L.scale_tensor])
    m.tensors[L.offset_tensor] = np.zeros_like(m.tensors[L.offset_tensor])
    assert np.all(np.abs(m.tensors[L.w_tensor]) < 2.0 ** -14)


def _weights(m, L, tc):
    K = L.kh * L.kw * L.in_c
    w = np.asarray(m.tensors[L.w_tensor], np.float32).reshape(K, L.n_pad)[:, :L.out_c]
    if tc:
        w = F.fp16_round(w)             # the tensor-core weights are rounded to fp16 once on the host
    return w.astype(np.float64).reshape(L.kh, L.kw, L.in_c, L.out_c)


@pytest.mark.parametrize('c', CASES, ids=lambda c: c.name + '-fp16')
def test_layer_kernel_fp16(c):
    m, li, inputs, (h, w) = LK.build(c.spec, seed=len(c.name))
    L = m.layers[li]
    if c is SUBNORMAL:
        _subnormal_weights(m, L, 7)
    sms = LK._sms()
    pre = np.random.default_rng(c.n).standard_normal((c.n, h, w, 3)).astype(np.float32)
    xs, (enc, lg, y), launches, kernels = LK._run(m, li, inputs, pre, FP16, c.env)

    # ---- the branch: plan(), launch count, kernel name (+ cluster split); the claims are bf16's (same plan)
    plans = [F.plan(Li, c.n, sms, c.env) for Li in m.layers[:li + 1]]
    p = plans[-1]
    want = LK.claim_for(c, 1 if 1 in c.precisions else FP16)
    assert {k: p[k] for k in want} == want, (p, want)
    assert launches == sum(q['launches'] for q in plans), (launches, plans)
    names = [k for k, _ in kernels]
    assert len(names) == launches, names
    last = len(kernels) - 1
    if p['kernel'] == 'k_gemm_cc' and p['splits'] > 1:
        assert 'k_splitk_reduce<__half>' in names[last], names
        last -= 1
    tested = kernels[last]
    assert F.kernel_name_pattern(p) in tested[0], (tested, p, names)
    if p['kernel'] == 'k_gemm_tc' and tested[1] is not None:
        assert tested[1][2] == p['splits'], (tested, p)

    # ---- the arithmetic
    kind = c.spec[0]
    f64 = [np.asarray(x, np.float64) for x in xs]
    if kind in ('pool', 'add', 'concat'):
        if kind == 'pool':
            want_y = F.pool_f32(xs[0], L.kh, L.stride, c.spec[5])
        elif kind == 'add':
            want_y = F.add_f32(xs[0], xs[1])
        else:
            cl = [m.layers[i] for i in range(li - 2, li + 1)]
            want_y = F.copy_channels_f32(xs, [q.row_off for q in cl], L.out_c)
        assert np.array_equal(y, want_y)
        assert np.abs(y).max() > 0
        return
    sc = np.asarray(m.tensors[L.scale_tensor], np.float64)[:L.out_c]
    of = np.asarray(m.tensors[L.offset_tensor], np.float64)[:L.out_c]
    if kind in ('stem', 'dw'):
        if kind == 'stem':
            a, wt, terms = pre.astype(np.float64), _weights(m, L, False), L.kh * L.kw * 3
            z, P = R.conv2d(a, wt, L.stride), R.conv2d(np.abs(a), np.abs(wt), L.stride)
        else:
            wt, terms = np.asarray(m.tensors[L.w_tensor], np.float64).reshape(3, 3, L.out_c), 9
            z, P = R.depthwise(f64[0], wt, L.stride), R.depthwise(np.abs(f64[0]), np.abs(wt), L.stride)
        yr = R.affine(z, sc, of, L.act)
        bound = F.chain_bound(P, z * sc, yr, sc, of, terms)
        err = np.abs(y - yr)
        _record(c.family, err, bound)
        assert np.all(err <= bound)
        return
    tc = p['kernel'] == 'k_gemm_tc'
    mode = FP16 if tc else 0

    def bound_for(q, P, z, sc, of, yr, is_head):
        if mode == 0:
            return F.dense_bound(P, z * sc, yr, sc, of, 0, K=L.kh * L.kw * L.in_c, splits=q['splits'], fp16_out=not is_head)
        return F.dense_bound(P, z * sc, yr, sc, of, mode, k_blocks=q['k_blocks'], splits=q['splits'], kb_per=q['kb_per'],
                             fp16_out=not is_head)

    if L.op == OP_HEAD:
        ref, bnd = [np.zeros(enc.shape), np.zeros(lg.shape)], [np.zeros(enc.shape), np.zeros(lg.shape)]
        for hl in (q for q in m.layers if q.op == OP_HEAD):
            hw_t = _weights(m, hl, tc)
            hsc = np.asarray(m.tensors[hl.scale_tensor], np.float64)[:hl.out_c]
            hof = np.asarray(m.tensors[hl.offset_tensor], np.float64)[:hl.out_c]
            z, P = R.conv2d(f64[0], hw_t, 1), R.conv2d(np.abs(f64[0]), np.abs(hw_t), 1)
            yr = R.affine(z, hsc, hof, hl.act)
            hq = F.plan(hl, c.n, sms, c.env)
            R.head_scatter(yr, hl.anchors_per_loc, hl.n_box, hl.row_off, *ref)
            R.head_scatter(bound_for(hq, P, z, hsc, hof, yr, True), hl.anchors_per_loc, hl.n_box, hl.row_off, *bnd)
        err = np.concatenate([np.abs(enc - ref[0]).ravel(), np.abs(lg - ref[1]).ravel()])
        yr = np.concatenate([r.ravel() for r in ref])
        bound = np.concatenate([b.ravel() for b in bnd])
    else:
        wt = _weights(m, L, tc)
        z, P = R.conv2d(f64[0], wt, L.stride), R.conv2d(np.abs(f64[0]), np.abs(wt), L.stride)
        yr = R.affine(z, sc, of, L.act)
        err = np.abs(y - yr)
        bound = bound_for(p, P, z, sc, of, yr, False)
    ratio = _record('subnormal_w' if c is SUBNORMAL else c.family, err, bound)
    assert np.all(err <= bound), (ratio, float(err.max()))
    assert np.abs(yr).max() > 0


# ------------------------------------------------------------------------------------------- (2) stem on frames
@pytest.mark.parametrize('group', FP.GROUPS)
@pytest.mark.parametrize('stem', list(FP.STEMS))
def test_stem_on_frames_fp16(batches, stem, group):  # noqa: F811
    """test_gpu_frame_path (a) in fp16: bit-identical to the stem on preprocess() of the same RGB images, and within
    the float64 bound on oracle.preprocess, for both stem kernels."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    m = FP._stem_model(stem)
    L = m.layers[0]
    shape = (L.out_h, L.out_w, L.out_c)
    plan = F.plan(L, 1, torch.cuda.get_device_properties(0).multi_processor_count)
    with Engine(m.to_blob(), device=0, max_batch=FP.MAX_IMAGES, precision=FP16) as e:
        runs = []
        for fmt, cams, frames, images in batches[group]:
            FP._configure(e, cams)
            runs += [(fmt, cams, frames, images, False, frames), (fmt, cams, frames, images, True, FP._to_device(frames))]
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                got = []
                for fmt, cams, _, images, on_dev, src in runs:
                    ptrs = [t.data_ptr() for t in src] if on_dev else src
                    _, _, y, n_img = e.backbone_frames(ptrs, list(cams), stop_layer=0, layer_shape=shape,
                                                       pixel_format=fmt, frames_on_device=on_dev)
                    assert n_img == len(images) and e.last_launch_count() == 1
                    got.append(y)
                torch.cuda.synchronize()
            kernels = [k for k, _ in LK._kernels(prof)]
            if len(kernels) == len(runs):
                break
        assert len(kernels) == len(runs), kernels
        assert all(F.kernel_name_pattern(plan) in k for k in kernels), (plan['kernel'], kernels)
        for b, (fmt, cams, frames, images) in enumerate(batches[group]):
            want = e.backbone(e.preprocess(images), stop_layer=0, layer_shape=shape)[2]
            for on_dev in (False, True):
                assert np.array_equal(got[2 * b + on_dev], want), (fmt, list(cams.values()), on_dev)
            key = (stem, group, b)
            if key not in FP.REFS:
                FP.REFS[key] = FP._stem_reference(m, images)
            zs, P, yr, sc, of = FP.REFS[key]
            bound = F.chain_bound(P, zs, yr, sc, of, L.kh * L.kw * 3)
            err = np.abs(got[2 * b] - yr)
            _record('frames:' + plan['kernel'], err, bound)
            assert np.all(err <= bound), (fmt, list(cams.values()), float(np.max(err / bound)))
            assert np.abs(yr).max() > 0


# ------------------------------------------------------------------------------------------------ (3) frame path
@pytest.mark.parametrize('net', list(FP.NETWORKS))
def test_network_frames_equal_stage_path_fp16(request, net):
    FP.test_network_frames_equal_stage_path(request, net, FP16)


def test_graph_replay_with_windows_fp16():
    FP.test_graph_replay_depends_only_on_its_key(FP16, True)


# ------------------------------------------------------------------------------------------------- (4) saturation
# Tiny models whose tested layer's exact output exceeds 65504: the stem's ReLU6 holds every input at exactly 6 (zero
# weights, offset 6), weights are powers of two, so the exact output is known and fp32 computes it exactly.  Channel
# scales alternate in sign, and a quarter of them keep the output in range.  A head reads the tested layer.
SAT_KINDS = {'k_gemm_tc': 32, 'k_gemm_cc': 36, 'k_dw_strip': 32, 'k_add': 32}


def _sat_scales(c, big):
    s = np.where(np.arange(c) % 2 == 0, big, -big).astype(np.float32)
    s[::4] = np.float32(1000.0) * np.sign(s[::4])
    return s


def _sat_model(kind, huge_weight=False):
    c = SAT_KINDS[kind]
    m = Model(name='sat-' + kind, input_h=20, input_w=20, num_classes=2, num_anchors=1)
    em = _Emitter(m)
    em.shape['image'] = (20, 20, 3)
    em.conv('stem', 'image', 's', np.zeros((3, 3, 3, c), np.float32), np.ones(c, np.float32),
            np.full(c, 6.0, np.float32), 1, ACT_RELU6)
    w1 = np.full((1, 1, c, c), 1.0 / 32, np.float32)
    if kind in ('k_gemm_tc', 'k_gemm_cc'):
        if huge_weight:
            w1[0, 0, 3, 5] = 1e5
        em.conv('tested', 's', 'y', w1, _sat_scales(c, 2e4), np.zeros(c, np.float32), 1, ACT_NONE)
    elif kind == 'k_dw_strip':
        # 4 / 6 / 9 in-image taps of 6 * 0.125: 3, 4.5 or 6.75, times 3e4: every scaled channel saturates
        em.conv('tested', 's', 'y', np.full((3, 3, c, 1), 0.125, np.float32), _sat_scales(c, 3e4),
                np.zeros(c, np.float32), 1, ACT_NONE, depthwise=True)
    else:
        # two 1x1 of 6 * 32 / 32 * 8000 = 48000 each (exact in fp16), summed: 96000
        for dst in ('a', 'b'):
            em.conv('mix_' + dst, 's', dst, w1, _sat_scales(c, 8000.0), np.zeros(c, np.float32), 1, ACT_NONE)
        em.add('tested', 'a', 'b', 'y')
    li = len(m.layers) - 1
    rng = np.random.default_rng(1)
    m.num_anchors = em.head('head', 'y', (rng.standard_normal((1, 1, c, 4)) * 1e-3).astype(np.float32),
                            np.zeros(4, np.float32), (rng.standard_normal((1, 1, c, 3)) * 1e-3).astype(np.float32),
                            np.zeros(3, np.float32), 0, 3)
    return LK._finish(m), li


def _sat_exact(kind, m, li):
    """the tested layer's exact output (float64) for the all-6 input"""
    L = m.layers[li]
    x = np.full((1, 20, 20, L.in_c), 6.0)
    if kind == 'k_add':
        mix = m.layers[li - 1]
        sc = np.asarray(m.tensors[mix.scale_tensor], np.float64)[:mix.out_c]
        one = R.affine(R.conv2d(x, np.full((1, 1, L.in_c, L.in_c), 1.0 / 32), 1), sc, 0.0, ACT_NONE)
        return one + one
    sc = np.asarray(m.tensors[L.scale_tensor], np.float64)[:L.out_c]
    if kind == 'k_dw_strip':
        return R.affine(R.depthwise(x, np.full((3, 3, L.out_c), 0.125), 1), sc, 0.0, ACT_NONE)
    return R.affine(R.conv2d(x, np.full((1, 1, L.in_c, L.out_c), 1.0 / 32), 1), sc, 0.0, ACT_NONE)


@pytest.mark.parametrize('kind', list(SAT_KINDS))
def test_saturation(kind):
    import torch
    from torch.profiler import ProfilerActivity, profile
    m, li = _sat_model(kind)
    L = m.layers[li]
    shape = (L.out_h, L.out_w, L.out_c)
    exact = _sat_exact(kind, m, li)
    assert np.abs(exact).max() > 65520 and np.abs(exact).min() < 65504        # both sides of the clamp
    pre = np.zeros((1, 20, 20, 3), np.float32)
    with Engine(m.to_blob(), device=0, max_batch=1, precision=FP16) as e:
        pattern = 'k_gemm_tc<3,' if kind == 'k_gemm_tc' else kind + '<__half'
        for _ in range(2):          # a short profiler session now and then misses the device activity: trace again
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                _, _, y = e.backbone(pre, stop_layer=li, layer_shape=shape)
                torch.cuda.synchronize()
            names = [k for k, _ in LK._kernels(prof)]
            if names:
                break
        assert any(pattern in k for k in names), names
        over = np.abs(exact) > F.FP16_MAX
        assert np.array_equal(y[over], np.sign(exact[over]) * F.FP16_MAX)    # exactly ±65504, with the sign
        assert np.any(y[over] > 0) and np.any(y[over] < 0)
        assert np.array_equal(y, F.fp16_store(exact.astype(np.float32)))      # and the rest rounded as usual
        enc, lg, _ = e.backbone(pre)
        assert np.all(np.isfinite(enc)) and np.all(np.isfinite(lg))
        assert np.abs(enc).max() > 0
    with Engine(m.to_blob(), device=0, max_batch=1, precision=PRECISION_BF16_TC) as e:
        _, _, yb = e.backbone(pre, stop_layer=li, layer_shape=shape)
        # bf16 keeps fp32's exponent range: the same layer stores the exact value rounded to bf16, no clamp
        assert np.array_equal(yb, R.bf16_round(exact.astype(np.float32)))
        assert np.abs(yb).max() > 65520


@pytest.mark.parametrize('kind', ['k_gemm_tc', 'k_gemm_cc'])
def test_weight_beyond_fp16_range(kind):
    """A tensor-core weight of 1e5 would become inf in fp16: wb_create refuses the model and names the layer.  The
    CUDA-core GEMM keeps fp32 weights, so a model whose 1x1 runs there (K % 8 != 0) is accepted; bf16 accepts both."""
    m, _ = _sat_model(kind, huge_weight=True)
    if kind == 'k_gemm_tc':
        with pytest.raises(WatsorB200Error, match='tested'):
            Engine(m.to_blob(), device=0, max_batch=1, precision=FP16)
    else:
        Engine(m.to_blob(), device=0, max_batch=1, precision=FP16).close()
    Engine(m.to_blob(), device=0, max_batch=1, precision=PRECISION_BF16_TC).close()


# ------------------------------------------------------------------------------------ (5) whole-network accuracy
def test_configs2_layer_error_fp16_vs_bf16():
    """test_v2_layer_by_layer's measure (max |GPU - fp32 oracle| over max(1, max |oracle|), per layer) on the
    configs[2] model and frames, in bf16 and fp16.  fp16's unit roundoff is 8x smaller and the accumulation is shared,
    so its worst layer must be at least 4x closer than bf16's."""
    from oracle.ssd_model import SsdModelOracle
    m = workload.v2_coco_model()
    oracle = SsdModelOracle(m)
    worst = {PRECISION_BF16_TC: 0.0, FP16: 0.0}
    peak = 0.0
    for cam in (0, 5):
        pre = oracle.preprocess(artist_frame(640, 480, cam, cam % 3))
        _, _, memo = oracle.raw_heads(pre, return_memo=True)
        want = {li: oracle.feature(memo, li) for li, layer in enumerate(m.layers) if layer.op != OP_HEAD}
        peak = max(peak, max(float(np.abs(v).max()) for v in want.values()))
        for precision in worst:
            with Engine(m.to_blob(), device=0, max_batch=1, precision=precision) as e:
                for li, w in want.items():
                    got = e.backbone(pre[None], stop_layer=li, layer_shape=w.shape)[2][0]
                    worst[precision] = max(worst[precision], float(np.abs(got - w).max()) / max(1.0, float(np.abs(w).max())))
    print('configs[2] worst per-layer error / range: bf16 %.3g, fp16 %.3g (ratio %.3g); largest |activation| %.4g'
          % (worst[PRECISION_BF16_TC], worst[FP16], worst[FP16] / worst[PRECISION_BF16_TC], peak))
    assert peak < F.FP16_MAX, 'the fp32 oracle activations leave the fp16 range: the comparison would measure the clamp'
    assert worst[FP16] <= worst[PRECISION_BF16_TC] / 4
