"""The fp16 mode (precision 4) on the GPU: every backbone kernel that runs in bf16 runs again in fp16 against the float64
restatement of tests/layer_reference.py, the stem on camera frames, the frame path's bit-identity with the stage path,
saturation of overflowing activations at ±65504, the refusal of weights beyond the fp16 range, and the whole-network
error of fp16 against bf16's on the configs[2] model."""
import numpy as np
import pytest

from tests import layer_reference as R
from tests import test_gpu_frame_path as FP
from tests import test_gpu_layer_kernels as LK
from tests import workload
from tests.artist import artist_frame
from tests.test_gpu_frame_path import batches  # noqa: F401  (the frame batches fixture, shared with that module)
from tests.test_gpu_layer_kernels import report  # noqa: F401  (the largest error / bound per family)
from watsor_b200._lib import WatsorB200Error
from watsor_b200.engine import PRECISION_BF16_TC, PRECISION_FP16_TC, Engine
from watsor_b200.model import ACT_NONE, ACT_RELU6, OP_HEAD, Model, _Emitter

pytestmark = pytest.mark.gpu
FP16 = PRECISION_FP16_TC


# --------------------------------------------------------------------------------------- (1) every kernel vs float64
def _subnormal_weights(m, L):
    """the tested 1x1's weights -> fp16 subnormals of both signs, scale 1, offset 0: y = z exactly"""
    rng = np.random.default_rng(7)
    w = m.tensors[L.w_tensor]
    m.tensors[L.w_tensor] = (rng.choice([-1.0, 1.0], w.shape) * rng.uniform(2.0 ** -24, 2.0 ** -15, w.shape)).astype(np.float32)
    m.tensors[L.scale_tensor] = np.ones_like(m.tensors[L.scale_tensor])
    m.tensors[L.offset_tensor] = np.zeros_like(m.tensors[L.offset_tensor])
    assert np.all(np.abs(m.tensors[L.w_tensor]) < 2.0 ** -14)


# every case that runs in bf16, and a 1x1 whose weights are all fp16 subnormals (|w| < 2^-14): the bound has no
# absolute term for the product chain, so a tensor core that flushed subnormal operands would fail it
SUBNORMAL = LK.case('pw_subnormal_weights_K64_N64_10_n2', 'subnormal_w', ('gemm', 10, 64, 64, 1, 1, ACT_NONE), 2,
                    (FP16,), {'all': {'kernel': 'k_gemm_tc', 'splits': 1}}, prepare=_subnormal_weights)
CASES = [c for c in LK.CASES if 1 in c.precisions] + [SUBNORMAL]


@pytest.mark.parametrize('c', CASES, ids=lambda c: c.name + '-fp16')
def test_layer_kernel_fp16(c):
    LK.check_layer(c, FP16)


# ------------------------------------------------------------------------------------------- (2) stem on frames
@pytest.mark.parametrize('group', FP.GROUPS)
@pytest.mark.parametrize('stem', list(FP.STEMS))
def test_stem_on_frames_fp16(batches, stem, group):  # noqa: F811
    FP.test_stem_on_frames(batches, stem, FP16, group)


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
        over = np.abs(exact) > R.FP16_MAX
        assert np.array_equal(y[over], np.sign(exact[over]) * R.FP16_MAX)    # exactly ±65504, with the sign
        assert np.any(y[over] > 0) and np.any(y[over] < 0)
        assert np.array_equal(y, R.fp16_store(exact.astype(np.float32)))      # and the rest rounded as usual
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
    assert peak < R.FP16_MAX, 'the fp32 oracle activations leave the fp16 range: the comparison would measure the clamp'
    assert worst[FP16] <= worst[PRECISION_BF16_TC] / 4
