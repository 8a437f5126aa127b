"""The fused depthwise -> 1x1 (-> residual Add) tensor-core kernel (csrc/kernels_fused.cu) against the unfused
kernels (WB_NO_FUSE=1: k_dw_strip, then k_gemm_tc with its own residual epilogue).  The accumulation orders are
the same, so every output must be bit-identical; the launch counts show that the groups really were fused."""
import os

import numpy as np
import pytest

from tests import workload
from tests.test_fusion_plan import fused_groups
from watsor_b200.engine import Engine
from watsor_b200.model import ACT_NONE, ACT_RELU6, Model, _Emitter, synthetic_ssd_mobilenet_v2

pytestmark = pytest.mark.gpu


def _run(blob, pre, no_fuse, **backbone_args):
    if no_fuse:
        os.environ['WB_NO_FUSE'] = '1'
    try:
        with Engine(blob, device=0, max_batch=pre.shape[0], precision=2) as e:
            out = e.backbone(pre, **backbone_args)
            return out, e.last_launch_count()
    finally:
        os.environ.pop('WB_NO_FUSE', None)


@pytest.fixture(scope='module')
def v2_models():
    return {'configs2': workload.v2_coco_model(),
            '3class': synthetic_ssd_mobilenet_v2(num_classes=3, seed=2, score_thr=0.3)}


@pytest.mark.parametrize('n', [1, 3, 8])
@pytest.mark.parametrize('which', ['configs2', '3class'])
def test_v2_heads_fused_equal_unfused(v2_models, which, n):
    from oracle.ssd_model import SsdModelOracle
    from tests.artist import artist_frame
    m = v2_models[which]
    oracle = SsdModelOracle(m)
    pre = np.stack([oracle.preprocess(artist_frame(640, 480, 3, f)) for f in range(n)])
    blob = m.to_blob()
    (enc_f, lg_f, _), launches_f = _run(blob, pre, False)
    (enc_u, lg_u, _), launches_u = _run(blob, pre, True)
    assert np.array_equal(enc_f, enc_u) and np.array_equal(lg_f, lg_u)
    # every group the kernel takes runs as one launch instead of two: a silent fall-back fails here.  The 19x19
    # groups (blocks 6..9) stay unfused (maps under 32 x 32 pixels, kernels_fused.cu)
    fused = [g for g in fused_groups(m) if g[0].out_h * g[0].out_w >= 32 * 32]
    assert launches_u - launches_f == len(fused) == 6


def _block_model(hw, stride, C, N, residual, seed):
    """1x1 stem -> 1x1 expand to C (ReLU6) -> 3x3 depthwise (stride, ReLU6) -> linear 1x1 projection to N
    [-> Add(stem output, projection)]."""
    rng = np.random.default_rng(seed)
    m = Model(name='dwpw-test', input_h=hw, input_w=hw, num_classes=1, num_anchors=1)
    em = _Emitter(m)
    em.shape['image'] = (hw, hw, 3)

    def bn(c):
        return (1.0 + 0.1 * rng.standard_normal(c)).astype(np.float32), (0.1 * rng.standard_normal(c)).astype(np.float32)

    def w(shape, fan_in):
        return (rng.standard_normal(shape) * np.sqrt(2.0 / fan_in)).astype(np.float32)

    em.conv('stem', 'image', 'x', w((1, 1, 3, N), 3), *bn(N), 1, ACT_RELU6)
    em.conv('expand', 'x', 'e', w((1, 1, N, C), N), *bn(C), 1, ACT_RELU6)
    em.conv('depthwise', 'e', 'd', w((3, 3, C, 1), 9), *bn(C), stride, ACT_RELU6, depthwise=True)
    em.conv('project', 'd', 'p', w((1, 1, C, N), C), *bn(N), 1, ACT_NONE)
    if residual:
        em.add('add', 'x', 'p', 'y')
    m.anchors_tensor = m.add_tensor(np.zeros((1, 4), np.float32))
    m.plan_arena()
    return m, em.shape['y' if residual else 'p']


# stride 2 on odd maps (75 -> 38, 63 -> 32) and stride 1 (partial edge tiles at 75 and 33); C = 48 / 144 leave a
# half-filled last k-block, C = 96 does not
@pytest.mark.parametrize('hw,stride,C,N,residual', [
    (75, 2, 48, 24, False), (75, 2, 144, 64, False), (63, 2, 96, 24, False),
    (75, 1, 144, 24, True), (38, 1, 48, 64, True), (33, 1, 144, 64, True), (75, 1, 48, 24, False), (38, 1, 96, 64, False)])
@pytest.mark.parametrize('n', [1, 3])
def test_block_fused_equals_unfused(hw, stride, C, N, residual, n):
    m, shape = _block_model(hw, stride, C, N, residual, seed=C + N + hw)
    pre = np.random.default_rng(n).standard_normal((n, hw, hw, 3)).astype(np.float32)
    last = len(m.layers) - 1
    (_, _, y_f), launches_f = _run(m.to_blob(), pre, False, stop_layer=last, layer_shape=shape)
    (_, _, y_u), launches_u = _run(m.to_blob(), pre, True, stop_layer=last, layer_shape=shape)
    assert launches_u - launches_f == 1
    assert np.array_equal(y_f, y_u)
    assert np.abs(y_f).max() > 0
    # and both are right: float64 depthwise -> projection [-> Add] on the depthwise layer's GPU input
    from tests import layer_reference as R
    (_, _, e), _ = _run(m.to_blob(), pre, False, stop_layer=1, layer_shape=(hw, hw, C))
    e = e.astype(np.float64)
    dw, pw = m.layers[2], m.layers[3]

    def vec(L, t):
        return np.asarray(m.tensors[t], np.float64)[:L.out_c]

    wd = np.asarray(m.tensors[dw.w_tensor], np.float64).reshape(3, 3, C)
    zd, Pd = R.depthwise(e, wd, stride), R.depthwise(np.abs(e), np.abs(wd), stride)
    d = R.affine(zd, vec(dw, dw.scale_tensor), vec(dw, dw.offset_tensor), dw.act)
    bd = R.chain_bound(Pd, zd * vec(dw, dw.scale_tensor), d, vec(dw, dw.scale_tensor), vec(dw, dw.offset_tensor), 9)
    wp = np.asarray(m.tensors[pw.w_tensor], np.float64).reshape(C, pw.n_pad)[:, :N]
    sp, op = vec(pw, pw.scale_tensor), vec(pw, pw.offset_tensor)
    z, P = d @ wp, (np.abs(d) + bd) @ np.abs(wp)
    want = R.affine(z, sp, op, pw.act)
    # the projection's own bound (tf32x3, no split below 16 k-blocks) plus the depthwise error carried through it
    bound = R.dense_bound(P, z * sp, want, sp, op, 2, k_blocks=-(-C // 32)) + (bd @ np.abs(wp)) * np.abs(sp) * (1 + 1e-6)
    if residual:
        (_, _, x), _ = _run(m.to_blob(), pre, False, stop_layer=0, layer_shape=(hw, hw, N))
        want = want + x
        bound = bound + R.U * (np.abs(want) + bound)
    assert np.all(np.abs(y_f - want) <= bound), float(np.max(np.abs(y_f - want) / bound))
