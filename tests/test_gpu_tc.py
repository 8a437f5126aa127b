"""The wgmma GEMM kernel (csrc/kernels_tc.cu) in isolation: one 1x1 convolution per precision mode
against a float64 reference computed from the very activations the GPU produced."""
import numpy as np
import pytest

from watsor_b200.engine import Engine
from watsor_b200.model import Model, _Emitter

pytestmark = pytest.mark.gpu


def tiny_model(K, N, hw, seed=0):
    rng = np.random.default_rng(seed)
    m = Model(name='gemm-test', input_h=hw, input_w=hw, num_classes=1, num_anchors=1)
    em = _Emitter(m)
    em.shape['image'] = (hw, hw, 3)
    w0 = rng.standard_normal((1, 1, 3, K)).astype(np.float32)
    em.conv('stem', 'image', 'a', w0, np.ones(K, np.float32), np.zeros(K, np.float32), 1, 0)
    w1 = (rng.standard_normal((1, 1, K, N)) / np.sqrt(K)).astype(np.float32)
    sc = (1.0 + 0.1 * rng.standard_normal(N)).astype(np.float32)
    of = (0.1 * rng.standard_normal(N)).astype(np.float32)
    em.conv('pw', 'a', 'b', w1, sc, of, 1, 1)
    m.anchors_tensor = m.add_tensor(np.zeros((1, 4), np.float32))
    m.plan_arena()
    return m, w1.reshape(K, N), sc, of


# (K, N, hw, batch): K = 32 is a half-filled swizzle row in bf16, N = 48 / 96 / 16 leave the last N tile ragged,
# M = 9 is a mostly out-of-bounds TMA box, 1024x1024 runs the full smem pipeline and the cluster split-K
CASES = [(512, 512, 19, 4), (32, 64, 32, 2), (1024, 1024, 10, 8), (256, 48, 3, 1), (64, 128, 20, 3),
         (128, 96, 7, 2), (16, 16, 5, 1),
         # more output tiles than SMs; the last row tile is partial in each (M = 22500, 28125, 20172) and
         # 256 columns make two N tiles
         (32, 64, 150, 1), (64, 128, 75, 5), (128, 256, 41, 12), (24, 128, 150, 2),
         # split-K clusters of 4, 3 (ragged N), 5 (the last k-block holds 20 of 32 values and the last split is
         # shorter) and 8 members (the portable cluster limit) on 132 SMs
         (1024, 128, 7, 1), (768, 96, 19, 2), (1300, 48, 10, 1), (2048, 64, 10, 1)]


@pytest.mark.parametrize('precision,rel_tol', [(2, 3e-6), (3, 4e-3), (1, 1.5e-2)],
                         ids=['tf32x3', 'tf32x1', 'bf16'])
@pytest.mark.parametrize('K,N,hw,n', CASES)
def test_pointwise_gemm(precision, rel_tol, K, N, hw, n):
    m, w1, sc, of = tiny_model(K, N, hw)
    pre = np.random.default_rng(1).standard_normal((n, hw, hw, 3)).astype(np.float32)
    with Engine(m.to_blob(), device=0, max_batch=n, precision=precision) as e:
        _, _, a = e.backbone(pre, stop_layer=0, layer_shape=(hw, hw, K))
        _, _, y = e.backbone(pre, stop_layer=1, layer_shape=(hw, hw, N))
    w = w1.astype(np.float64)
    if precision == 1:
        # the weights are rounded to bf16 once on the host; activations already are bf16
        import torch
        w = torch.from_numpy(w1).to(torch.bfloat16).to(torch.float64).numpy()
    ref = a.reshape(-1, K).astype(np.float64) @ w
    ref = np.clip(ref * sc.astype(np.float64) + of.astype(np.float64), 0.0, 6.0)
    err = np.abs(y.reshape(-1, N) - ref).max()
    assert err <= rel_tol * max(1.0, np.abs(ref).max()) * (4 if precision == 1 else 1), (err, np.abs(ref).max())


def test_fused_depthwise_pointwise_equals_unfused(shapes_model):
    """k_dwpw_tc_x3 (depthwise fused into the GEMM's A-operand producer, csrc/kernels_fused.cu) against
    the two-kernel path (WB_NO_FUSE=1): same accumulation orders, so the head outputs are bit-identical."""
    import os
    from tests.artist import artist_frame
    from oracle.ssd_model import SsdModelOracle
    oracle = SsdModelOracle(shapes_model)
    pres = np.stack([oracle.preprocess(artist_frame(640, 480, 3, f)) for f in range(4)])
    outs = []
    for no_fuse in (False, True):
        if no_fuse:
            os.environ['WB_NO_FUSE'] = '1'
        else:
            os.environ.pop('WB_NO_FUSE', None)
        try:
            with Engine(shapes_model.to_blob(), device=0, max_batch=4, precision=2) as e:
                enc, lg, _ = e.backbone(pres)
                launches = e.last_launch_count()
        finally:
            os.environ.pop('WB_NO_FUSE', None)
        outs.append((enc, lg, launches))
    assert outs[0][2] < outs[1][2]                      # fewer launches: pairs really were fused
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
