"""Host checks of the fp16 mode (precision 4) in tests/layer_reference.py: the restatement of fp16 storage against
numpy's and torch's float16, its bounds and kernel dispatch against bf16's, and the WATSOR_B200_PRECISION names."""
import numpy as np
import pytest

from tests import layer_reference as R
from tests.test_gpu_layer_kernels import CASES, build
from watsor_b200.detection.b200 import default_precision
from watsor_b200.engine import PRECISION_BF16_TC, PRECISION_FP16_TC


def _probe_values():
    """Every fp16 value, the midpoints between neighbours (ties), points just off the midpoints, the subnormal range,
    and values around and beyond the overflow threshold 65520."""
    h = np.arange(0, 0x7C00, dtype=np.uint16).view(np.float16).astype(np.float64)      # +0 .. 65504
    mid = (h[:-1] + h[1:]) / 2
    nxt = np.nextafter(mid.astype(np.float32), np.float32(np.inf)).astype(np.float64)
    prv = np.nextafter(mid.astype(np.float32), np.float32(0)).astype(np.float64)
    rng = np.random.default_rng(0)
    sub = rng.uniform(0, 2.0 ** -14, 20000)
    big = np.array([65504.0, 65519.0, 65519.996, 65520.0, 65536.0, 1e5, 3.0e38])
    x = np.concatenate([h, mid, nxt, prv, sub, big, 2.0 ** -25 * np.arange(0, 8)]).astype(np.float32)
    return np.concatenate([x, -x])


def test_fp16_round_equals_numpy_and_torch():
    import torch
    x = _probe_values()
    got = R.fp16_round(x)
    with np.errstate(over='ignore'):
        want = x.astype(np.float16).astype(np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))        # bit-equal: -0 and inf included
    tw = torch.from_numpy(x).to(torch.float16).to(torch.float32).numpy()
    assert np.array_equal(got.view(np.uint32), tw.view(np.uint32))
    # the probe reaches ties both ways, subnormal results and overflow
    assert np.any(got == np.float32(2.0 ** -24)) and np.any(np.isinf(got)) and np.any((got != 0) & (np.abs(got) < 2.0 ** -14))


def test_fp16_store_saturates():
    x = np.array([65504.0, 65505.0, 65519.0, 65520.0, 1e5, 3.0e38, -65505.0, -1e5, -3.0e38, 1.0, -2.5], np.float32)
    y = R.fp16_store(x)
    assert np.array_equal(y, [65504, 65504, 65504, 65504, 65504, 65504, -65504, -65504, -65504, 1.0, -2.5])
    big = _probe_values()
    assert np.all(np.isfinite(R.fp16_store(big)))
    inside = np.abs(big) <= R.FP16_MAX
    assert np.array_equal(R.fp16_store(big)[inside], R.fp16_round(big)[inside])


def test_fp16_output_bound_covers_rounding():
    """dense_bound's fp16 output term covers the rounding of every probe value that fits (normal and subnormal)."""
    x = _probe_values()
    x = x[np.abs(x) <= R.FP16_MAX].astype(np.float64)
    err = np.abs(R.fp16_round(x).astype(np.float64) - x)
    assert np.all(err <= R.U_FP16 * np.abs(x) + R.FP16_SUB_HALF)


@pytest.mark.parametrize('c', CASES, ids=lambda c: c.name)
def test_plan_fp16_equals_bf16(c):
    """Precision 4 takes bf16's dispatch: the restated fp16 tensor-core gate (2-byte elements) admits exactly the
    layers bf16's does, and the plan differs from bf16's only in the tensor-core GEMM's MODE (3 for fp16, 0 for
    bf16).  The GPU test proves the plan against the device (launch count, kernel names, cluster split)."""
    m, li, _, _ = build(c.spec, seed=len(c.name))
    pair = c.spec[0] == 'pw_add'
    for sms in (132, 114):
        for i, L in enumerate(m.layers[:li + 1]):
            if pair and i == li:
                continue
            kw = dict(env=c.env, fuse_add_next=pair and i == li - 1)
            assert R.tc_supported(L, 4, c.env) == R.tc_supported(L, 1, c.env), (c.name, L.name)
            p1, p4 = R.plan(L, c.n, 1, sms, **kw), R.plan(L, c.n, 4, sms, **kw)
            assert (p4['kernel'] == 'k_gemm_tc') == R.tc_supported(L, 4, c.env)
            if p1['kernel'] == 'k_gemm_tc':
                assert (p1.pop('mode'), p4.pop('mode')) == (0, 3)
            assert p1 == p4, (c.name, L.name, p1, p4)


def test_fp16_bounds_add_the_output_rounding():
    """fp16's dense and chain bounds are bf16's chain / the fp32 chain plus the fp16 output rounding; heads
    (head=True) keep the bound of the chain alone."""
    rng = np.random.default_rng(3)
    P, zs, y, sc, of = (np.abs(rng.standard_normal(50)) for _ in range(5))
    b1 = R.dense_bound(P, zs, y, sc, of, 1, k_blocks=4, splits=2, kb_per=2, head=True)
    b4 = R.dense_bound(P, zs, y, sc, of, 4, k_blocks=4, splits=2, kb_per=2)
    assert np.array_equal(b4, b1 + R.U_FP16 * (np.abs(y) + b1) + R.FP16_SUB_HALF)
    assert np.array_equal(R.dense_bound(P, zs, y, sc, of, 4, k_blocks=4, splits=2, kb_per=2, head=True), b1)
    b0 = R.chain_bound(P, zs, y, sc, of, 9)
    assert np.array_equal(R.chain_bound(P, zs, y, sc, of, 9, 4), b0 + R.U_FP16 * (np.abs(y) + b0) + R.FP16_SUB_HALF)


def test_kernel_name_pattern_fp16():
    assert R.kernel_name_pattern(dict(kernel='k_gemm_tc', mode=3, bn=64), 4) == 'k_gemm_tc<3, 64>'
    assert R.kernel_name_pattern(dict(kernel='k_dw_strip', stride=2), 4) == 'k_dw_strip<__half, 2>'
    assert R.kernel_name_pattern(dict(kernel='k_gemm_cc', tile=64), 4) == 'k_gemm_cc<__half, 64, 64, 4, 4>'
    assert R.kernel_name_pattern(dict(kernel='k_stem_3x3s2_c32'), 4) == 'k_stem_3x3s2_c32<__half'
    assert R.kernel_name_pattern(dict(kernel='k_add'), 4) == 'k_add<__half'


def test_fp16_storage_restatements():
    """k_add / k_copy_channels / k_pool in fp16: the float32 result, clamped and rounded."""
    x = np.array([[[[40000.0, -40000.0, 1.0 + 2.0 ** -12, 3.0e-8]]]], np.float32)
    assert np.array_equal(R.add_f32(x, x, 4), R.fp16_store(2 * x))
    assert np.array_equal(R.add_f32(x, x, 4)[0, 0, 0], [65504, -65504, 2.0, 2.0 ** -24])
    assert np.array_equal(R.copy_channels_f32([x], [0], 4, 4), R.fp16_round(x))
    assert np.array_equal(R.pool_f32(x, 1, 1, 'max', 4), R.fp16_round(x))


@pytest.mark.parametrize('value,want', [('fp16', PRECISION_FP16_TC), ('FP16', PRECISION_FP16_TC),
                                        ('half', PRECISION_FP16_TC), ('16', PRECISION_BF16_TC),
                                        ('bf16', PRECISION_BF16_TC)])
def test_default_precision_names(monkeypatch, value, want):
    monkeypatch.setenv('WATSOR_B200_PRECISION', value)
    assert default_precision() == want
    assert PRECISION_FP16_TC == 4
