"""tests/layer_reference.py on the CPU: its float64 operations against torch's, its bounds against known-wrong
results, and its dispatch restatement against the GPU case table (tests/test_gpu_layer_kernels.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import layer_reference as R
from tests.test_gpu_layer_kernels import CASES, build, claim_for
from tests.test_gpu_tc import CASES as PW_CASES
from watsor_b200.model import OP_PW, Layer, same_pad

SMS = 132       # H100 SXM


def _torch_same_pad(x, k, s, fill=0.0):
    """x NCHW padded as TF SAME with an explicit, possibly asymmetric F.pad."""
    H, W = x.shape[2:]
    oh, pt = same_pad(H, k, s)
    ow, pl = same_pad(W, k, s)
    th, tw = max((oh - 1) * s + k - H, 0), max((ow - 1) * s + k - W, 0)
    return F.pad(x, (pl, tw - pl, pt, th - pt), value=fill)


def _nchw(x):
    return torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2)))


def _nhwc(t):
    return t.numpy().transpose(0, 2, 3, 1)


SHAPES = [(1, 1), (2, 2), (3, 3), (4, 4), (5, 7), (10, 10), (11, 11), (19, 19), (38, 38)]


@pytest.mark.parametrize('k,s', [(1, 1), (1, 2), (3, 1), (3, 2), (7, 2), (7, 1)])
@pytest.mark.parametrize('h,w', SHAPES)
def test_conv_and_depthwise_equal_torch(h, w, k, s):
    rng = np.random.default_rng(h * 31 + w + k + s)
    x = rng.standard_normal((2, h, w, 5))
    wt = rng.standard_normal((k, k, 5, 6))
    want = F.conv2d(_torch_same_pad(_nchw(x), k, s), torch.from_numpy(wt.transpose(3, 2, 0, 1).copy()), stride=s)
    assert np.allclose(R.conv2d(x, wt, s), _nhwc(want), rtol=1e-12, atol=1e-12)
    wd = rng.standard_normal((k, k, 5))
    want = F.conv2d(_torch_same_pad(_nchw(x), k, s), torch.from_numpy(wd.transpose(2, 0, 1)[:, None].copy()),
                    stride=s, groups=5)
    assert np.allclose(R.depthwise(x, wd, s), _nhwc(want), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('k,s', [(3, 1), (3, 2), (1, 1), (2, 2)])
@pytest.mark.parametrize('h,w', SHAPES + [(75, 75)])
def test_pools_equal_torch(h, w, k, s):
    x = np.random.default_rng(h + w).standard_normal((2, h, w, 4))
    want = F.max_pool2d(_torch_same_pad(_nchw(x), k, s, -np.inf), k, s)
    assert np.array_equal(R.pool(x, k, s, 'max'), _nhwc(want))
    # AvgPool SAME: SAME pads pt before and pt or pt + 1 after, i.e. torch's symmetric padding pt with ceil_mode
    # adding the odd window; count_include_pad=False divides by the in-image taps
    _, pt = same_pad(h, k, s)
    _, pl = same_pad(w, k, s)
    want = F.avg_pool2d(_nchw(x), k, s, padding=(pt, pl), count_include_pad=False, ceil_mode=True)
    got = R.pool(x, k, s, 'avg')
    assert got.shape == _nhwc(want).shape and np.allclose(got, _nhwc(want), rtol=1e-12, atol=1e-12)
    # the float32 restatements: max exactly, average within its two float32 roundings per tap
    x32 = x.astype(np.float32)
    assert np.array_equal(R.pool_f32(x32, k, s, 'max'), R.pool(x32, k, s, 'max').astype(np.float32))
    assert np.allclose(R.pool_f32(x32, k, s, 'avg'), R.pool(x32, k, s, 'avg'), rtol=0, atol=1e-5)


def test_bf16_round_is_nearest_even():
    x = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -9), 3.14159, -0.0], np.float32)
    want = torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy()
    assert np.array_equal(R.bf16_round(x), want)


def test_head_scatter_layout():
    n, h, w, a, ncp1 = 2, 2, 3, 3, 4
    y = np.arange(n * h * w * a * (4 + ncp1), dtype=np.float64).reshape(n, h, w, -1)
    enc, lg = np.zeros((n, 5 + h * w * a, 4)), np.zeros((n, 5 + h * w * a, ncp1))
    R.head_scatter(y, a, 4 * a, 5, enc, lg)
    f, py, px, j = 1, 1, 2, 2
    row = 5 + (py * w + px) * a + j
    assert np.array_equal(enc[f, row], y[f, py, px, 4 * j:4 * j + 4])
    assert np.array_equal(lg[f, row], y[f, py, px, 4 * a + ncp1 * j:4 * a + ncp1 * (j + 1)])
    assert not enc[:, :5].any() and not lg[:, :5].any()


# ---------------------------------------------------------------------------------------------- negative controls
def _dense_case(k, s, cin, cout, seed=0):
    rng = np.random.default_rng(seed)
    x = np.clip(rng.standard_normal((2, 10, 10, cin)) * 2 + 0.5, -6, 6)
    wt = rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)
    sc, of = 1 + 0.1 * rng.standard_normal(cout), 0.1 * rng.standard_normal(cout)
    z, P = R.conv2d(x, wt, s), R.conv2d(np.abs(x), np.abs(wt), s)
    yr = R.affine(z, sc, of, 0)
    K = k * k * cin
    kb = -(-K // 32)
    bounds = {0: R.dense_bound(P, z * sc, yr, sc, of, 0, K=K),
              2: R.dense_bound(P, z * sc, yr, sc, of, 2, k_blocks=kb),
              3: R.dense_bound(P, z * sc, yr, sc, of, 3, k_blocks=kb)}
    return x, wt, sc, of, yr, bounds


def _rejected(got, yr, bounds, modes=(0, 2)):
    return all(np.any(np.abs(got - yr) > bounds[md]) for md in modes)


@pytest.mark.parametrize('s', [1, 2])
def test_bound_rejects_shifted_padding(s):
    x, wt, sc, of, yr, bounds = _dense_case(3, s, 64, 48)
    shifted = np.pad(x, ((0, 0), (1, 0), (0, 0), (0, 0)))[:, :-1]     # the window one pixel off at the top
    assert _rejected(R.affine(R.conv2d(shifted, wt, s), sc, of, 0), yr, bounds)


def test_bound_rejects_dropped_tap():
    x, wt, sc, of, yr, bounds = _dense_case(3, 1, 64, 48)
    w2 = wt.copy()
    w2[2, 1] = 0
    assert _rejected(R.affine(R.conv2d(x, w2, 1), sc, of, 0), yr, bounds)


def test_bound_rejects_dropped_k_block():
    x, wt, sc, of, yr, bounds = _dense_case(1, 1, 256, 64)
    x2 = x.copy()
    x2[..., 32:64] = 0
    assert _rejected(R.affine(R.conv2d(x2, wt, 1), sc, of, 0), yr, bounds)


def test_bound_rejects_head_row_off_by_one():
    rng = np.random.default_rng(3)
    y0, y1 = rng.standard_normal((1, 3, 3, 3 * 8)), rng.standard_normal((1, 2, 2, 6 * 8))
    rows = 27 + 24

    def scatter(off0):
        enc, lg = np.zeros((1, rows, 4)), np.zeros((1, rows, 4))
        R.head_scatter(y0, 3, 12, off0, enc, lg)
        R.head_scatter(y1, 6, 24, 27, enc, lg)
        return np.concatenate([enc.ravel(), lg.ravel()])

    want = scatter(0)
    bound = R.dense_bound(np.abs(want) + 1, want, want, 1.0, 0.0, 2, k_blocks=8)
    assert np.any(np.abs(scatter(1) - want) > bound)


def _tf32(v):
    return (np.ascontiguousarray(v, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)


def test_bound_rejects_missing_lo_correction():
    """Simulated tf32x3 products in float64: the full split passes the tf32x3 bound, hi·hi alone (a lost correction
    term, also what tf32x1 computes) fails it and passes the tf32x1 bound."""
    x, wt, sc, of, _, _ = _dense_case(1, 1, 256, 64, seed=5)
    x32, w32 = x.astype(np.float32), wt.astype(np.float32)
    x, wt = x32.astype(np.float64), w32.astype(np.float64)
    z, P = R.conv2d(x, wt, 1), R.conv2d(np.abs(x), np.abs(wt), 1)
    yr = R.affine(z, sc, of, 0)
    bounds = {md: R.dense_bound(P, z * sc, yr, sc, of, md, k_blocks=8) for md in (2, 3)}
    xh, wh = _tf32(x32), _tf32(w32)
    xl, wl = _tf32((x - xh).astype(np.float32)), _tf32((wt - wh).astype(np.float32))
    full = R.affine(R.conv2d(xh, wh, 1) + R.conv2d(xl, wh, 1) + R.conv2d(xh, wl, 1), sc, of, 0)
    hi_only = R.affine(R.conv2d(xh, wh, 1), sc, of, 0)
    assert np.all(np.abs(full - yr) <= bounds[2])
    assert np.all(np.abs(hi_only - yr) <= bounds[3])
    assert np.any(np.abs(hi_only - yr) > bounds[2])


# ------------------------------------------------------------------------------------------------ case coverage
def _claims():
    """(case, precision, plan of the tested layer) for every GPU case, on 132 SMs."""
    out = []
    for c in CASES:
        m, li, _, _ = build(c.spec, seed=len(c.name))
        L, pair = m.layers[li], c.spec[0] == 'pw_add'
        if pair:
            L = m.layers[li - 1]
        for p in c.precisions:
            out.append((c, p, R.plan(L, c.n, p, SMS, c.env, fuse_add_next=pair)))
    return out


def test_every_case_reaches_the_branch_it_claims():
    for c, p, pl in _claims():
        want = claim_for(c, p)
        assert {k: pl[k] for k in want} == want, (c.name, p, pl)


def test_every_gate_branch_is_claimed():
    seen = set()
    for _, _, pl in _claims():
        seen |= pl['branches']
    missing = R.BRANCHES - seen
    assert not missing, sorted(missing)
    assert not (seen & R.UNREACHABLE)


def test_pointwise_cases_reach_every_split_width():
    """test_gpu_tc.py::test_pointwise_gemm's 1x1 shapes: 2- to 8-way clusters except 6 and 7 (tf32, 132 SMs)."""
    got = {}
    for K, N, hw, n in PW_CASES:
        L = Layer(op=OP_PW, in_h=hw, in_w=hw, in_c=K, out_h=hw, out_w=hw, out_c=N, n_pad=-(-N // 16) * 16)
        got[(K, N, hw, n)] = R.plan(L, n, 2, SMS)['splits']
    assert got[(1024, 128, 7, 1)] == 4 and got[(768, 96, 19, 2)] == 3
    assert got[(1300, 48, 10, 1)] == 5 and got[(2048, 64, 10, 1)] == 8
    assert {2, 3, 4, 5, 8} <= set(got.values())


def test_cc_split_scratch_cap_cannot_bind():
    """launch_gemm_cc's scratch cap: splits·M·ldw never exceeds 4 M floats when a split is taken (tiles < 120)."""
    for tiles in range(1, R.CC_SPLIT_TILES):
        splits = -(-R.CC_SPLIT_CTAS // tiles)
        assert splits * 64 * 64 * tiles <= R.PARTIAL_FLOATS_MIN
