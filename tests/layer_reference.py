"""Float64 restatement of the backbone layer operations, per-element error bounds for the CUDA kernels that run them,
bit-exact float32 restatements where a kernel's order of operations is defined, and `plan()`, the kernel dispatch of
csrc/ restated so that a test can prove which branch a layer reaches.  Everything that depends on the precision mode
reads its row of `PRECISIONS`.

Everything is numpy on NHWC arrays.  The reference operations follow the TensorFlow op definitions (Conv2D,
DepthwiseConv2dNative, MaxPool, AvgPool with padding SAME; ConcatV2; Add; the box-predictor Reshape + concat), not the
CUDA code.

Error bounds
------------
A dense layer computes y = act(z·s + o) with z = Σ_k a_k·w_k over K = kh·kw·C_in terms.  Its bound is per output
element, in terms of P = Σ_k |a_k|·|w_k| (the `(|A|·|W|)_ij` of the layer), so a wrong element of a layer with a large
range cannot hide behind that range:

    |ŷ - y| <= B_acc·|s| + (epilogue roundings),     B_acc = (c_mode + steps·t_step + γ_n) · P + 1e-30

with u = 2^-24 and γ_n = n·u / (1 - n·u).  The epilogue `fl(fl(ẑ·s) + o)` adds u·|ẑ·s| and u·|ẑ·s + o|; ReLU6 is
1-Lipschitz, so the bound passes through it; 16-bit storage adds the final rounding of the stored value (below).
Heads write fp32 in every mode.  The mode terms:

* fp32 FFMA (precision 0, `k_gemm_cc`, the stem, depthwise): every product enters an fmaf chain (split-K: chains
  of a split, then an ordered sum of the splits), one rounding per step and at most K + splits steps:
  c = 0, no truncating steps, n = K + splits.
* tf32x3 (precision 2, `k_gemm_tc<2>`, DESIGN.md §4.1).  a = hi + lo + r with hi = a & 0xffffe000 (|a - hi| < 2^-10·|a|,
  computed exactly) and lo = (a - hi) & 0xffffe000 (|r| < 2^-10·|a - hi| < 2^-20·|a|); the same for w.  The kernel
  forms hi·hi + lo·hi + hi·lo; each of those products is exact in fp32 (11 × 11 significant bits), and what it drops,
  lo_a·lo_w + r_a·w + (a - r_a)·r_w, is below 3·2^-20·|a·w|: c = 3.01·2^-20.  The tensor core accumulates each
  32-value k-block into a fresh register tile with 12 `wgmma.k8` steps; a step adds 8 exact products to its fp32
  accumulator, aligning the 9 addends to the largest one and truncating, so it errs by less than 9 units of the 24th
  bit of the largest addend, and a product passes through at most 12 steps: 12 steps of t_step = 9·2^-23 on the
  k-block's own Σ|a·w|.  The k-block partials are added with round-to-nearest, then the split-K cluster sums its
  members in rank order: n = k_blocks + splits.  One constant per mode, whatever K, N or the split.
* tf32x1 (precision 3, diagnostic): the tensor core reads the fp32 operands as TF32 (each within 2^-10 relative):
  c = 2^-9 + 2^-20; the accumulator runs across the whole k range of a split: steps = 4 per k-block; n = splits.
* bf16 (precision 1): the same truncating chain (`wgmma.k16`: 17 addends, t_step = 17·2^-23, 4 steps per 64-value
  k-block) on the bf16-rounded activations and weights, c = 0, n = splits; then one bf16 rounding of the output, at
  most 2^-8 of the stored value.
* fp16 (precision 4, `k_gemm_tc<3>`) runs bf16's MMA sequence on fp16 operands (`wgmma.k16.f32.f16.f16`): bf16's chain
  constants.  A product of two fp16 values (11 × 11 significant bits) is exact in fp32, and so is a product with a
  subnormal fp16 factor (at least 2^-48, far above fp32's normal range floor): the chain needs no absolute term as long
  as the tensor core keeps subnormal operands (tests/test_gpu_fp16.py checks a 1x1 whose weights are all fp16
  subnormals against this bound).  The output rounding to fp16 (round to nearest even, subnormals kept) errs by at
  most 2^-11·|y| for a normal result and by half the subnormal spacing, 2^-25, for a subnormal one: 2^-11·|y| + 2^-25.
  That holds below the clamp (|y| <= 65504); above it the store saturates at ±65504 by design.

The CUDA-core kernels (stem, depthwise, `k_gemm_cc`) keep their fp32 arithmetic in every mode and only store the
mode's type: their bound is the fp32 one plus the output rounding.  The depthwise kernels are fmaf chains of at most 9
terms; they are bounded like the fp32 GEMM (γ_9), not emulated, because float64 cannot reproduce a fused multiply-add's
single rounding without double rounding.

Dispatch: fp16 and bf16 elements are both 2 bytes, which is all the tensor-core gate and the GEMM's k-block count
depend on, and both modes refuse residual and dw→1×1 fusion, so precision 4's plan is bf16's but for the GEMM's MODE.
"""
from collections import namedtuple

import numpy as np

from watsor_b200.model import (ACT_RELU6, OP_ADD, OP_AVGPOOL, OP_CONV, OP_COPY, OP_DW, OP_HEAD, OP_MAXPOOL, OP_PW,
                               OP_STEM, same_pad)

U = 2.0 ** -24            # fp32 unit roundoff
U_BF16 = 2.0 ** -8        # bf16 unit roundoff (8 significant bits)
U_FP16 = 2.0 ** -11       # fp16 unit roundoff (11 significant bits)
FP16_SUB_HALF = 2.0 ** -25  # half the spacing of fp16 subnormals: the absolute rounding error of a subnormal result
FP16_MAX = 65504.0        # largest finite fp16: the activation stores clamp to it
TINY = 1e-30              # absolute floor: products of subnormal TF32 halves may be flushed to zero

# (c, truncating steps per k-block, t_step) of a tensor-core accumulation chain, by PRECISIONS' `chain` key; 0 is the
# fp32 FFMA chain of the CUDA-core kernels: see the module docstring
MODE_CONSTANTS = {
    0: (0.0, 0, 0.0),
    2: (3.01 * 2.0 ** -20, 12, 9 * 2.0 ** -23),
    3: (2.0 ** -9 + 2.0 ** -20, 4, 9 * 2.0 ** -23),
    1: (0.0, 4, 17 * 2.0 ** -23),
}


def gamma(n):
    return n * U / (1.0 - n * U)


# ------------------------------------------------------------------------------------------- reference operations
def _same_padded(x, kh, kw, stride, fill=0.0):
    """x [n, H, W, C] padded as TF SAME does (the odd pixel after), and the output size."""
    _, H, W, _ = x.shape
    oh, pt = same_pad(H, kh, stride)
    ow, pl = same_pad(W, kw, stride)
    pb = max((oh - 1) * stride + kh - H, 0) - pt
    pr = max((ow - 1) * stride + kw - W, 0) - pl
    xp = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)), constant_values=fill)
    return xp, oh, ow


def _taps(xp, kh, kw, stride, oh, ow):
    for ky in range(kh):
        for kx in range(kw):
            yield ky, kx, xp[:, ky:ky + stride * (oh - 1) + 1:stride, kx:kx + stride * (ow - 1) + 1:stride, :]


def conv2d(x, w, stride):
    """TF Conv2D, padding SAME: x [n, H, W, C], w [kh, kw, C, O] -> [n, oh, ow, O] (float64)."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    kh, kw = w.shape[:2]
    xp, oh, ow = _same_padded(x, kh, kw, stride)
    out = np.zeros(x.shape[:1] + (oh, ow, w.shape[3]))
    for ky, kx, xs in _taps(xp, kh, kw, stride, oh, ow):
        out += xs @ w[ky, kx]
    return out


def depthwise(x, w, stride):
    """TF DepthwiseConv2dNative (multiplier 1), padding SAME: x [n, H, W, C], w [kh, kw, C]."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    kh, kw = w.shape[:2]
    xp, oh, ow = _same_padded(x, kh, kw, stride)
    out = np.zeros(x.shape[:1] + (oh, ow, x.shape[3]))
    for ky, kx, xs in _taps(xp, kh, kw, stride, oh, ow):
        out += xs * w[ky, kx]
    return out


def pool(x, k, stride, kind):
    """TF MaxPool / AvgPool, padding SAME; the average divides by the number of in-image taps."""
    x = np.asarray(x, np.float64)
    if kind == 'max':
        xp, oh, ow = _same_padded(x, k, k, stride, fill=-np.inf)
        return np.max([xs for _, _, xs in _taps(xp, k, k, stride, oh, ow)], axis=0)
    xp, oh, ow = _same_padded(x, k, k, stride)
    mp, _, _ = _same_padded(np.ones(x.shape[:3] + (1,)), k, k, stride)
    total = sum(xs for _, _, xs in _taps(xp, k, k, stride, oh, ow))
    count = sum(ms for _, _, ms in _taps(mp, k, k, stride, oh, ow))
    return total / count


def concat(parts, row_offs, total_c):
    """ConcatV2 along channels: part i lands in channels [row_offs[i], row_offs[i] + C_i)."""
    out = np.zeros(parts[0].shape[:3] + (total_c,), np.asarray(parts[0]).dtype)
    for p, off in zip(parts, row_offs):
        out[..., off:off + p.shape[3]] = p
    return out


def add(a, b):
    return np.asarray(a, np.float64) + np.asarray(b, np.float64)


def affine(z, scale, offset, act):
    """Folded BatchNorm / bias y = z·s + o, then ReLU6 when act says so."""
    y = z * np.asarray(scale, np.float64) + np.asarray(offset, np.float64)
    return np.clip(y, 0.0, 6.0) if act == ACT_RELU6 else y


def head_scatter(y, anchors_per_loc, n_box, row_off, enc, logits):
    """The box-predictor Reshape + concat as `copy_out_row` / `k_splitk_reduce` document it: y [n, h, w, N]; column c of
    pixel p goes to enc[f, row_off + p·a + c // 4, c % 4] when c < n_box, else to
    logits[f, row_off + p·a + (c - n_box) // (C + 1), (c - n_box) % (C + 1)].  Writes into enc / logits in place."""
    n, h, w, _ = y.shape
    a = anchors_per_loc
    ncp1 = logits.shape[2]
    flat = y.reshape(n, h * w, -1)
    enc[:, row_off:row_off + h * w * a, :] = flat[:, :, :n_box].reshape(n, h * w * a, 4)
    logits[:, row_off:row_off + h * w * a, :] = flat[:, :, n_box:].reshape(n, h * w * a, ncp1)
    return enc, logits


# ------------------------------------------------------------------------------------------------- error bounds
def dense_bound(P, zs, y_ref, scale, offset, precision, k_blocks=1, splits=1, kb_per=None, K=None, tc=True, head=False):
    """Per-element bound on |kernel - reference| of a dense layer of a `precision` engine (module docstring).  P =
    Σ|a|·|w|, zs = the exact z·s and y_ref = act(z·s + o), all broadcast to the output's shape.  tc: the layer runs on
    the tensor-core GEMM (else on the CUDA cores' fp32 chain); K: length of the fp32 chain; k_blocks / kb_per:
    tensor-core k-blocks of the layer / of one split; head: the output is written as fp32, not stored as an
    activation."""
    mode = PRECISIONS[precision]
    chain = mode.chain if tc else 0
    c, steps, t_step = MODE_CONSTANTS[chain]
    kb_per = k_blocks if kb_per is None else kb_per
    if chain == 0:
        rel = gamma(K + splits)
    elif chain == 2:
        rel = c + steps * t_step + gamma(k_blocks + splits)
    else:
        rel = c + steps * kb_per * t_step + gamma(splits)
    s = np.abs(np.asarray(scale, np.float64))
    b = rel * P * s + TINY
    b = b + U * (np.abs(zs) + b)                                             # fl(ẑ·s)
    b = b + U * (np.abs(zs + np.asarray(offset, np.float64)) + b)           # fl(· + o)
    if mode.out_round and not head:
        rel_out, abs_out = mode.out_round
        b = b + rel_out * (np.abs(y_ref) + b) + abs_out
    return b


def chain_bound(P, zs, y_ref, scale, offset, terms, precision=0):
    """An fmaf chain of `terms` products (stem, depthwise), the affine epilogue, then the store of `precision`."""
    return dense_bound(P, zs, y_ref, scale, offset, precision, K=terms - 1, splits=1, tc=False)


# -------------------------------------------------------------------------------------- bit-exact restatements
def bf16_round(x):
    """float32 -> bf16 (round to nearest even) -> float32, as __float2bfloat16_rn (no NaN inputs here)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def fp16_round(x):
    """float32 -> fp16 (round to nearest even, subnormals kept) -> float32, as __float2half_rn (no NaN inputs here).
    Magnitudes from 65520 up become inf, as they do there; the activation stores clamp first (fp16_store)."""
    x = np.asarray(x, np.float32).astype(np.float64)
    a = np.abs(x)
    _, ex = np.frexp(a)                             # a = m·2^ex with m in [0.5, 1): exponent ex - 1
    q = 2.0 ** (np.maximum(ex - 1, -14) - 10)       # the fp16 spacing at a: 2^(e - 10), 2^-24 among the subnormals
    r = np.round(a / q) * q                         # a / q is exact; np.round rounds half to even
    r = np.where(r > FP16_MAX, np.inf, r)
    return np.copysign(r, x).astype(np.float32)


def fp16_store(x):
    """ActIO<__half>::st / st4: clamp to ±65504, then round to fp16."""
    return fp16_round(np.clip(np.asarray(x, np.float32), -FP16_MAX, FP16_MAX))


def f32_store(x):
    return np.asarray(x, np.float32)


# The precision modes by wb_create's number; csrc/wb_api.cu has the same table for the library.
#   name: in test IDs.  storage: the activation type in kernel names.  store: its bit-exact store.
#   out_round: (relative, absolute) rounding of a stored activation, or None.
#   tc_bytes, tc_mode, tc_round: the tensor-core GEMM's operand bytes, k_gemm_tc MODE and the host rounding of its
#   weights, or None: no tensor cores.  chain: the MODE_CONSTANTS key of its accumulation.
#   fuse_add: a linear 1x1 -> residual Add runs as one GEMM (fp32 storage: the shortcut is added in the epilogue).
Precision = namedtuple('Precision', 'name storage store out_round tc_bytes tc_mode tc_round chain fuse_add')
PRECISIONS = [
    Precision('fp32', 'float', f32_store, None, None, None, None, 0, False),
    Precision('bf16', '__nv_bfloat16', bf16_round, (U_BF16, 0.0), 2, 0, bf16_round, 1, False),
    Precision('tf32x3', 'float', f32_store, None, 4, 2, f32_store, 2, True),
    Precision('tf32x1', 'float', f32_store, None, 4, 1, f32_store, 3, True),
    Precision('fp16', '__half', fp16_store, (U_FP16, FP16_SUB_HALF), 2, 3, fp16_round, 1, False),
]


def add_f32(a, b, precision=0):
    """k_add: one float32 addition per element, stored as T."""
    return PRECISIONS[precision].store(np.asarray(a, np.float32) + np.asarray(b, np.float32))


def copy_channels_f32(parts, row_offs, total_c, precision=0):
    """k_copy_channels: a copy (16-bit storage holds 16-bit values already)."""
    return PRECISIONS[precision].store(concat([np.asarray(p, np.float32) for p in parts], row_offs, total_c))


def pool_f32(x, k, stride, kind, precision=0):
    """k_pool: the max of the in-image taps, or their __fadd_rn sum in (ky, kx) order from +0, then __fdiv_rn by the
    number of in-image taps, stored as T."""
    store = PRECISIONS[precision].store
    x = np.asarray(x, np.float32)
    xp, oh, ow = _same_padded(x, k, k, stride)
    mp, _, _ = _same_padded(np.ones(x.shape[:3] + (1,), np.float32), k, k, stride)
    taps = list(zip(_taps(xp, k, k, stride, oh, ow), _taps(mp, k, k, stride, oh, ow)))
    if kind == 'max':
        acc = np.full(x.shape[:1] + (oh, ow, x.shape[3]), -np.inf, np.float32)
        for (_, _, xs), (_, _, ms) in taps:
            acc = np.where(ms > 0, np.maximum(acc, xs), acc)
        return store(acc)
    acc = np.zeros(x.shape[:1] + (oh, ow, x.shape[3]), np.float32)
    cnt = np.zeros(x.shape[:1] + (oh, ow, 1), np.float32)
    for (_, _, xs), (_, _, ms) in taps:
        acc = np.where(ms > 0, (acc + xs).astype(np.float32), acc)
        cnt = cnt + ms
    return store((acc / cnt).astype(np.float32))


# ----------------------------------------------------------------------------------------------------- dispatch
BLOCK_M, ROW_BYTES = 128, 128
CC_SPLIT_TILES, CC_SPLIT_CTAS = 120, 296      # launch_gemm_cc: split below 120 tiles, aim at ~296 CTAs

# every branch of every gate that plan() can report; a test case has to claim each of them
BRANCHES = frozenset(
    ['stem:3x3s2_c32', 'stem:generic', 'dw:strip_s1', 'dw:strip_s2',
     'tc:pw', 'tc:head', 'tc:conv', 'tc:unsupported_conv', 'tc:unsupported_1x1', 'tc:bn32', 'tc:bn64', 'tc:bn128',
     'tc:no_split_tiles', 'tc:no_split_kblocks', 'tc:no_split_env'] +
    ['tc:split%d' % s for s in range(2, 9)] +
    ['cc:big', 'cc:small', 'cc:split', 'cc:no_split_tiles', 'cc:no_split_ktiles',
     'fuse_add:yes', 'fuse_add:no', 'pool:max', 'pool:avg', 'add', 'copy'])
# launch_gemm_cc lowers the split count while splits·M·ldw exceeds the split-K scratch (>= 4 M floats).  A split needs
# fewer than 120 tiles of 64 x 64, so M·ldw <= 4096·tiles and splits <= ceil(296 / tiles): at most 4096·(296 + 119)
# floats.  The cap cannot bind (test_layer_reference_host.py checks this for every tile count).
UNREACHABLE = frozenset(['cc:partial_cap'])
PARTIAL_FLOATS_MIN = 4 * 1024 * 1024


def tc_supported(L, precision, env=()):
    """tc_layer_supported (csrc/kernels_tc.cu) in a mode with tensor cores: a 1x1 needs K-major rows of a multiple of
    16 bytes."""
    elem = PRECISIONS[precision].tc_bytes
    if L.op in (OP_PW, OP_HEAD) and L.kh == 1 and L.kw == 1 and L.stride == 1 and L.in_c * elem % 16 == 0:
        return True
    return (L.op == OP_CONV and L.in_c % 64 == 0 and L.out_h * L.out_w <= BLOCK_M and L.stride <= 8 and
            'WB_NO_TC_CONV' not in env)


def pick_block_n(n_pad):
    return 32 if n_pad <= 32 else (64 if n_pad <= 64 else 128)


def _ceil(a, b):
    return -(-a // b)


def plan(L, n, precision, sms, env=(), fuse_add_next=False):
    """Which kernel runs layer L of a batch of n, and how: a dict with 'kernel', 'launches' and the gate 'branches' it
    took, plus the launch parameters of the GEMMs.  `fuse_add_next`: the next layer is a residual Add of L's output
    that the same call also runs (`fused_span` in csrc/wb_api.cu)."""
    if L.op == OP_STEM:
        big = L.kh == 3 and L.kw == 3 and L.stride == 2 and L.out_c == 32
        return dict(kernel='k_stem_3x3s2_c32' if big else 'k_stem', launches=1,
                    branches={'stem:3x3s2_c32' if big else 'stem:generic'})
    if L.op == OP_DW:
        if L.stride not in (1, 2):
            raise ValueError('wb_create refuses a depthwise stride of %d' % L.stride)
        return dict(kernel='k_dw_strip', stride=L.stride, launches=1, branches={'dw:strip_s%d' % L.stride})
    if L.op in (OP_MAXPOOL, OP_AVGPOOL):
        return dict(kernel='k_pool', launches=1, branches={'pool:max' if L.op == OP_MAXPOOL else 'pool:avg'})
    if L.op == OP_ADD:
        return dict(kernel='k_add', launches=1, branches={'add'})
    if L.op == OP_COPY:
        return dict(kernel='k_copy_channels', launches=1, branches={'copy'})
    M, K = n * L.out_h * L.out_w, L.kh * L.kw * L.in_c
    mode = PRECISIONS[precision]
    if mode.tc_mode is not None and tc_supported(L, precision, env):
        conv = L.op == OP_CONV
        elem = mode.tc_bytes
        hw = L.out_h * L.out_w
        rpt = (BLOCK_M // hw) * hw if conv else BLOCK_M
        bn = pick_block_n(L.n_pad)
        tiles = _ceil(M, rpt) * _ceil(L.n_pad, bn)
        kb = _ceil(K * elem, ROW_BYTES)
        splits, kb_per = 1, kb
        br = {'tc:conv' if conv else ('tc:head' if L.op == OP_HEAD else 'tc:pw'), 'tc:bn%d' % bn}
        if not tiles < sms // 2:
            br.add('tc:no_split_tiles')
        elif kb < 16:
            br.add('tc:no_split_kblocks')
        elif 'WB_NO_SPLITK' in env:
            br.add('tc:no_split_env')
        else:
            # tiles < sms / 2 and kb >= 16 make this at least 2
            kb_per = _ceil(kb, min(sms // tiles, kb // 8, 8))
            splits = _ceil(kb, kb_per)
            br.add('tc:split%d' % splits)
        fused = fuse_add_next and mode.fuse_add and L.op == OP_PW and L.act != ACT_RELU6 and \
            'WB_NO_FUSE_ADD' not in env
        if fuse_add_next:
            br.add('fuse_add:yes' if fused else 'fuse_add:no')
        return dict(kernel='k_gemm_tc', mode=mode.tc_mode, bn=bn, tiles=tiles, k_blocks=kb,
                    kb_per=kb_per, splits=splits, rows_per_tile=rpt, launches=1 + (fuse_add_next and not fused),
                    fused_add=fused, branches=br)
    br = set()
    if mode.tc_mode is not None:
        br.add('tc:unsupported_conv' if L.op == OP_CONV else 'tc:unsupported_1x1')
    if fuse_add_next:
        br.add('fuse_add:no')
    N = L.out_c
    if _ceil(M, 128) * _ceil(N, 128) >= sms and N >= 128:
        br.add('cc:big')
        return dict(kernel='k_gemm_cc', tile=128, splits=1, launches=1 + fuse_add_next, branches=br)
    br.add('cc:small')
    tiles, kt = _ceil(N, 64) * _ceil(M, 64), _ceil(K, 16)
    splits = 1
    if tiles >= CC_SPLIT_TILES:
        br.add('cc:no_split_tiles')
    elif kt < 16:
        br.add('cc:no_split_ktiles')
    else:
        s = min(_ceil(CC_SPLIT_CTAS, tiles), kt // 8)
        assert s * M * L.n_pad <= PARTIAL_FLOATS_MIN          # the scratch cap (UNREACHABLE) cannot bind
        if s > 1:
            splits = _ceil(kt, _ceil(kt, s))
            br.add('cc:split')
        else:
            br.add('cc:no_split_ktiles')
    return dict(kernel='k_gemm_cc', tile=64, splits=splits, launches=1 + (splits > 1) + fuse_add_next, branches=br)


def kernel_name_pattern(p, precision):
    """Substring of the demangled name of the kernel plan() names (as torch.profiler reports it)."""
    t = PRECISIONS[precision].storage
    k = p['kernel']
    if k == 'k_gemm_tc':
        return 'k_gemm_tc<%d, %d>' % (p['mode'], p['bn'])
    if k == 'k_gemm_cc':
        return 'k_gemm_cc<%s, %s>' % (t, '128, 128, 8, 8' if p['tile'] == 128 else '64, 64, 4, 4')
    if k == 'k_dw_strip':
        return 'k_dw_strip<%s, %d>' % (t, p['stride'])
    return '%s<%s' % (k, t)
