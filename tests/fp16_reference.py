"""The fp16 mode (precision 4) in terms of tests/layer_reference.py: fp16 storage restated bit-exactly, the per-element
error bounds of the kernels that store fp16, and the kernel dispatch of precision 4.

Error bounds
------------
fp16 (precision 4, `k_gemm_tc<3>`) runs bf16's MMA sequence on fp16 operands (`wgmma.k16.f32.f16.f16`): the same
truncating chain as bf16 (17 addends per step, t_step = 17·2^-23, 4 steps per 64-value k-block), c = 0, n = splits.
A product of two fp16 values (11 × 11 significant bits) is exact in fp32, and so is a product with a subnormal fp16
factor (at least 2^-48, far above fp32's normal range floor): the chain needs no absolute term as long as the tensor
core keeps subnormal operands (tests/test_gpu_fp16.py checks a 1x1 whose weights are all fp16 subnormals against this
bound).  The output rounding to fp16 (round to nearest even, subnormals kept) errs by at most 2^-11·|y| for a normal
result and by half the subnormal spacing, 2^-25, for a subnormal one: 2^-11·|y| + 2^-25.  That holds below the clamp
(|y| <= 65504); above it the store saturates at ±65504 by design.  Heads write fp32 in every mode.

The CUDA-core kernels (stem, depthwise, `k_gemm_cc`) keep their fp32 arithmetic and only store fp16: their bound is
the fp32 one plus the output rounding.

Dispatch
--------
Precision 4 takes bf16's plan everywhere: fp16 and bf16 elements are both 2 bytes, which is all the tensor-core gate
and the GEMM's k-block count depend on, and both modes refuse residual and dw→1×1 fusion.  Only the tensor-core GEMM's
MODE differs (3 for fp16, 0 for bf16).
"""
import numpy as np

from tests import layer_reference as R
from watsor_b200.model import OP_CONV, OP_HEAD, OP_PW

PRECISION = 4
GEMM_MODE = 3               # k_gemm_tc<3, BN>
U_FP16 = 2.0 ** -11         # fp16 unit roundoff (11 significant bits)
FP16_SUB_HALF = 2.0 ** -25  # half the spacing of fp16 subnormals: the absolute rounding error of a subnormal result
FP16_MAX = 65504.0          # largest finite fp16: the activation stores clamp to it
MODE_CONSTANTS = (0.0, 4, 17 * 2.0 ** -23)   # (c, truncating steps per k-block, t_step): bf16's chain


# -------------------------------------------------------------------------------------- bit-exact restatements
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


def add_f32(a, b):
    """k_add<__half>: one float32 addition per element, stored as fp16."""
    return fp16_store(R.add_f32(a, b))


def copy_channels_f32(parts, row_offs, total_c):
    """k_copy_channels<__half>: a copy (fp16 storage holds fp16 values already)."""
    return fp16_store(R.copy_channels_f32(parts, row_offs, total_c))


def pool_f32(x, k, stride, kind):
    """k_pool<__half>: the float32 pooling of R.pool_f32, stored as fp16."""
    return fp16_store(R.pool_f32(x, k, stride, kind))


# ------------------------------------------------------------------------------------------------- error bounds
def _out_rounding(b, y_ref):
    return b + U_FP16 * (np.abs(y_ref) + b) + FP16_SUB_HALF


def dense_bound(P, zs, y_ref, scale, offset, mode, k_blocks=1, splits=1, kb_per=None, K=None, fp16_out=True):
    """R.dense_bound for a layer of an fp16 engine: mode 4 (the tensor-core GEMM, bf16's chain constants) or 0 (the
    CUDA-core GEMM's fp32 chain); fp16_out adds the rounding of the stored output (heads write fp32)."""
    if mode == PRECISION:
        assert R.MODE_CONSTANTS[1] == MODE_CONSTANTS, 'fp16 shares bf16 chain constants'
        mode = 1
    b = R.dense_bound(P, zs, y_ref, scale, offset, mode, k_blocks=k_blocks, splits=splits, kb_per=kb_per, K=K)
    return _out_rounding(b, y_ref) if fp16_out else b


def chain_bound(P, zs, y_ref, scale, offset, terms):
    """An fmaf chain of `terms` products (stem, depthwise), the affine epilogue, then the fp16 store."""
    return _out_rounding(R.chain_bound(P, zs, y_ref, scale, offset, terms), y_ref)


# ----------------------------------------------------------------------------------------------------- dispatch
def tc_supported(L, env=()):
    """tc_layer_supported (csrc/kernels_tc.cu) with 2-byte fp16 elements: a 1x1's K-major rows must be a multiple of
    16 bytes (K % 8); KxK convs as in every mode."""
    if L.op in (OP_PW, OP_HEAD) and L.kh == 1 and L.kw == 1 and L.stride == 1 and L.in_c * 2 % 16 == 0:
        return True
    return (L.op == OP_CONV and L.in_c % 64 == 0 and L.out_h * L.out_w <= R.BLOCK_M and L.stride <= 8 and
            'WB_NO_TC_CONV' not in env)


def plan(L, n, sms, env=(), fuse_add_next=False):
    """R.plan for precision 4: bf16's plan (module docstring) with the tensor-core GEMM's MODE 3."""
    p = R.plan(L, n, 1, sms, env, fuse_add_next)
    if p['kernel'] == 'k_gemm_tc':
        p['mode'] = GEMM_MODE
    return p


def kernel_name_pattern(p):
    """Substring of the demangled name of the fp16 kernel that plan() names (as torch.profiler reports it)."""
    if p['kernel'] == 'k_gemm_tc':
        return R.kernel_name_pattern(p, False)
    return R.kernel_name_pattern(p, True).replace('__nv_bfloat16', '__half')
