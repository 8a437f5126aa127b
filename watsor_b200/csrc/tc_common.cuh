// tc_common.cuh -- inline PTX wrappers shared by the tensor-core kernels (kernels_tc.cu, kernels_fused.cu):
// mbarrier, TMA (cp.async.bulk.tensor load / store), the consumer warpgroups' named barrier, wgmma (warpgroup MMA with
// the accumulator in registers) and the shared-memory matrix descriptor (bit layout as in cute/arch/mma_sm90_desc.hpp).  sm_90a.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
          "r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// barrier among the 128 threads of consumer warpgroup `wg` (hardware barriers 2 and 3)
__device__ __forceinline__ void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory"); }
// One elected lane of a converged warp.  Unlike `lane == 0`, ptxas knows the guarded region runs in a single
// thread, so the TMA operands move to uniform registers without a per-instruction uniformisation loop.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(pred));
  return pred != 0;
}

// Explicit shared-window accesses: the carve-up of the dynamic buffer goes through integer alignment, after
// which nvcc no longer proves the address space and would emit generic LD.E/ST.E in the hottest loops.
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ uint4 lds128u(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (cute::GMMA::DescriptorSm90 bit layout):
// start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major) | SBO>>4 [32,46) | layout_type=1 (SW128) [62,64).
// Rows are 128 B apart, 8-row swizzle atoms 1024 B apart (SBO).  A k-step inside the 128-byte row advances the start
// address by its byte offset; tiles start on 1024-byte boundaries, so the base offset field stays 0.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (+)= A[64 x K] * B[N x K]^T, both operands K-major in shared memory, fp32 accumulators in registers.
// Op: the operand type, float (read as TF32: k = 8 per instruction), __nv_bfloat16 or __half (k = 16).  Either way one instruction covers 32 bytes of a 128-byte row.
// Accumulator i of a thread holds row 16 * (warp % 4) + lane / 4 + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (lane % 4) + i % 2.
// scale_d = 0 overwrites D instead of adding to it.
template <typename Op, int N> struct Wgmma;
template <> struct Wgmma<float, 32> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
  }
};
template <> struct Wgmma<float, 64> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
  }
};
template <> struct Wgmma<float, 128> {
  static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
  }
};
// The bf16 and f16 forms differ only in the operand type's PTX name.
#define WB_WGMMA_16BIT(OP, PTX_T) \
  template <> struct Wgmma<OP, 32> { \
    static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) { \
      asm volatile( \
          "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n" \
          "wgmma.mma_async.sync.aligned.m64n32k16.f32." PTX_T "." PTX_T " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n" \
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
          : "l"(da), "l"(db), "r"(scale_d)); \
    } \
  }; \
  template <> struct Wgmma<OP, 64> { \
    static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) { \
      asm volatile( \
          "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n" \
          "wgmma.mma_async.sync.aligned.m64n64k16.f32." PTX_T "." PTX_T " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n" \
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
          : "l"(da), "l"(db), "r"(scale_d)); \
    } \
  }; \
  template <> struct Wgmma<OP, 128> { \
    static __device__ __forceinline__ void mma(float* d, uint64_t da, uint64_t db, uint32_t scale_d) { \
      asm volatile( \
          "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n" \
          "wgmma.mma_async.sync.aligned.m64n128k16.f32." PTX_T "." PTX_T " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n" \
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
          : "l"(da), "l"(db), "r"(scale_d)); \
    } \
  };
WB_WGMMA_16BIT(__nv_bfloat16, "bf16")
WB_WGMMA_16BIT(__half, "f16")
#undef WB_WGMMA_16BIT

// One 128-byte k-block (32 fp32 / 64 bf16 or fp16 along K) of a warpgroup's 64 x N tile: four k-steps.  X3 (3xTF32) issues
// the small correction products lo(A)*hi(B) and hi(A)*lo(B) of all four k-steps first and the hi(A)*hi(B) products
// last: the tensor core's accumulation rounds toward zero, and this order leaves four such roundings at the magnitude
// of the k-block's partial sum instead of twelve.  The GEMM and the fused depthwise kernel both issue their MMAs
// through here, so equal inputs give bit-equal outputs.
template <typename Op, bool X3, int N>
__device__ __forceinline__ void wg_mma_kblock(float* d, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                              uint32_t scale_first) {
  if (X3) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t koff = (uint32_t)(k * 32);
      Wgmma<Op, N>::mma(d, make_sw128_desc(a_lo + koff), make_sw128_desc(b_hi + koff), k == 0 ? scale_first : 1u);
      Wgmma<Op, N>::mma(d, make_sw128_desc(a_hi + koff), make_sw128_desc(b_lo + koff), 1u);
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t koff = (uint32_t)(k * 32);
    Wgmma<Op, N>::mma(d, make_sw128_desc(a_hi + koff), make_sw128_desc(b_hi + koff), (X3 || k > 0) ? 1u : scale_first);
  }
}

// 3xTF32 k-block into the running sum: the k-block's partial sum lands in `part` (overwritten), then is added to
// `acc` with round-to-nearest, so the tensor core's truncating accumulation never spans more than one k-block.
template <int N>
__device__ __forceinline__ void wg_x3_kblock_sum(float* acc, float* part, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                                 uint32_t b_lo) {
  wgmma_fence();
  wg_mma_kblock<float, true, N>(part, a_hi, a_lo, b_hi, b_lo, 0u);
  wgmma_commit();
  wgmma_wait_all();
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = __fadd_rn(acc[i], part[i]);
}

// Split one 16-byte chunk of fp32 in place into hi = a & 0xffffe000 (written back) and lo = (a - hi) & 0xffffe000:
// both exactly representable in TF32, so the tensor core's own input conversion never matters.
__device__ __forceinline__ void split_tf32(uint32_t hi_addr, uint32_t lo_addr) {
  const uint4 x = lds128u(hi_addr);
  uint4 h, l;
  h.x = x.x & 0xFFFFE000u;
  h.y = x.y & 0xFFFFE000u;
  h.z = x.z & 0xFFFFE000u;
  h.w = x.w & 0xFFFFE000u;
  l.x = __float_as_uint(__fsub_rn(__uint_as_float(x.x), __uint_as_float(h.x))) & 0xFFFFE000u;
  l.y = __float_as_uint(__fsub_rn(__uint_as_float(x.y), __uint_as_float(h.y))) & 0xFFFFE000u;
  l.z = __float_as_uint(__fsub_rn(__uint_as_float(x.z), __uint_as_float(h.z))) & 0xFFFFE000u;
  l.w = __float_as_uint(__fsub_rn(__uint_as_float(x.w), __uint_as_float(h.w))) & 0xFFFFE000u;
  sts128(hi_addr, h);
  sts128(lo_addr, l);
}

constexpr int BLOCK_M = 128;
constexpr int ROW_BYTES = 128;                     // one swizzle row = 64 bf16 / fp16 or 32 fp32 along K
constexpr int A_TILE_BYTES = BLOCK_M * ROW_BYTES;  // 16 KB


}  // namespace
