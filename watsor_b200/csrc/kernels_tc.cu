// kernels_tc.cu -- tensor-core path for the dense 1x1 convolutions and heads (K4/K6):
// TMA (cp.async.bulk.tensor) -> 128B-swizzled shared memory -> wgmma with the fp32 accumulators in registers ->
// staging tile -> epilogue (folded BatchNorm / bias, ReLU6) -> global.  sm_90a.
//
// Four operand modes share one warp-specialised kernel:
//   TC_BF16    A, W in bf16, bf16 activations out                        -- "fast" mode
//   TC_FP16    A, W in fp16, fp16 activations out (saturated at +-65504) -- "fast" mode, 3 more significant bits
//   TC_TF32X1  A, W in fp32, one TF32 MMA per product                     -- diagnostic
//   TC_TF32X3  A, W in fp32, every product formed as three TF32 MMAs
//              (A_hi*W_hi + A_lo*W_hi + A_hi*W_lo, fp32 accumulate)      -- fp32-faithful "parity" mode
// In TF32X3 the activation tile lands in shared memory as raw fp32; each consumer warpgroup splits its own 64 rows in
// place into hi = a & 0xffffe000 and lo = (a - hi) & 0xffffe000 (both exactly representable in TF32); the weights
// are split once on the host.
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (rows 0..63 / 64..127 of the 128-row tile: split,
// wgmma, epilogue), warp 8 = TMA producer.
#include <cuda.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "kernels_tc.cuh"
#include "tc_common.cuh"

namespace {

struct TcArgs {
  const float* scale;
  const float* offset;
  void* out;  // [M][N] activations: fp32, bf16 or fp16 by mode
  float* enc;
  float* logits;
  int M, N, n_pad, K;  // K in elements
  int block_n, stages, k_blocks;
  int splits, kb_per;  // split-K over blockIdx.z (one thread-block cluster per tile, reduced in distributed smem)
  const void* residual;  // != NULL: y = (acc*scale + offset) + residual[m][n]  (MobileNet-v2 bottleneck `Add`)
  // KxK / strided convolutions: the A tile of k-block kb is the tap (kb / cpb) of the filter window, channel block
  // kb % cpb, fetched by a 4-D TMA box {32 ch, OW, OH, imgs} whose traversal strides are the conv stride
  int conv, cpb, conv_kw, conv_pad_t, conv_pad_l;
  int ring_bytes;     // bytes of the stage ring (re-used as the epilogue's staging tile)
  int rows_per_tile;  // GEMM rows one CTA produces (128, or imgs_per_tile*OH*OW for conv tiles)
  int act, is_head, anchors_per_loc, row_off, n_box, num_anchors, ncp1, hw;
};

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// float4 at shared-memory address `addr` of cluster member `rank` (distributed shared memory)
__device__ __forceinline__ float4 ld_dsmem128(uint32_t addr, uint32_t rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(addr), "r"(rank));
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(ra));
  return v;
}

// One output row of the tile from the staging tile(s) to global memory, lanes along the columns (coalesced).
// The row's raw accumulators are this CTA's own (members == 1) or, in a split-K cluster, the sum of the members'
// partial rows in rank order; then folded BN / bias, ReLU6, the optional bottleneck shortcut, and the store: dense
// [M][N] of OutT (float in the TF32 modes), or the head scatter into the concatenated box-encoding / class-logit tensors.
template <typename OutT>
__device__ __forceinline__ void copy_out_row(const TcArgs& g, const uint8_t* smem, int pitch, int r, int m0, int n0,
                                             int lane, int members) {
  const int mm = m0 + r;
  const uint32_t src = smem_u32(smem) + (uint32_t)(r * pitch * 4);
  size_t hr = 0;
  if (g.is_head) {
    const int f = mm / g.hw;
    hr = (size_t)f * g.num_anchors + g.row_off + (size_t)(mm - f * g.hw) * g.anchors_per_loc;
  }
  for (int j = lane * 4; j < g.block_n; j += 128) {
    const int nn = n0 + j;
    if (nn >= g.N) break;
    float4 p[8];  // members <= 8 (portable cluster size): all remote loads in flight, then the ordered sum
    if (members == 1) {
      p[0] = lds128(src + (uint32_t)(j * 4));
    } else {
#pragma unroll
      for (int z = 0; z < 8; ++z)
        if (z < members) p[z] = ld_dsmem128(src + (uint32_t)(j * 4), (uint32_t)z);
    }
    float4 y = p[0];
#pragma unroll
    for (int z = 1; z < 8; ++z)
      if (z < members) y = make_float4(__fadd_rn(y.x, p[z].x), __fadd_rn(y.y, p[z].y), __fadd_rn(y.z, p[z].z), __fadd_rn(y.w, p[z].w));
    const float4 sc = *reinterpret_cast<const float4*>(g.scale + nn), of = *reinterpret_cast<const float4*>(g.offset + nn);
    y = make_float4(affine_rn(y.x, sc.x, of.x), affine_rn(y.y, sc.y, of.y), affine_rn(y.z, sc.z, of.z), affine_rn(y.w, sc.w, of.w));
    if (g.act == WB_ACT_RELU6) y = make_float4(relu6f(y.x), relu6f(y.y), relu6f(y.z), relu6f(y.w));
    if (g.is_head) {
      const float ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = nn + e;
        if (c >= g.N) break;
        if (c < g.n_box)
          g.enc[hr * 4 + c] = ys[e];
        else
          g.logits[hr * g.ncp1 + (c - g.n_box)] = ys[e];
      }
    } else if (std::is_same<OutT, float>::value) {
      if (g.residual != nullptr) {
        const float4 rr = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(g.residual) + (size_t)mm * g.N + nn);
        y = make_float4(__fadd_rn(y.x, rr.x), __fadd_rn(y.y, rr.y), __fadd_rn(y.z, rr.z), __fadd_rn(y.w, rr.w));
      }
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(g.out) + (size_t)mm * g.N + nn) = y;
    } else {
      ActIO<OutT>::st4(reinterpret_cast<OutT*>(g.out) + (size_t)mm * g.N + nn, y);
    }
  }
}

constexpr int GEMM_THREADS = 288;
constexpr int GEMM_PRODUCER_WARP = 8;

// MODE 0: bf16 operands; MODE 1: tf32 single product (diagnostic); MODE 2: tf32 x3 split; MODE 3: fp16 operands.
// BN: N tile (32 / 64 / 128).
template <int MODE, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    k_gemm_tc(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
              const __grid_constant__ CUtensorMap map_b_lo, TcArgs g) {
  constexpr bool TF32 = MODE == 1 || MODE == 2;
  constexpr bool X3 = MODE == 2;
  // activation type: the MMAs' operand type and the dense output's element type
  using ActT = typename std::conditional<TF32, float, typename std::conditional<MODE == 3, __half, __nv_bfloat16>::type>::type;
  constexpr int ELEM = TF32 ? 4 : 2;
  constexpr int K_PER_BLOCK = ROW_BYTES / ELEM;
  constexpr int B_TILE_BYTES = BN * ROW_BYTES;
  constexpr int SLOTS = X3 ? 2 : 1;  // raw / hi tile (+ lo tile)
  constexpr int STAGE_BYTES = (A_TILE_BYTES + B_TILE_BYTES) * SLOTS;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)g.ring_bytes);  // TMA landed
  uint64_t* empty = full + g.stages;                                           // both warpgroups done with the stage

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * g.rows_per_tile, n0 = blockIdx.y * BN;
  const int kb0 = blockIdx.z * g.kb_per;
  const int nkb = min(g.k_blocks, kb0 + g.kb_per) - kb0;  // k-blocks of this split (>= 1)

  if (threadIdx.x == 0) {
    for (int s = 0; s < g.stages; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      mbar_init(smem_u32(&empty[s]), 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

  if (warp == GEMM_PRODUCER_WARP) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
      for (int it = 0; it < nkb; ++it) {
        const int kb = kb0 + it;
        const int s = it % g.stages;
        const uint32_t ph = (it / g.stages) & 1;
        mbar_wait(smem_u32(&empty[s]), ph ^ 1);
        uint8_t* st = smem + (size_t)s * STAGE_BYTES;
        const uint32_t bar = smem_u32(&full[s]);
        if (g.conv) {
          // rows_per_tile = imgs * OH * OW rows arrive (the box never leaves the image range: whole images per tile);
          // taps that fall outside the input are zero-filled by TMA = TF SAME padding
          mbar_expect_tx(bar, g.rows_per_tile * ROW_BYTES + B_TILE_BYTES * SLOTS);
          const int tap = kb / g.cpb, cb = kb - tap * g.cpb;
          const int ky = tap / g.conv_kw, kx = tap - ky * g.conv_kw;
          tma_load_4d(smem_u32(st), &map_a, bar, cb * K_PER_BLOCK, kx - g.conv_pad_l, ky - g.conv_pad_t, m0 / g.hw);
        } else {
          mbar_expect_tx(bar, A_TILE_BYTES + B_TILE_BYTES * SLOTS);
          tma_load_2d(smem_u32(st), &map_a, bar, kb * K_PER_BLOCK, m0);
        }
        uint8_t* sb = st + A_TILE_BYTES * SLOTS;
        tma_load_2d(smem_u32(sb), &map_b, bar, kb * K_PER_BLOCK, n0);
        if (X3) tma_load_2d(smem_u32(sb + B_TILE_BYTES), &map_b_lo, bar, kb * K_PER_BLOCK, n0);
      }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups
    const int wg = warp >> 2, t = threadIdx.x & 127;
    float part[X3 ? BN / 2 : 1];
    for (int it = 0; it < nkb; ++it) {
      const int s = it % g.stages;
      mbar_wait(smem_u32(&full[s]), (it / g.stages) & 1);
      const uint32_t st = smem_u32(smem + (size_t)s * STAGE_BYTES);
      const uint32_t a_hi = st + (uint32_t)(wg * 64 * ROW_BYTES), a_lo = a_hi + A_TILE_BYTES;
      const uint32_t b_hi = st + (uint32_t)(A_TILE_BYTES * SLOTS), b_lo = b_hi + B_TILE_BYTES;
      if (X3) {
#pragma unroll
        for (int i = t; i < 64 * ROW_BYTES / 16; i += 128) split_tf32(a_hi + (uint32_t)(i * 16), a_lo + (uint32_t)(i * 16));
        fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
        wg_bar_sync(wg);
        wg_x3_kblock_sum<BN>(acc, part, a_hi, a_lo, b_hi, b_lo);
      } else {
        wgmma_fence();
        wg_mma_kblock<ActT, false, BN>(acc, a_hi, a_lo, b_hi, b_lo, 1u);
        wgmma_commit();
        wgmma_wait_all();
      }
      wg_bar_sync(wg);  // every warp of the warpgroup has seen its MMAs complete: the stage may be refilled
      if (t == 0) mbar_arrive(smem_u32(&empty[s]));
    }
  }

  // ------------------------------------------------------------------ epilogue
  // Every MMA has completed, so the stage ring is dead: it becomes a [128][BN + 4] fp32 staging tile (row pitch = 4
  // mod 16 words).  Phase 1 (consumer threads): raw accumulators -> staging.  Phase 2 (all warps, lanes along the
  // columns): staging -> folded BN / bias, ReLU6, optional bottleneck shortcut -> coalesced stores (dense [M][N], or
  // the head scatter into the concatenated box-encoding / class-logit tensors).
  // Split-K: the `splits` CTAs of an output tile form one thread-block cluster; after a cluster barrier CTA z
  // reduces rows z, z + splits, ... over all members' staging tiles through distributed shared memory, always in the
  // order z' = 0, 1, ... (deterministic), then runs the same phase 2 arithmetic.
  const int pitch = BN + 4;
  __syncthreads();  // both warpgroups are past their last MMA: the ring may be overwritten
  if (warp < GEMM_PRODUCER_WARP) {
    const int row = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
    const uint32_t stg = smem_u32(smem) + (uint32_t)((row * pitch + 2 * (lane & 3)) * 4);
#pragma unroll
    for (int i = 0; i < BN / 2; i += 4) {
      const uint32_t c = (uint32_t)((i >> 2) * 8 * 4);
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg + c), "f"(acc[i]), "f"(acc[i + 1]) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg + c + (uint32_t)(8 * pitch * 4)), "f"(acc[i + 2]), "f"(acc[i + 3])
                   : "memory");
    }
  }
  __syncthreads();  // the staging tile is complete
  const int n_warps = blockDim.x >> 5;
  const int rows = min(g.rows_per_tile, g.M - m0);
  if (g.splits > 1) {
    // all `splits` CTAs of this tile (one cluster) have staged their partial tiles
    cluster_sync_all();
    const int z = (int)cluster_ctarank();
    for (int r = z + g.splits * warp; r < rows; r += n_warps * g.splits)
      copy_out_row<ActT>(g, smem, pitch, r, m0, n0, lane, g.splits);
    __syncwarp();
    cluster_sync_all();  // nobody exits while a peer still reads its staging tile
  } else if (g.is_head) {
    for (int r = warp; r < rows; r += n_warps) copy_out_row<ActT>(g, smem, pitch, r, m0, n0, lane, 1);
  } else {
    // dense [M][N] output: the thread count is a multiple of the row's BN / 4 float4 columns, so a thread keeps its 4
    // columns and walks down the rows -- folded BN / bias in registers, pointers advanced by a constant, ~20
    // instructions per float4 (this phase is issue bound: 2.5 warps per scheduler)
    static_assert(GEMM_THREADS % (BN / 4) == 0, "every thread of the dense epilogue keeps its 4 columns");
    constexpr int C4N = BN / 4, ROW_STEP = GEMM_THREADS / C4N;
    const int r_it = (int)threadIdx.x / C4N, c_it = (int)threadIdx.x % C4N;
    const int nn = n0 + c_it * 4;
    if (nn < g.N && r_it < rows) {
      const float4 sc = __ldg(reinterpret_cast<const float4*>(g.scale + nn)), of = __ldg(reinterpret_cast<const float4*>(g.offset + nn));
      const bool relu = g.act == WB_ACT_RELU6;
      uint32_t sp = smem_u32(smem) + (uint32_t)((r_it * pitch + c_it * 4) * 4);
      constexpr uint32_t sstep = (uint32_t)(ROW_STEP * pitch * 4);
      ActT* op = reinterpret_cast<ActT*>(g.out) + (size_t)(m0 + r_it) * g.N + nn;
      // the bottleneck shortcut is fused in the fp32 modes only
      const float* rp = TF32 && g.residual != nullptr ? reinterpret_cast<const float*>(g.residual) + (size_t)(m0 + r_it) * g.N + nn : nullptr;
      const size_t gstep = (size_t)ROW_STEP * g.N;
      int r = r_it;
      for (; r + 3 * ROW_STEP < rows; r += 4 * ROW_STEP) {
        float4 y[4], rs[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          y[u] = lds128(sp + u * sstep);
          if (rp != nullptr) rs[u] = *reinterpret_cast<const float4*>(rp + u * gstep);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float4 v = make_float4(affine_rn(y[u].x, sc.x, of.x), affine_rn(y[u].y, sc.y, of.y), affine_rn(y[u].z, sc.z, of.z),
                                 affine_rn(y[u].w, sc.w, of.w));
          if (relu) v = make_float4(relu6f(v.x), relu6f(v.y), relu6f(v.z), relu6f(v.w));
          if (rp != nullptr) v = make_float4(__fadd_rn(v.x, rs[u].x), __fadd_rn(v.y, rs[u].y), __fadd_rn(v.z, rs[u].z), __fadd_rn(v.w, rs[u].w));
          ActIO<ActT>::st4(op + u * gstep, v);
        }
        sp += 4 * sstep;
        op += 4 * gstep;
        if (rp != nullptr) rp += 4 * gstep;
      }
      for (; r < rows; r += ROW_STEP) {
        const float4 y = lds128(sp);
        float4 v = make_float4(affine_rn(y.x, sc.x, of.x), affine_rn(y.y, sc.y, of.y), affine_rn(y.z, sc.z, of.z), affine_rn(y.w, sc.w, of.w));
        if (relu) v = make_float4(relu6f(v.x), relu6f(v.y), relu6f(v.z), relu6f(v.w));
        if (rp != nullptr) {
          const float4 r4 = *reinterpret_cast<const float4*>(rp);
          v = make_float4(__fadd_rn(v.x, r4.x), __fadd_rn(v.y, r4.y), __fadd_rn(v.z, r4.z), __fadd_rn(v.w, r4.w));
          rp += gstep;
        }
        ActIO<ActT>::st4(op, v);
        sp += sstep;
        op += gstep;
      }
    }
  }
}


// -------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

CUtensorMapDataType map_dtype(int mode) {
  return mode == TC_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                         : (mode == TC_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
}

// 2-D K-major matrix [rows][k] of operand mode `mode` -> tensor map with a (128 B x box_rows) box, 128B swizzle
bool make_map(CUtensorMap* map, const void* base, int mode, int rows, int k, int box_rows, std::string* err) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    *err = "cuTensorMapEncodeTiled is not available from the driver";
    return false;
  }
  const int elem_bytes = tc_elem_bytes(mode);
  cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)k * elem_bytes};
  cuuint32_t box[2] = {(cuuint32_t)(ROW_BYTES / elem_bytes), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, map_dtype(mode), 2,
                  const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    *err = "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r) + " (rows " + std::to_string(rows) +
           ", k " + std::to_string(k) + ", box_rows " + std::to_string(box_rows) + ")";
    return false;
  }
  return true;
}

}  // namespace

bool tc_encode_map(void* map, const void* base, int mode, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box, bool swizzle128, std::string* err,
                   const unsigned* elem_strides) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    *err = "cuTensorMapEncodeTiled is not available from the driver";
    return false;
  }
  cuuint64_t d[5], st[4];
  cuuint32_t b[5], es[5];
  for (int i = 0; i < rank; ++i) {
    d[i] = dims[i];
    b[i] = box[i];
    es[i] = elem_strides ? elem_strides[i] : 1;
    if (i + 1 < rank) st[i] = strides_bytes[i];
  }
  CUresult r = fn(reinterpret_cast<CUtensorMap*>(map), map_dtype(mode), (cuuint32_t)rank,
                  const_cast<void*>(base), d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    *err = "cuTensorMapEncodeTiled (rank " + std::to_string(rank) + ") failed with code " + std::to_string((int)r);
    return false;
  }
  return true;
}

namespace {

int num_sms_hint() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// N tile of the GEMM: the narrowest of the compiled wgmma widths (32 / 64 / 128) that covers N, else 128 with a ragged
// last tile (TMA zero-fills the weight rows beyond n_pad; the epilogue skips the columns beyond N).
int pick_block_n(int n_pad) { return n_pad <= 32 ? 32 : (n_pad <= 64 ? 64 : 128); }

}  // namespace

bool tc_layer_supported(const wb_layer& L, int mode, bool conv) {
  // 1x1: the activation and weight rows are K-major tensor maps, whose row stride must be a multiple of 16 bytes
  // (K % 4 in fp32, K % 8 in bf16 / fp16)
  const int elem = tc_elem_bytes(mode);
  if ((L.op == WB_OP_PW || L.op == WB_OP_HEAD) && L.kh == 1 && L.kw == 1 && L.stride == 1 && (L.in_c * elem) % 16 == 0)
    return true;
  // KxK / strided dense convolutions (the SSD extra layers): implicit GEMM, one filter tap x 32 (64 bf16 / fp16) channels
  // per k-block; a CTA's tile is a whole number of output images, so the maps must be small (<= 128 pixels)
  return L.op == WB_OP_CONV && L.in_c % 64 == 0 && L.out_h * L.out_w <= (uint32_t)BLOCK_M && L.stride <= 8 && conv;
}

int tc_prepare_weights(const std::vector<wb_layer>& layers, const std::vector<wb_tensor_entry>& tensors,
                       const float* host_data, int mode, bool conv, TcWeights* out, std::string* err) {
  out->mode = mode;
  out->layers = std::vector<TcLayerWeights>(layers.size());
  for (size_t li = 0; li < layers.size(); ++li) {
    const wb_layer& L = layers[li];
    if (!tc_layer_supported(L, mode, conv)) continue;
    TcLayerWeights& w = out->layers[li];
    const int K = L.kh * L.kw * L.in_c, NP = L.n_pad;             // conv: k = tap * in_c + channel
    const float* src = host_data + tensors[L.w_tensor].offset;  // [K][NP]
    w.k = K;
    w.n_pad = NP;
    w.block_n = pick_block_n(NP);
    const int elem = tc_elem_bytes(mode);
    const size_t bytes = (size_t)NP * K * elem;
    std::vector<uint8_t> hi(bytes), lo(mode == TC_TF32X3 ? bytes : 0);
    for (int n = 0; n < NP; ++n)
      for (int k = 0; k < K; ++k) {
        float v = src[(size_t)k * NP + n];
        if (mode == TC_BF16) {
          __nv_bfloat16 b = __float2bfloat16_rn(v);
          memcpy(&hi[((size_t)n * K + k) * 2], &b, 2);
        } else if (mode == TC_FP16) {
          // round to nearest even, subnormals kept; a weight that rounds beyond 65504 would become inf
          __half h = __float2half_rn(v);
          if (std::isinf(__half2float(h))) {
            *err = std::string("layer ") + L.name + ": weight " + std::to_string(v) +
                   " is outside the fp16 range (|w| <= 65504); run this model in bf16 or an fp32 mode";
            return 1;
          }
          memcpy(&hi[((size_t)n * K + k) * 2], &h, 2);
        } else {
          uint32_t u;
          memcpy(&u, &v, 4);
          uint32_t h = mode == TC_TF32X3 ? (u & 0xFFFFE000u) : u;
          memcpy(&hi[((size_t)n * K + k) * 4], &h, 4);
          if (mode == TC_TF32X3) {
            float hf;
            memcpy(&hf, &h, 4);
            float lf = v - hf;
            uint32_t l;
            memcpy(&l, &lf, 4);
            l &= 0xFFFFE000u;
            memcpy(&lo[((size_t)n * K + k) * 4], &l, 4);
          }
        }
      }
    // copies `host` to `dev`, and encodes the tensor map of the copy into `tmap`
    auto upload = [&](DevBuf<void>& dev, const std::vector<uint8_t>& host, unsigned char* tmap) {
      cudaError_t e = alloc(dev, bytes);
      if (e == cudaSuccess) e = cudaMemcpy(dev, host.data(), bytes, cudaMemcpyHostToDevice);
      if (e != cudaSuccess) {
        *err = std::string("cudaMalloc/cudaMemcpy of tensor-core weights failed: ") + cudaGetErrorString(e);
        return false;
      }
      return make_map(reinterpret_cast<CUtensorMap*>(tmap), dev, mode, NP, K, w.block_n, err);
    };
    if (!upload(w.w, hi, w.tmap_b)) return 1;
    if (mode == TC_TF32X3) {
      if (!upload(w.w_lo, lo, w.tmap_b_lo)) return 1;
    } else {
      memcpy(w.tmap_b_lo, w.tmap_b, sizeof(w.tmap_b));
    }
    w.ready = true;
  }
  return 0;
}

int tc_launch_gemm(const LaunchCtx& lc, const TcWeights& tw, int layer_index, int n, const wb_layer& L, const void* in,
                   const float* scale, const float* offset, void* out, float* enc, float* logits, int num_anchors,
                   int num_classes_p1, const void* residual, bool split_k, std::string* err) {
  const TcLayerWeights& w = tw.layers[layer_index];
  if (!w.ready) {
    *err = "no tensor-core weights for this layer";
    return 1;
  }
  const int mode = tw.mode;
  const int elem = tc_elem_bytes(mode);
  TcArgs g;
  g.scale = scale;
  g.offset = offset;
  g.out = out;
  g.enc = enc;
  g.logits = logits;
  g.M = n * L.out_h * L.out_w;
  g.N = L.out_c;
  g.n_pad = L.n_pad;
  g.K = L.kh * L.kw * L.in_c;
  g.block_n = w.block_n;
  g.residual = elem == 2 ? nullptr : residual;
  g.conv = L.op == WB_OP_CONV;
  g.cpb = (L.in_c * elem) / ROW_BYTES;
  g.conv_kw = L.kw;
  g.conv_pad_t = L.pad_t;
  g.conv_pad_l = L.pad_l;
  g.rows_per_tile = g.conv ? (BLOCK_M / (int)(L.out_h * L.out_w)) * (int)(L.out_h * L.out_w) : BLOCK_M;
  if (elem == 2 && residual != nullptr) {
    *err = "residual fusion is not available in the 16-bit modes";
    return 1;
  }
  g.k_blocks = (g.K * elem + ROW_BYTES - 1) / ROW_BYTES;
  g.act = L.act;
  g.is_head = L.op == WB_OP_HEAD;
  g.anchors_per_loc = L.anchors_per_loc;
  g.row_off = L.row_off;
  g.n_box = L.n_box;
  g.num_anchors = num_anchors;
  g.ncp1 = num_classes_p1;
  g.hw = L.out_h * L.out_w;
  const int x3 = mode == TC_TF32X3 ? 2 : 1;
  const int stage_bytes = (A_TILE_BYTES + g.block_n * ROW_BYTES) * x3;
  dim3 grid((g.M + g.rows_per_tile - 1) / g.rows_per_tile, (g.n_pad + g.block_n - 1) / g.block_n);
  // latency-bound shapes: split K so that about one wave of CTAs exists (deterministic cluster reduce)
  g.splits = 1;
  g.kb_per = g.k_blocks;
  const long tiles = (long)grid.x * grid.y;
  // the cluster barriers + DSMEM reduction of a split cost several k-blocks' worth of time: splitting only pays for
  // long accumulation chains, and every split keeps >= 8 k-blocks
  if (tiles < num_sms_hint() / 2 && g.k_blocks >= 16 && split_k) {
    int want = std::max(1, (int)(num_sms_hint() / tiles));  // at most one wave: tiles * splits <= SMs (a second wave of a
                                                            // few CTAs doubles the kernel's duration)
    int splits = std::min(std::min(want, g.k_blocks / 8), 8);  // 8 = portable thread-block cluster size
    if (splits > 1) {
      g.kb_per = (g.k_blocks + splits - 1) / splits;
      g.splits = (g.k_blocks + g.kb_per - 1) / g.kb_per;
      grid.z = g.splits;
    }
  }
  int stages = std::min(6, (200 * 1024) / stage_bytes);
  if (stages > g.kb_per) stages = g.kb_per;
  if (stages < 1) stages = 1;
  g.stages = stages;
  const int staging = BLOCK_M * (g.block_n + 4) * 4;  // epilogue staging tile re-uses the stage ring
  g.ring_bytes = ((std::max(stages * stage_bytes, staging) + 1023) / 1024) * 1024;
  const size_t smem = (size_t)g.ring_bytes + 1024 /*align*/ + 16 * stages;
  alignas(64) CUtensorMap map_a;
  if (g.conv) {
    const int imgs = BLOCK_M / (int)(L.out_h * L.out_w);
    unsigned long long dims[4] = {L.in_c, L.in_w, L.in_h, (unsigned long long)n};
    unsigned long long st[3] = {(unsigned long long)L.in_c * elem, (unsigned long long)L.in_w * L.in_c * elem,
                                (unsigned long long)L.in_h * L.in_w * L.in_c * elem};
    // boxDim counts tensor elements traversed; ceil(boxDim / elementStride) elements are loaded per dimension
    unsigned box[4] = {(unsigned)(ROW_BYTES / elem), (unsigned)((L.out_w - 1) * L.stride + 1),
                       (unsigned)((L.out_h - 1) * L.stride + 1), (unsigned)imgs};
    unsigned es[4] = {1, L.stride, L.stride, 1};
    if (!tc_encode_map(&map_a, in, mode, 4, dims, st, box, true, err, es)) return 1;
  } else if (!make_map(&map_a, in, mode, g.M, g.K, BLOCK_M, err)) {
    return 1;
  }
  CUtensorMap map_b, map_b_lo;
  memcpy(&map_b, w.tmap_b, sizeof(map_b));
  memcpy(&map_b_lo, w.tmap_b_lo, sizeof(map_b_lo));
  // split-K launches: the `splits` CTAs of a tile are one thread-block cluster (1, 1, splits)
  auto launch = [&](auto kern, PerDeviceFlag& attr_done) {
    if (cudaError_t e = max_dynamic_smem_once(kern, 227 * 1024, attr_done)) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = lc.stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 1;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = (unsigned)g.splits;
    cfg.attrs = at;
    cfg.numAttrs = g.splits > 1 ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, map_a, map_b, map_b_lo, g);
  };
  // the instantiations by [TcMode][block_n 32 / 64 / 128]
  struct Instance {
    void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, TcArgs);
    PerDeviceFlag attr_done;
  };
  static Instance instances[4][3] = {
      {{k_gemm_tc<TC_BF16, 32>}, {k_gemm_tc<TC_BF16, 64>}, {k_gemm_tc<TC_BF16, 128>}},
      {{k_gemm_tc<TC_TF32X1, 32>}, {k_gemm_tc<TC_TF32X1, 64>}, {k_gemm_tc<TC_TF32X1, 128>}},
      {{k_gemm_tc<TC_TF32X3, 32>}, {k_gemm_tc<TC_TF32X3, 64>}, {k_gemm_tc<TC_TF32X3, 128>}},
      {{k_gemm_tc<TC_FP16, 32>}, {k_gemm_tc<TC_FP16, 64>}, {k_gemm_tc<TC_FP16, 128>}},
  };
  Instance& k = instances[mode][g.block_n == 32 ? 0 : (g.block_n == 64 ? 1 : 2)];
  const cudaError_t e = launch(k.kern, k.attr_done);
  if (e != cudaSuccess) {
    *err = std::string("tensor-core GEMM launch: ") + cudaGetErrorString(e);
    return 1;
  }
  ++*lc.launch_counter;
  return 0;
}

