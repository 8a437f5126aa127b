// kernels_fused.cu -- depthwise 3x3 conv (+BN+ReLU6) fused into the A-operand producer of the tensor-core
// 1x1 conv (+BN+ReLU6): the depthwise activation never exists in HBM (K3+K4 of SURVEY.md 2.2).
//
// Restates the layer pairs `Conv2d_i_depthwise` -> `Conv2d_i_pointwise` of the frozen graph
// (watsor/detection/tensorflow_cpu.py:114 runs them inside sess.run).  fp32-faithful mode only (TF32X3).
//
// Persistent kernel, one CTA per SM, output tile = 8 x 16 pixels of one image x all N (<= 64) channels:
//   warp 16     TMA producer: per 32-channel k-block a 4-D box {32 ch, halo_w, halo_h, 1 image} of the
//               depthwise INPUT (halo included; out-of-image coordinates and channels >= C are zero-filled by
//               TMA = TF SAME padding) and the 1x1 weight tiles (hi, lo; weight rows >= K zero-filled)
//   warps 8..15 depthwise producers: thread = 4 adjacent pixels x 4 channels; a 3 x (3S + 3) window of the halo tile
//               is read once from shared memory (8 lanes = the 8 channel quads of one pixel -> conflict-free
//               128-byte rows, the 9 tap weights live in registers), BN + ReLU6, TF32 hi/lo split, written
//               straight into the 128B-swizzled wgmma A tiles
//   warps 0..7  two consumer warpgroups (tile rows 0..63 / 64..127): wgmma (3 TF32 MMAs per product, accumulators in
//               registers, k-block partial sums added with round-to-nearest), then BN (+ ReLU6) (+ the residual
//               shortcut of a following Add) and the stores of their rows
// The depthwise accumulation order (ky, kx) and the GEMM's MMA sequence (wg_mma_kblock) are those of the unfused
// kernels, so the result is bit-identical to running k_dw_strip followed by k_gemm_tc (with its residual epilogue).
//
// Stride 2: the halo of an 8 x 16 tile is 17 x 33 pixels x 128 B = 71 KB per stage.  Three of them do not fit beside
// the A/B ring, so make_plan picks 2 halo stages and 1 A/B stage: the TMA of the next k-block's halo still overlaps the
// depthwise work, and the MMAs of one 32-channel k-block (128 x N x 32, x3) are short next to the producers'
// 128 x 32 x 9 FMAs, so the single A/B stage costs little.  The other ways out (a 16-channel half-k-block halo, or a
// different 128-pixel tile shape) would need a second producer mapping and do not shrink the halo per output pixel.
// A partial last k-block (C % 32 != 0): the producers write zeros into the A columns of channels >= C, as TMA's zero
// fill does for k_gemm_tc, so the MMA sequence is the same on the zero-filled K tail (see s_dw below).
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "kernels_tc.cuh"
#include "tc_common.cuh"

namespace {

constexpr int F_TH = 8, F_TW = 16;  // output tile (pixels) = 128 GEMM rows

struct FusedArgs {
  const float* dw_w;  // [9][C]
  const float* dw_scale;
  const float* dw_offset;
  const float* scale;  // 1x1 layer, [n_pad]
  const float* offset;
  float* out;  // [n_img][OH][OW][N]
  const float* residual;  // nullptr, or the shortcut of a following Add: added after BN, laid out like `out`
  int dw_act, act;
  int C, S, pad_t, pad_l;
  int OH, OW, n_img;
  int N, n_pad, block_n, k_blocks;
  int tiles_x, tiles_y;
  int stages, halo_stages;
  int th_in, tw_in;
};

constexpr int F_CONSUMER_WARPS = 8;
constexpr int F_PRODUCER_WARPS = 8;
constexpr int F_FIRST_PRODUCER_THREAD = 32 * F_CONSUMER_WARPS;                   // 256
constexpr int F_TMA_WARP = F_CONSUMER_WARPS + F_PRODUCER_WARPS;                  // 16
constexpr int F_THREADS = F_FIRST_PRODUCER_THREAD + 32 * F_PRODUCER_WARPS + 32;  // 544

template <int S, int BN>
__global__ void __launch_bounds__(F_THREADS, 1)
    k_dwpw_tc_x3(const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_b_lo, FusedArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int halo_bytes = ((g.th_in * g.tw_in * ROW_BYTES + 1023) / 1024) * 1024;
  constexpr int B_TILE_BYTES = BN * ROW_BYTES;
  constexpr int AB_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
  uint8_t* halo0 = smem;
  uint8_t* ab0 = halo0 + (size_t)g.halo_stages * halo_bytes;
  uint64_t* halo_full = reinterpret_cast<uint64_t*>(ab0 + (size_t)g.stages * AB_BYTES);
  uint64_t* halo_empty = halo_full + g.halo_stages;
  uint64_t* b_full = halo_empty + g.halo_stages;
  uint64_t* a_ready = b_full + g.stages;
  uint64_t* empty = a_ready + g.stages;
  float* s_dw = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(empty + g.stages) + 15) & ~(uintptr_t)15);  // [11][cs]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = g.tiles_x * g.tiles_y;
  const int num_tiles = tiles_per_img * g.n_img;

  if (threadIdx.x == 0) {
    for (int h = 0; h < g.halo_stages; ++h) {
      mbar_init(smem_u32(&halo_full[h]), 1);
      mbar_init(smem_u32(&halo_empty[h]), F_PRODUCER_WARPS);  // one arrive per depthwise producer warp
    }
    for (int s = 0; s < g.stages; ++s) {
      mbar_init(smem_u32(&b_full[s]), 1);
      mbar_init(smem_u32(&a_ready[s]), F_PRODUCER_WARPS);
      mbar_init(smem_u32(&empty[s]), 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  // depthwise taps + folded BN of every channel: loaded once per CTA, read by the producers every k-block.  Rows are
  // padded with zeros to whole k-blocks: on the zero-filled halo channels >= C (a partial last k-block) the
  // producers then compute +0, the value TMA's zero fill puts into k_gemm_tc's A tiles there.
  const int cs = g.k_blocks * 32;  // row stride of s_dw
  for (int i = threadIdx.x; i < 9 * cs; i += blockDim.x) {
    const int k = i / cs, ch = i - k * cs;
    s_dw[i] = ch < g.C ? g.dw_w[k * g.C + ch] : 0.f;
  }
  for (int i = threadIdx.x; i < cs; i += blockDim.x) {
    s_dw[9 * cs + i] = i < g.C ? g.dw_scale[i] : 0.f;
    s_dw[10 * cs + i] = i < g.C ? g.dw_offset[i] : 0.f;
  }
  float* s_pw = s_dw + 11 * cs;  // [2][BN]: folded BN of the pointwise output channels
  for (int i = threadIdx.x; i < BN; i += blockDim.x) {  // BN may exceed n_pad (N = 16 / 24: one 32-wide tile)
    s_pw[i] = i < g.n_pad ? g.scale[i] : 1.f;
    s_pw[BN + i] = i < g.n_pad ? g.offset[i] : 0.f;
  }
  __syncthreads();

  if (warp == F_TMA_WARP) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      int it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int img = t / tiles_per_img, r = t - img * tiles_per_img;
        const int oy0 = (r / g.tiles_x) * F_TH, ox0 = (r % g.tiles_x) * F_TW;
        for (int kb = 0; kb < g.k_blocks; ++kb, ++it) {
          const int h = it % g.halo_stages, s = it % g.stages;
          mbar_wait(smem_u32(&halo_empty[h]), ((it / g.halo_stages) & 1) ^ 1);
          const uint32_t hb = smem_u32(&halo_full[h]);
          mbar_expect_tx(hb, (uint32_t)(g.th_in * g.tw_in * ROW_BYTES));
          tma_load_4d(smem_u32(halo0 + (size_t)h * halo_bytes), &map_in, hb, kb * 32, ox0 * S - g.pad_l,
                      oy0 * S - g.pad_t, img);
          mbar_wait(smem_u32(&empty[s]), ((it / g.stages) & 1) ^ 1);
          const uint32_t bb = smem_u32(&b_full[s]);
          uint8_t* sb = ab0 + (size_t)s * AB_BYTES + 2 * A_TILE_BYTES;
          mbar_expect_tx(bb, 2 * B_TILE_BYTES);
          tma_load_2d(smem_u32(sb), &map_b, bb, kb * 32, 0);
          tma_load_2d(smem_u32(sb + B_TILE_BYTES), &map_b_lo, bb, kb * 32, 0);
        }
      }
    }
  } else if (warp < F_CONSUMER_WARPS) {
    // ------------------------------------------------------------------ consumer warpgroups
    const int wg = warp >> 2;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // tile row of accumulators 0, 1 (+8: 2, 3)
    const int col = 2 * (lane & 3);
    int it = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int img = t / tiles_per_img, r = t - img * tiles_per_img;
      const int oy0 = (r / g.tiles_x) * F_TH, ox0 = (r % g.tiles_x) * F_TW;
      float acc[BN / 2], part[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < g.k_blocks; ++kb, ++it) {
        const int s = it % g.stages;
        const uint32_t ph = (it / g.stages) & 1;
        mbar_wait(smem_u32(&a_ready[s]), ph);
        mbar_wait(smem_u32(&b_full[s]), ph);
        const uint32_t a_hi = smem_u32(ab0 + (size_t)s * AB_BYTES) + (uint32_t)(wg * 64 * ROW_BYTES);
        const uint32_t a_lo = a_hi + A_TILE_BYTES;
        const uint32_t b_hi = smem_u32(ab0 + (size_t)s * AB_BYTES) + 2 * A_TILE_BYTES, b_lo = b_hi + B_TILE_BYTES;
        wg_x3_kblock_sum<BN>(acc, part, a_hi, a_lo, b_hi, b_lo);
        wg_bar_sync(wg);  // every warp of the warpgroup has seen its MMAs complete: the stage may be refilled
        if ((threadIdx.x & 127) == 0) mbar_arrive(smem_u32(&empty[s]));
      }
      // folded BN + ReLU6 of this thread's two rows, 8-byte stores (a lane quad covers 32 contiguous bytes)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rr = row + 8 * h;
        const int oy = oy0 + rr / F_TW, ox = ox0 + rr % F_TW;
        if (oy >= g.OH || ox >= g.OW) continue;
        const size_t po = (((size_t)img * g.OH + oy) * g.OW + ox) * g.N;
        float* op = g.out + po;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + col;
          if (c >= g.N) break;
          float y0 = affine_rn(acc[4 * j + 2 * h], s_pw[c], s_pw[BN + c]);
          float y1 = affine_rn(acc[4 * j + 2 * h + 1], s_pw[c + 1], s_pw[BN + c + 1]);
          if (g.act == WB_ACT_RELU6) {
            y0 = relu6f(y0);
            y1 = relu6f(y1);
          }
          if (g.residual != nullptr) {  // same order as k_gemm_tc's TF32 epilogue: BN, activation, then the shortcut
            const float2 r2 = *reinterpret_cast<const float2*>(g.residual + po + c);
            y0 = __fadd_rn(y0, r2.x);
            y1 = __fadd_rn(y1, r2.y);
          }
          *reinterpret_cast<float2*>(op + c) = make_float2(y0, y1);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ depthwise producers
    const int pt = threadIdx.x - F_FIRST_PRODUCER_THREAD;
    const int q = pt & 7, slot = pt >> 3;  // channel quad of the k-block, pixel slot
    int it = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      for (int kb = 0; kb < g.k_blocks; ++kb, ++it) {
        const int h = it % g.halo_stages, s = it % g.stages;
        const int cch = kb * 32 + q * 4;
        float4 wr[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) wr[k] = lds128(smem_u32(s_dw + k * cs + cch));
        const float4 sc = lds128(smem_u32(s_dw + 9 * cs + cch));
        const float4 of = lds128(smem_u32(s_dw + 10 * cs + cch));
        mbar_wait(smem_u32(&halo_full[h]), (it / g.halo_stages) & 1);
        mbar_wait(smem_u32(&empty[s]), ((it / g.stages) & 1) ^ 1);  // A tiles of this stage are free again
        const uint32_t hal = smem_u32(halo0 + (size_t)h * halo_bytes);
        const uint32_t a_hi = smem_u32(ab0 + (size_t)s * AB_BYTES);
        const uint32_t a_lo = a_hi + A_TILE_BYTES;
        // One thread = 4 horizontally adjacent output pixels of one channel quad: a 3 x (3S + 3) input window is
        // read once (18 / 27 LDS.128 instead of 36) and every input feeds up to 3 / S outputs.  Per output the taps
        // still accumulate in (ky, kx) order, so the result is bit-identical to the stand-alone depthwise kernel.
        static_assert((S == 1 || S == 2) && F_PRODUCER_WARPS == 8 && F_TW == 16 && F_TH == 8, "producer mapping");
        constexpr int TW_IN = (F_TW - 1) * S + 3, NC = 3 * S + 3;
        const int ty = slot >> 2, x0 = (slot & 3) * 4;
        const uint32_t win = hal + (uint32_t)((ty * S * TW_IN + x0 * S) * 128 + q * 16);
        float4 acc[4];
#pragma unroll
        for (int o = 0; o < 4; ++o) acc[o] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const float4 x = lds128(win + (uint32_t)((ky * TW_IN + c) * 128));
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const int o = (c - kx) / S;
              if (c >= kx && (c - kx) % S == 0 && o < 4) {
                const float4 ww = wr[ky * 3 + kx];
                acc[o].x = fmaf(x.x, ww.x, acc[o].x);
                acc[o].y = fmaf(x.y, ww.y, acc[o].y);
                acc[o].z = fmaf(x.z, ww.z, acc[o].z);
                acc[o].w = fmaf(x.w, ww.w, acc[o].w);
              }
            }
          }
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const int r = ty * F_TW + x0 + o;
          float v[4] = {affine_rn(acc[o].x, sc.x, of.x), affine_rn(acc[o].y, sc.y, of.y),
                        affine_rn(acc[o].z, sc.z, of.z), affine_rn(acc[o].w, sc.w, of.w)};
          uint4 hi, lo;
          uint32_t* hp = &hi.x;
          uint32_t* lp = &lo.x;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float a = g.dw_act == WB_ACT_RELU6 ? relu6f(v[e]) : v[e];
            const uint32_t hb = __float_as_uint(a) & 0xFFFFE000u;
            hp[e] = hb;
            lp[e] = __float_as_uint(__fsub_rn(a, __uint_as_float(hb))) & 0xFFFFE000u;
          }
          const uint32_t off = (uint32_t)r * 128u + (uint32_t)((q ^ (r & 7)) << 4);  // 128B swizzle
          sts128(a_hi + off, hi);
          sts128(a_lo + off, lo);
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(smem_u32(&a_ready[s]));
          mbar_arrive(smem_u32(&halo_empty[h]));
        }
      }
    }
  }
}

struct FusedPlan {
  int block_n, stages, halo_stages, th_in, tw_in, tiles_x, tiles_y;
  size_t smem;
};

bool make_plan(const wb_layer& dw, const wb_layer& pw, FusedPlan* p) {
  p->block_n = pw.n_pad <= 32 ? 32 : 64;  // the GEMM's N tile (weight rows beyond N: zero-filled)
  p->th_in = (F_TH - 1) * dw.stride + 3;
  p->tw_in = (F_TW - 1) * dw.stride + 3;
  p->tiles_x = (dw.out_w + F_TW - 1) / F_TW;
  p->tiles_y = (dw.out_h + F_TH - 1) / F_TH;
  const size_t halo = ((size_t)p->th_in * p->tw_in * ROW_BYTES + 1023) / 1024 * 1024;
  const size_t ab = 2 * A_TILE_BYTES + 2 * (size_t)p->block_n * ROW_BYTES;
  const size_t dw_bytes = 44 * (size_t)((dw.out_c + 31) / 32 * 32);  // s_dw: [11][C rounded up to 32] floats
  const size_t budget = 224 * 1024 - dw_bytes;
  // prefer two A/B stages, then as many halo buffers as fit (at least two)
  for (int st = 2; st >= 1; --st)
    for (int hs = 3; hs >= 2; --hs) {
      if (hs * halo + st * ab <= budget) {
        p->stages = st;
        p->halo_stages = hs;
        p->smem = hs * halo + st * ab + 1024 + 8 * (2 * hs + 3 * st) + 16 + dw_bytes + 8 * (size_t)p->block_n;
        return true;
      }
    }
  return false;
}


}  // namespace

bool fused_dwpw_supported(const TcWeights& tw, int pw_layer_index, const wb_layer& dw, const wb_layer& pw) {
  if (tw.mode != TC_TF32X3) return false;
  if (dw.op != WB_OP_DW || pw.op != WB_OP_PW) return false;
  if (dw.kh != 3 || dw.kw != 3 || (dw.stride != 1 && dw.stride != 2)) return false;
  // Small maps stay unfused.  A tile runs its C / 32 k-blocks one after another, so a map of few tiles is one long
  // chain per CTA, while k_dw_strip spreads the depthwise work over every SM.  Measured on an H100 80GB HBM3 (400 W
  // limit), SSD-MobileNet-v2 at batch 8: fused is slower on the 19x19 maps (6 tiles per image, C = 192 / 384; 28 us
  // against 23 us stand-alone) and faster from 38x38 (15 tiles per image) up.
  if (dw.out_h * dw.out_w < 32 * 32) return false;
  // N <= 64: the running sum and the k-block partial (2 x N / 2 registers per consumer thread) fit beside the
  // depthwise producers' registers.  Fewer than 16 k-blocks: from 16 on k_gemm_tc may split K, which changes the
  // summation order.
  if (dw.out_c % 4 != 0 || (dw.out_c + 31) / 32 >= 16 || pw.in_c != dw.out_c || pw.n_pad > 64 || pw.out_c % 4 != 0)
    return false;
  if (!tw.layers[pw_layer_index].ready) return false;
  FusedPlan p;
  return make_plan(dw, pw, &p);
}

int fused_launch_dwpw(const LaunchCtx& lc, const TcWeights& tw, int pw_layer_index, int n, const wb_layer& dw,
                      const wb_layer& pw, const void* in, const float* dw_w, const float* dw_scale, const float* dw_offset,
                      const float* scale, const float* offset, const float* residual, void* out, std::string* err) {
  const TcLayerWeights& w = tw.layers[pw_layer_index];
  FusedPlan p;
  if (!make_plan(dw, pw, &p)) {
    *err = "fused depthwise+pointwise: no shared-memory plan";
    return 1;
  }
  FusedArgs g;
  g.dw_w = dw_w;
  g.dw_scale = dw_scale;
  g.dw_offset = dw_offset;
  g.scale = scale;
  g.offset = offset;
  g.dw_act = dw.act;
  g.act = pw.act;
  g.C = dw.out_c;
  g.S = dw.stride;
  g.pad_t = dw.pad_t;
  g.pad_l = dw.pad_l;
  g.OH = dw.out_h;
  g.OW = dw.out_w;
  g.n_img = n;
  g.N = pw.out_c;
  g.n_pad = pw.n_pad;
  g.block_n = p.block_n;
  g.k_blocks = (dw.out_c + 31) / 32;
  g.out = static_cast<float*>(out);
  g.residual = residual;
  g.tiles_x = p.tiles_x;
  g.tiles_y = p.tiles_y;
  g.stages = p.stages;
  g.halo_stages = p.halo_stages;
  g.th_in = p.th_in;
  g.tw_in = p.tw_in;
  alignas(64) CUtensorMap map_in, map_b, map_b_lo;
  {
    unsigned long long dims[4] = {(unsigned long long)dw.in_c, dw.in_w, dw.in_h, (unsigned long long)n};
    unsigned long long st[3] = {(unsigned long long)dw.in_c * 4, (unsigned long long)dw.in_w * dw.in_c * 4,
                                (unsigned long long)dw.in_h * dw.in_w * dw.in_c * 4};
    unsigned box[4] = {32, (unsigned)p.tw_in, (unsigned)p.th_in, 1};
    if (!tc_encode_map(&map_in, in, TC_TF32X3, 4, dims, st, box, false, err)) return 1;
  }
  {
    unsigned long long dims[2] = {(unsigned long long)w.k, (unsigned long long)w.n_pad};
    unsigned long long st[1] = {(unsigned long long)w.k * 4};
    unsigned box[2] = {32, (unsigned)p.block_n};
    if (!tc_encode_map(&map_b, w.w, TC_TF32X3, 2, dims, st, box, true, err)) return 1;
    if (!tc_encode_map(&map_b_lo, w.w_lo, TC_TF32X3, 2, dims, st, box, true, err)) return 1;
  }
  static PerDeviceFlag attr_done[4];
  static int ctas = 0;
  if (ctas == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&ctas, cudaDevAttrMultiProcessorCount, dev);
  }
  const long tiles = (long)p.tiles_x * p.tiles_y * n;
  const dim3 grid((unsigned)std::min<long>(tiles, ctas));
  auto launch = [&](auto kern, PerDeviceFlag& done) {
    if (cudaError_t e = max_dynamic_smem_once(kern, 227 * 1024, done)) return e;
    kern<<<grid, F_THREADS, p.smem, lc.stream>>>(map_in, map_b, map_b_lo, g);
    return cudaGetLastError();
  };
  const int ki = (dw.stride == 2 ? 2 : 0) + (p.block_n == 32 ? 0 : 1);
  const cudaError_t e = ki == 0   ? launch(k_dwpw_tc_x3<1, 32>, attr_done[0])
                        : ki == 1 ? launch(k_dwpw_tc_x3<1, 64>, attr_done[1])
                        : ki == 2 ? launch(k_dwpw_tc_x3<2, 32>, attr_done[2])
                                  : launch(k_dwpw_tc_x3<2, 64>, attr_done[3]);
  if (e != cudaSuccess) {
    *err = std::string("fused depthwise+pointwise launch: ") + cudaGetErrorString(e);
    return 1;
  }
  ++*lc.launch_counter;
  return 0;
}

