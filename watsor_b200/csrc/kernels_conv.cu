// kernels_conv.cu -- fp32 (parity-mode) convolution kernels of the SSD backbone and heads.
//
// Restates `FeatureExtractor/...` (DepthwiseConv2dNative / Conv2D + FusedBatchNormV3 + Relu6) and
// `BoxPredictor_i/{BoxEncodingPredictor,ClassPredictor}` (Conv2D + BiasAdd, Reshape, concat) of the
// frozen graph run by watsor/detection/tensorflow_cpu.py:114.  All tensors are NHWC, TF `SAME`
// padding (asymmetric).  The 1x1 / KxK dense convolutions are one tiled SGEMM with an optional
// im2col row gather; the wgmma path lives in kernels_tc.cu.
#include <algorithm>

#include "common.cuh"

// ---------------------------------------------------------------------------------------------------
// depthwise 3x3, stride S = 1 or 2 (wb_create refuses others), + affine + ReLU6; one thread = 4 consecutive output
// pixels x 4 channels; the (4-1)*S+3 input columns of a row are loaded once and reused by the four outputs (2x fewer
// loads at stride 1).  Columns outside the input are zeros, and outputs beyond out_w are not stored, so any width works.
template <typename T, int S>
__global__ void __launch_bounds__(256)
    k_dw_strip(int n, wb_layer L, const T* __restrict__ in, const float* __restrict__ w, const float* __restrict__ scale,
               const float* __restrict__ offset, T* __restrict__ out) {
  constexpr int NC = 3 * S + 3;
  const int c4n = L.out_c >> 2;
  const int xs_n = (L.out_w + 3) >> 2;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)n * L.out_h * xs_n * c4n;
  if (idx >= total) return;
  const int c = (int)(idx % c4n) * 4;
  size_t p = idx / c4n;
  const int ox0 = (int)(p % xs_n) * 4;
  p /= xs_n;
  const int oy = (int)(p % L.out_h);
  const int f = (int)(p / L.out_h);
  float4 wr[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wr[t] = __ldg(reinterpret_cast<const float4*>(w + t * L.out_c + c));
  float4 acc[4];
#pragma unroll
  for (int o = 0; o < 4; ++o) acc[o] = make_float4(0.f, 0.f, 0.f, 0.f);
  const T* base = in + (size_t)f * L.in_h * L.in_w * L.in_c + c;
  const int iy0 = oy * S - (int)L.pad_t, ix0 = ox0 * S - (int)L.pad_l;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = iy0 + ky;
    if (iy < 0 || iy >= (int)L.in_h) continue;
    float4 col[NC];
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      const int ix = ix0 + j;
      col[j] = (ix >= 0 && ix < (int)L.in_w) ? ActIO<T>::ld4(base + ((size_t)iy * L.in_w + ix) * L.in_c)
                                             : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4 x = col[o * S + kx], ww = wr[ky * 3 + kx];
        acc[o].x = fmaf(x.x, ww.x, acc[o].x);
        acc[o].y = fmaf(x.y, ww.y, acc[o].y);
        acc[o].z = fmaf(x.z, ww.z, acc[o].z);
        acc[o].w = fmaf(x.w, ww.w, acc[o].w);
      }
  }
  const float4 sc = __ldg(reinterpret_cast<const float4*>(scale + c));
  const float4 of = __ldg(reinterpret_cast<const float4*>(offset + c));
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    const int ox = ox0 + o;
    if (ox >= (int)L.out_w) break;
    float4 v = make_float4(affine_rn(acc[o].x, sc.x, of.x), affine_rn(acc[o].y, sc.y, of.y),
                           affine_rn(acc[o].z, sc.z, of.z), affine_rn(acc[o].w, sc.w, of.w));
    if (L.act == WB_ACT_RELU6) v = make_float4(relu6f(v.x), relu6f(v.y), relu6f(v.z), relu6f(v.w));
    ActIO<T>::st4(out + (((size_t)f * L.out_h + oy) * L.out_w + ox) * L.out_c + c, v);
  }
}

template <typename T>
void launch_dw(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, const float* w, const float* scale,
               const float* offset, T* out) {
  size_t total = (size_t)n * L.out_h * ((L.out_w + 3) >> 2) * (L.out_c >> 2);
  unsigned blocks = (unsigned)((total + 255) / 256);
  if (L.stride == 1)
    k_dw_strip<T, 1><<<blocks, 256, 0, lc.stream>>>(n, L, in, w, scale, offset, out);
  else
    k_dw_strip<T, 2><<<blocks, 256, 0, lc.stream>>>(n, L, in, w, scale, offset, out);
  ++*lc.launch_counter;
}
template void launch_dw<float>(const LaunchCtx&, int, const wb_layer&, const float*, const float*, const float*,
                               const float*, float*);
template void launch_dw<__nv_bfloat16>(const LaunchCtx&, int, const wb_layer&, const __nv_bfloat16*, const float*,
                                       const float*, const float*, __nv_bfloat16*);
template void launch_dw<__half>(const LaunchCtx&, int, const wb_layer&, const __half*, const float*, const float*,
                                const float*, __half*);

// residual add (MobileNet-v2 style bottlenecks)
template <typename T>
__global__ void __launch_bounds__(256) k_add(size_t n4, const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 x = ActIO<T>::ld4(a + i * 4), y = ActIO<T>::ld4(b + i * 4);
  ActIO<T>::st4(out + i * 4, make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w));
}
template <typename T>
void launch_add(const LaunchCtx& lc, size_t elems, const T* a, const T* b, T* out) {
  size_t n4 = elems / 4;
  k_add<T><<<(unsigned)((n4 + 255) / 256), 256, 0, lc.stream>>>(n4, a, b, out);
  ++*lc.launch_counter;
}
template void launch_add<float>(const LaunchCtx&, size_t, const float*, const float*, float*);
template void launch_add<__nv_bfloat16>(const LaunchCtx&, size_t, const __nv_bfloat16*, const __nv_bfloat16*, __nv_bfloat16*);
template void launch_add<__half>(const LaunchCtx&, size_t, const __half*, const __half*, __half*);

// TF MaxPool / AvgPool with padding SAME (Inception modules): thread = (pixel, 4 channels).  The maximum ignores the
// padding; the average is the fp32 sum of the in-image taps in (ky, kx) order divided by their count.
template <typename T, bool MAX>
__global__ void __launch_bounds__(256) k_pool(int n, wb_layer L, const T* __restrict__ in, T* __restrict__ out) {
  const int c4n = L.out_c >> 2;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)n * L.out_h * L.out_w * c4n;
  if (idx >= total) return;
  const int c = (int)(idx % c4n) * 4;
  size_t p = idx / c4n;
  const int ox = (int)(p % L.out_w);
  p /= L.out_w;
  const int oy = (int)(p % L.out_h);
  const int f = (int)(p / L.out_h);
  const T* base = in + (size_t)f * L.in_h * L.in_w * L.in_c + c;
  const int iy0 = oy * (int)L.stride - (int)L.pad_t, ix0 = ox * (int)L.stride - (int)L.pad_l;
  float4 acc = MAX ? make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY) : make_float4(0.f, 0.f, 0.f, 0.f);
  int cnt = 0;
  for (int ky = 0; ky < (int)L.kh; ++ky) {
    const int iy = iy0 + ky;
    if (iy < 0 || iy >= (int)L.in_h) continue;
    for (int kx = 0; kx < (int)L.kw; ++kx) {
      const int ix = ix0 + kx;
      if (ix < 0 || ix >= (int)L.in_w) continue;
      const float4 x = ActIO<T>::ld4(base + ((size_t)iy * L.in_w + ix) * L.in_c);
      if (MAX) {
        acc = make_float4(fmaxf(acc.x, x.x), fmaxf(acc.y, x.y), fmaxf(acc.z, x.z), fmaxf(acc.w, x.w));
      } else {
        acc = make_float4(__fadd_rn(acc.x, x.x), __fadd_rn(acc.y, x.y), __fadd_rn(acc.z, x.z), __fadd_rn(acc.w, x.w));
      }
      ++cnt;
    }
  }
  if (!MAX) {
    const float d = (float)cnt;
    acc = make_float4(__fdiv_rn(acc.x, d), __fdiv_rn(acc.y, d), __fdiv_rn(acc.z, d), __fdiv_rn(acc.w, d));
  }
  ActIO<T>::st4(out + idx * 4, acc);
}
template <typename T>
void launch_pool(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, T* out) {
  size_t total = (size_t)n * L.out_h * L.out_w * (L.out_c >> 2);
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (L.op == WB_OP_MAXPOOL)
    k_pool<T, true><<<blocks, 256, 0, lc.stream>>>(n, L, in, out);
  else
    k_pool<T, false><<<blocks, 256, 0, lc.stream>>>(n, L, in, out);
  ++*lc.launch_counter;
}
template void launch_pool<float>(const LaunchCtx&, int, const wb_layer&, const float*, float*);
template void launch_pool<__nv_bfloat16>(const LaunchCtx&, int, const wb_layer&, const __nv_bfloat16*, __nv_bfloat16*);
template void launch_pool<__half>(const LaunchCtx&, int, const wb_layer&, const __half*, __half*);

// ConcatV2 along channels, one input: [n*h*w][in_c] -> channels [row_off, row_off + in_c) of [n*h*w][out_c]
template <typename T>
__global__ void __launch_bounds__(256) k_copy_channels(size_t pixels, int in_c, int out_c, int coff, const T* __restrict__ in,
                                                       T* __restrict__ out) {
  const int c4n = in_c >> 2;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= pixels * c4n) return;
  const size_t p = idx / c4n;
  const int c = (int)(idx - p * c4n) * 4;
  ActIO<T>::st4(out + p * out_c + coff + c, ActIO<T>::ld4(in + p * in_c + c));
}
template <typename T>
void launch_copy_channels(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, T* out) {
  const size_t pixels = (size_t)n * L.out_h * L.out_w;
  const size_t total = pixels * (L.in_c >> 2);
  k_copy_channels<T><<<(unsigned)((total + 255) / 256), 256, 0, lc.stream>>>(pixels, (int)L.in_c, (int)L.out_c, (int)L.row_off, in, out);
  ++*lc.launch_counter;
}
template void launch_copy_channels<float>(const LaunchCtx&, int, const wb_layer&, const float*, float*);
template void launch_copy_channels<__nv_bfloat16>(const LaunchCtx&, int, const wb_layer&, const __nv_bfloat16*, __nv_bfloat16*);
template void launch_copy_channels<__half>(const LaunchCtx&, int, const wb_layer&, const __half*, __half*);

// ---------------------------------------------------------------------------------------------------
// SGEMM  C[M,N] = A[M,K] * W[K,N]  (+ per-column affine, ReLU6)
//   M = n*out_h*out_w rows (NHWC pixels), K = kh*kw*in_c, N = out_c.
//   A rows are gathered: 1x1 -> the pixel's channel vector; KxK -> im2col on the fly (a BK=16 slice of
//   K never straddles a filter tap because in_c % 16 == 0).
//   Head layers scatter their columns straight into the concatenated [n][anchors][4] /
//   [n][anchors][C+1] tensors (graph nodes `concat`, `concat_1`).
template <typename T>
struct GemmArgs {
  const T* in;
  const float* w;
  const float* scale;
  const float* offset;
  T* out;
  float* enc;
  float* logits;
  int M, N, K, ldw;
  int in_h, in_w, in_c, out_h, out_w, kh, kw, stride, pad_t, pad_l;
  int act;
  int is_head, anchors_per_loc, row_off, n_box, num_anchors, ncp1;
  int splits;      // split-K: blockIdx.z handles k-tiles [z*kt_per, ...) and writes raw partial sums
  float* partial;  // [splits][M][ldw]
};

template <typename T, int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__(256) k_gemm_cc(GemmArgs<T> g) {
  constexpr int BK = 16;
  constexpr int NT = 256;
  static_assert((BM / TM) * (BN / TN) == NT, "thread tiling");
  constexpr int A_F4 = BM * BK / 4 / NT;  // float4 loads of A per thread
  constexpr int B_F4 = BK * BN / 4 / NT;
  static_assert(A_F4 >= 1 && B_F4 >= 1, "tile too small");
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const bool im2col = (g.kh != 1 || g.kw != 1 || g.stride != 1);

  // A loader: thread -> (row, k-quad)
  int a_row[A_F4], a_kq[A_F4];
  int a_f[A_F4], a_oy[A_F4], a_ox[A_F4];
  bool a_ok[A_F4];
#pragma unroll
  for (int i = 0; i < A_F4; ++i) {
    int e = tid + i * NT;
    a_row[i] = e >> 2;
    a_kq[i] = e & 3;
    int m = m0 + a_row[i];
    a_ok[i] = m < g.M;
    int mm = a_ok[i] ? m : 0;
    int hw = g.out_h * g.out_w;
    a_f[i] = mm / hw;
    int p = mm - a_f[i] * hw;
    a_oy[i] = p / g.out_w;
    a_ox[i] = p - a_oy[i] * g.out_w;
  }
  int b_k[B_F4], b_n[B_F4];
#pragma unroll
  for (int i = 0; i < B_F4; ++i) {
    int e = tid + i * NT;
    b_k[i] = e / (BN / 4);
    b_n[i] = (e % (BN / 4)) * 4;
  }

  float4 a_reg[A_F4], b_reg[B_F4];
  auto load_tile = [&](int kt) {
    const int k0 = kt * BK;
#pragma unroll
    for (int i = 0; i < A_F4; ++i) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a_ok[i]) {
        if (!im2col) {
          if (k0 + a_kq[i] * 4 < g.K) v = ActIO<T>::ld4(g.in + (size_t)(m0 + a_row[i]) * g.K + k0 + a_kq[i] * 4);
        } else {
          int tap = k0 / g.in_c, ci = k0 - tap * g.in_c;
          int ky = tap / g.kw, kx = tap - ky * g.kw;
          int iy = a_oy[i] * g.stride - g.pad_t + ky, ix = a_ox[i] * g.stride - g.pad_l + kx;
          if (iy >= 0 && iy < g.in_h && ix >= 0 && ix < g.in_w)
            v = ActIO<T>::ld4(g.in + (((size_t)a_f[i] * g.in_h + iy) * g.in_w + ix) * g.in_c + ci + a_kq[i] * 4);
        }
      }
      a_reg[i] = v;
    }
#pragma unroll
    for (int i = 0; i < B_F4; ++i) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      int n = n0 + b_n[i];
      if (n < g.ldw && k0 + b_k[i] < g.K) v = __ldg(reinterpret_cast<const float4*>(g.w + (size_t)(k0 + b_k[i]) * g.ldw + n));
      b_reg[i] = v;
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_F4; ++i) {
      As[buf][a_kq[i] * 4 + 0][a_row[i]] = a_reg[i].x;
      As[buf][a_kq[i] * 4 + 1][a_row[i]] = a_reg[i].y;
      As[buf][a_kq[i] * 4 + 2][a_row[i]] = a_reg[i].z;
      As[buf][a_kq[i] * 4 + 3][a_row[i]] = a_reg[i].w;
    }
#pragma unroll
    for (int i = 0; i < B_F4; ++i) *reinterpret_cast<float4*>(&Bs[buf][b_k[i]][b_n[i]]) = b_reg[i];
  };

  // compute mapping: TM rows as TM/4 groups of 4 spaced BM/(TM/4) apart, same for columns
  constexpr int TY = BM / TM, TX = BN / TN;
  const int ty = tid / TX, tx = tid % TX;
  constexpr int RG = TM / 4, CG = TN / 4;
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int KT_all = (g.K + BK - 1) / BK;
  const int kt_per = (KT_all + g.splits - 1) / g.splits;
  const int kt0 = blockIdx.z * kt_per;
  const int KT = min(KT_all, kt0 + kt_per);
  load_tile(kt0);
  store_tile(kt0 & 1);
  __syncthreads();
  for (int kt = kt0; kt < KT; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < KT) load_tile(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int r = 0; r < RG; ++r) {
        float4 v = *reinterpret_cast<const float4*>(&As[buf][k][r * (TY * 4) + ty * 4]);
        a[r * 4 + 0] = v.x;
        a[r * 4 + 1] = v.y;
        a[r * 4 + 2] = v.z;
        a[r * 4 + 3] = v.w;
      }
#pragma unroll
      for (int c = 0; c < CG; ++c) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][c * (TX * 4) + tx * 4]);
        b[c * 4 + 0] = v.x;
        b[c * 4 + 1] = v.y;
        b[c * 4 + 2] = v.z;
        b[c * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < KT) {
      store_tile(buf ^ 1);
      __syncthreads();
    }
  }

  // epilogue
#pragma unroll
  for (int r = 0; r < RG; ++r)
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const int i = r * 4 + ii;
      const int m = m0 + r * (TY * 4) + ty * 4 + ii;
      if (m >= g.M) continue;
#pragma unroll
      for (int c = 0; c < CG; ++c) {
        const int n = n0 + c * (TX * 4) + tx * 4;
        if (n >= g.N) continue;
        if (g.splits > 1) {
          *reinterpret_cast<float4*>(g.partial + ((size_t)blockIdx.z * g.M + m) * g.ldw + n) =
              make_float4(acc[i][c * 4 + 0], acc[i][c * 4 + 1], acc[i][c * 4 + 2], acc[i][c * 4 + 3]);
          continue;
        }
        float v[4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          int nn = n + jj;
          float s = nn < g.ldw ? __ldg(g.scale + nn) : 1.f, o = nn < g.ldw ? __ldg(g.offset + nn) : 0.f;
          float x = affine_rn(acc[i][c * 4 + jj], s, o);
          v[jj] = g.act == WB_ACT_RELU6 ? relu6f(x) : x;
        }
        if (!g.is_head) {
          ActIO<T>::st4(g.out + (size_t)m * g.N + n, make_float4(v[0], v[1], v[2], v[3]));
        } else {
          const int hw = g.out_h * g.out_w;
          const int f = m / hw, p = m - f * hw;
          const size_t row = (size_t)f * g.num_anchors + g.row_off + (size_t)p * g.anchors_per_loc;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            int nn = n + jj;
            if (nn >= g.N) break;
            if (nn < g.n_box)
              g.enc[row * 4 + nn] = v[jj];
            else
              g.logits[row * g.ncp1 + (nn - g.n_box)] = v[jj];
          }
        }
      }
    }
}

namespace {

struct SplitKReduceArgs {
  const float* partial;  // [splits][M][ld] raw accumulators
  const float* scale;
  const float* offset;
  void* out;  // T [M][N]
  float* enc;
  float* logits;
  int M, N, ld, splits, act;
  int is_head, anchors_per_loc, row_off, n_box, num_anchors, ncp1, hw;
};

// sums the split-K partial tiles in split order and applies the layer epilogue (affine, ReLU6, store
// or head scatter) with the activation type T.  One thread per 4 output columns.
template <typename T>
__global__ void __launch_bounds__(256) k_splitk_reduce(SplitKReduceArgs r) {
  const int n4 = r.ld >> 2;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)r.M * n4) return;
  const int m = (int)(idx / n4), n = (int)(idx % n4) * 4;
  if (n >= r.N) return;
  float4 acc = *reinterpret_cast<const float4*>(r.partial + (size_t)m * r.ld + n);
  for (int z = 1; z < r.splits; ++z) {
    float4 p = *reinterpret_cast<const float4*>(r.partial + ((size_t)z * r.M + m) * r.ld + n);
    acc.x = __fadd_rn(acc.x, p.x);
    acc.y = __fadd_rn(acc.y, p.y);
    acc.z = __fadd_rn(acc.z, p.z);
    acc.w = __fadd_rn(acc.w, p.w);
  }
  float v[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float x = affine_rn(v[j], __ldg(r.scale + n + j), __ldg(r.offset + n + j));
    v[j] = r.act == WB_ACT_RELU6 ? relu6f(x) : x;
  }
  if (r.is_head) {
    const int f = m / r.hw, p = m - f * r.hw;
    const size_t row = (size_t)f * r.num_anchors + r.row_off + (size_t)p * r.anchors_per_loc;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int nn = n + j;
      if (nn >= r.N) break;
      if (nn < r.n_box)
        r.enc[row * 4 + nn] = v[j];
      else
        r.logits[row * r.ncp1 + (nn - r.n_box)] = v[j];
    }
  } else {
    ActIO<T>::st4(reinterpret_cast<T*>(r.out) + (size_t)m * r.N + n, make_float4(v[0], v[1], v[2], v[3]));
  }
}

template <typename T>
void launch_splitk_reduce(const LaunchCtx& lc, const SplitKReduceArgs& r) {
  size_t total = (size_t)r.M * (r.ld >> 2);
  k_splitk_reduce<T><<<(unsigned)((total + 255) / 256), 256, 0, lc.stream>>>(r);
  ++*lc.launch_counter;
}

}  // namespace

template <typename T>
void launch_gemm_cc(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, const float* w,
                    const float* scale, const float* offset, T* out, float* enc, float* logits,
                    int num_anchors, int num_classes_p1, float* partial, size_t partial_floats) {
  GemmArgs<T> g;
  g.in = in;
  g.w = w;
  g.scale = scale;
  g.offset = offset;
  g.out = out;
  g.enc = enc;
  g.logits = logits;
  g.M = n * L.out_h * L.out_w;
  g.N = L.out_c;
  g.K = L.kh * L.kw * L.in_c;
  g.ldw = L.n_pad;
  g.in_h = L.in_h;
  g.in_w = L.in_w;
  g.in_c = L.in_c;
  g.out_h = L.out_h;
  g.out_w = L.out_w;
  g.kh = L.kh;
  g.kw = L.kw;
  g.stride = L.stride;
  g.pad_t = L.pad_t;
  g.pad_l = L.pad_l;
  g.act = L.act;
  g.is_head = L.op == WB_OP_HEAD;
  g.anchors_per_loc = L.anchors_per_loc;
  g.row_off = L.row_off;
  g.n_box = L.n_box;
  g.num_anchors = num_anchors;
  g.ncp1 = num_classes_p1;
  g.splits = 1;
  g.partial = partial;
  // big tiles when they still fill every SM, small tiles otherwise
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  long big = (long)((g.M + 127) / 128) * ((g.N + 127) / 128);
  if (big >= sms && g.N >= 128) {
    dim3 grid((g.N + 127) / 128, (g.M + 127) / 128);
    k_gemm_cc<T, 128, 128, 8, 8><<<grid, 256, 0, lc.stream>>>(g);
    ++*lc.launch_counter;
    return;
  }
  dim3 grid((g.N + 63) / 64, (g.M + 63) / 64);
  // latency-bound shapes (few tiles, long K): split K over blockIdx.z so that ~2 waves of CTAs exist;
  // partial sums go to scratch and are reduced in a fixed order (deterministic) with the epilogue fused
  const int kt_all = (g.K + 15) / 16;
  const long tiles = (long)grid.x * grid.y;
  if (partial != nullptr && tiles < 120 && kt_all >= 16) {
    int want = (int)((296 + tiles - 1) / tiles);
    int splits = std::min(want, kt_all / 8);
    while (splits > 1 && (size_t)splits * g.M * g.ldw > partial_floats) --splits;
    if (splits > 1) {
      const int kt_per = (kt_all + splits - 1) / splits;
      splits = (kt_all + kt_per - 1) / kt_per;  // no empty split
      g.splits = splits;
      grid.z = splits;
    }
  }
  k_gemm_cc<T, 64, 64, 4, 4><<<grid, 256, 0, lc.stream>>>(g);
  ++*lc.launch_counter;
  if (g.splits > 1) {
    SplitKReduceArgs r;
    r.partial = partial;
    r.scale = scale;
    r.offset = offset;
    r.out = out;
    r.enc = enc;
    r.logits = logits;
    r.M = g.M;
    r.N = g.N;
    r.ld = g.ldw;
    r.splits = g.splits;
    r.act = g.act;
    r.is_head = g.is_head;
    r.anchors_per_loc = g.anchors_per_loc;
    r.row_off = g.row_off;
    r.n_box = g.n_box;
    r.num_anchors = g.num_anchors;
    r.ncp1 = g.ncp1;
    r.hw = g.out_h * g.out_w;
    launch_splitk_reduce<T>(lc, r);
  }
}

template void launch_gemm_cc<float>(const LaunchCtx&, int, const wb_layer&, const float*, const float*, const float*,
                                    const float*, float*, float*, float*, int, int, float*, size_t);
template void launch_gemm_cc<__nv_bfloat16>(const LaunchCtx&, int, const wb_layer&, const __nv_bfloat16*, const float*,
                                            const float*, const float*, __nv_bfloat16*, float*, float*, int, int, float*,
                                            size_t);
template void launch_gemm_cc<__half>(const LaunchCtx&, int, const wb_layer&, const __half*, const float*, const float*,
                                     const float*, __half*, float*, float*, int, int, float*, size_t);
