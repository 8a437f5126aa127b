// kernels_pre.cu -- K1 (resize + normalise) and the fused K1+K2 stem convolution.
//
// Restates graph nodes `Cast`, `Preprocessor/map/while/ResizeImage/resize/ResizeBilinear`
// (align_corners=false, half_pixel_centers=false), `Preprocessor/mul`, `Preprocessor/sub` and
// `FeatureExtractor/.../Conv2d_0/{Conv2D,BatchNorm,Relu6}` of the frozen graph that
// watsor/detection/tensorflow_cpu.py:114 runs.  The bilinear lerp is written with the explicit
// round-to-nearest intrinsics (__fadd_rn / __fsub_rn / __fmul_rn / __fdiv_rn), which the compiler never
// contracts into a multiply-add: a chain of separately rounded fp32 ops, exactly like TF's CPU kernel, so K1
// is bit-exact against the oracle, and the fused stem's resize equals K1 bit for bit.
#include "common.cuh"

struct AxisTap {
  int lo, hi;
  float lerp;
};

// TF legacy sampling: scale = in/(float)out; pos = dst*scale; lo = floor(pos);
// hi = min(ceil(pos), in-1); lerp = pos - floor(pos).
__device__ __forceinline__ float axis_scale(int in_size, int out_size) {
  return __fdiv_rn((float)in_size, (float)out_size);
}
__device__ __forceinline__ AxisTap axis_tap(int dst, int in_size, float scale) {
  float pos = __fmul_rn((float)dst, scale);
  float fl = floorf(pos);
  AxisTap t;
  t.lo = max((int)fl, 0);
  t.hi = min((int)ceilf(pos), in_size - 1);
  t.lerp = __fsub_rn(pos, fl);
  return t;
}

__device__ __forceinline__ float lerp_px(float tl, float tr, float bl, float br, float lx, float ly) {
  float top = __fadd_rn(tl, __fmul_rn(__fsub_rn(tr, tl), lx));
  float bot = __fadd_rn(bl, __fmul_rn(__fsub_rn(br, bl), lx));
  return __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), ly));
}

// The 12 source bytes one resized pixel interpolates: channel c of tap k (tl, tr, bl, br) goes to raw[c * 4 + k].
// For a YUV frame (4:2:0 or 4:2:2) the slots hold Y, U, V of each tap, and resized_pixel_lerp converts them to the
// RGB24 bytes of cv2.cvtColor first, so the interpolation sees the same bytes as for the converted RGB frame.  The
// other RGB byte orders put each tap's R, G and B in the same slots as RGB24 does, so their lerp is RGB24's.
__device__ __forceinline__ void resized_pixel_load(const FrameDesc& fd, const AxisTap& ty, const AxisTap& tx,
                                                   uint32_t (&raw)[12]) {
  if (fd.fmt == WB_FMT_RGB24) {
    const uint8_t* r0 = fd.ptr + (size_t)ty.lo * fd.pitch;
    const uint8_t* r1 = fd.ptr + (size_t)ty.hi * fd.pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      raw[c * 4 + 0] = __ldg(r0 + tx.lo * 3 + c);
      raw[c * 4 + 1] = __ldg(r0 + tx.hi * 3 + c);
      raw[c * 4 + 2] = __ldg(r1 + tx.lo * 3 + c);
      raw[c * 4 + 3] = __ldg(r1 + tx.hi * 3 + c);
    }
  } else if (fmt_rgb(fd.fmt)) {
    // BGR24, RGBA, BGRA: each call below sees its layout as constants
    const uint8_t* r0 = fd.ptr + (size_t)ty.lo * fd.pitch;
    const uint8_t* r1 = fd.ptr + (size_t)ty.hi * fd.pitch;
    auto bytes = [&](const RgbLayout& L) {
      const uint8_t* const p[4] = {r0 + tx.lo * L.bpp, r0 + tx.hi * L.bpp, r1 + tx.lo * L.bpp, r1 + tx.hi * L.bpp};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        raw[0 + k] = __ldg(p[k] + L.r);
        raw[4 + k] = __ldg(p[k] + L.g);
        raw[8 + k] = __ldg(p[k] + L.b);
      }
    };
    // 4-byte pixels of a frame whose every row is word-aligned: one 32-bit load per tap
    auto words = [&](const RgbLayout& L) {
      const uint32_t* q0 = reinterpret_cast<const uint32_t*>(r0);
      const uint32_t* q1 = reinterpret_cast<const uint32_t*>(r1);
      const uint32_t px[4] = {__ldg(q0 + tx.lo), __ldg(q0 + tx.hi), __ldg(q1 + tx.lo), __ldg(q1 + tx.hi)};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        raw[0 + k] = (px[k] >> (8 * L.r)) & 255u;
        raw[4 + k] = (px[k] >> (8 * L.g)) & 255u;
        raw[8 + k] = (px[k] >> (8 * L.b)) & 255u;
      }
    };
    // row y starts at ptr + y * pitch: word-aligned on every row only when both are multiples of 4
    const bool aligned = ((reinterpret_cast<uintptr_t>(fd.ptr) | (uintptr_t)fd.pitch) & 3) == 0;
    if (fd.fmt == WB_FMT_BGR24)
      bytes(rgb_layout(WB_FMT_BGR24));
    else if (fd.fmt == WB_FMT_RGBA)
      aligned ? words(rgb_layout(WB_FMT_RGBA)) : bytes(rgb_layout(WB_FMT_RGBA));
    else
      aligned ? words(rgb_layout(WB_FMT_BGRA)) : bytes(rgb_layout(WB_FMT_BGRA));
  } else {
    // 4:2:2 and 4:2:0 branch apart so that each sees its layout's steps and shifts as constants (a layout chosen at
    // run time kept them in registers, and the generic stem spilled)
    auto taps = [&](const ChromaLayout& cl) {
      yuv_load(fd.ptr, fd.pitch, fd.chroma, cl, tx.lo, ty.lo, raw[0], raw[4], raw[8]);
      yuv_load(fd.ptr, fd.pitch, fd.chroma, cl, tx.hi, ty.lo, raw[1], raw[5], raw[9]);
      yuv_load(fd.ptr, fd.pitch, fd.chroma, cl, tx.lo, ty.hi, raw[2], raw[6], raw[10]);
      yuv_load(fd.ptr, fd.pitch, fd.chroma, cl, tx.hi, ty.hi, raw[3], raw[7], raw[11]);
    };
    if (fmt_422(fd.fmt))
      taps(chroma_layout_of(WB_FMT_YUYV422, fd.pitch, 2));
    else
      taps(chroma_layout_of(fd.fmt == WB_FMT_NV12 ? WB_FMT_NV12 : WB_FMT_YUV420P, fd.chroma_pitch, fd.v_off));
  }
}
__device__ __forceinline__ void resized_pixel_lerp(uint32_t (&raw)[12], bool yuv, float lx, float ly, float mul,
                                                   float sub, float* out3) {
  if (yuv) {
#pragma unroll
    for (int k = 0; k < 4; ++k) yuv_to_rgb(raw[k], raw[4 + k], raw[8 + k], raw[k], raw[4 + k], raw[8 + k]);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = lerp_px((float)raw[c * 4 + 0], (float)raw[c * 4 + 1], (float)raw[c * 4 + 2], (float)raw[c * 4 + 3], lx, ly);
    out3[c] = __fsub_rn(__fmul_rn(mul, v), sub);
  }
}

// one resized + normalised pixel (3 channels).  The two halves above are split so that a thread can have the loads of
// a second pixel in flight while it lerps the first one.
__device__ __forceinline__ void resized_pixel(const FrameDesc& fd, const AxisTap& ty, const AxisTap& tx, float mul,
                                              float sub, float* out3) {
  uint32_t raw[12];
  resized_pixel_load(fd, ty, tx, raw);
  resized_pixel_lerp(raw, !fmt_rgb(fd.fmt), tx.lerp, ty.lerp, mul, sub, out3);
}

// ---------------------------------------------------------------------------------------------------
// K1 stand-alone: u8 HWC (any size) -> f32 [n][oh][ow][3].  Used by wb_preprocess (parity tests)
// and by wb_backbone-less debugging; the production path is the fused stem below.
constexpr int PP_TY = 8, PP_TX = 32;  // resized pixels per CTA of the stand-alone kernel

__global__ void __launch_bounds__(PP_TY* PP_TX) k_preprocess_f32(const FrameDesc* __restrict__ frames,
                                                                  float* __restrict__ out, int oh, int ow, float mul,
                                                                  float sub) {
  const FrameDesc fd = frames[blockIdx.z];
  const float sy = axis_scale(fd.h, oh), sx = axis_scale(fd.w, ow);
  const int oy = blockIdx.y * PP_TY + (int)threadIdx.x / PP_TX, ox = blockIdx.x * PP_TX + (int)threadIdx.x % PP_TX;
  if (oy >= oh || ox >= ow) return;
  AxisTap ty = axis_tap(oy, fd.h, sy), tx = axis_tap(ox, fd.w, sx);
  float v[3];
  resized_pixel(fd, ty, tx, mul, sub, v);
  float* o = out + (((size_t)blockIdx.z * oh + oy) * ow + ox) * 3;
  o[0] = v[0];
  o[1] = v[1];
  o[2] = v[2];
}

void launch_preprocess_f32(const LaunchCtx& lc, const FrameDesc* frames, int n, float* out, int oh, int ow,
                           float mul, float sub) {
  dim3 grid((ow + PP_TX - 1) / PP_TX, (oh + PP_TY - 1) / PP_TY, n);
  k_preprocess_f32<<<grid, PP_TY * PP_TX, 0, lc.stream>>>(frames, out, oh, ow, mul, sub);
  ++*lc.launch_counter;
}

// ---------------------------------------------------------------------------------------------------
// Fused stem: resized tile built in shared memory (the 300x300x3 tensor never reaches HBM), then the
// first KxK stride-S convolution (C_in = 3) + folded BatchNorm + ReLU6.
// Tile = 8 x 32 output pixels, one thread per output pixel, output channels in chunks of 16.
constexpr int ST_TY = 8, ST_TX = 32;

template <typename T>
__global__ void __launch_bounds__(ST_TY* ST_TX)
    k_stem(const FrameDesc* __restrict__ frames, const float* __restrict__ pre, wb_layer L, int in_h, int in_w,
           float mul, float sub, const float* __restrict__ w, const float* __restrict__ scale,
           const float* __restrict__ offset, T* __restrict__ out) {
  extern __shared__ float smem[];
  const int K = L.kh, S = L.stride;
  const int tile_h = (ST_TY - 1) * S + K, tile_w = (ST_TX - 1) * S + K;
  float* s_in = smem;                              // [tile_h][tile_w][3]
  float* s_w = smem + ((tile_h * tile_w * 3 + 3) & ~3);  // [K*K*3][n_pad], 16-byte aligned
  const int f = blockIdx.z;
  const int oy0 = blockIdx.y * ST_TY, ox0 = blockIdx.x * ST_TX;
  const int tid = threadIdx.x;

  for (int i = tid; i < K * K * 3 * (int)L.n_pad; i += blockDim.x) s_w[i] = w[i];

  // resized tile; rows/cols outside the 300x300 image are the SAME-padding zeros
  const int ry0 = oy0 * S - (int)L.pad_t, rx0 = ox0 * S - (int)L.pad_l;
  FrameDesc fd;
  float sy = 1.f, sx = 1.f;
  if (pre == nullptr) {
    fd = frames[f];
    sy = axis_scale(fd.h, in_h);  // hoisted: one division per thread, not per sampled pixel
    sx = axis_scale(fd.w, in_w);
  }
  for (int i = tid; i < tile_h * tile_w; i += blockDim.x) {
    int ly = i / tile_w, lx = i - ly * tile_w;
    int ry = ry0 + ly, rx = rx0 + lx;
    float v[3] = {0.f, 0.f, 0.f};
    if (ry >= 0 && ry < in_h && rx >= 0 && rx < in_w) {
      if (pre != nullptr) {
        const float* p = pre + (((size_t)f * in_h + ry) * in_w + rx) * 3;
        v[0] = p[0];
        v[1] = p[1];
        v[2] = p[2];
      } else {
        AxisTap ty = axis_tap(ry, fd.h, sy), tx = axis_tap(rx, fd.w, sx);
        resized_pixel(fd, ty, tx, mul, sub, v);
      }
    }
    s_in[i * 3 + 0] = v[0];
    s_in[i * 3 + 1] = v[1];
    s_in[i * 3 + 2] = v[2];
  }
  __syncthreads();

  const int ty = tid / ST_TX, tx = tid - ty * ST_TX;
  const int oy = oy0 + ty, ox = ox0 + tx;
  if (oy >= (int)L.out_h || ox >= (int)L.out_w) return;
  T* o = out + (((size_t)f * L.out_h + oy) * L.out_w + ox) * L.out_c;
  const int taps = K * K * 3;
  for (int oc0 = 0; oc0 < (int)L.out_c; oc0 += 16) {
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    for (int ky = 0; ky < K; ++ky)
      for (int kx = 0; kx < K; ++kx) {
        const float* ip = s_in + ((ty * S + ky) * tile_w + tx * S + kx) * 3;
        const float* wp = s_w + (size_t)((ky * K + kx) * 3) * L.n_pad + oc0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          float x = ip[c];
          const float4* w4 = reinterpret_cast<const float4*>(wp + c * L.n_pad);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float4 ww = w4[q];
            acc[q * 4 + 0] = fmaf(x, ww.x, acc[q * 4 + 0]);
            acc[q * 4 + 1] = fmaf(x, ww.y, acc[q * 4 + 1]);
            acc[q * 4 + 2] = fmaf(x, ww.z, acc[q * 4 + 2]);
            acc[q * 4 + 3] = fmaf(x, ww.w, acc[q * 4 + 3]);
          }
        }
      }
    (void)taps;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      int oc = oc0 + q * 4;
      if (oc >= (int)L.out_c) break;
      float4 v;
      v.x = affine_rn(acc[q * 4 + 0], scale[oc + 0], offset[oc + 0]);
      v.y = affine_rn(acc[q * 4 + 1], scale[oc + 1], offset[oc + 1]);
      v.z = affine_rn(acc[q * 4 + 2], scale[oc + 2], offset[oc + 2]);
      v.w = affine_rn(acc[q * 4 + 3], scale[oc + 3], offset[oc + 3]);
      if (L.act == WB_ACT_RELU6) {
        v.x = relu6f(v.x);
        v.y = relu6f(v.y);
        v.z = relu6f(v.z);
        v.w = relu6f(v.w);
      }
      ActIO<T>::st4(o + oc, v);
    }
  }
}

// Register-tiled variant for the common 3x3 / stride-2 / 32-channel stem: one thread = 4 consecutive output
// pixels x 8 output channels, so every weight vector read from shared memory feeds 4 pixels (the generic
// kernel re-reads all 27x32 weights per pixel: `LDS.128` broadcasts cost 4 wavefronts each and dominated).
// Same tile (8 x 32 pixels), same resize code, same (ky, kx, c) accumulation order => identical results.
template <typename T>
__global__ void __launch_bounds__(256)
    k_stem_3x3s2_c32(const FrameDesc* __restrict__ frames, const float* __restrict__ pre, wb_layer L, int in_h, int in_w,
                     float mul, float sub, const float* __restrict__ w, const float* __restrict__ scale,
                     const float* __restrict__ offset, T* __restrict__ out) {
  constexpr int K = 3, S = 2, OC = 32;
  constexpr int tile_h = (ST_TY - 1) * S + K, tile_w = (ST_TX - 1) * S + K;  // 17 x 65
  __shared__ __align__(16) float s_in[tile_h * tile_w * 3];
  __shared__ __align__(16) float s_w[K * K * 3 * OC];
  const int f = blockIdx.z;
  const int oy0 = blockIdx.y * ST_TY, ox0 = blockIdx.x * ST_TX;
  const int tid = threadIdx.x;
  // the 864 weights go through registers: the loads are issued here and waited for after the tile has been built
  // (13 % of the kernel's stall samples sat on this copy when it stored right away)
  constexpr int WREGS = (K * K * 3 * OC + 255) / 256;
  float wreg[WREGS];
#pragma unroll
  for (int j = 0; j < WREGS; ++j) {
    const int i = tid + j * 256;
    wreg[j] = i < K * K * 3 * OC ? __ldg(w + (i / OC) * L.n_pad + (i % OC)) : 0.f;
  }
  const int ry0 = oy0 * S - (int)L.pad_t, rx0 = ox0 * S - (int)L.pad_l;
  if (pre == nullptr) {
    const FrameDesc fd = frames[f];
    const float sy = axis_scale(fd.h, in_h), sx = axis_scale(fd.w, in_w);
    // two pixels per round: the byte loads of both are in flight before either is interpolated
    for (int i0 = tid; i0 < tile_h * tile_w; i0 += 512) {
      uint32_t raw[2][12];
      AxisTap tys[2], txs[2];
      bool inside[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = i0 + u * 256;
        const int ly = i / tile_w, lx = i - ly * tile_w;
        const int ry = ry0 + ly, rx = rx0 + lx;
        inside[u] = i < tile_h * tile_w && ry >= 0 && ry < in_h && rx >= 0 && rx < in_w;
        if (inside[u]) {
          tys[u] = axis_tap(ry, fd.h, sy);
          txs[u] = axis_tap(rx, fd.w, sx);
          resized_pixel_load(fd, tys[u], txs[u], raw[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = i0 + u * 256;
        if (i < tile_h * tile_w) {
          float v[3] = {0.f, 0.f, 0.f};
          if (inside[u]) resized_pixel_lerp(raw[u], !fmt_rgb(fd.fmt), txs[u].lerp, tys[u].lerp, mul, sub, v);
          s_in[i * 3 + 0] = v[0];
          s_in[i * 3 + 1] = v[1];
          s_in[i * 3 + 2] = v[2];
        }
      }
    }
  } else {
    for (int i = tid; i < tile_h * tile_w; i += 256) {
      int ly = i / tile_w, lx = i - ly * tile_w;
      int ry = ry0 + ly, rx = rx0 + lx;
      float v[3] = {0.f, 0.f, 0.f};
      if (ry >= 0 && ry < in_h && rx >= 0 && rx < in_w) {
        const float* p = pre + (((size_t)f * in_h + ry) * in_w + rx) * 3;
        v[0] = p[0];
        v[1] = p[1];
        v[2] = p[2];
      }
      s_in[i * 3 + 0] = v[0];
      s_in[i * 3 + 1] = v[1];
      s_in[i * 3 + 2] = v[2];
    }
  }
#pragma unroll
  for (int j = 0; j < WREGS; ++j) {
    const int i = tid + j * 256;
    if (i < K * K * 3 * OC) s_w[i] = wreg[j];
  }
  __syncthreads();

  const int ocg = tid & 3, quad = tid >> 2;  // 4 channel groups of 8, 64 pixel quads (8 rows x 8 quads)
  const int ty = quad >> 3, tx0 = (quad & 7) * 4;
  float acc[4][8];
#pragma unroll
  for (int o = 0; o < 4; ++o)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[o][j] = 0.f;
#pragma unroll
  for (int ky = 0; ky < K; ++ky)
#pragma unroll
    for (int kx = 0; kx < K; ++kx)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float4 w0 = *reinterpret_cast<const float4*>(&s_w[((ky * K + kx) * 3 + c) * OC + ocg * 8]);
        const float4 w1 = *reinterpret_cast<const float4*>(&s_w[((ky * K + kx) * 3 + c) * OC + ocg * 8 + 4]);
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const float x = s_in[((ty * S + ky) * tile_w + (tx0 + o) * S + kx) * 3 + c];
          acc[o][0] = fmaf(x, w0.x, acc[o][0]);
          acc[o][1] = fmaf(x, w0.y, acc[o][1]);
          acc[o][2] = fmaf(x, w0.z, acc[o][2]);
          acc[o][3] = fmaf(x, w0.w, acc[o][3]);
          acc[o][4] = fmaf(x, w1.x, acc[o][4]);
          acc[o][5] = fmaf(x, w1.y, acc[o][5]);
          acc[o][6] = fmaf(x, w1.z, acc[o][6]);
          acc[o][7] = fmaf(x, w1.w, acc[o][7]);
        }
      }
  const int oy = oy0 + ty;
  if (oy >= (int)L.out_h) return;
  float sc[8], of[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sc[j] = __ldg(scale + ocg * 8 + j);
    of[j] = __ldg(offset + ocg * 8 + j);
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    const int ox = ox0 + tx0 + o;
    if (ox >= (int)L.out_w) break;
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = affine_rn(acc[o][j], sc[j], of[j]);
      y[j] = L.act == WB_ACT_RELU6 ? relu6f(v) : v;
    }
    T* dst = out + (((size_t)f * L.out_h + oy) * L.out_w + ox) * OC + ocg * 8;
    ActIO<T>::st4(dst, make_float4(y[0], y[1], y[2], y[3]));
    ActIO<T>::st4(dst + 4, make_float4(y[4], y[5], y[6], y[7]));
  }
}

template <typename T>
void launch_stem(const LaunchCtx& lc, const FrameDesc* frames, const float* pre, int n, const wb_layer& L,
                 int in_h, int in_w, float mul, float sub, const float* w, const float* scale,
                 const float* offset, T* out) {
  dim3 grid((L.out_w + ST_TX - 1) / ST_TX, (L.out_h + ST_TY - 1) / ST_TY, n);
  if (L.kh == 3 && L.kw == 3 && L.stride == 2 && L.out_c == 32) {
    k_stem_3x3s2_c32<T><<<grid, 256, 0, lc.stream>>>(frames, pre, L, in_h, in_w, mul, sub, w, scale, offset, out);
    ++*lc.launch_counter;
    return;
  }
  const int tile_h = (ST_TY - 1) * L.stride + L.kh, tile_w = (ST_TX - 1) * L.stride + L.kw;
  const size_t smem = ((((size_t)tile_h * tile_w * 3 + 3) & ~(size_t)3) +
                       (((size_t)L.kh * L.kw * 3 * L.n_pad + 3) & ~(size_t)3)) * sizeof(float);
  static PerDeviceFlag attr_done;
  max_dynamic_smem_once(k_stem<T>, 200 * 1024, attr_done);
  k_stem<T><<<grid, ST_TY * ST_TX, smem, lc.stream>>>(frames, pre, L, in_h, in_w, mul, sub, w, scale, offset, out);
  ++*lc.launch_counter;
}

template void launch_stem<float>(const LaunchCtx&, const FrameDesc*, const float*, int, const wb_layer&, int,
                                 int, float, float, const float*, const float*, const float*, float*);
template void launch_stem<__nv_bfloat16>(const LaunchCtx&, const FrameDesc*, const float*, int,
                                         const wb_layer&, int, int, float, float, const float*, const float*,
                                         const float*, __nv_bfloat16*);
template void launch_stem<__half>(const LaunchCtx&, const FrameDesc*, const float*, int, const wb_layer&, int, int,
                                  float, float, const float*, const float*, const float*, __half*);
