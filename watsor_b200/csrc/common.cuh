// common.cuh -- shared device-side types of libwatsor_b200 (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/watsor_b200.h"
#include "model_format.h"
#include "yuv420.cuh"

// One model image of a batch: where its pixels are and which camera it belongs to.  The image is a whole frame or a
// detection window of one (wb_set_camera_windows); either way its rows start at `ptr`, `pitch` bytes apart, and its
// chroma rows at `chroma`, `chroma_pitch` bytes apart.  The planes are the caller's device frame (read in place) or
// the packed copy of a host frame.  Replaces the (image_shape, image_np) pair of ObjectDetector.detect
// (tensorflow_cpu.py:74).
struct FrameDesc {
  const uint8_t* ptr;     // device pointer to pixel (0, 0): RGB24 HWC (share.py:68-73), or its Y sample in a YUV frame
  const uint8_t* chroma;  // YUV: the U sample of pixel (0, 0) (4:2:0: in the U or UV plane; 4:2:2: the U byte of the
                          // pixel's macropixel)
  int64_t v_off;          // YUV: bytes from a U sample to its V sample (yuv420p: V plane - U plane, either sign; NV12:
                          // 1; 4:2:2: 2)
  int32_t w, h;
  int32_t pitch;          // bytes between rows of the RGB / luma plane / macropixels (packed frame: bpp*w / w / 2w)
  int32_t chroma_pitch;   // YUV: bytes between chroma rows (packed frame: w/2 yuv420p, w NV12, 2w 4:2:2)
  int32_t cam;            // -1: no camera (a window's rows are filtered after the merge, k_window_merge)
  int32_t fmt;            // WB_FMT_* (yuv420.cuh)
};

// The model images of one frame of a windowed batch, for k_window_merge: images [first, first + count) are its
// windows, whose rows are shifted by the window's origin.
struct WindowFrame {
  int32_t first, count;
  int32_t cam;
  int32_t _pad;
  double merge_thr;  // a row is dropped when a kept row of another window covers more than this share of the smaller box
  int32_t x[WB_MAX_WINDOWS], y[WB_MAX_WINDOWS];
};

// Per-camera filter state resident in HBM (ConfidenceFilter / AreaFilter / MaskFilter __init__).
#define WB_MAX_LABELS 128
struct CameraCfg {
  int32_t width, height;
  int32_t n_zones;
  int32_t has_mask;
  int32_t check_label;      // require label > 0 (track.py:26)
  int32_t default_present;  // entry used for labels without one of their own
  int32_t default_has_zone_list;
  uint32_t default_zone_bits;
  double default_conf, default_area;
  const int32_t* sat;  // [n_zones][(height+1)*(width+1)] inclusive-exclusive summed-area tables
  double conf[WB_MAX_LABELS];
  double area[WB_MAX_LABELS];
  uint32_t zone_bits[WB_MAX_LABELS];
  uint8_t present[WB_MAX_LABELS];
  uint8_t has_zone_list[WB_MAX_LABELS];
};

struct PostParams {
  int32_t num_anchors, num_classes;  // classes without background
  float scale_y, scale_x, scale_h, scale_w, logit_scale;
  float iou_thr, score_thr;
  int32_t max_per_class, max_total;
  float class_offset;
};

// activation element type helpers (fp32 parity path / bf16 and fp16 tensor-core paths)
template <typename T> struct ActIO;
template <> struct ActIO<float> {
  static __device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
  static __device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <> struct ActIO<__nv_bfloat16> {
  static __device__ __forceinline__ float4 ld4(const __nv_bfloat16* p) {
    uint2 r = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&r.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&r.y);
    float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
  }
  static __device__ __forceinline__ void st4(__nv_bfloat16* p, float4 v) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 r;
    r.x = *reinterpret_cast<uint32_t*>(&a);
    r.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = r;
  }
  static __device__ __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
};
// fp16 storage (precision 4): round to nearest even, subnormals kept.  A value beyond the largest finite half is
// clamped to +-65504 first, so an overflowing activation saturates instead of becoming +-inf and poisoning every layer
// after it.  Only stores clamp: loads widen exactly.
constexpr float FP16_MAX = 65504.0f;
__device__ __forceinline__ float sat_fp16(float v) { return fminf(fmaxf(v, -FP16_MAX), FP16_MAX); }
template <> struct ActIO<__half> {
  static __device__ __forceinline__ float4 ld4(const __half* p) {
    uint2 r = *reinterpret_cast<const uint2*>(p);
    float2 fa = __half22float2(*reinterpret_cast<__half2*>(&r.x)), fb = __half22float2(*reinterpret_cast<__half2*>(&r.y));
    return make_float4(fa.x, fa.y, fb.x, fb.y);
  }
  static __device__ __forceinline__ void st4(__half* p, float4 v) {
    __half2 a = __floats2half2_rn(sat_fp16(v.x), sat_fp16(v.y)), b = __floats2half2_rn(sat_fp16(v.z), sat_fp16(v.w));
    uint2 r;
    r.x = *reinterpret_cast<uint32_t*>(&a);
    r.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = r;
  }
  static __device__ __forceinline__ float ld(const __half* p) { return __half2float(*p); }
  static __device__ __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(sat_fp16(v)); }
};

__device__ __forceinline__ float relu6f(float v) { return fminf(fmaxf(v, 0.0f), 6.0f); }

// y = acc*scale + offset exactly as two roundings (the graph runs Conv2D and
// FusedBatchNormV3 / BiasAdd as separate fp32 ops)
__device__ __forceinline__ float affine_rn(float acc, float s, float o) {
  return __fadd_rn(__fmul_rn(acc, s), o);
}

// ---- launchers implemented in the .cu files -------------------------------------------------------
// cudaFuncSetAttribute applies to the current device only: "already done" is remembered per device, so that
// several contexts on different GPUs can live in one process (the reference runs one process per detector,
// detector.py:12-55, but nothing in the C-ABI forbids the other arrangement).
struct PerDeviceFlag {
  bool done[64] = {};
  static int dev() {
    int d = 0;
    cudaGetDevice(&d);
    return d & 63;
  }
  bool get() const { return done[dev()]; }
  void set() { done[dev()] = true; }
};

// lets `kern` use up to `bytes` of dynamic shared memory on the current device; `done` remembers a success, so that
// only the first launch on a device pays for the call and a failed call is made again by the next launch
template <typename Kernel>
cudaError_t max_dynamic_smem_once(Kernel kern, int bytes, PerDeviceFlag& done) {
  if (done.get()) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done.set();
  return e;
}

struct LaunchCtx {
  cudaStream_t stream;
  int* launch_counter;  // host-side counter of kernel launches (bench: gpu_launches)
};

void launch_preprocess_f32(const LaunchCtx& lc, const FrameDesc* frames, int n, float* out, int oh, int ow,
                           float mul, float sub);
template <typename T>
void launch_stem(const LaunchCtx& lc, const FrameDesc* frames, const float* pre, int n, const wb_layer& L,
                 int in_h, int in_w, float mul, float sub, const float* w, const float* scale,
                 const float* offset, T* out);
template <typename T>
void launch_dw(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, const float* w, const float* scale,
               const float* offset, T* out);
template <typename T>
void launch_add(const LaunchCtx& lc, size_t elems, const T* a, const T* b, T* out);
template <typename T>
void launch_pool(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, T* out);
template <typename T>
void launch_copy_channels(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, T* out);
template <typename T>
void launch_gemm_cc(const LaunchCtx& lc, int n, const wb_layer& L, const T* in, const float* w,
                    const float* scale, const float* offset, T* out, float* enc, float* logits,
                    int num_anchors, int num_classes_p1, float* partial, size_t partial_floats);
void launch_post(const LaunchCtx& lc, int n, const PostParams& pp, const float* enc, const float* logits,
                 const float* anchors, const FrameDesc* frames, const CameraCfg* cams, uint32_t flags,
                 int* sel_count, unsigned long long* sel_key, float4* sel_box, wb_detection* out, uint32_t* verdicts,
                 float* raw_boxes, float* raw_scores, float* raw_classes, int* raw_num, int* kept_hist);
void launch_window_merge(const LaunchCtx& lc, int n_frames, const PostParams& pp, const WindowFrame* win,
                         const wb_detection* rows, const int* raw_num, const CameraCfg* cams, uint32_t flags,
                         wb_detection* out, uint32_t* verdicts);
void launch_filter_rows(const LaunchCtx& lc, const CameraCfg* cam, int n_rows, wb_detection* rows,
                        uint32_t* verdicts);
void launch_build_sat(const LaunchCtx& lc, const uint8_t* raster, int n_zones, int h, int w, int32_t* sat);
