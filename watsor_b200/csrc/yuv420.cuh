// yuv420.cuh -- 4:2:0 frames (what video decoders emit) converted to the RGB24 bytes the kernels read, and RGB24
// pixels converted to the 4:2:0 frames the effects pass can write for an encoder.
//
// A 4:2:0 frame of w x h pixels (w, h even) is packed in w*h*3/2 bytes: the full-resolution luma plane, then the
// chroma at half resolution in both directions.  The two layouts differ only in where the chroma lives, which
// ChromaLayout holds as data:
//   yuv420p (ffmpeg's software decoders): U plane [h/2][w/2], then V plane [h/2][w/2]
//   NV12 (NVDEC): one plane [h/2][w/2] of interleaved (U, V) pairs
// The arithmetic is BT.601 limited range in 20-bit fixed point, which equals cv2.cvtColor(COLOR_YUV2RGB_I420 /
// COLOR_YUV2RGB_NV12) on every (Y, U, V) triple (tests/test_yuv_host.py, tests/test_gpu_yuv.py).  Integer only, so
// the result does not depend on the file's -fmad setting.
#pragma once
#include <stddef.h>
#include <stdint.h>

#define WB_FMT_RGB24 0
#define WB_FMT_YUV420P 1
#define WB_FMT_NV12 2

struct ChromaLayout {
  int step;      // bytes between horizontally adjacent U samples
  int row;       // bytes between chroma rows
  size_t v_off;  // V sample = U sample + v_off
};

__host__ __device__ __forceinline__ ChromaLayout chroma_layout(int fmt, int w, int h) {
  if (fmt == WB_FMT_NV12) return ChromaLayout{2, w, 1};
  return ChromaLayout{1, w / 2, (size_t)(w / 2) * (h / 2)};
}

// bytes of one packed frame
__host__ __device__ __forceinline__ size_t frame_bytes(int fmt, int w, int h) {
  return fmt == WB_FMT_RGB24 ? (size_t)w * h * 3 : (size_t)w * h * 3 / 2;
}

// address of the U sample of pixel (x, y) given that of pixel (0, 0); the V sample is at + v_off.  A window of a frame
// (x0, y0 even) has its own origin `chroma` and keeps the parent frame's layout.  T: uint8_t or const uint8_t.
template <typename T>
__device__ __forceinline__ T* chroma_ptr(T* chroma, const ChromaLayout& cl, int x, int y) {
  return chroma + (size_t)(y >> 1) * cl.row + (size_t)(x >> 1) * cl.step;
}

// Y, U, V bytes of pixel (x, y) of the frame whose luma rows start at `luma`, `pitch` bytes apart; yuv_to_rgb below
// converts them (two halves, so that a caller can have the loads of several pixels in flight before it converts any)
__device__ __forceinline__ void yuv420_load(const uint8_t* __restrict__ luma, int pitch, const uint8_t* __restrict__ chroma,
                                            const ChromaLayout& cl, int x, int y, uint32_t& Y, uint32_t& U, uint32_t& V) {
  const uint8_t* c = chroma_ptr(chroma, cl, x, y);
  Y = __ldg(luma + (size_t)y * pitch + x);
  U = __ldg(c);
  V = __ldg(c + cl.v_off);
}

__device__ __forceinline__ uint32_t yuv_sat(int v) { return (uint32_t)min(max(v >> 20, 0), 255); }

// RGB of one (Y, U, V) triple
__device__ __forceinline__ void yuv_to_rgb(uint32_t Y, uint32_t U, uint32_t V, uint32_t& r, uint32_t& g, uint32_t& b) {
  const int y = max((int)Y - 16, 0) * 1220542 + (1 << 19);
  const int u = (int)U - 128, v = (int)V - 128;
  r = yuv_sat(y + 1673527 * v);
  g = yuv_sat(y - 852492 * v - 409993 * u);
  b = yuv_sat(y + 2116026 * u);
}

// The other direction, for the frames the effects pass writes: Y, U, V of one RGB pixel, BT.601 limited range in 20-bit
// fixed point, which equals cv2.cvtColor(COLOR_RGB2YUV_I420) on every (R, G, B) triple (tests/test_yuv_out_host.py,
// tests/test_gpu_yuv_out.py).  OpenCV takes a 2x2 block's U and V from its top-left pixel alone, without averaging,
// so a caller converts every pixel for Y and only the top-left ones for U and V.  The results lie in 16..240 and every
// intermediate fits in int32; integer only, so the result does not depend on the file's -fmad setting.
__device__ __forceinline__ void rgb_to_yuv(uint32_t r, uint32_t g, uint32_t b, uint32_t& Y, uint32_t& U, uint32_t& V) {
  const int R = (int)r, G = (int)g, B = (int)b;
  Y = yuv_sat(269484 * R + 528482 * G + 102760 * B + (1 << 19) + (16 << 20));
  U = yuv_sat(-155188 * R - 305135 * G + 460324 * B + (1 << 19) + (128 << 20));
  V = yuv_sat(460324 * R - 385875 * G - 74448 * B + (1 << 19) + (128 << 20));
}
