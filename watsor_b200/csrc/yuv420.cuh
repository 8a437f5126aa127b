// yuv420.cuh -- the frame layouts the kernels read: YUV frames (what video decoders and capture devices emit) converted
// to the RGB24 bytes the kernels work on, RGB24 pixels converted to the 4:2:0 frames the effects pass can write for an
// encoder, and the packed RGB byte orders (RGB24, BGR24, RGBA, BGRA) described by one table, rgb_layout below.
//
// A 4:2:0 frame of w x h pixels (w, h even) is packed in w*h*3/2 bytes: the full-resolution luma plane, then the
// chroma at half resolution in both directions.  A packed 4:2:2 frame (w even, any h) is [h][w][2] bytes: each pair of
// pixels (2k, 2k+1) of a row shares one 4-byte macropixel, and every row has its own chroma.  The layouts differ only
// in where the samples live, which ChromaLayout holds as data:
//   yuv420p (ffmpeg's software decoders): U plane [h/2][w/2], then V plane [h/2][w/2]
//   NV12 (NVDEC): one plane [h/2][w/2] of interleaved (U, V) pairs
//   YUYV (ffmpeg yuyv422, UVC webcams): macropixel Y0 U Y1 V
//   UYVY (ffmpeg uyvy422, HDMI / SDI capture cards): macropixel U Y0 V Y1
// The arithmetic is BT.601 limited range in 20-bit fixed point, which equals cv2.cvtColor(COLOR_YUV2RGB_I420 /
// COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_YUYV / COLOR_YUV2RGB_UYVY) on every (Y, U, V) triple (tests/test_yuv_host.py,
// tests/test_yuv422_host.py and their GPU counterparts).  Integer only, so the result does not depend on the file's
// -fmad setting.
#pragma once
#include <stddef.h>
#include <stdint.h>

#define WB_FMT_RGB24 0
#define WB_FMT_YUV420P 1
#define WB_FMT_NV12 2
#define WB_FMT_YUYV422 3
#define WB_FMT_UYVY422 4
#define WB_FMT_BGR24 5
#define WB_FMT_RGBA 6  // also rgb0: the fourth byte is not read
#define WB_FMT_BGRA 7  // also bgr0

__host__ __device__ __forceinline__ bool fmt_422(int fmt) { return fmt == WB_FMT_YUYV422 || fmt == WB_FMT_UYVY422; }

// Packed RGB frames [h][w][bpp], one byte per channel, in any of four byte orders.  These facts are all that the
// detection path (resized_pixel_load) and the effects pass (k_fx_render) know about the orders; converting one to
// RGB24 is a byte permutation, so the kernels' results equal cv2.cvtColor(COLOR_BGR2RGB / RGBA2RGB / BGRA2RGB) of the
// frame exactly.
struct RgbLayout {
  int bpp;      // bytes per pixel
  int r, g, b;  // byte offsets of R, G and B within a pixel
};
__host__ __device__ __forceinline__ bool fmt_rgb(int fmt) {
  return fmt == WB_FMT_RGB24 || fmt == WB_FMT_BGR24 || fmt == WB_FMT_RGBA || fmt == WB_FMT_BGRA;
}
// the layout of a packed RGB format (fmt_rgb(fmt)); a constant where fmt is one
__host__ __device__ __forceinline__ constexpr RgbLayout rgb_layout(int fmt) {
  return fmt == WB_FMT_BGR24  ? RgbLayout{3, 2, 1, 0}
         : fmt == WB_FMT_RGBA ? RgbLayout{4, 0, 1, 2}
         : fmt == WB_FMT_BGRA ? RgbLayout{4, 2, 1, 0}
                              : RgbLayout{3, 0, 1, 2};
}

// the format's name, as ffmpeg's -pix_fmt and the Python layer spell it (for error messages)
inline const char* fmt_name(int fmt) {
  static const char* const names[] = {"rgb24", "yuv420p", "nv12", "yuyv422", "uyvy422", "bgr24", "rgba", "bgra"};
  return fmt >= 0 && fmt < 8 ? names[fmt] : "unknown";
}

struct ChromaLayout {
  int luma_step;  // bytes between horizontally adjacent Y samples: 1 (4:2:0 luma plane), 2 (4:2:2 macropixels)
  int step;       // bytes between horizontally adjacent U samples
  int row;        // bytes between chroma rows
  int row_shift;  // luma row y has chroma row y >> row_shift: 1 (4:2:0, one per two luma rows), 0 (4:2:2, one per row)
  ptrdiff_t v_off;  // V sample = U sample + v_off
};

// the layout of a YUV frame, or of a window of one, whose chroma rows are `row` bytes apart (4:2:2: the macropixel
// rows); v_off is only read for yuv420p, where it is the distance from the U plane to the V plane, of either sign
__host__ __device__ __forceinline__ ChromaLayout chroma_layout_of(int fmt, int row, ptrdiff_t v_off) {
  if (fmt_422(fmt)) return ChromaLayout{2, 4, row, 0, 2};
  if (fmt == WB_FMT_NV12) return ChromaLayout{1, 2, row, 1, 1};
  return ChromaLayout{1, 1, row, 1, v_off};
}

// the layout of a packed w x h frame
__host__ __device__ __forceinline__ ChromaLayout chroma_layout(int fmt, int w, int h) {
  return chroma_layout_of(fmt, fmt_422(fmt) ? 2 * w : fmt == WB_FMT_NV12 ? w : w / 2, (ptrdiff_t)(w / 2) * (h / 2));
}

// byte offsets, from the first byte of a packed w x h frame, of the Y and the U sample of pixel (0, 0)
__host__ __device__ __forceinline__ size_t luma_origin(int fmt) { return fmt == WB_FMT_UYVY422 ? 1 : 0; }
__host__ __device__ __forceinline__ size_t chroma_origin(int fmt, int w, int h) {
  return fmt == WB_FMT_YUYV422 ? 1 : fmt == WB_FMT_UYVY422 ? 0 : (size_t)w * h;
}

// bytes of one packed frame
__host__ __device__ __forceinline__ size_t frame_bytes(int fmt, int w, int h) {
  return fmt_rgb(fmt) ? (size_t)w * h * rgb_layout(fmt).bpp : fmt_422(fmt) ? (size_t)w * h * 2 : (size_t)w * h * 3 / 2;
}

// A frame as planes (wb_frame_planes): the RGB formats and 4:2:2 have one plane, the pixel rows; NV12 two, Y and the
// interleaved UV pairs; yuv420p three, Y, U and V.  A packed frame is its planes stored back to back, each with rows of
// plane_row_bytes, so plane k starts plane_offset(k) bytes after plane 0.
__host__ __device__ __forceinline__ int plane_count(int fmt) {
  return fmt == WB_FMT_YUV420P ? 3 : fmt == WB_FMT_NV12 ? 2 : 1;
}
__host__ __device__ __forceinline__ int plane_rows(int h, int k) { return k > 0 ? h / 2 : h; }
__host__ __device__ __forceinline__ size_t plane_row_bytes(int fmt, int w, int k) {
  return fmt_rgb(fmt) ? (size_t)w * rgb_layout(fmt).bpp : fmt_422(fmt) ? (size_t)w * 2
         : k == 0 || fmt == WB_FMT_NV12 ? (size_t)w : (size_t)(w / 2);
}
__host__ __device__ __forceinline__ size_t plane_offset(int fmt, int w, int h, int k) {
  size_t off = 0;
  for (int j = 0; j < k; ++j) off += plane_row_bytes(fmt, w, j) * plane_rows(h, j);
  return off;
}

// address of the U sample of pixel (x, y) given that of pixel (0, 0); the V sample is at + v_off.  A window of a frame
// (x0 even, and y0 even for 4:2:0) has its own origin `chroma` and keeps the parent frame's layout.  T: uint8_t or
// const uint8_t.
template <typename T>
__device__ __forceinline__ T* chroma_ptr(T* chroma, const ChromaLayout& cl, int x, int y) {
  return chroma + (size_t)(y >> cl.row_shift) * cl.row + (size_t)(x >> 1) * cl.step;
}

// Y, U, V bytes of pixel (x, y) of the frame whose luma rows start at `luma`, `pitch` bytes apart; yuv_to_rgb below
// converts them (two halves, so that a caller can have the loads of several pixels in flight before it converts any)
__device__ __forceinline__ void yuv_load(const uint8_t* __restrict__ luma, int pitch, const uint8_t* __restrict__ chroma,
                                         const ChromaLayout& cl, int x, int y, uint32_t& Y, uint32_t& U, uint32_t& V) {
  const uint8_t* c = chroma_ptr(chroma, cl, x, y);
  Y = __ldg(luma + (size_t)y * pitch + (size_t)x * cl.luma_step);
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
