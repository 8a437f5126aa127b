// kernels_fx.cu -- the reference's output-stage visual effects as one CUDA pass per batch of frames
// (SURVEY.md section 8 (f)4), behind the wb_fx_* entry points of include/watsor_b200.h:
//
//   CopyImageEffect            watsor/output/copy.py:14-18     image_out = image_in
//   BlendEffect                watsor/output/blend.py:8-32     image_out = u8(f32(image_in) * a/255 + 255 * (1 - a/255))
//   DrawEffect                 watsor/output/draw.py:9-88      per detection with label > 0, in row order:
//                                                              cv2.rectangle, the alpha-blended label box
//                                                              (cv2.addWeighted) and the label text (cv2.putText)
//   DrawEffectWithContours     watsor/output/draw.py:91-103    + the zone contours of the detections' zones
//
// Every byte equals what the reference computes with numpy / OpenCV on the CPU (tests/test_gpu_effects.py).  Where
// the arithmetic is OpenCV's, it is either restated after being pinned on all inputs (addWeighted: one fused
// multiply-add in float, round half to even) or taken over by construction as tables the host builds with the
// installed OpenCV (glyph tables: watsor_b200/output/font.py; contour pixels: cv2.drawContours on an empty raster).
// Compiled with the default -fmad=true: the float arithmetic that must not be contracted uses the _rn intrinsics.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/watsor_b200.h"
#include "host.cuh"
#include "yuv420.cuh"

namespace {

// wb_fx_last_error's message, kept apart from wb_last_error's
thread_local std::string g_fx_err;
int fail(const std::string& m) {
  g_fx_err = m;
  return 1;
}

constexpr int FX_MAX_GLYPHS = 48;  // "traffic light: 100%" is 19; prefix <= 40 + up to 7 digits + '%'

struct FxDet {                 // one drawable detection, computed by k_fx_prepare
  int32_t x0, y0, x1, y1;      // rectangle corners, min/max ordered (cv2.rectangle draws the same pixels either way)
  int32_t bx0, by0, bx1, by1;  // label box [bx0, bx1) x [by0, by1), clamped to the image; empty: no box and no text
  int32_t ox, oy;              // text origin (cv2.putText org)
  int32_t style;               // label style index
  int32_t n_glyphs;
  int32_t text_x1;             // one past the last column any glyph can touch
  uint8_t glyph[FX_MAX_GLYPHS];
  uint16_t pen2[FX_MAX_GLYPHS];  // pen offset from ox in half pixels
};

struct FxFrame {           // per frame, after k_fx_prepare
  int32_t n_active;        // detections with label > 0, in row order
  uint32_t zone_sel;       // bit z-1: some active detection lists zone z (draw.py:100-103)
  uint8_t order[WB_MAX_DETECTIONS];
  FxDet det[WB_MAX_DETECTIONS];
};

struct FxFont {  // device copies
  int32_t n_glyphs, rows, cols, y0, text_height, baseline, margin;
  const int32_t* advance;
  const uint8_t* lut;  // [n_glyphs][2][cols + 1][rows][cols][256]
};

struct FxLabel {
  uint8_t box_color[3];
  uint8_t n_prefix;
  uint8_t prefix[60];
};

struct FxCamera {
  int32_t w, h;
  const uint8_t* alpha;      // [h][w] or nullptr
  const uint32_t* contours;  // [h][w] or nullptr
};

// a camera of wb_fx_set_camera: the view the kernels receive, and the rasters it points to
struct FxCameraEntry {
  FxCamera view{};
  DevBuf<uint8_t> alpha;
  DevBuf<uint32_t> contours;
};

struct FxFrameDesc {
  const uint8_t* in;  // frame_bytes(fmt, w, h) bytes
  uint8_t* out;       // frame_bytes(out_fmt, w, h) bytes
  FxCamera cam;
  int32_t fmt;        // WB_FMT_* (yuv420.cuh) of `in`
  int32_t out_fmt;    // WB_FMT_* of `out`
};

// ---------------------------------------------------------------------------------------------------
// one block per frame, thread t = detection row t.  Restates the geometry of DrawEffect._draw (draw.py:51-88).
__global__ void __launch_bounds__(128)
    k_fx_prepare(const wb_detection* __restrict__ rows, const FxFrameDesc* __restrict__ frames, FxFont font,
                 const FxLabel* __restrict__ labels, int n_labels, const uint8_t* __restrict__ digit_glyphs,
                 FxFrame* __restrict__ out) {
  const int f = blockIdx.x, t = threadIdx.x;
  const int W = frames[f].cam.w, H = frames[f].cam.h;
  FxFrame& fr = out[f];
  __shared__ uint32_t s_zone;
  __shared__ uint32_t s_active[4];
  if (t == 0) s_zone = 0u;
  __syncthreads();
  bool active = false;
  if (t < WB_MAX_DETECTIONS) {
    const wb_detection d = rows[(size_t)f * WB_MAX_DETECTIONS + t];
    active = d.label > 0;  // draw.py:13 `filter(lambda d: d.label > 0, ...)`
    if (active) {
      FxDet& r = fr.det[t];
      const int left = d.bounding_box.x_min, top = d.bounding_box.y_min;
      const int right = d.bounding_box.x_max, bottom = d.bounding_box.y_max;
      r.x0 = min(left, right);
      r.x1 = max(left, right);
      r.y0 = min(top, bottom);
      r.y1 = max(top, bottom);
      const int style = d.label < n_labels ? d.label : 0;  // coco.py:124-131: unknown index -> 'unlabeled'
      r.style = style;
      // display_str = "{}: {}".format(label, "{0:.0%}".format(confidence))      draw.py:15
      const FxLabel lb = labels[style];
      int ng = 0, pen = 0;
      for (int i = 0; i < lb.n_prefix && ng < FX_MAX_GLYPHS; ++i) {
        r.glyph[ng] = lb.prefix[i];
        r.pen2[ng] = (uint16_t)pen;
        pen += font.advance[lb.prefix[i]];
        ++ng;
      }
      // '.0%': confidence * 100 rounded to the nearest integer, ties to even, on the double product (Python float
      // formatting is correctly rounded); confidences outside [0, 9999.99] have no counterpart in the detector's output
      const double pct = rint(d.confidence * 100.0);
      long long n = pct >= 0.0 && pct < 1.0e6 ? (long long)pct : 0;
      uint8_t digits[8];
      int nd = 0;
      do {
        digits[nd++] = (uint8_t)(n % 10);
        n /= 10;
      } while (n > 0 && nd < 8);
      for (int i = nd - 1; i >= 0 && ng < FX_MAX_GLYPHS; --i) {
        const uint8_t g = digit_glyphs[digits[i]];
        r.glyph[ng] = g;
        r.pen2[ng] = (uint16_t)pen;
        pen += font.advance[g];
        ++ng;
      }
      if (ng < FX_MAX_GLYPHS) {
        const uint8_t g = digit_glyphs[10];  // '%'
        r.glyph[ng] = g;
        r.pen2[ng] = (uint16_t)pen;
        pen += font.advance[g];
        ++ng;
      }
      r.n_glyphs = ng;
      // cv2.getTextSize: width = cvRound(sum(advance) * 0.5 + thickness), half to even      draw.py:55-59
      const int text_width = (int)rint((double)pen * 0.5 + 1.0);
      const int text_height = font.text_height, baseline = font.baseline, margin = font.margin;
      const int total = text_height + 2 * margin;  // draw.py:67
      int text_bottom;
      if (top - baseline > total)
        text_bottom = top;
      else if (bottom + total + baseline < H)
        text_bottom = bottom + total + baseline;
      else
        text_bottom = top + total + baseline;
      const int p1x = left, p1y = text_bottom - baseline - text_height - 2 * margin;  // draw.py:76-77
      const int p2x = left + text_width + 2 * margin, p2y = text_bottom;
      // image[p1y:p2y, p1x:p2x]: non-negative indices clamp to the image.  (Negative ones would wrap around in numpy;
      // the detector never produces them and such rows get no label here.)
      const bool valid = p1x >= 0 && p1y >= 0;
      r.bx0 = min(p1x, W);
      r.bx1 = min(p2x, W);
      r.by0 = min(p1y, H);
      r.by1 = min(p2y, H);
      if (!valid || r.by0 >= r.by1) {  // draw.py:80 `if len(cropped_image) == 0: return`
        r.bx0 = r.bx1 = r.by0 = r.by1 = 0;
        r.n_glyphs = 0;
      }
      r.ox = left + margin;  // draw.py:86-87
      r.oy = text_bottom - baseline - margin;
      r.text_x1 = r.ox + (pen >> 1) + font.cols;
      // draw.py:100-103: zones of the active detections select the contours to outline
      uint32_t z = 0;
      for (int i = 0; i < WB_MAX_ZONES; ++i)
        if (d.zones[i] > 0 && d.zones[i] <= 32) z |= 1u << (d.zones[i] - 1);
      if (z) atomicOr(&s_zone, z);
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, active);
  if ((t & 31) == 0) s_active[t >> 5] = m;
  __syncthreads();
  if (active) {
    int pos = __popc(m & ((1u << (t & 31)) - 1u));
    for (int w = 0; w < (t >> 5); ++w) pos += __popc(s_active[w]);
    fr.order[pos] = (uint8_t)t;
  }
  if (t == 0) {
    fr.n_active = __popc(s_active[0]) + __popc(s_active[1]) + __popc(s_active[2]) + __popc(s_active[3]);
    fr.zone_sel = s_zone;
  }
}

// ---------------------------------------------------------------------------------------------------
// grid (ceil(W / 128), ceil(H / 8), frames), 256 threads; thread = 4 consecutive pixels of one row.  (32-row tiles with
// four rows per thread and a quarter of the blocks measured 45 % slower: the pass is bound by the latency of dependent
// loads, and more resident threads hide it better than fewer culling preambles.)  For the same reason a thread issues
// the loads of its pixels, alpha values and outline bits first and only then takes part in building the tile's list of
// detections, so that the two chains of global round trips overlap.
constexpr int FX_TW = 128, FX_TH = 8;

// (forcing 32 registers for 8 blocks per SM instead of 5 spills and measured 8 % slower)
// YUV_OUT: the frames' out_fmt is yuv420p or NV12.  The RGB24 pass has an instantiation of its own because the 4:2:0
// store, as a run-time branch, made it 0.8 % slower.
// RGB_ORDERS: the input is BGR24, RGBA or BGRA, or the output is BGR24 (fx_rgb_orders).  Those byte orders have
// instantiations of their own for the same reason, so the <false, false> pass compiles to what it was without them.
template <bool YUV_OUT, bool RGB_ORDERS>
__global__ void __launch_bounds__(256, 5)
    k_fx_render(const FxFrameDesc* __restrict__ frames, const FxFrame* __restrict__ prep, FxFont font,
                const FxLabel* __restrict__ labels, const uint8_t* __restrict__ aw_lut, uint32_t flags) {
  __shared__ FxDet s_det[WB_MAX_DETECTIONS];
  __shared__ int s_n;
  __shared__ uint32_t s_hit[4];
  const FxFrameDesc fd = frames[blockIdx.z];
  const FxFrame& fr = prep[blockIdx.z];
  const int W = fd.cam.w, H = fd.cam.h;
  const int tx0 = blockIdx.x * FX_TW, ty0 = blockIdx.y * FX_TH;
  if (tx0 >= W || ty0 >= H) return;
  const int tx1 = min(tx0 + FX_TW, W), ty1 = min(ty0 + FX_TH, H);
  const int t = threadIdx.x;
  const int y = ty0 + t / (FX_TW / 4);
  const int xb = tx0 + (t % (FX_TW / 4)) * 4;
  const bool live = y < H && xb < W;  // threads outside the frame still take part in the barriers below
  const size_t row = (size_t)(live ? y : 0) * W;
  const int npx = live ? min(4, W - xb) : 0;
  const size_t px0 = row + (live ? xb : 0);
  const bool yuv = RGB_ORDERS ? !fmt_rgb(fd.fmt) : fd.fmt != WB_FMT_RGB24;
  // the packed RGB input's byte order (rgb_layout: G is byte 1 of every order, R and B bytes 0 and 2)
  const RgbLayout il = rgb_layout(RGB_ORDERS ? fd.fmt : WB_FMT_RGB24);
  const bool quad = RGB_ORDERS && !yuv && il.bpp == 4;  // RGBA / BGRA input
  const uint8_t* src = fd.in + px0 * (quad ? 4 : 3);  // RGB pixels (a YUV frame's samples are addressed below)
  const bool rgb_out = !YUV_OUT;
  uint8_t* dst = fd.out + px0 * (rgb_out ? 3 : 1);  // RGB24 / BGR24 pixels, or the luma of a 4:2:0 frame
  const bool blend = (flags & WB_FX_BLEND) && fd.cam.alpha != nullptr;
  const bool outline = (flags & WB_FX_CONTOURS) && fd.cam.contours != nullptr;
  // 3-byte loads and stores are whole words when every 4-pixel group of the thread's input and output is aligned
  const bool vec = npx == 4 && (((yuv || quad ? 0 : reinterpret_cast<uintptr_t>(src)) |
                                 (rgb_out ? reinterpret_cast<uintptr_t>(dst) : 0)) & 3) == 0;
  // 4-byte input: the 16 bytes of the thread's pixels are one uint4 when they are 16-byte aligned
  const bool vec4 = quad && npx == 4 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  // ---- loads first
  // RGB24 / BGR24: the 12 bytes; RGBA / BGRA: the 16 bytes; YUV: 4 Y bytes, then U and V of the 2 chroma samples
  uint32_t ws[RGB_ORDERS ? 4 : 3] = {0u, 0u, 0u};
  uint8_t v[4][3];
  uint8_t al[4] = {255, 255, 255, 255};
  uint32_t cb[4] = {0u, 0u, 0u, 0u};
  if (yuv) {
    // 4 pixels starting at a multiple of 4 in an even-width frame: exactly 2 chroma samples (4:2:2: two macropixels,
    // or one when the width is 2 mod 4).  4:2:2 and 4:2:0 branch apart so that each sees its layout as constants.
    auto load = [&](const ChromaLayout& cl, const uint8_t* luma, const uint8_t* chroma) {
      const uint8_t* c = chroma_ptr(chroma, cl, live ? xb : 0, live ? y : 0);
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (p < npx) ws[0] |= (uint32_t)__ldg(luma + (px0 + p) * cl.luma_step) << (8 * p);
#pragma unroll
      for (int q = 0; q < 2; ++q)
        if (2 * q < npx) {
          ws[1] |= (uint32_t)__ldg(c + q * cl.step) << (8 * q);
          ws[2] |= (uint32_t)__ldg(c + q * cl.step + cl.v_off) << (8 * q);
        }
    };
    if (fmt_422(fd.fmt)) {
      load(chroma_layout(WB_FMT_YUYV422, W, H), fd.in + luma_origin(fd.fmt), fd.in + chroma_origin(fd.fmt, W, H));
    } else {
      load(chroma_layout(fd.fmt == WB_FMT_NV12 ? WB_FMT_NV12 : WB_FMT_YUV420P, W, H), fd.in, fd.in + (size_t)W * H);
    }
  } else if (quad) {
    if (vec4) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(src));
      ws[0] = q.x;
      ws[1] = q.y;
      ws[2] = q.z;
      ws[RGB_ORDERS ? 3 : 0] = q.w;
    } else {
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (p < npx) {
#pragma unroll
          for (int c = 0; c < 3; ++c) v[p][c] = __ldg(src + p * 4 + c);
        }
    }
  } else if (vec) {
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
    ws[0] = __ldg(s32);
    ws[1] = __ldg(s32 + 1);
    ws[2] = __ldg(s32 + 2);
  } else {
#pragma unroll
    for (int p = 0; p < 4; ++p)
      if (p < npx) {
#pragma unroll
        for (int c = 0; c < 3; ++c) v[p][c] = __ldg(src + p * 3 + c);
      }
  }
  if (blend) {
    const uint8_t* ap = fd.cam.alpha + px0;
    if (npx == 4 && (reinterpret_cast<uintptr_t>(ap) & 3) == 0) {
      const uint32_t a4 = __ldg(reinterpret_cast<const uint32_t*>(ap));
#pragma unroll
      for (int p = 0; p < 4; ++p) al[p] = (uint8_t)(a4 >> (8 * p));
    } else {
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (p < npx) al[p] = __ldg(ap + p);
    }
  }
  if (outline) {
    const uint32_t* cp = fd.cam.contours + px0;
    if (npx == 4 && (reinterpret_cast<uintptr_t>(cp) & 15) == 0) {
      const uint4 c4 = __ldg(reinterpret_cast<const uint4*>(cp));
      cb[0] = c4.x;
      cb[1] = c4.y;
      cb[2] = c4.z;
      cb[3] = c4.w;
    } else {
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (p < npx) cb[p] = __ldg(cp + p);
    }
  }
  // ---- detections that can touch this tile, in row order
  int n_here = 0;
  uint32_t zone_sel = 0u;
  if (flags & WB_FX_DRAW) {
    const int na = fr.n_active;
    zone_sel = fr.zone_sel;
    if (na > 0) {  // uniform
      bool hit = false;
      int idx = 0;
      if (t < na) {
        idx = fr.order[t];
        const FxDet& d = fr.det[idx];
        // the tile holds outline pixels unless it misses the box or lies strictly inside it
        const bool rect = d.x0 < tx1 && d.x1 >= tx0 && d.y0 < ty1 && d.y1 >= ty0 &&
                          !(tx0 > d.x0 && tx1 - 1 < d.x1 && ty0 > d.y0 && ty1 - 1 < d.y1);
        const bool box = d.bx0 < tx1 && max(d.bx1, d.text_x1) > tx0 && d.by0 < ty1 && d.by1 > ty0 && d.by1 > d.by0;
        hit = rect || box;
      }
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (t < 128 && (t & 31) == 0) s_hit[t >> 5] = m;
      __syncthreads();
      if (hit) {
        int pos = __popc(m & ((1u << (t & 31)) - 1u));
        for (int w = 0; w < (t >> 5); ++w) pos += __popc(s_hit[w]);
        s_det[pos] = fr.det[idx];
      }
      if (t == 0) s_n = __popc(s_hit[0]) + __popc(s_hit[1]) + __popc(s_hit[2]) + __popc(s_hit[3]);
      __syncthreads();
      n_here = s_n;
    }
  }
  if (!live) return;
  if (yuv) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      uint32_t r, g, b;
      yuv_to_rgb((ws[0] >> (8 * p)) & 255u, (ws[1] >> (8 * (p >> 1))) & 255u, (ws[2] >> (8 * (p >> 1))) & 255u, r, g, b);
      v[p][0] = (uint8_t)r;
      v[p][1] = (uint8_t)g;
      v[p][2] = (uint8_t)b;
    }
  } else if (vec4) {
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int c = 0; c < 3; ++c) v[p][c] = (uint8_t)(ws[RGB_ORDERS ? p : 0] >> (8 * c));
  } else if (vec && !quad) {
#pragma unroll
    for (int i = 0; i < 12; ++i) v[i / 3][i % 3] = (uint8_t)(ws[i >> 2] >> (8 * (i & 3)));
  }
  // BGR24 / BGRA input: v holds bytes 0, 1, 2 of each pixel; R is byte 2
  if (RGB_ORDERS && !yuv && il.r == 2) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const uint8_t t = v[p][0];
      v[p][0] = v[p][2];
      v[p][2] = t;
    }
  }
  // CopyImageEffect / BlendEffect
  if (blend) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      if (p >= npx) continue;
      const float af = __fdiv_rn((float)al[p], 255.f);         // blend.py:15
      const float wi = __fmul_rn(255.f, __fsub_rn(1.f, af));   // blend.py:21-22
#pragma unroll
      for (int c = 0; c < 3; ++c)
        v[p][c] = (uint8_t)__float2int_rz(__fadd_rn(__fmul_rn((float)v[p][c], af), wi));  // blend.py:28-32
    }
  }
  // DrawEffect: detections in row order; within one detection rectangle, label box, text (draw.py:51-88)
  for (int i = 0; i < n_here; ++i) {
    const FxDet& d = s_det[i];
    const uint8_t* col = labels[d.style].box_color;
    const bool on_h = (y == d.y0 || y == d.y1);
    const bool in_y = y >= d.y0 && y <= d.y1;
    const bool box_y = y >= d.by0 && y < d.by1;
    const int gy = y - (d.oy + font.y0);
    const bool text_y = d.n_glyphs > 0 && gy >= 0 && gy < font.rows;
    if (!in_y && !box_y && !text_y) continue;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      if (p >= npx) continue;
      const int x = xb + p;
      if ((on_h && x >= d.x0 && x <= d.x1) || (in_y && (x == d.x0 || x == d.x1))) {  // cv2.rectangle, thickness 1
        v[p][0] = col[0];
        v[p][1] = col[1];
        v[p][2] = col[2];
      }
      if (box_y && x >= d.bx0 && x < d.bx1) {  // cv2.addWeighted(cropped, alpha, solid, 1 - alpha, 0)   draw.py:81-85
        const uint8_t* lut = aw_lut + (size_t)d.style * 768;
        v[p][0] = lut[v[p][0]];
        v[p][1] = lut[256 + v[p][1]];
        v[p][2] = lut[512 + v[p][2]];
      }
      if (text_y && x >= d.ox && x < d.text_x1) {  // cv2.putText, glyph after glyph                       draw.py:86-88
        for (int g = 0; g < d.n_glyphs; ++g) {
          const int pen2 = d.pen2[g];
          const int px = d.ox + (pen2 >> 1);
          const int gc = x - px;
          if (gc < 0) break;  // pens only move right
          if (gc >= font.cols) continue;
          const int k = W - px;  // distance from the pen to the right border: OpenCV clips the strokes there
          const int clip = min(k, font.cols + 1) - 1;
          const uint8_t* tab =
              font.lut + ((((size_t)(d.glyph[g] * 2 + (pen2 & 1)) * (font.cols + 1) + clip) * font.rows + gy) * font.cols + gc) * 256;
          v[p][0] = __ldg(tab + v[p][0]);
          v[p][1] = __ldg(tab + v[p][1]);
          v[p][2] = __ldg(tab + v[p][2]);
        }
      }
    }
  }
  // DrawEffectWithContours: outline every zone some drawn detection lies in (draw.py:100-103), colour (255, 255, 0)
  if (outline && zone_sel != 0u) {
#pragma unroll
    for (int p = 0; p < 4; ++p)
      if (p < npx && (cb[p] & zone_sel)) {
        v[p][0] = 255;
        v[p][1] = 255;
        v[p][2] = 0;
      }
  }
  // BGR24 output: the RGB24 result with R and B swapped, stored as RGB24 is
  if (RGB_ORDERS && rgb_out && rgb_layout(fd.out_fmt).r == 2) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const uint8_t t = v[p][0];
      v[p][0] = v[p][2];
      v[p][2] = t;
    }
  }
  if (!rgb_out) {
    // 4:2:0 as cv2.cvtColor(COLOR_RGB2YUV_I420) computes it: Y of every pixel; U and V of a 2x2 block from its top-left
    // pixel, which is pixel 0 or 2 of a thread on an even row, so each thread writes only what it holds
    uint32_t y4 = 0u, us[2], vs[2];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      uint32_t Y, U, V;
      rgb_to_yuv(v[p][0], v[p][1], v[p][2], Y, U, V);
      y4 |= Y << (8 * p);
      if ((p & 1) == 0) {
        us[p >> 1] = U;
        vs[p >> 1] = V;
      }
    }
    if (npx == 4 && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
      *reinterpret_cast<uint32_t*>(dst) = y4;
    } else {
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (p < npx) dst[p] = (uint8_t)(y4 >> (8 * p));
    }
    if ((y & 1) == 0) {
      // out_fmt is yuv420p or NV12: spelt out, so that the layout's 4:2:0 steps and shifts are constants here
      const ChromaLayout co = chroma_layout(fd.out_fmt == WB_FMT_NV12 ? WB_FMT_NV12 : WB_FMT_YUV420P, W, H);
      uint8_t* c = chroma_ptr(fd.out + (size_t)W * H, co, xb, y);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        if (2 * q >= npx) continue;  // npx == 2: one chroma sample
        uint8_t* cq = c + q * co.step;
        if (fd.out_fmt == WB_FMT_NV12 && (reinterpret_cast<uintptr_t>(cq) & 1) == 0) {
          *reinterpret_cast<uint16_t*>(cq) = (uint16_t)(us[q] | (vs[q] << 8));
        } else {
          cq[0] = (uint8_t)us[q];
          cq[co.v_off] = (uint8_t)vs[q];
        }
      }
    }
  } else if (vec) {
    uint32_t wo[3] = {0u, 0u, 0u};
#pragma unroll
    for (int i = 0; i < 12; ++i) wo[i >> 2] |= (uint32_t)v[i / 3][i % 3] << (8 * (i & 3));
    uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
    d32[0] = wo[0];
    d32[1] = wo[1];
    d32[2] = wo[2];
  } else {
#pragma unroll
    for (int p = 0; p < 4; ++p)
      if (p < npx) {
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[p * 3 + c] = v[p][c];
      }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
struct wb_fx {
  int device = 0;
  std::mutex mu;
  Stream stream;
  Event ev0, ev1;
  FxFont font{};
  DevBuf<int32_t> d_advance;
  DevBuf<uint8_t> d_lut;
  DevBuf<FxLabel> d_labels;
  int n_labels = 0;
  DevBuf<uint8_t> d_digits;
  DevBuf<uint8_t> d_aw;
  std::map<int, FxCameraEntry> cams;
  // staging
  int cap_n = 0;
  size_t cap_bytes = 0;
  DevBuf<uint8_t> d_in, d_out;
  DevBuf<wb_detection> d_rows;
  PinnedBuf<wb_detection> h_rows;
  DevBuf<FxFrameDesc> d_desc;
  PinnedBuf<FxFrameDesc> h_desc;
  DevBuf<FxFrame> d_prep;
};

const char* wb_fx_last_error(void) { return g_fx_err.c_str(); }

int wb_fx_create(int device, const wb_fx_font* font, int n_labels, const wb_fx_label* labels, const uint8_t* digit_glyphs,
                 double alpha, wb_fx** out) {
  REQUIRE(font && labels && digit_glyphs && out, "NULL argument");
  REQUIRE(font->n_glyphs > 0 && font->n_glyphs <= 128 && font->rows > 0 && font->cols > 0 && font->cols <= 64,
          "bad font geometry");
  REQUIRE(n_labels > 0 && n_labels <= 256, "n_labels must be in 1..256");
  for (int i = 0; i < n_labels; ++i) {
    REQUIRE(labels[i].n_prefix <= sizeof(labels[i].prefix), "label prefix too long");
    for (int j = 0; j < labels[i].n_prefix; ++j) REQUIRE(labels[i].prefix[j] < font->n_glyphs, "glyph index out of range");
  }
  for (int i = 0; i < 11; ++i) REQUIRE(digit_glyphs[i] < font->n_glyphs, "digit glyph index out of range");
  int count = 0;
  CK(cudaGetDeviceCount(&count));
  REQUIRE(device >= 0 && device < count, "no such CUDA device");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  const std::string unsupported = unsupported_device(prop);
  REQUIRE(unsupported.empty(), unsupported);
  std::unique_ptr<wb_fx> fx(new wb_fx());  // every REQUIRE / CK early return below releases what it holds
  fx->device = device;
  CK(create(fx->stream));
  CK(create(fx->ev0));
  CK(create(fx->ev1));
  const size_t lut_bytes = (size_t)font->n_glyphs * 2 * (font->cols + 1) * font->rows * font->cols * 256;
  CK(alloc(fx->d_advance, sizeof(int32_t) * font->n_glyphs));
  CK(alloc(fx->d_lut, lut_bytes));
  CK(cudaMemcpy(fx->d_advance, font->advance, sizeof(int32_t) * font->n_glyphs, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(fx->d_lut, font->lut, lut_bytes, cudaMemcpyHostToDevice));
  fx->font.n_glyphs = font->n_glyphs;
  fx->font.rows = font->rows;
  fx->font.cols = font->cols;
  fx->font.y0 = font->y0;
  fx->font.text_height = font->text_height;
  fx->font.baseline = font->baseline;
  fx->font.margin = font->margin;
  fx->font.advance = fx->d_advance;
  fx->font.lut = fx->d_lut;
  static_assert(sizeof(FxLabel) == sizeof(wb_fx_label), "label style layout");
  fx->n_labels = n_labels;
  CK(alloc(fx->d_labels, sizeof(FxLabel) * n_labels));
  CK(cudaMemcpy(fx->d_labels, labels, sizeof(FxLabel) * n_labels, cudaMemcpyHostToDevice));
  CK(alloc(fx->d_digits, 16));
  CK(cudaMemcpy(fx->d_digits, digit_glyphs, 11, cudaMemcpyHostToDevice));
  // cv2.addWeighted(src1, alpha, src2, beta = 1 - alpha, 0) on 8-bit images:  saturate(rint(fmaf(a, alpha, b * beta)))
  // in float -- pinned against OpenCV on all 256 x 256 inputs (tests/test_effects_host.py)
  std::vector<uint8_t> aw((size_t)n_labels * 768);
  const float fa = (float)alpha, fb = (float)(1.0 - alpha);
  for (int l = 0; l < n_labels; ++l)
    for (int c = 0; c < 3; ++c)
      for (int a = 0; a < 256; ++a) {
        const float t = (float)labels[l].box_color[c] * fb;
        const float r = nearbyintf(fmaf((float)a, fa, t));
        aw[(size_t)l * 768 + c * 256 + a] = (uint8_t)(r < 0.f ? 0.f : (r > 255.f ? 255.f : r));
      }
  CK(alloc(fx->d_aw, aw.size()));
  CK(cudaMemcpy(fx->d_aw, aw.data(), aw.size(), cudaMemcpyHostToDevice));
  *out = fx.release();
  return 0;
}

int wb_fx_set_camera(wb_fx* fx, int cam_id, int width, int height, const uint8_t* alpha, const uint32_t* contour_bits) {
  REQUIRE(fx, "NULL fx");
  REQUIRE(width > 0 && height > 0, "bad frame size");
  std::lock_guard<std::mutex> lock(fx->mu);
  CK(cudaSetDevice(fx->device));
  CK(cudaStreamSynchronize(fx->stream));
  FxCameraEntry cam;
  cam.view = FxCamera{width, height, nullptr, nullptr};
  const size_t px = (size_t)width * height;
  if (alpha) {
    CK(alloc(cam.alpha, px));
    CK(cudaMemcpy(cam.alpha, alpha, px, cudaMemcpyHostToDevice));
    cam.view.alpha = cam.alpha;
  }
  if (contour_bits) {
    CK(alloc(cam.contours, px * 4));
    CK(cudaMemcpy(cam.contours, contour_bits, px * 4, cudaMemcpyHostToDevice));
    cam.view.contours = cam.contours;
  }
  fx->cams[cam_id] = std::move(cam);  // an earlier configuration's rasters move to `cam`, which releases them
  return 0;
}

int wb_fx_render(wb_fx* fx, int n, const uint8_t* const* images_in, uint8_t* const* images_out, const int32_t* cam_ids,
                 const wb_detection* const* rows, uint32_t flags, float* gpu_ms) {
  REQUIRE(fx, "NULL fx");
  REQUIRE(n > 0 && n <= 4096, "n out of range");
  REQUIRE(images_in && images_out && cam_ids && rows, "NULL argument");
  std::lock_guard<std::mutex> lock(fx->mu);
  CK(cudaSetDevice(fx->device));
  const bool on_device = (flags & WB_FX_ON_DEVICE) != 0;
  static const FormatFlag in_formats[] = {{WB_FX_YUV420P, WB_FMT_YUV420P, "WB_FX_YUV420P"},
                                          {WB_FX_NV12, WB_FMT_NV12, "WB_FX_NV12"},
                                          {WB_FX_YUYV422, WB_FMT_YUYV422, "WB_FX_YUYV422"},
                                          {WB_FX_UYVY422, WB_FMT_UYVY422, "WB_FX_UYVY422"},
                                          {WB_FX_BGR24, WB_FMT_BGR24, "WB_FX_BGR24"},
                                          {WB_FX_RGBA, WB_FMT_RGBA, "WB_FX_RGBA"},
                                          {WB_FX_BGRA, WB_FMT_BGRA, "WB_FX_BGRA"}};
  static const FormatFlag out_formats[] = {{WB_FX_OUT_YUV420P, WB_FMT_YUV420P, "WB_FX_OUT_YUV420P"},
                                           {WB_FX_OUT_NV12, WB_FMT_NV12, "WB_FX_OUT_NV12"},
                                           {WB_FX_OUT_BGR24, WB_FMT_BGR24, "WB_FX_OUT_BGR24"}};
  std::string err;
  const int fmt = pixel_format(flags, in_formats, err);
  REQUIRE(fmt >= 0, err);
  const int out_fmt = pixel_format(flags, out_formats, err);
  REQUIRE(out_fmt >= 0, err);
  const bool yuv420 = fmt == WB_FMT_YUV420P || fmt == WB_FMT_NV12 || !fmt_rgb(out_fmt);
  // in place only between packed RGB layouts of one pixel size: a thread then writes exactly the bytes it read
  const bool in_place_ok = fmt_rgb(fmt) && fmt_rgb(out_fmt) && rgb_layout(fmt).bpp == rgb_layout(out_fmt).bpp;
  // the BGR24 / RGBA / BGRA passes are instantiations of their own (k_fx_render)
  const bool rgb_orders = (fmt_rgb(fmt) && fmt != WB_FMT_RGB24) || out_fmt == WB_FMT_BGR24;
  // host staging: one slot per frame, 256-byte aligned, of the RGB24 output's size or the input's if that is larger
  auto slot_bytes = [&](const FxCamera& cam) {
    return (std::max((size_t)cam.w * cam.h * 3, frame_bytes(fmt, cam.w, cam.h)) + 255) / 256 * 256;
  };
  size_t total = 0;
  int max_w = 0, max_h = 0;
  for (int i = 0; i < n; ++i) {
    auto it = fx->cams.find(cam_ids[i]);
    REQUIRE(it != fx->cams.end(), "cam_id " + std::to_string(cam_ids[i]) + " has not been configured with wb_fx_set_camera");
    REQUIRE(images_in[i] && images_out[i] && rows[i], "NULL frame / rows pointer");
    const FxCamera& cam = it->second.view;
    const std::string size = "cam_id " + std::to_string(cam_ids[i]) + " is " + std::to_string(cam.w) + "x" +
                             std::to_string(cam.h);
    REQUIRE(!yuv420 || (cam.w % 2 == 0 && cam.h % 2 == 0), size + ": 4:2:0 frames need an even width and height");
    REQUIRE(!fmt_422(fmt) || cam.w % 2 == 0, size + ": 4:2:2 frames need an even width");
    // in place, the stores of some threads would overwrite bytes that others still read
    REQUIRE(in_place_ok || images_in[i] != images_out[i],
            std::string(fmt_422(fmt)             ? "4:2:2 input"
                        : !fmt_rgb(fmt)          ? "4:2:0 input"
                        : !fmt_rgb(out_fmt)      ? "4:2:0 output"
                                                 : "input and output of different pixel sizes") +
                " cannot be rendered in place: images_out must be another buffer (cam_id " +
                std::to_string(cam_ids[i]) + ", " + fmt_name(fmt) + " input, " + fmt_name(out_fmt) + " output)");
    // labels are placed inside the frame only if it is high enough for one above/below/inside a box (draw.py:68-73);
    // lower frames would need OpenCV's re-capping of strokes cut by the bottom border, which the tables do not hold
    const int min_h = 2 * (fx->font.text_height + 2 * fx->font.margin + fx->font.baseline) + 1;
    REQUIRE(!(flags & WB_FX_DRAW) || cam.h >= min_h,
            "the draw effect needs frames of at least " + std::to_string(min_h) + " rows");
    total += slot_bytes(cam);
    max_w = std::max(max_w, cam.w);
    max_h = std::max(max_h, cam.h);
  }
  // staging that is too small is replaced once the stream is done with it; after a failed allocation the capacity is 0
  if (n > fx->cap_n) {
    CK(cudaStreamSynchronize(fx->stream));
    fx->cap_n = 0;
    CK(alloc(fx->d_rows, sizeof(wb_detection) * WB_MAX_DETECTIONS * n));
    CK(alloc(fx->d_desc, sizeof(FxFrameDesc) * n));
    CK(alloc(fx->d_prep, sizeof(FxFrame) * n));
    CK(alloc(fx->h_rows, sizeof(wb_detection) * WB_MAX_DETECTIONS * n));
    CK(alloc(fx->h_desc, sizeof(FxFrameDesc) * n));
    fx->cap_n = n;
  }
  if (!on_device && total > fx->cap_bytes) {
    CK(cudaStreamSynchronize(fx->stream));
    fx->cap_bytes = 0;
    CK(alloc(fx->d_in, total));
    CK(alloc(fx->d_out, total));
    fx->cap_bytes = total;
  }
  cudaStream_t st = fx->stream;
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    const FxCamera& cam = fx->cams[cam_ids[i]].view;
    memcpy(fx->h_rows + (size_t)i * WB_MAX_DETECTIONS, rows[i], sizeof(wb_detection) * WB_MAX_DETECTIONS);
    FxFrameDesc d;
    d.cam = cam;
    d.fmt = fmt;
    d.out_fmt = out_fmt;
    if (on_device) {
      d.in = images_in[i];
      d.out = images_out[i];
    } else {
      CK(cudaMemcpyAsync(fx->d_in + off, images_in[i], frame_bytes(fmt, cam.w, cam.h), cudaMemcpyHostToDevice, st));
      d.in = fx->d_in + off;
      d.out = fx->d_out + off;
    }
    fx->h_desc[i] = d;
    off += slot_bytes(cam);
  }
  CK(cudaMemcpyAsync(fx->d_rows, fx->h_rows, sizeof(wb_detection) * WB_MAX_DETECTIONS * n, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(fx->d_desc, fx->h_desc, sizeof(FxFrameDesc) * n, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(fx->ev0, st));
  if (flags & WB_FX_DRAW)
    k_fx_prepare<<<n, 128, 0, st>>>(fx->d_rows, fx->d_desc, fx->font, fx->d_labels, fx->n_labels, fx->d_digits, fx->d_prep);
  dim3 grid((max_w + FX_TW - 1) / FX_TW, (max_h + FX_TH - 1) / FX_TH, n);
  const bool yuv_out = !fmt_rgb(out_fmt);
  if (!rgb_orders && !yuv_out)
    k_fx_render<false, false><<<grid, 256, 0, st>>>(fx->d_desc, fx->d_prep, fx->font, fx->d_labels, fx->d_aw, flags);
  else if (!rgb_orders)
    k_fx_render<true, false><<<grid, 256, 0, st>>>(fx->d_desc, fx->d_prep, fx->font, fx->d_labels, fx->d_aw, flags);
  else if (!yuv_out)
    k_fx_render<false, true><<<grid, 256, 0, st>>>(fx->d_desc, fx->d_prep, fx->font, fx->d_labels, fx->d_aw, flags);
  else
    k_fx_render<true, true><<<grid, 256, 0, st>>>(fx->d_desc, fx->d_prep, fx->font, fx->d_labels, fx->d_aw, flags);
  CK(cudaGetLastError());
  CK(cudaEventRecord(fx->ev1, st));
  if (!on_device) {
    off = 0;
    for (int i = 0; i < n; ++i) {
      const FxCamera& cam = fx->cams[cam_ids[i]].view;
      CK(cudaMemcpyAsync(images_out[i], fx->d_out + off, frame_bytes(out_fmt, cam.w, cam.h), cudaMemcpyDeviceToHost, st));
      off += slot_bytes(cam);
    }
  }
  CK(cudaStreamSynchronize(st));
  if (gpu_ms) CK(cudaEventElapsedTime(gpu_ms, fx->ev0, fx->ev1));
  return 0;
}

int wb_fx_destroy(wb_fx* fx) {
  if (!fx) return 0;
  cudaSetDevice(fx->device);
  cudaStreamSynchronize(fx->stream);
  delete fx;  // releases the owned buffers, rasters, stream and events
  return 0;
}
