/*
 * watsor_b200.h -- C-ABI of libwatsor_b200.so: the H100-native (sm_90a) detection hot path of
 * asmirnou/watsor behind plain pointers and sizes.  No torch / CUDA types appear in any signature;
 * device pointers and streams travel as void* / integers.
 *
 * Every entry point states the reference interface it replaces (paths relative to the watsor
 * repository, asmirnou/watsor @127f125).  The reference is pure Python, so "the FFI a maintainer
 * would bind" is ctypes: see INTEGRATION.md for the stub that goes into watsor/detection/.
 *
 * Conventions: every function returns 0 on success, non-zero on failure; wb_last_error() then
 * returns a message for the calling thread.  No C++ exception crosses this boundary (the reference
 * reports failures as Python exceptions raised inside the detector process,
 * watsor/detection/detector.py:86-100 -- the Python shim turns a non-zero status into one).
 */
#ifndef WATSOR_B200_H
#define WATSOR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WB_ABI_VERSION 1
#define WB_MAX_DETECTIONS 100 /* watsor/stream/share.py:31  ("detections", Detection * 100) */
#define WB_MAX_ZONES 10       /* watsor/stream/share.py:22  ('zones', c_int * 10)           */
#define WB_MAX_CAMERA_ZONES 32

/* Result ABI -- byte-identical to the ctypes structs of watsor/stream/share.py:11-24.
 * sizeof(wb_bounding_box) == 16, sizeof(wb_detection) == 72 (label @0, zones @4, confidence @48,
 * bounding_box @56).  wb_detect() writes straight into addressof(frame.header.detections). */
typedef struct wb_bounding_box {
  int32_t x_min, y_min, x_max, y_max;
} wb_bounding_box;

typedef struct wb_detection {
  int32_t label;
  int32_t zones[WB_MAX_ZONES];
  double confidence;
  wb_bounding_box bounding_box;
} wb_detection;

/* Verdict bits produced by the fused per-camera filter stage (one uint32 per detection row).
 * They restate the lazily evaluated predicate chain of watsor/filter/track.py:26
 * `d.label > 0 and all(f(d) for f in [ConfidenceFilter, AreaFilter, MaskFilter])`. */
#define WB_V_LABEL 1u      /* detection.label > 0                          track.py:26        */
#define WB_V_CONFIDENCE 2u /* watsor/filter/confidence.py:17-19                                 */
#define WB_V_AREA 4u       /* watsor/filter/area.py:20-26                                       */
#define WB_V_MASK 8u       /* watsor/filter/mask.py:44-59 (bit set when a mask is configured and hit) */
#define WB_V_PASS 16u      /* every configured predicate passed -> TrackFilter keeps the row    */

/* Per-label thresholds of one camera = one entry of the reference's camera_config['detect']
 * (watsor/config/schema.py:75-105): confidence/100, area/100*W*H, allowed zones. */
typedef struct wb_class_filter {
  int32_t label;         /* COCO index, watsor/config/coco.py:14-105                        */
  int32_t has_zone_list; /* 0: every zone of the mask counts (mask.py:36-37 `continue`)      */
  uint32_t zone_bits;    /* bit (z-1) set <=> zone z listed                                   */
  int32_t _pad;
  double confidence;     /* confidence.py:15  entry['confidence'] / 100                      */
  double area;           /* area.py:18        entry['area'] / 100 * max_area                 */
} wb_class_filter;

typedef struct wb_ctx wb_ctx;

/* ---- library / device ------------------------------------------------------------------------- */
int wb_abi_version(void);
const char* wb_last_error(void);
/* replaces the pycuda device probe of watsor/detection/devices.py:39-49 (cuda.init, Device.count) */
int wb_device_count(int* count);

/* ---- detector life cycle ---------------------------------------------------------------------- */
/* replaces TensorRTObjectDetector.__init__ / __enter__ (watsor/detection/tensorrt_gpu.py:23-57) and
 * TensorFlowObjectDetector.__init__ (tensorflow_cpu.py:13-25): builds the device-resident model from
 * a compiled model blob (watsor_b200/model.py writes it from frozen_inference_graph.pb / cpu.pb).
 * precision: 0 = fp32 storage, dense convs on CUDA cores (FFMA); 1 = bf16 storage, bf16 wgmma (fast mode, not
 * a parity mode); 2 = fp32 storage, dense convs as 3xTF32 wgmma MMAs with fp32 accumulation (fp32-faithful: the
 * default of the Python host and what bench.py reports); 3 = single TF32 MMA (diagnostic); 4 = fp16 storage, fp16
 * wgmma (fast mode with 11 significant bits, the analogue of TensorRT's FP16 flag; not a parity mode).
 * Precision 4's numerical policy: activations are stored as IEEE half, rounded to nearest even with subnormals kept,
 * after a clamp to +-65504, so an activation that overflows saturates at +-65504 and never becomes inf.  Tensor-core
 * weights are rounded to fp16 once, here; a model with a weight whose magnitude rounds beyond 65504 is refused, and
 * wb_last_error names the layer.  Accumulation, folded BatchNorm, bias and the heads stay fp32; the stem, depthwise
 * and CUDA-core GEMM weights stay fp32, as in precision 1. */
int wb_create(int device, const void* model_blob, size_t blob_bytes, int max_batch, int precision,
              wb_ctx** out);
/* replaces __exit__ (tensorrt_gpu.py:59-63) */
int wb_destroy(wb_ctx* ctx);
/* replaces the `device_name` property (tensorrt_gpu.py:53-57, tensorflow_cpu.py:64-66) */
int wb_device_name(wb_ctx* ctx, char* buf, size_t buf_bytes);
/* use an externally owned CUDA stream (e.g. torch.cuda.current_stream().cuda_stream); 0 = own */
int wb_set_stream(wb_ctx* ctx, uint64_t cuda_stream);
int wb_model_info(wb_ctx* ctx, int32_t* input_h, int32_t* input_w, int32_t* num_classes,
                  int32_t* num_anchors, int32_t* num_layers);

/* ---- per-camera filter state ------------------------------------------------------------------ */
/* replaces ConfidenceFilter.__init__ (confidence.py:10-15), AreaFilter.__init__ (area.py:10-18) and
 * MaskFilter.__init__ (mask.py:17-42).  zone_raster: n_zones filled-contour rasters, uint8
 * [n_zones][height][width] (1 = pixel belongs to the zone, zones already in mask.py:87 order), or
 * NULL when the camera has no mask.  The library builds the per-zone summed-area tables on the GPU.
 * A filter entry with label == -1 is the default for every label that has no entry of its own
 * (MaskFilter alone treats an unlisted label as "all zones", mask.py:50); without it an unlisted
 * label fails the confidence predicate (confidence.py:18 `confidence is not None`).
 * flags: WB_CAM_NO_LABEL_CHECK drops the `label > 0` test (a filter object called on its own). */
#define WB_CAM_NO_LABEL_CHECK 1u
int wb_set_camera(wb_ctx* ctx, int cam_id, int width, int height, int n_zones,
                  const uint8_t* zone_raster, int n_filters, const wb_class_filter* filters,
                  uint32_t flags);

/* Detection windows of a camera (no counterpart in the reference, whose frames are always squeezed whole into the
 * model's input).  xywh: n_windows rectangles (x, y, w, h) in the camera's pixels, each inside the frame set by
 * wb_set_camera; (0, 0, width, height) is the whole frame.  Every window of every frame of the camera becomes one model
 * image; max_batch counts model images.  A window's rows are those of the frame cropped to the window, shifted by
 * (x, y).  The rows of a frame's windows are then merged into its 100 rows (k_window_merge, DESIGN.md 4.4): sorted by
 * (confidence descending, window, row); a row is dropped when an already kept row of the same label from another
 * window covers more than merge_threshold (in [0, 1]) of the smaller of the two inclusive pixel boxes; the first 100
 * kept rows are filtered as the camera's rows always are.  In a batch with windows, a camera without any is one
 * full-frame window.  4:2:0 batches need even window origins and sizes, 4:2:2 batches an even x and width.
 * n_windows = 0 removes the windows;
 * wb_set_camera clears them. */
#define WB_MAX_WINDOWS 16
int wb_set_camera_windows(wb_ctx* ctx, int cam_id, int n_windows, const int32_t* xywh, double merge_threshold);

/* ---- the hot path ----------------------------------------------------------------------------- */
/* pin host frame memory (multiprocessing shared ctypes arrays, share.py:40) for async H2D */
int wb_register_host(wb_ctx* ctx, void* ptr, size_t bytes);
int wb_unregister_host(wb_ctx* ctx, void* ptr);

/* replaces ObjectDetector.detect (tensorflow_cpu.py:74-92 / tensorrt_gpu.py:65-91) for a batch:
 *   frames[i]   frame of camera cam_ids[i], host or device memory, packed (no row padding; wb_detect_planes below
 *               takes frames whose rows are padded or whose planes are separate buffers):
 *               uint8 RGB24 HWC [h][w][3] (share.py:68-73) by default; with WB_F_YUV420P or WB_F_NV12 a
 *               4:2:0 frame [h*3/2][w]: the luma plane [h][w], then the chroma ([h/2][w/2] U, then [h/2][w/2] V
 *               for yuv420p; [h/2][w/2] interleaved (U, V) pairs for NV12).  4:2:0 needs an even w and h; the
 *               conversion to RGB (BT.601 limited range) is fused into the resize and equals cv2.cvtColor's
 *               COLOR_YUV2RGB_I420 / COLOR_YUV2RGB_NV12 byte for byte, so the rows equal those of the RGB frame
 *               cvtColor makes.  With WB_F_YUYV422 or WB_F_UYVY422 a
 *               packed 4:2:2 frame [h][w][2]: each pixel pair (2k, 2k+1) of a row shares one macropixel, Y0 U Y1 V
 *               (YUYV) or U Y0 V Y1 (UYVY), and every row has its own chroma.  4:2:2 needs an even w (any h); its
 *               conversion equals COLOR_YUV2RGB_YUYV / COLOR_YUV2RGB_UYVY the same way.  With WB_F_BGR24 a
 *               BGR24 frame [h][w][3] (OpenCV's order: cv2.VideoCapture, cv2.imread); with WB_F_RGBA / WB_F_BGRA a
 *               4-byte frame [h][w][4], R G B A / B G R A (also rgb0 / bgr0: the fourth byte is not read).  These
 *               are read as the RGB24 frame cv2.cvtColor(COLOR_BGR2RGB / COLOR_RGBA2RGB / COLOR_BGRA2RGB) makes,
 *               so the rows equal that frame's; any size, any window.  The format is one per batch: at most one of
 *               the seven format flags.
 *   out[i]      Detection[100] block of that frame's header (share.py:27-32); all 100 rows written
 *   verdicts[i] optional uint32[100] filter verdicts (NULL to skip)
 *   flags       WB_F_* below
 *   gpu_ms      device time of the batch (CUDA events), the value `detect` returns (in ms)
 * Runs resize+normalise -> SSD convs -> heads -> decode -> per-class NMS -> top-100 ->
 * int conversion -> confidence/area/mask predicates, then copies results to `out`. */
#define WB_F_FRAMES_ON_DEVICE 1u /* frames[] are device pointers (no H2D)                        */
#define WB_F_FUSE_FILTERS 2u     /* also write zones[] of rows that pass (state after track.py:26) */
#define WB_F_OUT_ON_DEVICE 4u    /* out[]/verdicts[] are device pointers (no D2H)                 */
/* n counts frames; a batch whose cameras have detection windows (wb_set_camera_windows) runs one model image per
 * window and needs n_images <= max_batch */
#define WB_F_YUV420P 8u          /* frames[] are yuv420p (ffmpeg -pix_fmt yuv420p)                */
#define WB_F_NV12 16u            /* frames[] are NV12 (NVDEC's output, packed)                    */
#define WB_F_YUYV422 32u         /* frames[] are YUYV 4:2:2 (ffmpeg yuyv422: UVC webcams)         */
#define WB_F_UYVY422 64u         /* frames[] are UYVY 4:2:2 (ffmpeg uyvy422: HDMI / SDI capture)  */
#define WB_F_BGR24 128u          /* frames[] are BGR24 [h][w][3] (OpenCV, ffmpeg bgr24)           */
#define WB_F_RGBA 256u           /* frames[] are RGBA [h][w][4] (also rgb0; the A byte is ignored) */
#define WB_F_BGRA 512u           /* frames[] are BGRA [h][w][4] (also bgr0; the A byte is ignored) */
int wb_detect(wb_ctx* ctx, int n, const uint8_t* const* frames, const int32_t* cam_ids,
              uint32_t flags, wb_detection* const* out, uint32_t* const* verdicts, float* gpu_ms);

/* asynchronous form of wb_detect over slots 0..5 (stream + arena + staging each): submit() enqueues H2D +
 * kernels + D2H on the slot's stream and returns; collect() waits and scatters results.  Lets host ingest of
 * batch k+1 overlap the kernels of batch k (the reference overlaps them with processes, detector.py:40-50),
 * and several batches in flight are what keeps the GPU's SMs busy (DESIGN.md 4.5).  Thread-safe: a mutex in
 * the context serialises the calls that touch shared state. */
int wb_submit(wb_ctx* ctx, int slot, int n, const uint8_t* const* frames, const int32_t* cam_ids,
              uint32_t flags);
int wb_collect(wb_ctx* ctx, int slot, wb_detection* const* out, uint32_t* const* verdicts,
               float* gpu_ms);

/* Frames given as planes with row pitches: hardware decoder surfaces (NV12 whose pitch, and so the start of the chroma
 * plane, is rounded up to the decoder's alignment), ffmpeg AVFrames (data[i] / linesize[i]: yuv420p has three separate
 * buffers), capture buffers with bytesperline > 2w, and views of part of a larger frame.  Each plane holds the rows of
 * the packed layout above, pitch[k] bytes apart:
 *   RGB24, BGR24, RGBA, BGRA, YUYV, UYVY   plane[0]: the h pixel rows (bpp*w or 2w bytes each)
 *   NV12                                   plane[0]: h rows of w Y bytes; plane[1]: h/2 rows of w/2 (U, V) pairs
 *                                          (w bytes)
 *   yuv420p                                plane[0]: Y as for NV12; plane[1] U, plane[2] V: h/2 rows of w/2 bytes each,
 *                                          in any order in memory, with the same pitch
 * Planes the format does not use are NULL.  Every pitch is at least the plane's row bytes and below 2^31; bytes
 * between the end of a row and the next row are never read. */
typedef struct wb_frame_planes {
  const uint8_t* plane[3];
  int64_t pitch[3]; /* bytes between the starts of two rows of plane[k] */
} wb_frame_planes;
/* wb_detect / wb_submit on frames given as planes, with the same flags and wb_collect to collect wb_submit_planes.
 * Host frames (no WB_F_FRAMES_ON_DEVICE; pageable or wb_register_host-pinned) are packed into the slot's staging
 * buffer as they are uploaded, one cudaMemcpy2DAsync per plane.  Device frames are read in place: the kernels read the
 * caller's planes through their pitches, without a copy.  Either way the planes must stay valid until wb_collect has
 * returned.  A batch whose planes do not match its format (a plane missing or one too many, a pitch out of range,
 * yuv420p U and V pitches that differ, or an odd size where 4:2:0 or 4:2:2 needs it even) is refused with a message
 * naming the frame, the format and the value, and nothing is enqueued. */
int wb_detect_planes(wb_ctx* ctx, int n, const wb_frame_planes* frames, const int32_t* cam_ids, uint32_t flags,
                     wb_detection* const* out, uint32_t* const* verdicts, float* gpu_ms);
int wb_submit_planes(wb_ctx* ctx, int slot, int n, const wb_frame_planes* frames, const int32_t* cam_ids,
                     uint32_t flags);

/* order the library's internal slot streams against a caller stream (0 = legacy default stream):
 * direction 0: every slot stream waits for the work already enqueued on `cuda_stream`;
 * direction 1: `cuda_stream` waits for everything enqueued on the slot streams.
 * Lets a caller bracket several in-flight wb_submit() batches with its own CUDA events. */
int wb_stream_fence(wb_ctx* ctx, uint64_t cuda_stream, int direction);

/* ---- engine frame scatter (BASELINE.json north star: "NCCL over NVLink only for the engine's frame scatter";
 * SURVEY.md section 8(b)/(e)).  The reference has no counterpart: its detectors pull frames from one queue
 * (detector.py:40-50).  One rank (the ingest rank) owns a tick's frames of every camera and sends each rank its slab;
 * the detection kernels read the receive buffer in place (wb_submit with WB_F_FRAMES_ON_DEVICE).
 * NCCL is bound at run time -- the libnccl.so.2 already loaded in the process, else the file WB_NCCL_LIB names, else
 * the system one; the library has no link-time dependency on it and every other entry point works without it.
 *   wb_comm_unique_id : rank `root` makes the 128-byte rendezvous id; ship it to the other ranks over any host channel
 *   wb_comm_init      : collective over the `world` contexts (one per process / GPU)
 *   wb_scatter_frames : root: send_per_rank[r] = device pointer of rank r's slab (bytes_per_rank bytes each; the
 *                       root's own slab is a device copy); other ranks pass NULL.  recv = this rank's device buffer.
 *                       cuda_stream = 0: runs on the context's communication stream and every later wb_submit on
 *                       this context is ordered after it; otherwise it is enqueued on the caller's stream (order the
 *                       slots with wb_stream_fence).  The caller guarantees that nothing still reads `recv`. */
#define WB_COMM_ID_BYTES 128
int wb_comm_unique_id(uint8_t* id_out);
int wb_comm_init(wb_ctx* ctx, int rank, int world, const uint8_t* id);
int wb_scatter_frames(wb_ctx* ctx, int root, const uint8_t* const* send_per_rank, uint8_t* recv,
                      size_t bytes_per_rank, uint64_t cuda_stream);
int wb_comm_destroy(wb_ctx* ctx);

/* ---- visual effects of the output stage, SURVEY.md section 8 (f)4 -------------------------------------------------
 * One CUDA pass per batch of frames replaces the effect chain of watsor/main.py:302-312:
 *   CopyImageEffect (output/copy.py:14-18) or BlendEffect (output/blend.py:8-32), then DrawEffect (output/draw.py:9-88)
 *   or DrawEffectWithContours (draw.py:91-103).  Output bytes equal the reference's (numpy + OpenCV on the CPU).
 * The label text is cv2.putText's: the host builds per-glyph tables with the installed OpenCV
 * (watsor_b200/output/font.py) and the kernel applies them; zone outlines are cv2.drawContours rasters made once per
 * camera.  An effects context is independent of a detector context (the reference runs effects in their own process
 * per camera, output/video.py:10-35). */
typedef struct wb_fx wb_fx;
typedef struct wb_fx_font {
  int32_t n_glyphs;
  int32_t rows, cols, y0;         /* glyph window: cols x rows pixels, first row at org.y + y0, first column at the pen */
  int32_t text_height, baseline;  /* cv2.getTextSize(...) of FONT_HERSHEY_DUPLEX, scale 0.5, thickness 1   draw.py:56-59 */
  int32_t margin;                 /* int(round(ceil(0.1 * text_height)))                                    draw.py:62 */
  const int32_t* advance;         /* [n_glyphs] pen advance in half pixels */
  const uint8_t* lut;             /* [n_glyphs][2 phases][cols + 1 clip distances][rows][cols][256] */
} wb_fx_font;
typedef struct wb_fx_label {      /* drawing attributes of one label index (config/coco.py:110-121) */
  uint8_t box_color[3];
  uint8_t n_prefix;               /* "<label>: " as glyph indices */
  uint8_t prefix[60];
} wb_fx_label;
#define WB_FX_BLEND 1u     /* BlendEffect for cameras that have an alpha channel (else the image is copied) */
#define WB_FX_DRAW 2u      /* DrawEffect */
#define WB_FX_CONTOURS 4u  /* ... WithContours */
#define WB_FX_ON_DEVICE 8u /* images_in / images_out are device pointers */
#define WB_FX_YUV420P 16u  /* images_in are yuv420p [h*3/2][w] (layouts as for wb_detect); images_out stay RGB24 */
#define WB_FX_NV12 32u     /* images_in are NV12 [h*3/2][w] */
#define WB_FX_OUT_YUV420P 64u /* images_out are yuv420p [h*3/2][w], for an encoder that takes 4:2:0 */
#define WB_FX_OUT_NV12 128u   /* images_out are NV12 [h*3/2][w]; not with WB_FX_OUT_YUV420P */
#define WB_FX_YUYV422 256u    /* images_in are YUYV 4:2:2 [h][w][2] (layouts as for wb_detect) */
#define WB_FX_UYVY422 512u    /* images_in are UYVY 4:2:2 [h][w][2] */
#define WB_FX_BGR24 1024u     /* images_in are BGR24 [h][w][3] */
#define WB_FX_RGBA 2048u      /* images_in are RGBA [h][w][4] (also rgb0) */
#define WB_FX_BGRA 4096u      /* images_in are BGRA [h][w][4] (also bgr0); at most one input format flag is set */
#define WB_FX_OUT_BGR24 8192u /* images_out are BGR24 [h][w][3], for cv2.imencode; at most one output format flag */
/* labels[0] is also the style of unknown label indices (coco.py:124-131); digit_glyphs = glyph indices of '0'..'9','%';
 * alpha = opacity of the label box (coco.py:119) */
int wb_fx_create(int device, const wb_fx_font* font, int n_labels, const wb_fx_label* labels,
                 const uint8_t* digit_glyphs, double alpha, wb_fx** out);
/* alpha: [height][width] alpha channel of the mask image (filter/mask.py:71-81) or NULL; contour_bits: [height][width]
 * uint32, bit z-1 set where cv2.drawContours(contours, z-1, thickness=1) paints, or NULL */
int wb_fx_set_camera(wb_fx* fx, int cam_id, int width, int height, const uint8_t* alpha, const uint32_t* contour_bits);
/* rows[i]: the 100 Detection rows of frame i (host memory: header.detections).  images: RGB24, host pointers unless
 * WB_FX_ON_DEVICE.  With WB_FX_YUV420P / WB_FX_NV12 images_in are 4:2:0 (even width and height), converted as
 * cv2.cvtColor does; with WB_FX_YUYV422 / WB_FX_UYVY422 they are packed 4:2:2 (even width, any height),
 * converted the same way; with WB_FX_BGR24 / WB_FX_RGBA / WB_FX_BGRA they are BGR24 [h][w][3] or RGBA / BGRA
 * [h][w][4] (alpha ignored: the blend alpha is the camera's), read as cv2.cvtColor's RGB24 of them.  With
 * WB_FX_OUT_BGR24 images_out are BGR24, the rendered RGB24 frame with R and B swapped (cv2.cvtColor(COLOR_RGB2BGR)),
 * which cv2.imencode takes as it is.  With WB_FX_OUT_YUV420P / WB_FX_OUT_NV12 images_out are 4:2:0 (even width and height), the
 * rendered RGB24 frame converted as cv2.cvtColor(COLOR_RGB2YUV_I420) does (U and V of a 2x2 block from its top-left
 * pixel; NV12 = the same bytes with U and V interleaved); host output then moves w*h*3/2 bytes per frame.  Any input
 * format goes with any output format and every effect flag.  images_out[i] may be images_in[i] only when both are
 * RGB24 or BGR24 (the same pixel size, no YUV); otherwise it must be another buffer.  Without effect flags the call
 * is a pure format converter.  gpu_ms: kernels only. */
int wb_fx_render(wb_fx* fx, int n, const uint8_t* const* images_in, uint8_t* const* images_out, const int32_t* cam_ids,
                 const wb_detection* const* rows, uint32_t flags, float* gpu_ms);
int wb_fx_destroy(wb_fx* fx);
const char* wb_fx_last_error(void);

/* ---- stage-level entry points (parity tests call the same kernels stage by stage) -------------- */
/* graph nodes Cast + Preprocessor/... : out = float32 [n][in_h][in_w][3] on the host */
int wb_preprocess(wb_ctx* ctx, int n, const uint8_t* const* frames, const int32_t* widths,
                  const int32_t* heights, float* out);
/* FeatureExtractor/... + BoxPredictor_i: pre = float32 [n][in_h][in_w][3] (host);
 * enc = [n][anchors][4], logits = [n][anchors][classes+1] (host).  stop_layer >= 0 additionally
 * copies that layer's activation (float32 NHWC) to layer_out. */
int wb_backbone(wb_ctx* ctx, int n, const float* pre, float* enc, float* logits, int stop_layer,
                float* layer_out, size_t layer_out_floats);
/* the product path's own input handling (frames as wb_submit takes them: host or device, rgb24 / yuv420p / nv12 /
 * yuyv422 / uyvy422 / bgr24 / rgba / bgra,
 * a camera's detection windows expanded into model images), run to stop_layer; n_images = model images of the batch.
 * flags: one format flag (WB_F_YUV420P, WB_F_NV12, WB_F_YUYV422, WB_F_UYVY422, WB_F_BGR24, WB_F_RGBA, WB_F_BGRA),
 * WB_F_FRAMES_ON_DEVICE,
 * WB_F_FUSE_FILTERS.  Runs on slot 0.
 *   stop_layer >= 0: the layers up to stop_layer, eagerly; layer_out as for wb_backbone, for n_images images.
 *   stop_layer == -1: the kernels of wb_submit (CUDA graph, post stage, window merge).
 * enc / logits (optional): [n_images][anchors][4] / [n_images][anchors][classes+1] as the run left them -- unlike
 * wb_backbone, they are not cleared first; size them from the cameras' windows. */
int wb_backbone_frames(wb_ctx* ctx, int n, const uint8_t* const* frames, const int32_t* cam_ids, uint32_t flags,
                       float* enc, float* logits, int stop_layer, float* layer_out, size_t layer_out_floats,
                       int32_t* n_images);
/* Postprocessor/... + tensorflow_cpu.py:79-90 + filters, from given head outputs (host);
 * boxes/scores/classes (optional, host): the graph outputs detection_boxes[n][100][4],
 * detection_scores[n][100], detection_classes[n][100], num[n] before integer conversion */
int wb_postprocess(wb_ctx* ctx, int n, const float* enc, const float* logits,
                   const int32_t* cam_ids, uint32_t flags, wb_detection* const* out,
                   uint32_t* const* verdicts, float* boxes, float* scores, float* classes,
                   int32_t* num);
/* the predicate chain alone on caller-provided rows (replaces ConfidenceFilter/AreaFilter/
 * MaskFilter.__call__): rows are updated in place (zones), verdicts[n_rows] written */
int wb_filter_rows(wb_ctx* ctx, int cam_id, int n_rows, wb_detection* rows, uint32_t* verdicts);
/* anchors as the library generated them: float32 [anchors][4] (ymin,xmin,ymax,xmax) */
int wb_anchors(wb_ctx* ctx, float* out);

/* ---- host side of the filter stage (no GPU involved) ---------------------------------------------- */
/* TrackFilter's centroid tracker, watsor/filter/track.py:19-23 (sensitivity, history) and :29-149.
 * One tracker per camera, like the reference's one TrackFilter per camera (main.py:293-299). */
typedef struct wb_tracker wb_tracker;
int wb_tracker_create(int sensitivity, int history, wb_tracker** out);
int wb_tracker_destroy(wb_tracker* tracker);
/* One frame: rows that passed stage 1 of track.py:26 are those with WB_V_PASS in verdicts[i] (from
 * wb_detect / wb_filter_rows), or, when verdicts is NULL, those with label > 0 (TrackFilter without
 * predicates).  Writes the envelopes of the objects seen >= sensitivity times to out[0..*n_out) in the
 * reference's order and sets *suspicious_activity (track.py:39).  Returns 2 if out_cap was too small. */
int wb_tracker_update(wb_tracker* tracker, const wb_detection* rows, int n_rows, const uint32_t* verdicts,
                      wb_detection* out, int out_cap, int* n_out, int* suspicious_activity);
/* DetectionSieve._incoming_frame with filters == [TrackFilter] (watsor/filter/sieve.py:21-52): the frame's
 * rows are replaced in place by the tracker's result, the remainder is zero-filled. */
int wb_sieve_rows(wb_tracker* tracker, wb_detection* rows, int n_rows, const uint32_t* verdicts,
                  int* suspicious_activity);
/* test hook: iteration order of a CPython set after adding keys[0..n) (restated in tracker.cpp) */
int wb_debug_pyset_order(const int32_t* keys, int n, int32_t* out, int* n_out);
/* test hook: np.argsort(keys) (default kind) as restated in tracker.cpp */
int wb_debug_argsort(const int64_t* keys, int n, int32_t* out);
/* test hook: iteration order of set(range(n)).difference({i : used[i] != 0}) (track.py:90,98) */
int wb_debug_unused_order(int n, const uint8_t* used, int32_t* out, int* n_out);

/* ---- introspection used by bench.py ------------------------------------------------------------ */
/* number of kernel launches the last wb_detect/wb_submit issued, and per-layer device time of the
 * last profiled run (wb_profile_layers runs the program once with events around every launch) */
int wb_last_launch_count(wb_ctx* ctx, int* launches);
int wb_profile_layers(wb_ctx* ctx, int n, const uint8_t* const* device_frames,
                      const int32_t* cam_ids, float* ms_per_launch, int32_t* kinds, int max_launches,
                      int* n_launches);

#ifdef __cplusplus
}
#endif
#endif /* WATSOR_B200_H */
