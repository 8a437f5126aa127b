// wb_api.cu -- the C-ABI of libwatsor_b200.so (include/watsor_b200.h): context, model upload,
// per-camera filter state, the layer-program executor, the asynchronous pipeline of WB_SLOTS slots and the
// stage-level entry points the parity tests use.
#include <dlfcn.h>
#include <nccl.h>  // types only: the functions are bound with dlopen in wb_comm_*

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "host.cuh"
#include "kernels_tc.cuh"

#define WB_MAX_CAMERAS 256
#define WB_SLOTS 6

static thread_local std::string g_err;
static int fail(const std::string& msg) {
  g_err = msg;
  return 1;
}

// The precision modes, indexed by wb_create's `precision` (include/watsor_b200.h).  Every precision-dependent choice of
// the executor reads the mode's row: the activation storage type and the tensor-core GEMMs' operand mode.
enum class Storage { F32, BF16, F16 };
struct PrecisionMode {
  const char* name;  // wb_device_name
  Storage storage;   // activations in the arena
  int tc_mode;       // TcMode of the dense layers that the tensor-core GEMM takes, or -1: CUDA cores only
};
static const PrecisionMode PRECISIONS[] = {
    {"fp32", Storage::F32, -1},
    {"bf16 wgmma", Storage::BF16, TC_BF16},
    {"fp32 3xTF32 wgmma", Storage::F32, TC_TF32X3},
    {"tf32 wgmma", Storage::F32, TC_TF32X1},
    {"fp16 wgmma", Storage::F16, TC_FP16},
};

struct Slot {
  Stream stream;
  Event ev0, ev1;
  PinnedBuf<FrameDesc> h_desc;
  DevBuf<FrameDesc> d_desc;
  DevBuf<uint8_t> d_frames;
  size_t d_frames_cap = 0;
  DevBuf<void> arena;
  DevBuf<float> d_enc, d_logits;
  DevBuf<float> d_partial;  // split-K scratch
  size_t partial_floats = 0;
  DevBuf<int> d_sel_count;
  DevBuf<int> d_kept_hist;  // [B][1024] per-frame histogram of kept scores (exact NMS early exit)
  DevBuf<unsigned long long> d_sel;  // [B][C][max_per_class] merge keys of the kept boxes
  DevBuf<float4> d_sel_box;          // ... and their decoded corners
  DevBuf<wb_detection> d_out;
  PinnedBuf<wb_detection> h_out;
  DevBuf<uint32_t> d_verdicts;
  PinnedBuf<uint32_t> h_verdicts;
  DevBuf<int> d_raw_num;  // valid rows per image: wb_postprocess's `num`, and k_window_merge's input
  // batches with detection windows: the frames' windows (copied before every launch) and their merged rows
  PinnedBuf<WindowFrame> h_win;
  DevBuf<WindowFrame> d_win;
  DevBuf<wb_detection> d_wout;
  DevBuf<uint32_t> d_wverd;
  int n = 0;         // frames of the batch in flight
  bool windowed = false;
  uint32_t flags = 0;
  bool busy = false;
  int launches = 0;
  // CUDA graph of the kernel sequence, keyed by (model images, flags, frames, windowed)
  GraphExec graph_exec;
  int graph_n = -1;
  int graph_frames = -1;
  bool graph_windowed = false;
  uint32_t graph_flags = 0;
};

struct wb_ctx {
  int device = 0;
  int max_batch = 0;
  int precision = 0;  // index into PRECISIONS
  // path switches (INTEGRATION.md §4), read from the environment once, in wb_create: an engine keeps the paths it was
  // created with, and routes to the tensor cores exactly the layers whose weights it prepared for them
  struct {
    bool graph, fuse_dwpw, fuse_add, tc_conv, split_k;
  } sw;
  // frame scatter (wb_comm_*): NCCL communicator bound at run time, its stream and the event the slots wait on
  void* comm = nullptr;
  int comm_rank = -1, comm_world = 0;
  Stream comm_stream;
  Event comm_ev;
  cudaDeviceProp prop;
  wb_model_header hdr;
  std::vector<wb_layer> layers;
  std::vector<wb_tensor_entry> tensors;
  DevBuf<float> d_weights;
  // the GEMM weights in the tensor cores' operand format (modes with a tc_mode).  Declared before `slots`, so the slots'
  // graph execs, whose kernels read these weights, are released first.
  TcWeights tc;
  PostParams pp;
  DevBuf<CameraCfg> d_cams;
  std::vector<CameraCfg> h_cams;
  DevBuf<int32_t> cam_sat[WB_MAX_CAMERAS];
  std::vector<std::vector<int4>> cam_windows;  // wb_set_camera_windows: (x, y, w, h) per window
  std::vector<double> cam_merge_thr;
  Slot slots[WB_SLOTS];
  cudaStream_t user_stream = nullptr;
  bool has_user_stream = false;
  int last_launches = 0;
  std::vector<void*> registered;
  // One lock for everything that touches shared per-context state: the camera table (h_cams / d_cams / SATs), slot 0's
  // staging buffers used by the stage-level calls, the filter staging buffers and the registration list.  The
  // reference runs one DetectionSieve thread per camera in one process (ref: watsor/main.py:378-384) and ctypes drops
  // the GIL, so wb_filter_rows / wb_set_camera DO get called concurrently.  Held for the host-side enqueue only,
  // except in the synchronous calls (filter_rows, set_camera, stage-level test hooks), which hold it until their
  // results are back.
  std::mutex mu;
  // wb_filter_rows: its own stream and staging buffers (never slot 0's: a detector batch may be in flight there)
  Stream fstream;
  DevBuf<wb_detection> d_frows;
  DevBuf<uint32_t> d_fverd;
  int frows_cap = 0;
  // read by the stage hooks only, which run on slot 0: wb_backbone's pre-processed input and wb_postprocess's float
  // outputs, boxes[n][100][4] scores[n][100] classes[n][100] and the valid rows per image
  DevBuf<float> d_pre;
  DevBuf<float> d_raw;
  PinnedBuf<float> h_raw;
  PinnedBuf<int> h_raw_num;

  const float* tensor(int idx) const { return d_weights + tensors[idx].offset; }
  const PrecisionMode& mode() const { return PRECISIONS[precision]; }
  size_t elem_size() const { return mode().storage == Storage::F32 ? 4 : 2; }
  cudaStream_t stream_of(int s) { return has_user_stream ? user_stream : slots[s].stream; }
  // whether layer L runs on the tensor-core GEMM
  bool tc_runs(const wb_layer& L) const { return mode().tc_mode >= 0 && tc_layer_supported(L, tc.mode, sw.tc_conv); }
};

extern "C" {

int wb_abi_version(void) { return WB_ABI_VERSION; }
const char* wb_last_error(void) { return g_err.c_str(); }

int wb_device_count(int* count) {
  REQUIRE(count != nullptr, "count is NULL");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    cudaGetLastError();
    n = 0;
  }
  *count = n;
  return 0;
}

static int alloc_slot(wb_ctx* c, Slot& s) {
  const int B = c->max_batch, N = c->hdr.num_anchors, C = c->hdr.num_classes, MP = c->hdr.max_per_class;
  CK(create(s.stream));
  CK(create(s.ev0));
  CK(create(s.ev1));
  CK(alloc(s.h_desc, sizeof(FrameDesc) * B));
  CK(alloc(s.d_desc, sizeof(FrameDesc) * B));
  CK(alloc(s.arena, (size_t)B * c->hdr.arena_elems * c->elem_size() + 1024));
  CK(alloc(s.d_enc, sizeof(float) * (size_t)B * N * 4));
  CK(alloc(s.d_logits, sizeof(float) * (size_t)B * N * (C + 1)));
  s.partial_floats = (size_t)4 * 1024 * 1024 + (size_t)B * 512 * 1024;
  CK(alloc(s.d_partial, sizeof(float) * s.partial_floats));
  CK(alloc(s.d_sel_count, sizeof(int) * (size_t)B * C));
  CK(alloc(s.d_kept_hist, sizeof(int) * (size_t)B * 1024));
  CK(alloc(s.d_sel, sizeof(unsigned long long) * (size_t)B * C * MP));
  CK(alloc(s.d_sel_box, sizeof(float4) * (size_t)B * C * MP));
  CK(alloc(s.d_out, sizeof(wb_detection) * (size_t)B * WB_MAX_DETECTIONS));
  CK(alloc(s.h_out, sizeof(wb_detection) * (size_t)B * WB_MAX_DETECTIONS));
  CK(alloc(s.d_verdicts, sizeof(uint32_t) * (size_t)B * WB_MAX_DETECTIONS));
  CK(alloc(s.h_verdicts, sizeof(uint32_t) * (size_t)B * WB_MAX_DETECTIONS));
  CK(alloc(s.d_raw_num, sizeof(int) * B));
  CK(alloc(s.h_win, sizeof(WindowFrame) * B));
  CK(alloc(s.d_win, sizeof(WindowFrame) * B));
  CK(alloc(s.d_wout, sizeof(wb_detection) * (size_t)B * WB_MAX_DETECTIONS));
  CK(cudaMemset(s.d_wout, 0, sizeof(wb_detection) * (size_t)B * WB_MAX_DETECTIONS));
  CK(alloc(s.d_wverd, sizeof(uint32_t) * (size_t)B * WB_MAX_DETECTIONS));
  return 0;
}

int wb_create(int device, const void* model_blob, size_t blob_bytes, int max_batch, int precision,
              wb_ctx** out) {
  REQUIRE(out != nullptr && model_blob != nullptr, "NULL argument");
  REQUIRE(blob_bytes >= sizeof(wb_model_header), "model blob too small");
  REQUIRE(max_batch >= 1 && max_batch <= 4096, "max_batch out of range");
  REQUIRE(precision >= 0 && precision < (int)std::size(PRECISIONS),
          "precision must be 0 (fp32 CUDA cores), 1 (bf16 wgmma), 2 (fp32 via 3xTF32 wgmma), 3 (1xTF32, diagnostic) or "
          "4 (fp16 wgmma)");
  CK(cudaSetDevice(device));
  struct CtxFree {
    void operator()(wb_ctx* p) const { wb_destroy(p); }
  };
  std::unique_ptr<wb_ctx, CtxFree> guard(new wb_ctx());  // every REQUIRE / CK early return below frees it
  wb_ctx* c = guard.get();
  c->device = device;
  c->max_batch = max_batch;
  c->precision = precision;
  const char* no_graph = getenv("WB_NO_GRAPH");
  c->sw.graph = !(no_graph && no_graph[0] == '1');
  c->sw.fuse_dwpw = getenv("WB_NO_FUSE") == nullptr;
  c->sw.fuse_add = getenv("WB_NO_FUSE_ADD") == nullptr;
  c->sw.tc_conv = getenv("WB_NO_TC_CONV") == nullptr;
  c->sw.split_k = getenv("WB_NO_SPLITK") == nullptr;
  CK(cudaGetDeviceProperties(&c->prop, device));
  const std::string unsupported = unsupported_device(c->prop);
  REQUIRE(unsupported.empty(), unsupported);
  memcpy(&c->hdr, model_blob, sizeof(wb_model_header));
  REQUIRE(memcmp(c->hdr.magic, WB_MODEL_MAGIC, 8) == 0, "bad model blob magic");
  const uint8_t* p = static_cast<const uint8_t*>(model_blob) + sizeof(wb_model_header);
  size_t need = sizeof(wb_model_header) + (size_t)c->hdr.n_layers * sizeof(wb_layer) +
                (size_t)c->hdr.n_tensors * sizeof(wb_tensor_entry);
  REQUIRE(blob_bytes >= need, "model blob truncated (tables)");
  c->layers.resize(c->hdr.n_layers);
  memcpy(c->layers.data(), p, c->layers.size() * sizeof(wb_layer));
  p += c->layers.size() * sizeof(wb_layer);
  c->tensors.resize(c->hdr.n_tensors);
  memcpy(c->tensors.data(), p, c->tensors.size() * sizeof(wb_tensor_entry));
  p += c->tensors.size() * sizeof(wb_tensor_entry);
  size_t floats = 0;
  for (auto& t : c->tensors) floats = std::max<size_t>(floats, t.offset + ((t.count + 63) / 64) * 64);
  REQUIRE(blob_bytes >= need + floats * sizeof(float), "model blob truncated (data)");
  REQUIRE(c->hdr.num_classes >= 1 && c->hdr.num_classes <= WB_MAX_LABELS, "num_classes must be in 1..128");
  REQUIRE(c->hdr.max_per_class >= 1 && c->hdr.max_per_class <= 128, "max_per_class must be in 1..128");
  REQUIRE(c->hdr.max_total >= 1 && c->hdr.max_total <= 128, "max_total must be in 1..128");
  REQUIRE(c->hdr.score_thr >= 0.f, "negative score threshold is not supported");
  REQUIRE(c->hdr.iou_thr >= 0.f, "negative IoU threshold is not supported");
  REQUIRE(c->hdr.num_anchors >= 1 && c->hdr.num_anchors <= 8192, "num_anchors must be in 1..8192 (NMS sort buffers live in shared memory)");
  for (auto& L : c->layers) {
    if (L.op == WB_OP_PW || L.op == WB_OP_HEAD)
      REQUIRE(L.in_c % 4 == 0, std::string("layer ") + L.name + ": in_c must be a multiple of 4");
    if (L.op == WB_OP_CONV)
      REQUIRE(L.in_c % 16 == 0, std::string("layer ") + L.name + ": KxK convs need in_c to be a multiple of 16");
    if (L.op == WB_OP_DW)
      REQUIRE(L.out_c % 4 == 0 && L.kh == 3 && L.kw == 3 && (L.stride == 1 || L.stride == 2),
              "depthwise must be 3x3 with stride 1 or 2, C%4==0");
    if (L.op == WB_OP_PW || L.op == WB_OP_CONV) REQUIRE(L.out_c % 4 == 0, "out_c must be a multiple of 4");
    if (L.op == WB_OP_MAXPOOL || L.op == WB_OP_AVGPOOL)
      REQUIRE(L.out_c % 4 == 0 && L.in_c == L.out_c && L.kh >= 1 && L.kw >= 1, "pooling needs C % 4 == 0");
    if (L.op == WB_OP_COPY)
      REQUIRE(L.in_c % 4 == 0 && L.out_c % 4 == 0 && L.row_off % 4 == 0 && L.row_off + L.in_c <= L.out_c,
              "channel copy: slice must be 4-aligned and inside the destination");
    REQUIRE(L.op >= WB_OP_STEM && L.op <= WB_OP_COPY, std::string("layer ") + L.name + ": unknown op");
  }
  CK(alloc(c->d_weights, floats * sizeof(float)));
  CK(cudaMemcpy(c->d_weights, p, floats * sizeof(float), cudaMemcpyHostToDevice));
  if (c->mode().tc_mode >= 0) {
    std::string err;
    if (tc_prepare_weights(c->layers, c->tensors, reinterpret_cast<const float*>(p), c->mode().tc_mode, c->sw.tc_conv,
                           &c->tc, &err))
      return fail("tensor-core weight preparation: " + err);
  }
  c->pp.num_anchors = c->hdr.num_anchors;
  c->pp.num_classes = c->hdr.num_classes;
  c->pp.scale_y = c->hdr.scale_y;
  c->pp.scale_x = c->hdr.scale_x;
  c->pp.scale_h = c->hdr.scale_h;
  c->pp.scale_w = c->hdr.scale_w;
  c->pp.logit_scale = c->hdr.logit_scale;
  c->pp.iou_thr = c->hdr.iou_thr;
  c->pp.score_thr = c->hdr.score_thr;
  c->pp.max_per_class = c->hdr.max_per_class;
  c->pp.max_total = c->hdr.max_total;
  c->pp.class_offset = c->hdr.class_offset;
  c->h_cams.assign(WB_MAX_CAMERAS, CameraCfg{});
  c->cam_windows.assign(WB_MAX_CAMERAS, {});
  c->cam_merge_thr.assign(WB_MAX_CAMERAS, 0.5);
  CK(alloc(c->d_cams, sizeof(CameraCfg) * WB_MAX_CAMERAS));
  CK(cudaMemset(c->d_cams, 0, sizeof(CameraCfg) * WB_MAX_CAMERAS));
  for (int s = 0; s < WB_SLOTS; ++s)
    if (alloc_slot(c, c->slots[s])) return 1;
  c->frows_cap = WB_MAX_DETECTIONS * max_batch;
  CK(create(c->fstream));
  CK(alloc(c->d_frows, sizeof(wb_detection) * (size_t)c->frows_cap));
  CK(alloc(c->d_fverd, sizeof(uint32_t) * (size_t)c->frows_cap));
  CK(alloc(c->d_pre, sizeof(float) * (size_t)max_batch * c->hdr.input_h * c->hdr.input_w * 3));
  CK(alloc(c->d_raw, sizeof(float) * (size_t)max_batch * WB_MAX_DETECTIONS * 6));
  CK(alloc(c->h_raw, sizeof(float) * (size_t)max_batch * WB_MAX_DETECTIONS * 6));
  CK(alloc(c->h_raw_num, sizeof(int) * max_batch));
  CK(cudaDeviceSynchronize());
  *out = guard.release();
  return 0;
}

int wb_destroy(wb_ctx* c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  wb_comm_destroy(c);
  for (void* r : c->registered) cudaHostUnregister(r);
  delete c;  // releases the owned buffers, streams, events and graph execs
  return 0;
}

int wb_device_name(wb_ctx* c, char* buf, size_t n) {
  REQUIRE(c && buf && n > 0, "NULL argument");
  snprintf(buf, n, "%s (cuda:%d, sm_%d%d, %s)", c->prop.name, c->device, c->prop.major, c->prop.minor,
           c->mode().name);
  return 0;
}

int wb_set_stream(wb_ctx* c, uint64_t stream) {
  REQUIRE(c, "NULL ctx");
  c->user_stream = reinterpret_cast<cudaStream_t>(stream);
  c->has_user_stream = stream != 0;
  for (auto& s : c->slots) s.graph_n = -1;  // graphs are stream-agnostic, but keep it simple
  return 0;
}

int wb_model_info(wb_ctx* c, int32_t* ih, int32_t* iw, int32_t* nc, int32_t* na, int32_t* nl) {
  REQUIRE(c, "NULL ctx");
  if (ih) *ih = c->hdr.input_h;
  if (iw) *iw = c->hdr.input_w;
  if (nc) *nc = c->hdr.num_classes;
  if (na) *na = c->hdr.num_anchors;
  if (nl) *nl = c->hdr.n_layers;
  return 0;
}

int wb_anchors(wb_ctx* c, float* out) {
  REQUIRE(c && out, "NULL argument");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpy(out, c->tensor(c->hdr.anchors_tensor), sizeof(float) * 4 * c->hdr.num_anchors,
                cudaMemcpyDeviceToHost));
  return 0;
}

int wb_set_camera(wb_ctx* c, int cam, int width, int height, int n_zones, const uint8_t* raster, int n_filters,
                  const wb_class_filter* filters, uint32_t cam_flags) {
  REQUIRE(c, "NULL ctx");
  REQUIRE(cam >= 0 && cam < WB_MAX_CAMERAS, "cam_id out of range (0..255)");
  REQUIRE(width > 0 && height > 0, "bad frame size");
  REQUIRE(n_zones >= 0 && n_zones <= WB_MAX_CAMERA_ZONES, "a mask may hold at most 32 zones");
  REQUIRE(n_zones == 0 || raster != nullptr, "zone_raster is NULL");
  REQUIRE(n_filters == 0 || filters != nullptr, "filters is NULL");
  std::lock_guard<std::mutex> lock(c->mu);
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());  // no batch may be reading the table while it changes
  CameraCfg cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.width = width;
  cfg.height = height;
  cfg.n_zones = n_zones;
  cfg.has_mask = raster != nullptr ? 1 : 0;
  cfg.check_label = (cam_flags & WB_CAM_NO_LABEL_CHECK) ? 0 : 1;
  for (int i = 0; i < n_filters; ++i) {
    const wb_class_filter& f = filters[i];
    if (f.label == -1) {
      cfg.default_present = 1;
      cfg.default_conf = f.confidence;
      cfg.default_area = f.area;
      cfg.default_has_zone_list = f.has_zone_list ? 1 : 0;
      cfg.default_zone_bits = f.zone_bits;
      continue;
    }
    REQUIRE(f.label >= 0 && f.label < WB_MAX_LABELS, "filter label out of range (0..127)");
    cfg.present[f.label] = 1;
    cfg.conf[f.label] = f.confidence;
    cfg.area[f.label] = f.area;
    cfg.has_zone_list[f.label] = f.has_zone_list ? 1 : 0;
    cfg.zone_bits[f.label] = f.zone_bits;
  }
  CK(c->cam_sat[cam].reset());
  if (n_zones > 0) {
    size_t sat_elems = (size_t)n_zones * (height + 1) * (width + 1);
    CK(alloc(c->cam_sat[cam], sat_elems * sizeof(int32_t)));
    DevBuf<uint8_t> d_r;
    size_t rb = (size_t)n_zones * height * width;
    CK(alloc(d_r, rb));
    CK(cudaMemcpy(d_r, raster, rb, cudaMemcpyHostToDevice));
    int lcnt = 0;
    LaunchCtx lc{c->slots[0].stream, &lcnt};
    launch_build_sat(lc, d_r, n_zones, height, width, c->cam_sat[cam]);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c->slots[0].stream));
    cfg.sat = c->cam_sat[cam];
  }
  c->h_cams[cam] = cfg;
  c->cam_windows[cam].clear();  // they were checked against the previous frame size
  CK(cudaMemcpy(c->d_cams + cam, &cfg, sizeof(cfg), cudaMemcpyHostToDevice));
  return 0;
}

int wb_set_camera_windows(wb_ctx* c, int cam, int n_windows, const int32_t* xywh, double merge_threshold) {
  REQUIRE(c, "NULL ctx");
  REQUIRE(cam >= 0 && cam < WB_MAX_CAMERAS, "cam_id out of range (0..255)");
  REQUIRE(n_windows >= 0 && n_windows <= WB_MAX_WINDOWS, "a camera may have at most 16 detection windows");
  REQUIRE(n_windows == 0 || xywh != nullptr, "xywh is NULL");
  REQUIRE(merge_threshold >= 0.0 && merge_threshold <= 1.0, "merge_threshold must be in [0, 1]");
  std::lock_guard<std::mutex> lock(c->mu);
  const CameraCfg& cc = c->h_cams[cam];
  REQUIRE(cc.width > 0, "cam_id " + std::to_string(cam) + " has not been configured with wb_set_camera");
  std::vector<int4> wins(n_windows);
  for (int i = 0; i < n_windows; ++i) {
    const int x = xywh[4 * i], y = xywh[4 * i + 1], w = xywh[4 * i + 2], h = xywh[4 * i + 3];
    REQUIRE(x >= 0 && y >= 0 && w >= 1 && h >= 1 && w <= cc.width - x && h <= cc.height - y,
            "cam_id " + std::to_string(cam) + " window " + std::to_string(i) + " (" + std::to_string(x) + ", " +
                std::to_string(y) + ", " + std::to_string(w) + ", " + std::to_string(h) + ") is not inside the " +
                std::to_string(cc.width) + "x" + std::to_string(cc.height) + " frame or is empty");
    wins[i] = make_int4(x, y, w, h);
  }
  c->cam_windows[cam] = wins;
  c->cam_merge_thr[cam] = merge_threshold;
  return 0;
}

int wb_register_host(wb_ctx* c, void* ptr, size_t bytes) {
  REQUIRE(c && ptr && bytes, "NULL argument");
  std::lock_guard<std::mutex> lock(c->mu);
  CK(cudaSetDevice(c->device));
  CK(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
  c->registered.push_back(ptr);
  return 0;
}
int wb_unregister_host(wb_ctx* c, void* ptr) {
  REQUIRE(c && ptr, "NULL argument");
  std::lock_guard<std::mutex> lock(c->mu);
  for (size_t i = 0; i < c->registered.size(); ++i)
    if (c->registered[i] == ptr) {
      CK(cudaHostUnregister(ptr));
      c->registered.erase(c->registered.begin() + i);
      return 0;
    }
  return fail("pointer was not registered");
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// Which layers run as one kernel.  Both the executor (run_layers) and the per-layer timer (wb_profile_layers) ask this,
// so the timing table covers exactly what runs.
enum SpanKind {
  SPAN_ONE,        // layer li alone
  SPAN_DW_PW,      // depthwise -> 1x1 (k_dwpw_tc_x3)
  SPAN_DW_PW_ADD,  // depthwise -> linear 1x1 -> residual Add (k_dwpw_tc_x3, shortcut added in its epilogue)
  SPAN_PW_ADD,     // linear 1x1 -> residual Add (k_gemm_tc, shortcut added in its epilogue)
};
struct Span {
  size_t last;  // last layer of the span
  SpanKind kind;
  uint32_t out_off;        // arena offset the span's kernel writes: the output of layer `last`
  long long residual_off;  // arena offset of the residual Add's other input (the shortcut), or -1: no Add
};

// a fused kernel reads the arena range of `reader`'s input while it writes that of `writer`'s output
static bool arena_disjoint(const wb_layer& reader, const wb_layer& writer) {
  const unsigned long long a0 = reader.in_off, a1 = a0 + (unsigned long long)reader.in_h * reader.in_w * reader.in_c;
  const unsigned long long b0 = writer.out_off, b1 = b0 + (unsigned long long)writer.out_h * writer.out_w * writer.out_c;
  return !(a0 < b1 && b0 < a1);
}

// the span of the program that starts at layer `li` (layers [li, end) are requested).  model.py plan_arena keeps each
// fused kernel's input alive through its output layer; older blobs may not, and their pairs run unfused.
static Span fused_span(const wb_ctx* c, size_t li, size_t end) {
  const std::vector<wb_layer>& Ls = c->layers;
  const wb_layer& L = Ls[li];
  // layer p + 1 is `Add(shortcut, output of p)` (tensor-core modes with fp32 storage: the shortcut can be added in an
  // fp32 epilogue)
  auto residual_add_after = [&](size_t p) {
    if (c->mode().tc_mode < 0 || c->mode().storage != Storage::F32 || p + 1 >= end || !c->sw.fuse_add) return false;
    const wb_layer& P = Ls[p], &A = Ls[p + 1];
    return P.op == WB_OP_PW && P.act == WB_ACT_NONE && A.op == WB_OP_ADD &&
           (A.in_off == P.out_off || A.in2_off == P.out_off) && A.in_off != A.in2_off;
  };
  // layers [li, last]; a span ending in an Add adds the Add's other input to the output of layer last - 1
  auto span = [&](size_t last, SpanKind kind) {
    const wb_layer& A = Ls[last];
    long long residual_off = -1;
    if (kind == SPAN_DW_PW_ADD || kind == SPAN_PW_ADD) residual_off = A.in_off == Ls[last - 1].out_off ? A.in2_off : A.in_off;
    return Span{last, kind, A.out_off, residual_off};
  };
  if (L.op == WB_OP_DW && li + 1 < end && c->sw.fuse_dwpw) {
    const wb_layer& P = Ls[li + 1];
    if (P.in_off == L.out_off && fused_dwpw_supported(c->tc, (int)li + 1, L, P)) {
      if (residual_add_after(li + 1)) {
        if (arena_disjoint(L, Ls[li + 2])) return span(li + 2, SPAN_DW_PW_ADD);
      } else if (arena_disjoint(L, P)) {
        return span(li + 1, SPAN_DW_PW);
      }
    }
  }
  if (L.op == WB_OP_PW && c->tc_runs(L) && residual_add_after(li) && arena_disjoint(L, Ls[li + 1]))
    return span(li + 1, SPAN_PW_ADD);
  return span(li, SPAN_ONE);
}

// the layer program.  `pre` != NULL feeds an already pre-processed input (wb_backbone); otherwise the
// fused stem samples the frames directly.
template <typename T>
static int run_layers(wb_ctx* c, Slot& s, cudaStream_t st, int n, const float* pre, int first_layer,
                      int last_layer) {
  LaunchCtx lc{st, &s.launches};
  // the n images' tensor at arena offset `off`
  auto at = [&](long long off) { return static_cast<T*>(s.arena.h) + (size_t)off * n; };
  const int NA = c->hdr.num_anchors, C1 = c->hdr.num_classes + 1;
  const size_t end = last_layer < 0 ? c->layers.size() : (size_t)last_layer + 1;
  for (size_t li = (size_t)first_layer; li < end; ++li) {
    const wb_layer& L = c->layers[li];
    const T* in = at(L.in_off);
    const T* in2 = at(L.in2_off);
    T* outp = at(L.out_off);
    const float* w = L.w_tensor >= 0 ? c->tensor(L.w_tensor) : nullptr;
    const float* sc = L.scale_tensor >= 0 ? c->tensor(L.scale_tensor) : nullptr;
    const float* of = L.offset_tensor >= 0 ? c->tensor(L.offset_tensor) : nullptr;
    switch (L.op) {
      case WB_OP_STEM:
        launch_stem<T>(lc, s.d_desc, pre, n, L, c->hdr.input_h, c->hdr.input_w, c->hdr.pre_mul, c->hdr.pre_sub, w,
                       sc, of, outp);
        break;
      case WB_OP_DW: {
        const Span sp = fused_span(c, li, end);
        if (sp.kind == SPAN_DW_PW || sp.kind == SPAN_DW_PW_ADD) {
          const wb_layer& P = c->layers[li + 1];
          const float* residual = sp.residual_off < 0 ? nullptr : reinterpret_cast<const float*>(at(sp.residual_off));
          std::string err;
          if (fused_launch_dwpw(lc, c->tc, (int)li + 1, n, L, P, static_cast<const void*>(in), w, sc, of,
                                c->tensor(P.scale_tensor), c->tensor(P.offset_tensor), residual,
                                static_cast<void*>(at(sp.out_off)), &err))
            return fail("layers " + std::string(L.name) + " .. " + c->layers[sp.last].name + ": " + err);
          li = sp.last;
          break;
        }
        launch_dw<T>(lc, n, L, in, w, sc, of, outp);
        break;
      }
      case WB_OP_ADD:
        launch_add<T>(lc, (size_t)n * L.out_h * L.out_w * L.out_c, in, in2, outp);
        break;
      case WB_OP_MAXPOOL:
      case WB_OP_AVGPOOL:
        launch_pool<T>(lc, n, L, in, outp);
        break;
      case WB_OP_COPY:
        launch_copy_channels<T>(lc, n, L, in, outp);
        break;
      case WB_OP_PW:
      case WB_OP_CONV:
      case WB_OP_HEAD:
        if (c->tc_runs(L)) {
          // MobileNet-v2 bottleneck: a linear projection followed by `Add(shortcut, projection)` runs as one kernel,
          // the shortcut is added in the GEMM epilogue (fp32 modes) and the Add layer is skipped
          const Span sp = fused_span(c, li, end);
          const void* residual = sp.residual_off < 0 ? nullptr : static_cast<const void*>(at(sp.residual_off));
          std::string err;
          if (tc_launch_gemm(lc, c->tc, (int)li, n, L, static_cast<const void*>(in), sc, of, static_cast<void*>(at(sp.out_off)),
                             s.d_enc, s.d_logits, NA, C1, residual, c->sw.split_k, &err))
            return fail("layer " + std::string(L.name) + ": " + err);
          li = sp.last;  // past the Add when it was fused
        } else {
          launch_gemm_cc<T>(lc, n, L, in, w, sc, of, outp, s.d_enc, s.d_logits, NA, C1, s.d_partial, s.partial_floats);
        }
        break;
      default:
        return fail("unknown layer op " + std::to_string(L.op));
    }
  }
  CK(cudaGetLastError());
  return 0;
}

// windowed batch (n_frames frames in n model images): the windows' rows go to s.d_out unfiltered, with their valid row
// counts in s.d_raw_num, and k_window_merge writes each frame's rows and verdicts to s.d_wout / s.d_wverd
static int run_post(wb_ctx* c, Slot& s, cudaStream_t st, int n, uint32_t flags, bool want_raw = false,
                    int n_frames = 0, bool windowed = false) {
  LaunchCtx lc{st, &s.launches};
  // the float boxes / scores / classes of `sess.run` are a test hook (wb_postprocess); the product path writes
  // Detection rows only
  float* rb = want_raw ? c->d_raw.h : nullptr;
  float* rs = want_raw ? rb + (size_t)c->max_batch * WB_MAX_DETECTIONS * 4 : nullptr;
  float* rc = want_raw ? rs + (size_t)c->max_batch * WB_MAX_DETECTIONS : nullptr;
  launch_post(lc, n, c->pp, s.d_enc, s.d_logits, c->tensor(c->hdr.anchors_tensor), s.d_desc,
              windowed ? nullptr : c->d_cams.h, flags, s.d_sel_count, s.d_sel, s.d_sel_box, s.d_out,
              s.d_verdicts, rb, rs, rc, (want_raw || windowed) ? s.d_raw_num.h : nullptr, s.d_kept_hist);
  if (windowed)
    launch_window_merge(lc, n_frames, c->pp, s.d_win, s.d_out, s.d_raw_num, c->d_cams, flags, s.d_wout, s.d_wverd);
  CK(cudaGetLastError());
  return 0;
}

// layers first..last (last < 0: to the end) in the engine's activation type
static int run_program(wb_ctx* c, Slot& s, cudaStream_t st, int n, const float* pre, int first, int last) {
  if (c->mode().storage == Storage::BF16) return run_layers<__nv_bfloat16>(c, s, st, n, pre, first, last);
  if (c->mode().storage == Storage::F16) return run_layers<__half>(c, s, st, n, pre, first, last);
  return run_layers<float>(c, s, st, n, pre, first, last);
}

static int run_all(wb_ctx* c, Slot& s, cudaStream_t st, int n, uint32_t flags, int n_frames, bool windowed) {
  if (int rc = run_program(c, s, st, n, nullptr, 0, -1)) return rc;
  return run_post(c, s, st, n, flags, false, n_frames, windowed);
}

// kernels of one batch, through a CUDA graph when possible (launch-bound at small batch).  The pixel format is not part
// of the graph's key: the kernels read it from the frame descriptors, which fill_desc copies to the device before every
// launch, so one graph serves batches of every pixel format alike.
static int enqueue_kernels(wb_ctx* c, Slot& s, cudaStream_t st, int n, uint32_t flags, int n_frames, bool windowed) {
  const uint32_t gflags = flags & WB_F_FUSE_FILTERS;
  if (!c->sw.graph) {
    s.launches = 0;
    return run_all(c, s, st, n, gflags, n_frames, windowed);
  }
  if (s.graph_exec == nullptr || s.graph_n != n || s.graph_flags != gflags || s.graph_frames != n_frames ||
      s.graph_windowed != windowed) {
    s.graph_exec.reset();
    // warm-up run outside capture (sets function attributes, validates launches)
    s.launches = 0;
    if (int rc = run_all(c, s, st, n, gflags, n_frames, windowed)) return rc;
    CK(cudaStreamSynchronize(st));
    cudaGraph_t graph = nullptr;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    s.launches = 0;
    int rc = run_all(c, s, st, n, gflags, n_frames, windowed);
    cudaError_t e = cudaStreamEndCapture(st, &graph);
    if (rc) return rc;
    if (e != cudaSuccess) return fail(std::string("cudaStreamEndCapture: ") + cudaGetErrorString(e));
    CK(cudaGraphInstantiate(&s.graph_exec.h, graph, 0));
    CK(cudaGraphDestroy(graph));
    s.graph_n = n;
    s.graph_flags = gflags;
    s.graph_frames = n_frames;
    s.graph_windowed = windowed;
  }
  CK(cudaGraphLaunch(s.graph_exec, st));
  return 0;
}

// the planes of the packed frame of format `fmt` and size w x h that starts at `base`
static wb_frame_planes packed_planes(const uint8_t* base, int fmt, int w, int h) {
  wb_frame_planes p{};
  for (int k = 0; k < plane_count(fmt); ++k) {
    p.plane[k] = base + plane_offset(fmt, w, h, k);
    p.pitch[k] = (int64_t)plane_row_bytes(fmt, w, k);
  }
  return p;
}

static bool same_planes(const wb_frame_planes& a, const wb_frame_planes& b, int fmt) {
  for (int k = 0; k < plane_count(fmt); ++k)
    if (a.plane[k] != b.plane[k] || a.pitch[k] != b.pitch[k]) return false;
  return true;
}

// Copies n host frames to s.d_frames, each packed into frame_bytes of its format and size (sizes[i] = (w, h)) at a
// 256-byte aligned offset, and replaces their planes with those of the copies.  A packed frame is one copy; any other
// is copied plane by plane, each plane's rows gathered from its pitch.  A buffer that is too small is replaced, once
// the stream is done with it, by one with 25 % headroom.
static int upload_frames(Slot& s, cudaStream_t st, int n, int fmt, const int2* sizes, wb_frame_planes* planes) {
  size_t total = 0;
  for (int i = 0; i < n; ++i) total += (frame_bytes(fmt, sizes[i].x, sizes[i].y) + 255) / 256 * 256;
  if (total > s.d_frames_cap) {
    CK(cudaStreamSynchronize(st));
    s.d_frames_cap = total + total / 4;
    CK(alloc(s.d_frames, s.d_frames_cap));
  }
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    const int w = sizes[i].x, h = sizes[i].y;
    const wb_frame_planes& src = planes[i];
    const wb_frame_planes dst = packed_planes(s.d_frames + off, fmt, w, h);
    if (same_planes(src, packed_planes(src.plane[0], fmt, w, h), fmt)) {
      CK(cudaMemcpyAsync(s.d_frames + off, src.plane[0], frame_bytes(fmt, w, h), cudaMemcpyHostToDevice, st));
    } else {
      for (int k = 0; k < plane_count(fmt); ++k)
        CK(cudaMemcpy2DAsync(const_cast<uint8_t*>(dst.plane[k]), (size_t)dst.pitch[k], src.plane[k],
                             (size_t)src.pitch[k], (size_t)dst.pitch[k], plane_rows(h, k), cudaMemcpyHostToDevice, st));
    }
    planes[i] = dst;
    off += (frame_bytes(fmt, w, h) + 255) / 256 * 256;
  }
  return 0;
}

// The descriptor of the window (x, y, w, h) = wd of a frame given as device planes (NULL planes: a descriptor without
// pixels, for the post stage alone).  The window's rows are the frame's, read through the planes' own pitches.
static FrameDesc frame_desc(const wb_frame_planes& p, int fmt, int4 wd, int cam) {
  FrameDesc d{};
  d.w = wd.z;
  d.h = wd.w;
  d.cam = cam;
  d.fmt = fmt;
  d.pitch = (int32_t)p.pitch[0];
  if (p.plane[0] == nullptr) return d;
  const uint8_t* row = p.plane[0] + wd.y * p.pitch[0];  // the window's first row, of pixels or macropixels
  if (fmt_rgb(fmt)) {
    d.ptr = row + (size_t)wd.x * rgb_layout(fmt).bpp;
  } else if (fmt_422(fmt)) {
    // macropixels Y0 U Y1 V (YUYV) or U Y0 V Y1 (UYVY), V two bytes after U
    d.ptr = row + luma_origin(fmt) + (size_t)wd.x * 2;
    d.chroma = row + (fmt == WB_FMT_YUYV422 ? 1 : 0) + (size_t)(wd.x >> 1) * 4;
    d.chroma_pitch = d.pitch;
    d.v_off = 2;
  } else {
    const bool nv12 = fmt == WB_FMT_NV12;
    d.ptr = row + wd.x;
    d.chroma = p.plane[1] + (wd.y >> 1) * p.pitch[1] + (size_t)(wd.x >> 1) * (nv12 ? 2 : 1);
    d.chroma_pitch = (int32_t)p.pitch[1];
    d.v_off = nv12 ? 1 : (int64_t)(reinterpret_cast<intptr_t>(p.plane[2]) - reinterpret_cast<intptr_t>(p.plane[1]));
  }
  return d;
}

// Refuses planes that do not match frame i's format and width: a used plane missing or an unused one given, a pitch
// below the plane's row bytes or at 2^31 or more (FrameDesc holds pitches as int32), yuv420p U and V pitches that
// differ (one chroma pitch serves both).
static int check_planes(int i, const wb_frame_planes& p, int fmt, int w) {
  const std::string at = "frame " + std::to_string(i) + " (" + fmt_name(fmt) + "): ";
  const int np = plane_count(fmt);
  for (int k = 0; k < 3; ++k) {
    const std::string pk = "plane[" + std::to_string(k) + "]";
    if (k >= np) {
      REQUIRE(p.plane[k] == nullptr, at + fmt_name(fmt) + " has " + std::to_string(np) +
                                         (np == 1 ? " plane" : " planes") + ", but " + pk + " is given");
      continue;
    }
    REQUIRE(p.plane[k] != nullptr, at + pk + " is NULL");
    const int64_t row = (int64_t)plane_row_bytes(fmt, w, k);
    const std::string pitch = "pitch[" + std::to_string(k) + "] = " + std::to_string(p.pitch[k]);
    REQUIRE(p.pitch[k] >= row, at + pitch + " is below the plane's row bytes (" + std::to_string(row) + ")");
    REQUIRE(p.pitch[k] < ((int64_t)1 << 31), at + pitch + " is 2^31 or more");
  }
  REQUIRE(fmt != WB_FMT_YUV420P || p.pitch[1] == p.pitch[2],
          at + "the U and V planes need the same pitch, not pitch[1] = " + std::to_string(p.pitch[1]) +
              " and pitch[2] = " + std::to_string(p.pitch[2]));
  return 0;
}

static int require_camera(wb_ctx* c, int cam) {
  REQUIRE(cam >= 0 && cam < WB_MAX_CAMERAS && c->h_cams[cam].width > 0,
          "cam_id " + std::to_string(cam) + " has not been configured with wb_set_camera");
  return 0;
}

// the planes of n packed frames (wb_detect / wb_submit, wb_backbone_frames, wb_profile_layers), sized by their cameras
static int packed_frames(wb_ctx* c, int n, const uint8_t* const* frames, const int32_t* cam_ids, int fmt,
                         std::vector<wb_frame_planes>& planes) {
  planes.resize(n);
  for (int i = 0; i < n; ++i) {
    if (int rc = require_camera(c, cam_ids[i])) return rc;
    REQUIRE(frames[i] != nullptr, "NULL frame pointer");
    const CameraCfg& cc = c->h_cams[cam_ids[i]];
    planes[i] = packed_planes(frames[i], fmt, cc.width, cc.height);
  }
  return 0;
}

// the frame formats of wb_detect / wb_submit / wb_backbone_frames
static const FormatFlag kFrameFormats[] = {{WB_F_YUV420P, WB_FMT_YUV420P, "WB_F_YUV420P"},
                                           {WB_F_NV12, WB_FMT_NV12, "WB_F_NV12"},
                                           {WB_F_YUYV422, WB_FMT_YUYV422, "WB_F_YUYV422"},
                                           {WB_F_UYVY422, WB_FMT_UYVY422, "WB_F_UYVY422"},
                                           {WB_F_BGR24, WB_FMT_BGR24, "WB_F_BGR24"},
                                           {WB_F_RGBA, WB_FMT_RGBA, "WB_F_RGBA"},
                                           {WB_F_BGRA, WB_FMT_BGRA, "WB_F_BGRA"}};

// One descriptor per model image.  With use_windows and at least one camera of the batch having detection windows, the
// batch is windowed: every window of a frame is one image (a camera without windows: one full-frame window, camera
// -1), and s.h_win / s.d_win describe the frames for k_window_merge.  Otherwise an image is a frame, as always.  A host
// frame is copied to the device once, packed, whatever its window count; the windows point into that copy (or into the
// caller's device planes).  frames == NULL: descriptors without pixels (wb_postprocess).  Every check comes before the
// first copy, so a refused batch enqueues nothing.
static int fill_desc(wb_ctx* c, Slot& s, int n, const wb_frame_planes* frames, const int32_t* cam_ids,
                     bool on_device, int fmt, cudaStream_t st, bool use_windows, int* n_images_out) {
  std::vector<int2> sizes(n);
  bool windowed = false;
  int n_images = 0;
  for (int i = 0; i < n; ++i) {
    int cam = cam_ids[i];
    if (int rc = require_camera(c, cam)) return rc;
    const CameraCfg& cc = c->h_cams[cam];
    // 4:2:0 chroma covers 2x2 pixels, 4:2:2 chroma a pixel pair of one row
    const bool yuv420 = fmt == WB_FMT_YUV420P || fmt == WB_FMT_NV12;
    const std::string size = "frame " + std::to_string(i) + " (" + fmt_name(fmt) + "): cam_id " + std::to_string(cam) +
                             " is " + std::to_string(cc.width) + "x" + std::to_string(cc.height);
    REQUIRE(!yuv420 || (cc.width % 2 == 0 && cc.height % 2 == 0), size + ": 4:2:0 frames need an even width and height");
    REQUIRE(!fmt_422(fmt) || cc.width % 2 == 0, size + ": 4:2:2 frames need an even width");
    if (frames != nullptr)
      if (int rc = check_planes(i, frames[i], fmt, cc.width)) return rc;
    sizes[i] = make_int2(cc.width, cc.height);
    const int nw = use_windows ? (int)c->cam_windows[cam].size() : 0;
    windowed |= nw > 0;
    n_images += std::max(nw, 1);
    for (int k = 0; k < nw; ++k) {
      const int4 wd = c->cam_windows[cam][k];
      const std::string win = "frame " + std::to_string(i) + " (" + fmt_name(fmt) + "): cam_id " + std::to_string(cam) +
                              " window " + std::to_string(k) + " (" + std::to_string(wd.x) + ", " +
                              std::to_string(wd.y) + ", " + std::to_string(wd.z) + ", " + std::to_string(wd.w) + ")";
      REQUIRE(!yuv420 || (wd.x % 2 == 0 && wd.y % 2 == 0 && wd.z % 2 == 0 && wd.w % 2 == 0),
              win + ": 4:2:0 frames need an even window origin, width and height");
      REQUIRE(!fmt_422(fmt) || (wd.x % 2 == 0 && wd.z % 2 == 0), win + ": 4:2:2 frames need an even window x and width");
    }
  }
  REQUIRE(n_images <= c->max_batch, "the batch's detection windows add up to " + std::to_string(n_images) +
                                        " model images, more than max_batch (" + std::to_string(c->max_batch) + ")");
  if (!windowed) n_images = n;
  std::vector<wb_frame_planes> dev(n, wb_frame_planes{});  // each frame's planes on the device
  if (frames != nullptr) {
    dev.assign(frames, frames + n);
    if (!on_device)
      if (int rc = upload_frames(s, st, n, fmt, sizes.data(), dev.data())) return rc;
  }
  int img = 0;
  for (int i = 0; i < n; ++i) {
    const int cam = cam_ids[i];
    const CameraCfg& cc = c->h_cams[cam];
    const std::vector<int4>& wins = c->cam_windows[cam];
    const int nw = windowed ? std::max((int)wins.size(), 1) : 1;
    if (windowed) {
      WindowFrame& wf = s.h_win[i];
      wf.first = img;
      wf.count = nw;
      wf.cam = cam;
      wf._pad = 0;
      wf.merge_thr = wins.empty() ? 0.5 : c->cam_merge_thr[cam];
    }
    for (int k = 0; k < nw; ++k) {
      const int4 wd = (windowed && !wins.empty()) ? wins[k] : make_int4(0, 0, cc.width, cc.height);
      if (windowed) {
        s.h_win[i].x[k] = wd.x;
        s.h_win[i].y[k] = wd.y;
      }
      s.h_desc[img++] = frame_desc(dev[i], fmt, wd, windowed ? -1 : cam);
    }
  }
  CK(cudaMemcpyAsync(s.d_desc, s.h_desc, sizeof(FrameDesc) * n_images, cudaMemcpyHostToDevice, st));
  if (windowed) CK(cudaMemcpyAsync(s.d_win, s.h_win, sizeof(WindowFrame) * n, cudaMemcpyHostToDevice, st));
  s.windowed = windowed;
  if (n_images_out) *n_images_out = n_images;
  return 0;
}

// The stage hooks (wb_preprocess, wb_backbone, wb_backbone_frames, wb_postprocess, wb_profile_layers) run
// synchronously on slot 0 and hold the context lock throughout.  The guard takes the lock and makes the context's
// device current; `rc` is non-zero when that fails, the batch of n images does not fit or slot 0 has a batch in flight.
struct StageHook {
  std::lock_guard<std::mutex> lock;
  Slot& s;
  cudaStream_t st;
  int rc;
  StageHook(wb_ctx* c, int n) : lock(c->mu), s(c->slots[0]), st(c->stream_of(0)), rc(enter(c, n)) {}
  static int enter(wb_ctx* c, int n) {
    REQUIRE(n >= 1 && n <= c->max_batch, "batch size out of range");
    CK(cudaSetDevice(c->device));
    REQUIRE(!c->slots[0].busy, "slot 0 is busy");
    return 0;
  }
};

// wb_submit (packed frames) and wb_submit_planes: exactly one of `packed` and `planes` is given
static int submit(wb_ctx* c, int slot, int n, const uint8_t* const* packed, const wb_frame_planes* planes,
                  const int32_t* cam_ids, uint32_t flags) {
  REQUIRE(c && (packed || planes) && cam_ids, "NULL argument");
  REQUIRE(slot >= 0 && slot < WB_SLOTS, "slot out of range");
  REQUIRE(n >= 1 && n <= c->max_batch, "batch size out of range (1..max_batch)");
  std::lock_guard<std::mutex> lock(c->mu);
  Slot& s = c->slots[slot];
  REQUIRE(!s.busy, "slot is busy: collect it first");
  CK(cudaSetDevice(c->device));
  cudaStream_t st = c->stream_of(slot);
  std::string err;
  const int fmt = pixel_format(flags, kFrameFormats, err);
  REQUIRE(fmt >= 0, err);
  std::vector<wb_frame_planes> packed_as_planes;
  if (packed) {
    if (int rc = packed_frames(c, n, packed, cam_ids, fmt, packed_as_planes)) return rc;
    planes = packed_as_planes.data();
  }
  CK(cudaEventRecord(s.ev0, st));
  int n_images = n;
  if (int rc = fill_desc(c, s, n, planes, cam_ids, (flags & WB_F_FRAMES_ON_DEVICE) != 0, fmt, st, true, &n_images))
    return rc;
  if (int rc = enqueue_kernels(c, s, st, n_images, flags, n, s.windowed)) return rc;
  if (!(flags & WB_F_OUT_ON_DEVICE)) {
    CK(cudaMemcpyAsync(s.h_out, s.windowed ? s.d_wout : s.d_out, sizeof(wb_detection) * (size_t)n * WB_MAX_DETECTIONS,
                       cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_verdicts, s.windowed ? s.d_wverd : s.d_verdicts,
                       sizeof(uint32_t) * (size_t)n * WB_MAX_DETECTIONS, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaEventRecord(s.ev1, st));
  s.n = n;
  s.flags = flags;
  s.busy = true;
  c->last_launches = s.launches;
  return 0;
}

extern "C" {

int wb_submit(wb_ctx* c, int slot, int n, const uint8_t* const* frames, const int32_t* cam_ids, uint32_t flags) {
  return submit(c, slot, n, frames, nullptr, cam_ids, flags);
}

int wb_submit_planes(wb_ctx* c, int slot, int n, const wb_frame_planes* frames, const int32_t* cam_ids,
                     uint32_t flags) {
  return submit(c, slot, n, nullptr, frames, cam_ids, flags);
}

int wb_collect(wb_ctx* c, int slot, wb_detection* const* out, uint32_t* const* verdicts, float* gpu_ms) {
  REQUIRE(c, "NULL ctx");
  REQUIRE(slot >= 0 && slot < WB_SLOTS, "slot out of range");
  Slot& s = c->slots[slot];
  {
    std::lock_guard<std::mutex> lock(c->mu);
    REQUIRE(s.busy, "slot has no batch in flight");
    s.busy = false;
  }
  CK(cudaSetDevice(c->device));
  CK(cudaEventSynchronize(s.ev1));  // not under the lock: other threads keep submitting to other slots
  if (gpu_ms) CK(cudaEventElapsedTime(gpu_ms, s.ev0, s.ev1));
  if (s.flags & WB_F_OUT_ON_DEVICE) {
    cudaStream_t st = c->stream_of(slot);
    const wb_detection* d_out = s.windowed ? s.d_wout : s.d_out;
    const uint32_t* d_verd = s.windowed ? s.d_wverd : s.d_verdicts;
    for (int i = 0; i < s.n; ++i) {
      if (out && out[i])
        CK(cudaMemcpyAsync(out[i], d_out + (size_t)i * WB_MAX_DETECTIONS, sizeof(wb_detection) * WB_MAX_DETECTIONS,
                           cudaMemcpyDeviceToDevice, st));
      if (verdicts && verdicts[i])
        CK(cudaMemcpyAsync(verdicts[i], d_verd + (size_t)i * WB_MAX_DETECTIONS,
                           sizeof(uint32_t) * WB_MAX_DETECTIONS, cudaMemcpyDeviceToDevice, st));
    }
    CK(cudaStreamSynchronize(st));
    return 0;
  }
  for (int i = 0; i < s.n; ++i) {
    if (out && out[i])
      memcpy(out[i], s.h_out + (size_t)i * WB_MAX_DETECTIONS, sizeof(wb_detection) * WB_MAX_DETECTIONS);
    if (verdicts && verdicts[i])
      memcpy(verdicts[i], s.h_verdicts + (size_t)i * WB_MAX_DETECTIONS, sizeof(uint32_t) * WB_MAX_DETECTIONS);
  }
  return 0;
}

int wb_stream_fence(wb_ctx* c, uint64_t stream, int direction) {
  REQUIRE(c, "NULL ctx");
  REQUIRE(direction == 0 || direction == 1, "direction must be 0 or 1");
  CK(cudaSetDevice(c->device));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  Event ev;
  CK(cudaEventCreateWithFlags(&ev.h, cudaEventDisableTiming));
  if (direction == 0) {
    CK(cudaEventRecord(ev, user));
    for (auto& s : c->slots) CK(cudaStreamWaitEvent(s.stream, ev, 0));
  } else {
    for (auto& s : c->slots) {
      CK(cudaEventRecord(ev, s.stream));
      CK(cudaStreamWaitEvent(user, ev, 0));
    }
  }
  return 0;
}

int wb_detect(wb_ctx* c, int n, const uint8_t* const* frames, const int32_t* cam_ids, uint32_t flags,
              wb_detection* const* out, uint32_t* const* verdicts, float* gpu_ms) {
  if (int rc = wb_submit(c, 0, n, frames, cam_ids, flags)) return rc;
  return wb_collect(c, 0, out, verdicts, gpu_ms);
}

int wb_detect_planes(wb_ctx* c, int n, const wb_frame_planes* frames, const int32_t* cam_ids, uint32_t flags,
                     wb_detection* const* out, uint32_t* const* verdicts, float* gpu_ms) {
  if (int rc = wb_submit_planes(c, 0, n, frames, cam_ids, flags)) return rc;
  return wb_collect(c, 0, out, verdicts, gpu_ms);
}

// ---------------------------------------------------------------------------------------------------
int wb_preprocess(wb_ctx* c, int n, const uint8_t* const* frames, const int32_t* widths, const int32_t* heights,
                  float* out) {
  REQUIRE(c && frames && widths && heights && out, "NULL argument");
  StageHook h(c, n);
  if (h.rc) return h.rc;
  Slot& s = h.s;
  cudaStream_t st = h.st;
  std::vector<int2> sizes(n);
  std::vector<wb_frame_planes> planes(n);
  for (int i = 0; i < n; ++i) {
    sizes[i] = make_int2(widths[i], heights[i]);
    planes[i] = packed_planes(frames[i], WB_FMT_RGB24, widths[i], heights[i]);
  }
  if (int rc = upload_frames(s, st, n, WB_FMT_RGB24, sizes.data(), planes.data())) return rc;
  for (int i = 0; i < n; ++i)
    s.h_desc[i] = frame_desc(planes[i], WB_FMT_RGB24, make_int4(0, 0, widths[i], heights[i]), -1);
  CK(cudaMemcpyAsync(s.d_desc, s.h_desc, sizeof(FrameDesc) * n, cudaMemcpyHostToDevice, st));
  LaunchCtx lc{st, &s.launches};
  launch_preprocess_f32(lc, s.d_desc, n, c->d_pre, c->hdr.input_h, c->hdr.input_w, c->hdr.pre_mul, c->hdr.pre_sub);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, c->d_pre, sizeof(float) * (size_t)n * c->hdr.input_h * c->hdr.input_w * 3,
                     cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

// the backbone hooks' outputs from slot s (n images): the head buffers (enc and logits may be NULL) and, for
// stop_layer >= 0 and a layer_out, that layer's activation (float32 NHWC; bf16 / fp16 storage is widened exactly)
static int copy_backbone_out(wb_ctx* c, Slot& s, cudaStream_t st, int n, float* enc, float* logits, int stop_layer,
                             float* layer_out, size_t layer_out_floats) {
  if (enc) CK(cudaMemcpyAsync(enc, s.d_enc, sizeof(float) * (size_t)n * c->hdr.num_anchors * 4, cudaMemcpyDeviceToHost, st));
  if (logits)
    CK(cudaMemcpyAsync(logits, s.d_logits, sizeof(float) * (size_t)n * c->hdr.num_anchors * (c->hdr.num_classes + 1),
                       cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (stop_layer < 0 || !layer_out) return 0;
  const wb_layer& L = c->layers[stop_layer];
  REQUIRE(L.op != WB_OP_HEAD, "head layers have no activation output");
  size_t elems = (size_t)n * L.out_h * L.out_w * L.out_c;
  REQUIRE(layer_out_floats >= elems, "layer_out too small");
  if (c->mode().storage == Storage::F32) {
    CK(cudaMemcpy(layer_out, static_cast<float*>(s.arena.h) + (size_t)L.out_off * n, elems * 4, cudaMemcpyDeviceToHost));
  } else {
    std::vector<uint16_t> tmp(elems);
    CK(cudaMemcpy(tmp.data(), static_cast<uint16_t*>(s.arena.h) + (size_t)L.out_off * n, elems * 2, cudaMemcpyDeviceToHost));
    if (c->mode().storage == Storage::F16) {
      for (size_t i = 0; i < elems; ++i) {
        __half h;
        memcpy(&h, &tmp[i], 2);
        layer_out[i] = __half2float(h);
      }
    } else {
      for (size_t i = 0; i < elems; ++i) {
        uint32_t u = (uint32_t)tmp[i] << 16;
        memcpy(&layer_out[i], &u, 4);
      }
    }
  }
  return 0;
}

extern "C" {

int wb_backbone(wb_ctx* c, int n, const float* pre, float* enc, float* logits, int stop_layer, float* layer_out,
                size_t layer_out_floats) {
  REQUIRE(c && pre, "NULL argument");
  REQUIRE(stop_layer < (int)c->layers.size(), "stop_layer out of range");
  StageHook h(c, n);
  if (h.rc) return h.rc;
  Slot& s = h.s;
  cudaStream_t st = h.st;
  const size_t pre_floats = (size_t)n * c->hdr.input_h * c->hdr.input_w * 3;
  CK(cudaMemcpyAsync(c->d_pre, pre, sizeof(float) * pre_floats, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(s.d_enc, 0, sizeof(float) * (size_t)n * c->hdr.num_anchors * 4, st));
  CK(cudaMemsetAsync(s.d_logits, 0, sizeof(float) * (size_t)n * c->hdr.num_anchors * (c->hdr.num_classes + 1), st));
  s.launches = 0;
  if (int rc = run_program(c, s, st, n, c->d_pre, 0, stop_layer)) return rc;
  if (int rc = copy_backbone_out(c, s, st, n, enc, logits, stop_layer, layer_out, layer_out_floats)) return rc;
  c->last_launches = s.launches;
  return 0;
}

int wb_backbone_frames(wb_ctx* c, int n, const uint8_t* const* frames, const int32_t* cam_ids, uint32_t flags,
                       float* enc, float* logits, int stop_layer, float* layer_out, size_t layer_out_floats,
                       int32_t* n_images) {
  REQUIRE(c && frames && cam_ids, "NULL argument");
  REQUIRE(stop_layer >= -1 && stop_layer < (int)c->layers.size(), "stop_layer out of range");
  uint32_t allowed = WB_F_FRAMES_ON_DEVICE | WB_F_FUSE_FILTERS;
  std::string names;
  for (const FormatFlag& f : kFrameFormats) {
    allowed |= f.bit;
    names += std::string(f.name) + ", ";
  }
  REQUIRE((flags & ~allowed) == 0, "flags may only hold " + names + "WB_F_FRAMES_ON_DEVICE and WB_F_FUSE_FILTERS");
  StageHook h(c, n);
  if (h.rc) return h.rc;
  Slot& s = h.s;
  cudaStream_t st = h.st;
  std::string err;
  const int fmt = pixel_format(flags, kFrameFormats, err);
  REQUIRE(fmt >= 0, err);
  std::vector<wb_frame_planes> planes;
  if (int rc = packed_frames(c, n, frames, cam_ids, fmt, planes)) return rc;
  int ni = n;
  if (int rc = fill_desc(c, s, n, planes.data(), cam_ids, (flags & WB_F_FRAMES_ON_DEVICE) != 0, fmt, st, true, &ni))
    return rc;
  if (stop_layer >= 0) {
    s.launches = 0;
    if (int rc = run_program(c, s, st, ni, nullptr, 0, stop_layer)) return rc;
  } else if (int rc = enqueue_kernels(c, s, st, ni, flags, n, s.windowed)) {
    return rc;
  }
  // the head buffers as the run left them: not cleared first, so a head row that no kernel wrote keeps stale values
  if (int rc = copy_backbone_out(c, s, st, ni, enc, logits, stop_layer, layer_out, layer_out_floats)) return rc;
  if (n_images) *n_images = ni;
  c->last_launches = s.launches;
  return 0;
}

int wb_postprocess(wb_ctx* c, int n, const float* enc, const float* logits, const int32_t* cam_ids, uint32_t flags,
                   wb_detection* const* out, uint32_t* const* verdicts, float* boxes, float* scores, float* classes,
                   int32_t* num) {
  REQUIRE(c && enc && logits && cam_ids, "NULL argument");
  StageHook h(c, n);
  if (h.rc) return h.rc;
  Slot& s = h.s;
  cudaStream_t st = h.st;
  const int NA = c->hdr.num_anchors, C1 = c->hdr.num_classes + 1;
  CK(cudaMemcpyAsync(s.d_enc, enc, sizeof(float) * (size_t)n * NA * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.d_logits, logits, sizeof(float) * (size_t)n * NA * C1, cudaMemcpyHostToDevice, st));
  if (int rc = fill_desc(c, s, n, nullptr, cam_ids, false, WB_FMT_RGB24, st, false, nullptr)) return rc;
  s.launches = 0;
  if (int rc = run_post(c, s, st, n, flags, true)) return rc;
  const size_t B = c->max_batch;
  CK(cudaMemcpyAsync(s.h_out, s.d_out, sizeof(wb_detection) * (size_t)n * WB_MAX_DETECTIONS, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(s.h_verdicts, s.d_verdicts, sizeof(uint32_t) * (size_t)n * WB_MAX_DETECTIONS, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(c->h_raw, c->d_raw, sizeof(float) * B * WB_MAX_DETECTIONS * 6, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(c->h_raw_num, s.d_raw_num, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    if (out && out[i]) memcpy(out[i], s.h_out + (size_t)i * WB_MAX_DETECTIONS, sizeof(wb_detection) * WB_MAX_DETECTIONS);
    if (verdicts && verdicts[i])
      memcpy(verdicts[i], s.h_verdicts + (size_t)i * WB_MAX_DETECTIONS, sizeof(uint32_t) * WB_MAX_DETECTIONS);
  }
  if (boxes) memcpy(boxes, c->h_raw, sizeof(float) * (size_t)n * WB_MAX_DETECTIONS * 4);
  if (scores) memcpy(scores, c->h_raw + B * WB_MAX_DETECTIONS * 4, sizeof(float) * (size_t)n * WB_MAX_DETECTIONS);
  if (classes) memcpy(classes, c->h_raw + B * WB_MAX_DETECTIONS * 5, sizeof(float) * (size_t)n * WB_MAX_DETECTIONS);
  if (num) memcpy(num, c->h_raw_num, sizeof(int) * n);
  c->last_launches = s.launches;
  return 0;
}

int wb_filter_rows(wb_ctx* c, int cam, int n_rows, wb_detection* rows, uint32_t* verdicts) {
  REQUIRE(c && rows && verdicts, "NULL argument");
  REQUIRE(n_rows >= 1 && n_rows <= c->frows_cap, "n_rows out of range");
  // thread-safe: one DetectionSieve thread per camera calls this concurrently (ref: watsor/main.py:378-384)
  std::lock_guard<std::mutex> lock(c->mu);
  REQUIRE(cam >= 0 && cam < WB_MAX_CAMERAS && c->h_cams[cam].width > 0, "camera has not been configured");
  CK(cudaSetDevice(c->device));
  cudaStream_t st = c->fstream;
  CK(cudaMemcpyAsync(c->d_frows, rows, sizeof(wb_detection) * n_rows, cudaMemcpyHostToDevice, st));
  int launches = 0;
  LaunchCtx lc{st, &launches};
  launch_filter_rows(lc, c->d_cams + cam, n_rows, c->d_frows, c->d_fverd);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(rows, c->d_frows, sizeof(wb_detection) * n_rows, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(verdicts, c->d_fverd, sizeof(uint32_t) * n_rows, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

int wb_last_launch_count(wb_ctx* c, int* launches) {
  REQUIRE(c && launches, "NULL argument");
  *launches = c->last_launches;
  return 0;
}

// runs the program once, un-graphed, with an event pair around every layer and one around the post
// stage: per-layer device times for bench.py's roofline (kinds[i] = layer op, 100 = post stage)
int wb_profile_layers(wb_ctx* c, int n, const uint8_t* const* device_frames, const int32_t* cam_ids,
                      float* ms, int32_t* kinds, int max_launches, int* n_out) {
  REQUIRE(c && device_frames && cam_ids && ms && kinds && n_out, "NULL argument");
  StageHook h(c, n);
  if (h.rc) return h.rc;
  Slot& s = h.s;
  cudaStream_t st = h.st;
  std::vector<wb_frame_planes> planes;
  if (int rc = packed_frames(c, n, device_frames, cam_ids, WB_FMT_RGB24, planes)) return rc;
  if (int rc = fill_desc(c, s, n, planes.data(), cam_ids, true, WB_FMT_RGB24, st, false, nullptr)) return rc;
  const int nl = (int)c->layers.size();
  REQUIRE(max_launches >= nl + 1, "max_launches too small");
  std::vector<Event> ev(nl + 2);  // entry i is timed from ev[i] to ev[i + 1]
  for (auto& e : ev) CK(create(e));
  // every layer is launched REPS times back to back between two events (layers are idempotent: they
  // never write their own input), so host launch gaps do not leak into the per-kernel time
  const int REPS = 10;
  s.launches = 0;
  if (int rc = run_all(c, s, st, n, 0, n, false)) return rc;  // warm-up, also fills every activation buffer
  s.launches = 0;
  CK(cudaEventRecord(ev[0], st));
  for (int li = 0; li < nl;) {
    // time each span the executor runs as one kernel REPS times, and report its time on its 1x1 (projection) entry,
    // or on its only layer; the span's other entries read 0
    const Span sp = fused_span(c, li, nl);
    const int last = (int)sp.last;
    const int timed = sp.kind == SPAN_DW_PW || sp.kind == SPAN_DW_PW_ADD ? li + 1 : li;
    for (int i = li; i <= last; ++i) {
      for (int r = 0; i == timed && r < REPS; ++r)
        if (int rc = run_program(c, s, st, n, nullptr, li, last)) return rc;
      CK(cudaEventRecord(ev[i + 1], st));
      kinds[i] = (int)c->layers[i].op;
    }
    li = last + 1;
  }
  for (int r = 0; r < REPS; ++r)
    if (int rc = run_post(c, s, st, n, 0)) return rc;
  CK(cudaEventRecord(ev[nl + 1], st));
  CK(cudaEventSynchronize(ev[nl + 1]));
  for (int li = 0; li <= nl; ++li) {
    CK(cudaEventElapsedTime(&ms[li], ev[li], ev[li + 1]));
    ms[li] /= REPS;
  }
  s.launches /= REPS;
  kinds[nl] = 100;
  *n_out = nl + 1;
  c->last_launches = s.launches;
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// Engine frame scatter over NCCL, bound with dlopen so that the library itself does not depend on libnccl.
namespace {
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string error;
};

NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    // one NCCL per process: the copy that is already loaded wins (torch brings its own libnccl.so.2 and cannot be
    // imported after a different one -- same SONAME); then WB_NCCL_LIB (the Python shim points it at the copy bundled
    // with torch, so a later `import torch` still works); then the system library
    api.handle = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    const char* override_path = getenv("WB_NCCL_LIB");
    if (!api.handle && override_path && override_path[0]) api.handle = dlopen(override_path, RTLD_NOW | RTLD_GLOBAL);
    if (!api.handle) api.handle = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!api.handle) api.handle = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!api.handle) {
      const char* e = dlerror();
      api.error = std::string("cannot load NCCL (libnccl.so.2): ") + (e ? e : "not found");
      return;
    }
    bool ok = true;
    auto sym = [&](const char* name) {
      void* p = dlsym(api.handle, name);
      if (!p) {
        ok = false;
        api.error = std::string("NCCL symbol missing: ") + name;
      }
      return p;
    };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(sym("ncclGroupStart"));
    api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(sym("ncclGroupEnd"));
    api.Send = reinterpret_cast<decltype(api.Send)>(sym("ncclSend"));
    api.Recv = reinterpret_cast<decltype(api.Recv)>(sym("ncclRecv"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    if (!ok) api.handle = nullptr;
  });
  return &api;
}
}  // namespace

#define NCCL_CK(api, call)                                                                      \
  do {                                                                                          \
    ncclResult_t _r = (call);                                                                   \
    if (_r != ncclSuccess) return fail(std::string(#call) + ": " + (api)->GetErrorString(_r));  \
  } while (0)

static_assert(sizeof(ncclUniqueId) == WB_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");

int wb_comm_unique_id(uint8_t* id_out) {
  REQUIRE(id_out, "NULL id_out");
  NcclApi* api = nccl_api();
  if (!api->handle) return fail(api->error);
  ncclUniqueId id;
  NCCL_CK(api, api->GetUniqueId(&id));
  memcpy(id_out, &id, sizeof(id));
  return 0;
}

int wb_comm_init(wb_ctx* c, int rank, int world, const uint8_t* id_bytes) {
  REQUIRE(c, "NULL ctx");
  REQUIRE(id_bytes, "NULL id");
  REQUIRE(world >= 1 && rank >= 0 && rank < world, "rank must be in [0, world)");
  NcclApi* api = nccl_api();
  if (!api->handle) return fail(api->error);
  std::lock_guard<std::mutex> lock(c->mu);
  REQUIRE(c->comm == nullptr, "the context already has a communicator (wb_comm_destroy first)");
  CK(cudaSetDevice(c->device));
  ncclUniqueId id;
  memcpy(&id, id_bytes, sizeof(id));
  ncclComm_t comm = nullptr;
  NCCL_CK(api, api->CommInitRank(&comm, world, id, rank));
  c->comm = comm;
  c->comm_rank = rank;
  c->comm_world = world;
  CK(create(c->comm_stream));
  CK(cudaEventCreateWithFlags(&c->comm_ev.h, cudaEventDisableTiming));
  return 0;
}

int wb_scatter_frames(wb_ctx* c, int root, const uint8_t* const* send_per_rank, uint8_t* recv, size_t bytes_per_rank,
                      uint64_t cuda_stream) {
  REQUIRE(c, "NULL ctx");
  REQUIRE(c->comm != nullptr, "wb_comm_init has not been called on this context");
  REQUIRE(root >= 0 && root < c->comm_world, "root out of range");
  REQUIRE(recv != nullptr && bytes_per_rank > 0, "NULL receive buffer / empty slab");
  const bool is_root = c->comm_rank == root;
  REQUIRE(!is_root || send_per_rank != nullptr, "the root rank must pass send_per_rank");
  if (is_root)
    for (int r = 0; r < c->comm_world; ++r) REQUIRE(send_per_rank[r] != nullptr, "NULL slab pointer");
  NcclApi* api = nccl_api();
  ncclComm_t comm = static_cast<ncclComm_t>(c->comm);
  std::lock_guard<std::mutex> lock(c->mu);
  CK(cudaSetDevice(c->device));
  const bool own = cuda_stream == 0;
  cudaStream_t st = own ? c->comm_stream : reinterpret_cast<cudaStream_t>(cuda_stream);
  if (is_root) {
    NCCL_CK(api, api->GroupStart());
    for (int r = 0; r < c->comm_world; ++r)
      if (r != root) NCCL_CK(api, api->Send(send_per_rank[r], bytes_per_rank, ncclUint8, r, comm, st));
    NCCL_CK(api, api->GroupEnd());
    if (send_per_rank[root] != recv)
      CK(cudaMemcpyAsync(recv, send_per_rank[root], bytes_per_rank, cudaMemcpyDeviceToDevice, st));
  } else {
    NCCL_CK(api, api->Recv(recv, bytes_per_rank, ncclUint8, root, comm, st));
  }
  if (own) {
    CK(cudaEventRecord(c->comm_ev, st));
    for (auto& s : c->slots) CK(cudaStreamWaitEvent(s.stream, c->comm_ev, 0));
  }
  return 0;
}

int wb_comm_destroy(wb_ctx* c) {
  if (!c || !c->comm) return 0;
  NcclApi* api = nccl_api();
  cudaSetDevice(c->device);
  if (c->comm_stream) cudaStreamSynchronize(c->comm_stream);
  if (api->handle) api->CommDestroy(static_cast<ncclComm_t>(c->comm));
  c->comm = nullptr;
  c->comm_rank = -1;
  c->comm_world = 0;
  c->comm_ev.reset();
  c->comm_stream.reset();
  return 0;
}
