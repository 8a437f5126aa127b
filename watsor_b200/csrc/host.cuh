// host.cuh -- host-side helpers of libwatsor_b200: owned CUDA handles, the error-return macros and the checks that the
// detector (wb_*) and the effects pass (wb_fx_*) share.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <utility>

#include "yuv420.cuh"

// CK(call) and REQUIRE(cond, msg) return fail(message) from the enclosing entry point.  Each translation unit defines
// its own `fail`, which stores the message where its C-ABI's last-error call reads it.
#define CK(call)                                                                              \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess)                                                                    \
      return fail(std::string(#call) + ": " + cudaGetErrorString(e_) + " (" + __FILE__ + ":" + \
                  std::to_string(__LINE__) + ")");                                            \
  } while (0)
#define REQUIRE(cond, msg) \
  do {                     \
    if (!(cond)) return fail(msg); \
  } while (0)

// An owned CUDA handle (a device or pinned allocation, a stream, an event or a graph exec), released with the object or
// scope that holds it, so that neither a destroy call nor an early error return has to list it.  It converts to the raw
// handle.  It cannot be copied; a move swaps the two handles, so the moved-from object releases what the target held.
template <typename H, auto Release>
struct Owned {
  H h = nullptr;
  Owned() = default;
  Owned(Owned&& o) noexcept { std::swap(h, o.h); }
  Owned& operator=(Owned&& o) noexcept {
    std::swap(h, o.h);
    return *this;
  }
  ~Owned() { reset(); }
  operator H() const { return h; }
  cudaError_t reset() {
    const cudaError_t e = h ? Release(h) : cudaSuccess;
    h = nullptr;
    return e;
  }
};
template <typename T>
using DevBuf = Owned<T*, cudaFree>;
template <typename T>
using PinnedBuf = Owned<T*, cudaFreeHost>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using GraphExec = Owned<cudaGraphExec_t, cudaGraphExecDestroy>;

// (re-)allocate `bytes` of device or pinned memory; the previous allocation is released first, and a failed allocation
// leaves the handle null
template <typename T, auto Release>
cudaError_t alloc(Owned<T*, Release>& b, size_t bytes) {
  if (cudaError_t e = b.reset()) return e;
  return Release == cudaFreeHost ? cudaMallocHost(&b.h, bytes) : cudaMalloc(&b.h, bytes);
}
inline cudaError_t create(Stream& s) { return cudaStreamCreateWithFlags(&s.h, cudaStreamNonBlocking); }
inline cudaError_t create(Event& e) { return cudaEventCreate(&e.h); }

// "" when the library's kernels, which are built for sm_90a only, run on the device of `prop`; otherwise why they do not
inline std::string unsupported_device(const cudaDeviceProp& prop) {
  if (prop.major == 9 && prop.minor == 0) return "";
  return std::string("libwatsor_b200 is built for sm_90a only; device is ") + prop.name + " (sm_" +
         std::to_string(prop.major) + std::to_string(prop.minor) + ")";
}

// the pixel format (WB_FMT_*) that a call's two 4:2:0 flag bits select, or -1 when both are set
inline int pixel_format(bool yuv420p, bool nv12) {
  if (yuv420p && nv12) return -1;
  return yuv420p ? WB_FMT_YUV420P : nv12 ? WB_FMT_NV12 : WB_FMT_RGB24;
}
