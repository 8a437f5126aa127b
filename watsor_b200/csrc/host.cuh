// host.cuh -- host-side helpers of libwatsor_b200: owned CUDA handles, the error-return macros and the checks that the
// detector (wb_*) and the effects pass (wb_fx_*) share.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <utility>
#include <vector>

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

// one pixel-format flag bit of a C-ABI call: the format (WB_FMT_*) it selects and its name for error messages
struct FormatFlag {
  uint32_t bit;
  int fmt;
  const char* name;
};

// the pixel format that the format bits of `flags` select (WB_FMT_RGB24 when none is set); -1 when more than one is
// set, with `err` naming them ("WB_F_YUV420P and WB_F_NV12 are mutually exclusive")
template <size_t N>
inline int pixel_format(uint32_t flags, const FormatFlag (&table)[N], std::string& err) {
  int fmt = WB_FMT_RGB24;
  std::vector<const char*> set;
  for (const FormatFlag& f : table)
    if (flags & f.bit) {
      fmt = f.fmt;
      set.push_back(f.name);
    }
  if (set.size() <= 1) return fmt;
  err.clear();
  for (size_t i = 0; i < set.size(); ++i) err += std::string(i == 0 ? "" : i + 1 == set.size() ? " and " : ", ") + set[i];
  err += " are mutually exclusive";
  return -1;
}
