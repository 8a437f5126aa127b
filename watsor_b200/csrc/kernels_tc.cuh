// kernels_tc.cuh -- tensor-core (wgmma + TMA) GEMM path for the dense 1x1 convolutions.
#pragma once
#include <string>
#include <vector>

#include "common.cuh"
#include "host.cuh"

enum TcMode { TC_BF16 = 0, TC_TF32X1 = 1, TC_TF32X3 = 2, TC_FP16 = 3 };
// bytes per operand element: 2 in the 16-bit modes, 4 (fp32 read as TF32) otherwise
inline int tc_elem_bytes(int mode) { return mode == TC_BF16 || mode == TC_FP16 ? 2 : 4; }

struct TcLayerWeights {
  DevBuf<void> w;     // [n_pad][K] K-major (bf16, fp16, or fp32 "hi" part)
  DevBuf<void> w_lo;  // fp32 "lo" part (TF32X3)
  int n_pad = 0, k = 0, block_n = 0;
  bool ready = false;
  alignas(64) unsigned char tmap_b[128];     // CUtensorMap of w
  alignas(64) unsigned char tmap_b_lo[128];  // CUtensorMap of w_lo
};

struct TcWeights {
  int mode = TC_BF16;
  std::vector<TcLayerWeights> layers;  // indexed by layer number (unset entries for non-GEMM layers)
};

// whether the tensor-core GEMM of operand mode `mode` (TcMode) runs layer L; KxK convs only with `conv`
bool tc_layer_supported(const wb_layer& L, int mode, bool conv);
int tc_prepare_weights(const std::vector<wb_layer>& layers, const std::vector<wb_tensor_entry>& tensors,
                       const float* host_data, int mode, bool conv, TcWeights* out, std::string* err);
// `split_k`: latency-bound shapes may split K over a thread-block cluster
int tc_launch_gemm(const LaunchCtx& lc, const TcWeights& tw, int layer_index, int n, const wb_layer& L, const void* in,
                   const float* scale, const float* offset, void* out, float* enc, float* logits, int num_anchors,
                   int num_classes_p1, const void* residual, bool split_k, std::string* err);

// generic tiled tensor-map encoder (rank <= 5) of elements of operand mode `mode` (TcMode); `map` points to 128 bytes
// aligned to 64
bool tc_encode_map(void* map, const void* base, int mode, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box, bool swizzle128, std::string* err,
                   const unsigned* elem_strides = nullptr);

// fused depthwise 3x3 (+BN+ReLU6) -> 1x1 conv (+BN+ReLU6) (+ residual Add) on tensor cores (kernels_fused.cu);
// TF32X3 only.  `supported` checks the layer shapes and sizes only: the caller checks the arena (the depthwise input
// must not overlap the output).  `residual` is nullptr or the Add's other operand; `out` is then the Add's output.
bool fused_dwpw_supported(const TcWeights& tw, int pw_layer_index, const wb_layer& dw, const wb_layer& pw);
int fused_launch_dwpw(const LaunchCtx& lc, const TcWeights& tw, int pw_layer_index, int n, const wb_layer& dw,
                      const wb_layer& pw, const void* in, const float* dw_w, const float* dw_scale, const float* dw_offset,
                      const float* scale, const float* offset, const float* residual, void* out, std::string* err);
