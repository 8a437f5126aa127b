// kernels_post.cu -- K8 (per-class sigmoid scores, anchor decode and NMS), K9 (global top-100, integer conversion +
// confidence / area / mask-zone predicates -> Detection[100]).
//
// Restates `Postprocessor/Decode/*`, `Postprocessor/convert_scores`, `Postprocessor/Slice`,
// `Postprocessor/BatchMultiClassNonMaxSuppression/*` and the final `add` of the frozen graph
// (watsor/detection/tensorflow_cpu.py:114), the python write loop tensorflow_cpu.py:79-90, and
// watsor/filter/{confidence,area,mask}.py as applied by watsor/filter/track.py:26.
//
// Every float op is an explicit round-to-nearest intrinsic (no FMA contraction) in the graph's op
// order, so that given identical head outputs the result is bit-identical to the oracle
// (up to the last-ulp difference between CUDA's expf and the host libm's).
#include <algorithm>

#include "common.cuh"

// `Postprocessor/Decode/*` for one anchor
__device__ __forceinline__ float4 decode_box(float4 e, float4 a, const PostParams& pp) {
  // anchors are corner boxes [ymin,xmin,ymax,xmax]  (get_center_coordinates_and_sizes)
  float wa = __fsub_rn(a.w, a.y), ha = __fsub_rn(a.z, a.x);
  float ycenter_a = __fadd_rn(a.x, __fdiv_rn(ha, 2.0f));
  float xcenter_a = __fadd_rn(a.y, __fdiv_rn(wa, 2.0f));
  float ty = __fdiv_rn(e.x, pp.scale_y), tx = __fdiv_rn(e.y, pp.scale_x);
  float th = __fdiv_rn(e.z, pp.scale_h), tw = __fdiv_rn(e.w, pp.scale_w);
  float w = __fmul_rn(expf(tw), wa), h = __fmul_rn(expf(th), ha);
  float ycenter = __fadd_rn(__fmul_rn(ty, ha), ycenter_a);
  float xcenter = __fadd_rn(__fmul_rn(tx, wa), xcenter_a);
  float hh = __fdiv_rn(h, 2.0f), hw = __fdiv_rn(w, 2.0f);
  return make_float4(__fsub_rn(ycenter, hh), __fsub_rn(xcenter, hw), __fadd_rn(ycenter, hh),
                     __fadd_rn(xcenter, hw));
}

// `Postprocessor/convert_scores`
__device__ __forceinline__ float sigmoid_score(float logit, float logit_scale) {
  float z = __fdiv_rn(logit, logit_scale);
  return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-z)));
}

// ------------------------------------------------------------------------------------------- K8
// `IOU(a, b) > thr` of TF non_max_suppression_op.cc (IOU<float>(): same op order, each operation separately rounded)
// for boxes whose corners were normalised (min/max) and whose areas were computed once: disjoint boxes are rejected
// after 4 min/max + 2 subtractions, without the IEEE division.  TF's inter = max(dy,0)*max(dx,0) is 0 when dy <= 0 or
// dx <= 0, so its IoU is 0 <= thr there; it also returns 0 when either area is <= 0.
struct NBox {
  float4 c;  // ymin, xmin, ymax, xmax (normalised)
  float area;
};
__device__ __forceinline__ NBox normalise_box(float4 b) {
  NBox r;
  r.c = make_float4(fminf(b.x, b.z), fminf(b.y, b.w), fmaxf(b.x, b.z), fmaxf(b.y, b.w));
  r.area = __fmul_rn(__fsub_rn(r.c.z, r.c.x), __fsub_rn(r.c.w, r.c.y));
  return r;
}
__device__ __forceinline__ bool suppresses(const float4& a, float area_a, const float4& b, float area_b, float thr) {
  const float iy0 = fmaxf(a.x, b.x), ix0 = fmaxf(a.y, b.y), iy1 = fminf(a.z, b.z), ix1 = fminf(a.w, b.w);
  const float dy = __fsub_rn(iy1, iy0), dx = __fsub_rn(ix1, ix0);
  if (!(dy > 0.f && dx > 0.f)) return false;
  if (area_a <= 0.f || area_b <= 0.f) return false;
  const float inter = __fmul_rn(dy, dx);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter)) > thr;
}

__device__ __forceinline__ float4 clip_unit(float4 b) {  // ClipToWindow [0,0,1,1]
  return make_float4(fmaxf(fminf(b.x, 1.f), 0.f), fmaxf(fminf(b.y, 1.f), 0.f), fmaxf(fminf(b.z, 1.f), 0.f),
                     fmaxf(fminf(b.w, 1.f), 0.f));
}

// descending bitonic sort of P (power of two) keys in shared memory, whole block
__device__ __forceinline__ void bitonic_desc(unsigned long long* a, int P) {
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long x = a[i], y = a[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? x < y : x > y) {
            a[i] = y;
            a[ixj] = x;
          }
        }
      }
      __syncthreads();
    }
}

// grid (classes, frames), 256 threads.  Per (frame, class):
//  0. scores: the block reads its class's column of the frame's logits (the heads' [N][C+1] output, L2-resident) and
//     keeps every anchor's sigmoid score in shared memory; anchors at or below the score threshold are marked as no
//     candidate.  A candidate's key  score_bits << 32 | ~anchor  is formed only when it is gathered (sorting keys
//     descending gives "score descending, lower anchor index first", the pop order of TF's NonMaxSuppressionV5).
//  1. candidate keys -> shared memory, in CHUNKS of descending score.  With many candidates (score threshold 1e-8
//     makes every anchor one) only the head of the order is ever visited before max_per_class boxes are kept or the
//     early exit fires (most classes stop after two rounds), so the keys are never sorted as a whole: a score
//     histogram (sign, exponent and 5 mantissa bits of the float: 32 bins per octave), built in the score pass, and
//     each chunk is "the highest remaining bins that hold >= want keys" (96 for the first chunk, 384 after), gathered
//     from the scores in shared memory and sorted (bitonic).  A chunk is a whole number of bins and every key of a
//     higher bin is larger than every key of a lower one, so the visiting order is exactly the descending key order.
//     A class with at most NMS_PREFILTER_MIN candidates is one chunk of every bin.
//  2. greedy suppression with exact sequential semantics, 32 candidates per round; warp 0 decodes the round's
//     candidate boxes from the box encodings and the anchors:
//     phase 1 (all 8 warps): candidate i vs every box kept in EARLIER rounds (warp w takes candidates
//     4w..4w+3, lanes stride over the kept list, a ballot decides);
//     phase 2 (warp 0): walk the 32 candidates in order; a surviving candidate is kept and immediately
//     suppresses the later candidates of the same round that it overlaps.
// Output: merge keys  score_bits << 32 | (0xFFFF - class) << 16 | (0xFFFF - rank)  for the kept boxes whose
// window-clipped area is positive (0 otherwise), plus the decoded corners of every kept box.
constexpr int KEPT_BINS = 1024;
// monotone non-decreasing in the score (scores are sigmoid outputs in [0, 1]); resolution 1/1024
__device__ __forceinline__ int score_bin(unsigned score_bits) {
  return min(KEPT_BINS - 1, max(0, (int)(__uint_as_float(score_bits) * (float)KEPT_BINS)));
}
constexpr int NMS_CHUNK0 = 96;   // keys wanted in the first chunk (three rounds of 32)
constexpr int NMS_CHUNK = 384;   // ... in every later chunk
constexpr int NMS_PREFILTER_MIN = 640;
constexpr int NMS_BINS = 1024;
// bin of a candidate key, monotone non-decreasing in the key: sign + exponent + 5 mantissa bits of the score, counted
// from 2^-27 (scores are in (0, 1]: exponents 100..127; anything smaller lands in bin 0)
__device__ __forceinline__ int nms_bin(unsigned long long key) {
  return min(NMS_BINS - 1, max(0, (int)(key >> 50) - (100 << 5)));
}
__device__ __forceinline__ unsigned long long nms_key(unsigned score_bits, int anchor) {
  return ((unsigned long long)score_bits << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)anchor);
}
constexpr unsigned NMS_NO_CAND = 0xFFFFFFFFu;  // score slot of an anchor that is no candidate (a NaN: never > thr)
constexpr int NMS_LOADS = 4;  // logits in flight per thread in the score pass (8 would spill at 40 registers)

// 720 blocks (8 frames x 90 classes) are one wave on 132 SMs at 6 blocks per SM: at most 40 registers per thread
__global__ void __launch_bounds__(256, 6)
    k_nms(PostParams pp, const float* __restrict__ enc, const float* __restrict__ logits,
          const float* __restrict__ anchors, int sort_cap, int* __restrict__ sel_count,
          unsigned long long* __restrict__ sel_key, float4* __restrict__ sel_box, int* __restrict__ kept_hist) {
  extern __shared__ unsigned long long s_a[];  // [sort_cap]: the current chunk, sorted; then the scores
  unsigned* s_score = reinterpret_cast<unsigned*>(s_a + sort_cap);  // [N]: score bits by anchor, or NMS_NO_CAND
  __shared__ float4 s_kept[128];  // normalised corners of the kept boxes
  __shared__ float s_karea[128];
  __shared__ float4 s_cbox[32];  // normalised corners of the round's candidates
  __shared__ float s_carea[32];
  __shared__ float4 s_craw[32];  // as decoded (for the clipped-area test and the output)
  __shared__ unsigned s_alive;   // bit i: candidate i of the round survived phase 1
  __shared__ int s_nkept_sh, s_na, s_cut, s_n;
  __shared__ int s_hist[NMS_BINS];
  __shared__ int s_above[8];
  int* fhist = kept_hist + (size_t)blockIdx.y * KEPT_BINS;  // this frame's histogram of kept, selectable scores
  const int c = blockIdx.x, f = blockIdx.y, C = pp.num_classes, N = pp.num_anchors;
  const int max_out = min(pp.max_per_class, N);
  unsigned long long* out_key = sel_key + ((size_t)f * C + c) * pp.max_per_class;
  float4* out_box = sel_box + ((size_t)f * C + c) * pp.max_per_class;
  for (int i = threadIdx.x; i < pp.max_per_class; i += blockDim.x) out_key[i] = 0ull;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < NMS_BINS; i += blockDim.x) s_hist[i] = 0;
  if (threadIdx.x == 0) {
    s_n = 0;
    s_nkept_sh = 0;
  }
  __syncthreads();
  // `Postprocessor/convert_scores` + `Postprocessor/Slice` (background column 0 dropped after the sigmoid) for column
  // c + 1: strided 4-byte loads, all of a thread's issued before any is used
  const float* col = logits + (size_t)f * N * (C + 1) + (c + 1);
  int ncand = 0;
  for (int a0 = 0; a0 < N; a0 += NMS_LOADS * blockDim.x) {
    float lg[NMS_LOADS];
#pragma unroll
    for (int k = 0; k < NMS_LOADS; ++k) {
      const int a = a0 + k * blockDim.x + threadIdx.x;
      lg[k] = a < N ? __ldg(col + (size_t)a * (C + 1)) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < NMS_LOADS; ++k) {
      const int a = a0 + k * blockDim.x + threadIdx.x;
      const unsigned sb = __float_as_uint(sigmoid_score(lg[k], pp.logit_scale));
      const bool cand = a < N && __uint_as_float(sb) > pp.score_thr;
      if (a < N) s_score[a] = cand ? sb : NMS_NO_CAND;
      // scores of one class crowd into few bins: aggregate equal bins inside the warp (__match_any_sync) so that one
      // lane per distinct bin issues the shared-memory atomic
      const int bin = cand ? nms_bin(nms_key(sb, a)) : -1;
      const unsigned peers = __match_any_sync(0xffffffffu, bin);
      if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_hist[bin], __popc(peers));
      ncand += cand;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ncand += __shfl_xor_sync(0xffffffffu, ncand, o);
  if (lane == 0 && ncand > 0) atomicAdd(&s_n, ncand);
  __syncthreads();
  const int n = s_n;
  if (n == 0) {
    if (threadIdx.x == 0) sel_count[f * C + c] = 0;
    return;
  }
  const bool chunked = n > NMS_PREFILTER_MIN;
  const float4* fenc = reinterpret_cast<const float4*>(enc) + (size_t)f * N;
  const float4* anc = reinterpret_cast<const float4*>(anchors);

  bool stop = false;
  int hi_bin = NMS_BINS;  // bins >= hi_bin have been visited
  for (int chunk = 0; !stop; ++chunk) {
    if (hi_bin <= 0 || s_nkept_sh >= max_out) break;  // uniform: both were published before a barrier
    const int want = chunk == 0 ? NMS_CHUNK0 : NMS_CHUNK;
    if (warp == 0) {  // highest remaining bins first until `want` keys are covered (or nothing is left: cut = 0)
      int acc = 0, cut = 0;
      for (int top = hi_bin - 1; chunked && top >= 0 && acc < want; top -= 32) {
        const int b = top - lane;
        const int v = b >= 0 ? s_hist[b] : 0;
        int incl = v;  // inclusive prefix over lanes (lane 0 = highest bin)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        const unsigned reach = __ballot_sync(0xffffffffu, acc + incl >= want);
        if (reach) {
          const int l = __ffs(reach) - 1;
          cut = top - l;
          acc += __shfl_sync(0xffffffffu, incl, l);
          break;
        }
        acc += __shfl_sync(0xffffffffu, incl, 31);
        cut = max(top - 31, 0);
      }
      if (lane == 0) {
        s_cut = cut;
        s_na = 0;
      }
    }
    __syncthreads();
    const int cut = s_cut;
    for (int i0 = 0; i0 < N; i0 += blockDim.x) {  // pass over the scores: the candidates in bins [cut, hi_bin)
      const int i = i0 + threadIdx.x;
      const unsigned sb = i < N ? s_score[i] : NMS_NO_CAND;
      const unsigned long long k = nms_key(sb, i);
      const int bin = nms_bin(k);
      const bool in = sb != NMS_NO_CAND && bin >= cut && bin < hi_bin;
      // warp-aggregated append: one shared-memory atomic per warp instead of one per key
      const unsigned m = __ballot_sync(0xffffffffu, in);
      int base_pos = 0;
      if (lane == 0 && m) base_pos = atomicAdd(&s_na, __popc(m));
      base_pos = __shfl_sync(0xffffffffu, base_pos, 0);
      if (in) s_a[base_pos + __popc(m & ((1u << lane) - 1u))] = k;
    }
    __syncthreads();
    const int count = s_na;
    hi_bin = cut;
    if (count == 0) continue;  // uniform; an empty range can only be the last one (cut == 0)
    int P = 32;
    while (P < count) P <<= 1;
    for (int i = count + threadIdx.x; i < P; i += blockDim.x) s_a[i] = 0ull;
    __syncthreads();
    bitonic_desc(s_a, P);
    const unsigned long long* sorted = s_a;
    for (int base = 0; base < count; base += 32) {
      const int nkept = s_nkept_sh;
      if (nkept >= max_out) break;
      if (base > 0 || chunk > 0) {
        // Early exit (exact): the frame-wide histogram counts boxes that some class has already KEPT with a positive
        // clipped area -- final facts.  If max_total of them sit in score bins strictly above this class's best
        // remaining candidate, neither it nor anything after it can reach the frame's top max_total, and whatever
        // this class would still select is never read.  Stale (smaller) counts only delay the exit.
        const int b = score_bin((unsigned)(sorted[base] >> 32));
        int above = 0;
        for (int i = threadIdx.x * 4; i < KEPT_BINS; i += blockDim.x * 4) {
          const int4 h = __ldcg(reinterpret_cast<const int4*>(fhist + i));
          above += (i > b ? h.x : 0) + (i + 1 > b ? h.y : 0) + (i + 2 > b ? h.z : 0) + (i + 3 > b ? h.w : 0);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) above += __shfl_xor_sync(0xffffffffu, above, o);
        if (lane == 0) s_above[warp] = above;
        __syncthreads();
        above = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) above += s_above[w];
        __syncthreads();
        if (above >= pp.max_total) {
          stop = true;
          break;
        }
      }
      const int cnt = min(32, count - base);
      if (threadIdx.x < 32) {
        if (lane < cnt) {
          const unsigned idx = 0xFFFFFFFFu - (unsigned)(sorted[base + lane] & 0xFFFFFFFFull);
          const float4 raw = decode_box(__ldg(fenc + idx), __ldg(anc + idx), pp);
          const NBox nb = normalise_box(raw);
          s_craw[lane] = raw;
          s_cbox[lane] = nb.c;
          s_carea[lane] = nb.area;
        }
        if (lane == 0) s_alive = 0u;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int i = warp * 4 + k;
        if (i < cnt) {
          const float4 bi = s_cbox[i];
          const float ai = s_carea[i];
          bool sup = false;
          for (int j = lane; j < nkept; j += 32) sup |= suppresses(bi, ai, s_kept[j], s_karea[j], pp.iou_thr);
          if (!__any_sync(0xffffffffu, sup) && lane == 0) atomicOr(&s_alive, 1u << i);
        }
      }
      __syncthreads();
      if (warp == 0) {
        unsigned alive = s_alive;
        const float4 box = lane < cnt ? s_cbox[lane] : make_float4(0.f, 0.f, 0.f, 0.f);
        const float barea = lane < cnt ? s_carea[lane] : 0.f;
        int nk = nkept;
        for (int t = 0; t < cnt && nk < max_out; ++t) {
          if (!((alive >> t) & 1u)) continue;  // warp-uniform
          float4 bt;
          bt.x = __shfl_sync(0xffffffffu, box.x, t);
          bt.y = __shfl_sync(0xffffffffu, box.y, t);
          bt.z = __shfl_sync(0xffffffffu, box.z, t);
          bt.w = __shfl_sync(0xffffffffu, box.w, t);
          const float at = __shfl_sync(0xffffffffu, barea, t);
          if (lane == t) {
            const unsigned long long key = sorted[base + t];
            s_kept[nk] = box;
            s_karea[nk] = barea;
            float4 cb = clip_unit(s_craw[t]);
            float area = __fmul_rn(__fsub_rn(cb.z, cb.x), __fsub_rn(cb.w, cb.y));
            out_box[nk] = s_craw[t];
            out_key[nk] = area > 0.f ? ((key & 0xFFFFFFFF00000000ull) | ((unsigned long long)(0xFFFFu - (unsigned)c) << 16) |
                                        (unsigned long long)(0xFFFFu - (unsigned)nk))
                                     : 0ull;
            if (area > 0.f) atomicAdd(&fhist[score_bin((unsigned)(key >> 32))], 1);
          }
          ++nk;
          const bool hit = lane > t && lane < cnt && suppresses(box, barea, bt, at, pp.iou_thr);
          alive &= ~__ballot_sync(0xffffffffu, hit);
        }
        if (lane == 0) s_nkept_sh = nk;
      }
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) sel_count[f * C + c] = s_nkept_sh;
}

// ------------------------------------------------------------------------------------------- K9
__device__ __forceinline__ int sat_count(const int32_t* s, int W1, int x0, int y0, int x1, int y1) {
  return s[(size_t)(y1 + 1) * W1 + (x1 + 1)] - s[(size_t)y0 * W1 + (x1 + 1)] - s[(size_t)(y1 + 1) * W1 + x0] +
         s[(size_t)y0 * W1 + x0];
}

// abs((x1 - x0 + 1) * (y1 - y0 + 1)) >= thr for any int32 corners, compared as Python compares an int with a float:
// exactly.  Each span is taken in 64 bits and is at most 2^32, so the area is at most 2^64: it overflows 64 bits only
// when both spans are 2^32, and then 2^64 >= thr is decided on its own.
__device__ __forceinline__ bool area_at_least(int x0, int y0, int x1, int y1, double thr) {
  const long long sx = (long long)x1 - x0 + 1, sy = (long long)y1 - y0 + 1;
  const unsigned long long ax = (unsigned long long)(sx < 0 ? -sx : sx), ay = (unsigned long long)(sy < 0 ? -sy : sy);
  if (thr <= 0.0) return true;
  if (!(thr <= 18446744073709551616.0)) return false;  // above 2^64, or NaN
  const double c = ceil(thr);                          // an integer area is >= thr iff it is >= ceil(thr)
  if (c == 18446744073709551616.0) return ax == (1ull << 32) && ay == (1ull << 32);
  return __umul64hi(ax, ay) != 0ull || ax * ay >= (unsigned long long)c;
}

// The lazily evaluated predicate chain of watsor/filter/track.py:26.
__device__ uint32_t apply_filters(const CameraCfg* __restrict__ cam, wb_detection* d, bool write_zones) {
  uint32_t v = 0;
  const int lab = d->label;
  if (cam == nullptr) return lab > 0 ? WB_V_LABEL : 0u;
  if (cam->check_label) {
    if (!(lab > 0)) return v;
    v |= WB_V_LABEL;
  }
  bool present = lab >= 0 && lab < WB_MAX_LABELS && cam->present[lab];
  double conf_thr, area_thr;
  uint32_t allowed;
  if (present) {
    conf_thr = cam->conf[lab];
    area_thr = cam->area[lab];
    allowed = cam->has_zone_list[lab] ? cam->zone_bits[lab] : 0xFFFFFFFFu;
  } else if (cam->default_present) {
    present = true;
    conf_thr = cam->default_conf;
    area_thr = cam->default_area;
    allowed = cam->default_has_zone_list ? cam->default_zone_bits : 0xFFFFFFFFu;
  } else {
    return v;  // confidence.py:18 / area.py:21: `... is not None and ...`
  }
  // confidence.py:17-19.  A -inf threshold is no confidence predicate: the stand-alone AreaFilter / MaskFilter tables
  // (area.py and mask.py never read the confidence, so a NaN confidence passes them)
  if (conf_thr != -INFINITY && !(d->confidence >= conf_thr)) return v;
  v |= WB_V_CONFIDENCE;
  // area.py:20-26  abs((x_max - x_min + 1) * (y_max - y_min + 1)) >= pct/100 * W*H
  const wb_bounding_box bb = d->bounding_box;
  if (!area_at_least(bb.x_min, bb.y_min, bb.x_max, bb.y_max, area_thr)) return v;
  v |= WB_V_AREA;
  if (cam->has_mask) {
    // mask.py:44-59: closed bbox rectangle intersects zone polygon  <=>  it covers >= 1 pixel of the
    // filled-contour raster (summed-area table, 4 loads per zone)
    int xa = min(bb.x_min, bb.x_max), xb = max(bb.x_min, bb.x_max);
    int ya = min(bb.y_min, bb.y_max), yb = max(bb.y_min, bb.y_max);
    xa = max(xa, 0);
    ya = max(ya, 0);
    xb = min(xb, cam->width - 1);
    yb = min(yb, cam->height - 1);
    bool hit = false;
    int z = 0;
    if (xa <= xb && ya <= yb) {
      const int W1 = cam->width + 1;
      const size_t plane = (size_t)(cam->height + 1) * W1;
      for (int p = 0; p < cam->n_zones && z < WB_MAX_ZONES; ++p) {
        if (!((allowed >> p) & 1u)) continue;
        if (sat_count(cam->sat + p * plane, W1, xa, ya, xb, yb) > 0) {
          if (write_zones) d->zones[z] = p + 1;
          ++z;
          hit = true;
        }
      }
    }
    if (!hit) return v;
    v |= WB_V_MASK;
  }
  return v | WB_V_PASS;
}

// One block per frame.  (1) the merge keys of all classes (C x max_per_class, zero = not selectable) are streamed
// once: a 2048-bin histogram of their top bits finds the bin that holds the max_total-th largest key; (2) the keys at or
// above that bin (normally ~max_total of them) are gathered into shared memory and sorted descending (bitonic) =
// `SortByField` (TopKV2, ties -> lower concat index: the keys carry (class, rank) below the score, so they are distinct
// and the descending key order IS the C-way merge order of the per-class lists) restricted to boxes with positive
// clipped area, top max_total; (3) one thread per output row: clip, `add` +1, tensorflow_cpu.py:79-90 integer
// conversion, predicates, Detection write.
constexpr int MERGE_THREADS = 512;
constexpr int MERGE_BINS = 2048;   // sign + exponent + 2 mantissa bits of the score
constexpr int MERGE_CAP = 4096;    // gathered keys that fit the fast path (ties in the cut bin can exceed max_total)

__global__ void __launch_bounds__(MERGE_THREADS)
    k_merge_filter(PostParams pp, const int* __restrict__ sel_count, const unsigned long long* __restrict__ sel_key,
                   const float4* __restrict__ sel_box,
                   const FrameDesc* __restrict__ frames, const CameraCfg* __restrict__ cams, uint32_t flags,
                   wb_detection* __restrict__ out, uint32_t* __restrict__ verdicts, float* __restrict__ raw_boxes,
                   float* __restrict__ raw_scores, float* __restrict__ raw_classes, int* __restrict__ raw_num) {
  extern __shared__ unsigned long long s_keys[];  // [cap]: gathered keys (cap = MERGE_CAP, or all keys in the slow path)
  __shared__ int s_hist[MERGE_BINS];
  __shared__ unsigned long long s_win[128];
  __shared__ int s_nvalid, s_cut, s_n;
  const int f = blockIdx.x, C = pp.num_classes, MP = pp.max_per_class;
  const unsigned long long* keys = sel_key + (size_t)f * C * MP;
  const int total = C * MP;
  const int want = min(pp.max_total, 128);
  for (int i = threadIdx.x; i < MERGE_BINS; i += blockDim.x) s_hist[i] = 0;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  // keys beyond a class's selection count were zeroed by k_nms, so the whole [C][MP] block can be read blindly
  for (int i0 = 0; i0 < total; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const unsigned long long k = i < total ? __ldg(keys + i) : 0ull;
    const int bin = k != 0ull ? (int)(k >> 53) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, bin);  // equal bins inside the warp: one atomic
    if (bin >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&s_hist[bin], __popc(peers));
  }
  __syncthreads();
  if (threadIdx.x < 32) {  // highest bins first until `want` keys are covered
    const int lane = threadIdx.x;
    int acc = 0, cut = 0;
    for (int top = MERGE_BINS - 1; top >= 0 && acc < want; top -= 32) {
      const int b = top - lane;
      const int v = b >= 0 ? s_hist[b] : 0;
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const unsigned reach = __ballot_sync(0xffffffffu, acc + incl >= want);
      if (reach) {
        cut = top - (__ffs(reach) - 1);
        acc = want;
        break;
      }
      acc += __shfl_sync(0xffffffffu, incl, 31);
      cut = max(top - 31, 0);
    }
    if (lane == 0) s_cut = cut;
  }
  __syncthreads();
  const int cut = s_cut;
  int cap = MERGE_CAP;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    const unsigned long long k = __ldg(keys + i);  // second pass, L2 / L1 resident
    if (k != 0ull && (int)(k >> 53) >= cut) {
      const int p = atomicAdd(&s_n, 1);
      if (p < cap) s_keys[p] = k;
    }
  }
  __syncthreads();
  int n_g = s_n;
  if (n_g > cap) {
    // pathological: thousands of keys share the cut bin (e.g. every score identical).  Sort everything; the
    // dynamic shared memory was sized for the whole [C][MP] block by the launcher.
    __syncthreads();
    int P = 32;
    while (P < total) P <<= 1;
    for (int i = threadIdx.x; i < P; i += blockDim.x) s_keys[i] = i < total ? __ldg(keys + i) : 0ull;
    n_g = total;
    __syncthreads();
    bitonic_desc(s_keys, P);
  } else {
    int P = 32;
    while (P < n_g) P <<= 1;
    for (int i = n_g + threadIdx.x; i < P; i += blockDim.x) s_keys[i] = 0ull;
    __syncthreads();
    bitonic_desc(s_keys, P);
  }
  if (threadIdx.x < 128) {
    const unsigned long long k = threadIdx.x < min(n_g, want) ? s_keys[threadIdx.x] : 0ull;
    s_win[threadIdx.x] = k;
  }
  if (threadIdx.x == 0) {
    // number of valid rows = non-zero keys among the first `want` (zeros sort last)
    int lo = 0, hi = min(n_g, want);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (s_keys[mid] != 0ull) lo = mid + 1; else hi = mid;
    }
    s_nvalid = lo;
  }
  __syncthreads();
  const int nvalid = s_nvalid;
  const int r = threadIdx.x;
  if (r == 0 && raw_num) raw_num[f] = nvalid;
  if (r >= WB_MAX_DETECTIONS) return;
  float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
  float score = 0.f, cls = 0.f;
  if (r < nvalid && r < pp.max_total) {
    unsigned long long k = s_win[r];
    int c = 0xFFFF - (int)((k >> 16) & 0xFFFFull), rank = 0xFFFF - (int)(k & 0xFFFFull);
    score = __uint_as_float((unsigned)(k >> 32));
    cls = (float)c;
    box = clip_unit(sel_box[((size_t)f * C + c) * MP + rank]);
  }
  cls = __fadd_rn(cls, pp.class_offset);  // graph node `add` (+1 also on the zero padding)
  if (raw_boxes) {
    reinterpret_cast<float4*>(raw_boxes)[(size_t)f * WB_MAX_DETECTIONS + r] = box;
    raw_scores[(size_t)f * WB_MAX_DETECTIONS + r] = score;
    raw_classes[(size_t)f * WB_MAX_DETECTIONS + r] = cls;
  }
  const FrameDesc fd = frames[f];
  wb_detection d;
  d.label = (int)cls;
  for (int z = 0; z < WB_MAX_ZONES; ++z) d.zones[z] = 0;
  d.confidence = (double)score;
  // int(np.float32 * int): exact product (float64), truncation toward zero
  const double mh = (double)(fd.h - 1), mw = (double)(fd.w - 1);
  d.bounding_box.y_min = (int)((double)box.x * mh);
  d.bounding_box.x_min = (int)((double)box.y * mw);
  d.bounding_box.y_max = (int)((double)box.z * mh);
  d.bounding_box.x_max = (int)((double)box.w * mw);
  const CameraCfg* cam = (cams != nullptr && fd.cam >= 0) ? cams + fd.cam : nullptr;
  uint32_t v = apply_filters(cam, &d, (flags & WB_F_FUSE_FILTERS) != 0);
  out[(size_t)f * WB_MAX_DETECTIONS + r] = d;
  if (verdicts) verdicts[(size_t)f * WB_MAX_DETECTIONS + r] = v;
}

void launch_post(const LaunchCtx& lc, int n, const PostParams& pp, const float* enc, const float* logits,
                 const float* anchors, const FrameDesc* frames, const CameraCfg* cams, uint32_t flags,
                 int* sel_count, unsigned long long* sel_key, float4* sel_box, wb_detection* out, uint32_t* verdicts,
                 float* raw_boxes, float* raw_scores, float* raw_classes, int* raw_num, int* kept_hist) {
  const int C = pp.num_classes, N = pp.num_anchors;
  cudaMemsetAsync(kept_hist, 0, sizeof(int) * (size_t)n * KEPT_BINS, lc.stream);
  int sort_cap = 32;
  while (sort_cap < N) sort_cap <<= 1;
  static PerDeviceFlag nms_attr, merge_attr;
  max_dynamic_smem_once(k_nms, 200 * 1024, nms_attr);
  max_dynamic_smem_once(k_merge_filter, 160 * 1024, merge_attr);
  // the chunk buffer (every key may land in one chunk) and the scores: 23.5 KB for 1917 anchors
  const size_t nms_smem = sizeof(unsigned long long) * sort_cap + sizeof(unsigned) * (size_t)N;
  k_nms<<<dim3(C, n), 256, nms_smem, lc.stream>>>(pp, enc, logits, anchors, sort_cap, sel_count, sel_key, sel_box,
                                                  kept_hist);
  ++*lc.launch_counter;
  {
    int P = 32;
    while (P < C * pp.max_per_class) P <<= 1;
    const size_t merge_smem = sizeof(unsigned long long) * (size_t)std::max(P, MERGE_CAP);
    k_merge_filter<<<n, MERGE_THREADS, merge_smem, lc.stream>>>(pp, sel_count, sel_key, sel_box, frames, cams, flags,
                                                                out, verdicts, raw_boxes, raw_scores, raw_classes,
                                                                raw_num);
  }
  ++*lc.launch_counter;
}

// ------------------------------------------------------------------------------------------- window merge
// One block per frame of a batch with detection windows (wb_set_camera_windows).  k_merge_filter has written every
// window's rows (camera -1: no predicates) and its number of valid rows (raw_num).  Those rows are sorted by the key
// score_bits << 32 | ~(window << 8 | row) -- confidence descending, then window, then row: scores are >= 0, so the
// float's bits order like its value, and padding keys (0) sort last.  One warp walks the sorted rows and keeps a row
// unless an already kept row with the same label from ANOTHER window covers more than merge_thr of the smaller box
// (intersection over the smaller of the two integer, inclusive pixel boxes, after the shift by the window's origin).
// Rows of one window never suppress each other: the model's NMS has decided between them.  IoS rather than IoU: a part
// of an object cut by a window border lies inside the whole box seen by a neighbouring or the full-frame window.  The
// first max_total kept rows, then padding rows as k_merge_filter writes them, go through the camera's predicates.
constexpr int WM_THREADS = 256;
constexpr int WM_KEYS = 2048;  // >= WB_MAX_WINDOWS * WB_MAX_DETECTIONS, a power of two
static_assert(WM_KEYS >= WB_MAX_WINDOWS * WB_MAX_DETECTIONS, "window merge keys");

__global__ void __launch_bounds__(WM_THREADS)
    k_window_merge(PostParams pp, const WindowFrame* __restrict__ win, const wb_detection* __restrict__ rows,
                   const int* __restrict__ raw_num, const CameraCfg* __restrict__ cams, uint32_t flags,
                   wb_detection* __restrict__ out, uint32_t* __restrict__ verdicts) {
  __shared__ unsigned long long s_keys[WM_KEYS];
  __shared__ int4 s_kbox[WB_MAX_DETECTIONS];  // kept rows: x_min, y_min, x_max, y_max in camera pixels
  __shared__ long long s_karea[WB_MAX_DETECTIONS];
  __shared__ int s_klab[WB_MAX_DETECTIONS], s_kid[WB_MAX_DETECTIONS];  // label, window << 8 | row
  __shared__ int s_nvalid[WB_MAX_WINDOWS];
  __shared__ int s_nkept;
  const int f = blockIdx.x;
  const WindowFrame& wf = win[f];
  const int first = wf.first, count = wf.count;
  const int max_out = min(pp.max_total, WB_MAX_DETECTIONS);
  if ((int)threadIdx.x < count) s_nvalid[threadIdx.x] = min(raw_num[first + threadIdx.x], WB_MAX_DETECTIONS);
  __syncthreads();
  int P = 32;
  while (P < count * WB_MAX_DETECTIONS) P <<= 1;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const int w = i / WB_MAX_DETECTIONS, r = i - w * WB_MAX_DETECTIONS;
    unsigned long long k = 0ull;
    if (w < count && r < s_nvalid[w]) {
      const float score = (float)rows[(size_t)(first + w) * WB_MAX_DETECTIONS + r].confidence;  // exact: it was a float
      k = ((unsigned long long)__float_as_uint(score) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)(w << 8 | r));
    }
    s_keys[i] = k;
  }
  __syncthreads();
  bitonic_desc(s_keys, P);
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    int total = 0;
    for (int w = 0; w < count; ++w) total += s_nvalid[w];
    const double thr = wf.merge_thr;
    int nk = 0;
    for (int base = 0; base < total && nk < max_out; base += 32) {
      // lane l fetches candidate base + l; the candidates are then decided one after another
      const int cnt = min(32, total - base);
      int id = 0, lab = 0;
      int4 b = make_int4(0, 0, 0, 0);
      long long area = 0;
      if (lane < cnt) {
        id = (int)(0xFFFFFFFFu - (unsigned)(s_keys[base + lane] & 0xFFFFFFFFull));
        const int w = id >> 8;
        const wb_detection& d = rows[(size_t)(first + w) * WB_MAX_DETECTIONS + (id & 255)];
        lab = d.label;
        b = make_int4(d.bounding_box.x_min + wf.x[w], d.bounding_box.y_min + wf.y[w], d.bounding_box.x_max + wf.x[w],
                      d.bounding_box.y_max + wf.y[w]);
        area = ((long long)b.z - b.x + 1) * ((long long)b.w - b.y + 1);
      }
      for (int t = 0; t < cnt && nk < max_out; ++t) {
        const int tid = __shfl_sync(0xffffffffu, id, t), tlab = __shfl_sync(0xffffffffu, lab, t);
        const int4 tb = make_int4(__shfl_sync(0xffffffffu, b.x, t), __shfl_sync(0xffffffffu, b.y, t),
                                  __shfl_sync(0xffffffffu, b.z, t), __shfl_sync(0xffffffffu, b.w, t));
        const long long tarea = __shfl_sync(0xffffffffu, area, t);
        bool sup = false;
        for (int j = lane; j < nk; j += 32) {
          if (s_klab[j] != tlab || (s_kid[j] >> 8) == (tid >> 8)) continue;
          const int4 kb = s_kbox[j];
          const long long iw = (long long)min(tb.z, kb.z) - max(tb.x, kb.x) + 1;
          const long long ih = (long long)min(tb.w, kb.w) - max(tb.y, kb.y) + 1;
          const long long inter = iw > 0 && ih > 0 ? iw * ih : 0;
          sup |= (double)inter > __dmul_rn(thr, (double)min(tarea, s_karea[j]));
        }
        if (__any_sync(0xffffffffu, sup)) continue;  // warp-uniform
        if (lane == t) {
          s_kbox[nk] = b;
          s_karea[nk] = area;
          s_klab[nk] = lab;
          s_kid[nk] = id;
        }
        ++nk;
        __syncwarp();
      }
    }
    if (lane == 0) s_nkept = nk;
  }
  __syncthreads();
  const int r = threadIdx.x;
  if (r >= WB_MAX_DETECTIONS) return;
  wb_detection d;
  for (int z = 0; z < WB_MAX_ZONES; ++z) d.zones[z] = 0;
  if (r < s_nkept) {
    const int id = s_kid[r];
    const wb_detection& src = rows[(size_t)(first + (id >> 8)) * WB_MAX_DETECTIONS + (id & 255)];
    const int4 b = s_kbox[r];
    d.label = src.label;
    d.confidence = src.confidence;
    d.bounding_box.x_min = b.x;
    d.bounding_box.y_min = b.y;
    d.bounding_box.x_max = b.z;
    d.bounding_box.y_max = b.w;
  } else {  // k_merge_filter's padding row
    d.label = (int)__fadd_rn(0.f, pp.class_offset);
    d.confidence = 0.0;
    d.bounding_box.x_min = d.bounding_box.y_min = d.bounding_box.x_max = d.bounding_box.y_max = 0;
  }
  const CameraCfg* cam = cams != nullptr && wf.cam >= 0 ? cams + wf.cam : nullptr;
  const uint32_t v = apply_filters(cam, &d, (flags & WB_F_FUSE_FILTERS) != 0);
  out[(size_t)f * WB_MAX_DETECTIONS + r] = d;
  if (verdicts) verdicts[(size_t)f * WB_MAX_DETECTIONS + r] = v;
}

void launch_window_merge(const LaunchCtx& lc, int n_frames, const PostParams& pp, const WindowFrame* win,
                         const wb_detection* rows, const int* raw_num, const CameraCfg* cams, uint32_t flags,
                         wb_detection* out, uint32_t* verdicts) {
  k_window_merge<<<n_frames, WM_THREADS, 0, lc.stream>>>(pp, win, rows, raw_num, cams, flags, out, verdicts);
  ++*lc.launch_counter;
}

// ---------------------------------------------------------------------------------------------------
// stand-alone predicate chain on caller rows (ConfidenceFilter / AreaFilter / MaskFilter __call__)
__global__ void k_filter_rows(const CameraCfg* __restrict__ cam, int n_rows, wb_detection* __restrict__ rows,
                              uint32_t* __restrict__ verdicts) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  wb_detection d = rows[r];
  uint32_t v = apply_filters(cam, &d, true);
  rows[r] = d;
  verdicts[r] = v;
}
void launch_filter_rows(const LaunchCtx& lc, const CameraCfg* cam, int n_rows, wb_detection* rows,
                        uint32_t* verdicts) {
  k_filter_rows<<<(n_rows + 127) / 128, 128, 0, lc.stream>>>(cam, n_rows, rows, verdicts);
  ++*lc.launch_counter;
}

// ---------------------------------------------------------------------------------------------------
// summed-area tables of the zone rasters (MaskFilter.__init__): sat[z][y][x] = #zone pixels in
// rows < y, cols < x.  Two passes (row scan, column scan); set-up time only.
__global__ void k_sat_rows(const uint8_t* __restrict__ raster, int n_zones, int h, int w, int32_t* __restrict__ sat) {
  int y = blockIdx.x * blockDim.x + threadIdx.x, z = blockIdx.y;
  if (y > h) return;
  int32_t* row = sat + ((size_t)z * (h + 1) + y) * (w + 1);
  row[0] = 0;
  if (y == 0) {
    for (int x = 1; x <= w; ++x) row[x] = 0;
    return;
  }
  const uint8_t* src = raster + ((size_t)z * h + (y - 1)) * w;
  int run = 0;
  for (int x = 0; x < w; ++x) {
    run += src[x] ? 1 : 0;
    row[x + 1] = run;
  }
}
__global__ void k_sat_cols(int n_zones, int h, int w, int32_t* __restrict__ sat) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, z = blockIdx.y;
  if (x > w) return;
  int32_t* base = sat + (size_t)z * (h + 1) * (w + 1) + x;
  int run = 0;
  for (int y = 0; y <= h; ++y) {
    run += base[(size_t)y * (w + 1)];
    base[(size_t)y * (w + 1)] = run;
  }
}
void launch_build_sat(const LaunchCtx& lc, const uint8_t* raster, int n_zones, int h, int w, int32_t* sat) {
  k_sat_rows<<<dim3((h + 1 + 127) / 128, n_zones), 128, 0, lc.stream>>>(raster, n_zones, h, w, sat);
  k_sat_cols<<<dim3((w + 1 + 127) / 128, n_zones), 128, 0, lc.stream>>>(n_zones, h, w, sat);
  *lc.launch_counter += 2;
}
