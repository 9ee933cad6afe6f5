// MultiProposalTarget on device, zero host round trips.
//
// Replaces SNIPER-mxnet/src/operator/multi_proposal_target.cu (MultiProposalTargetGPUOp::Forward,
// :362-589): getProps (:263-331) -> mpt_decode_kernel; NonMaximumSuppression (:117-260) plus the
// host-side GT-append / IoU / label / bbox-target section (:435-588) -> mpt_nms_assign_kernel.
// Semantics are the reference GPU operator's (not the .cc CPU operator's); arithmetic is written
// with explicit round-to-nearest intrinsics so that no FMA contraction can change a bit relative
// to oracle/mpt.c.
//
// Layout in HBM (per call workspace):  boxes float4[B*A*H*W] | score float[B*A*H*W] | area float[..]
// (SoA instead of the reference's 6-float AoS rows: 16-byte box loads, coalesced score scans).
#include "common.cuh"
#include <math.h>
#include <stdlib.h>

namespace {

constexpr int kMaxAnchors = 64;
struct AnchorTable {
  float v[4 * kMaxAnchors];
};

// Same fixed operation sequence as oracle_expf (oracle/mpt.c): double arithmetic, one rounding.
__device__ __forceinline__ float sn_expf(float x) {
  if (x != x) return x;
  double xd = (double)x;
  if (xd > 100.0) return __int_as_float(0x7f800000);
  if (xd < -110.0) return 0.0f;
  double k = rint(__dmul_rn(xd, 1.4426950408889634));
  double r = __fma_rn(-k, 0.6931471803691238, xd);
  r = __fma_rn(-k, 1.9082149292705877e-10, r);
  double p = 1.0 / 39916800.0;
  p = __fma_rn(p, r, 1.0 / 3628800.0);
  p = __fma_rn(p, r, 1.0 / 362880.0);
  p = __fma_rn(p, r, 1.0 / 40320.0);
  p = __fma_rn(p, r, 1.0 / 5040.0);
  p = __fma_rn(p, r, 1.0 / 720.0);
  p = __fma_rn(p, r, 1.0 / 120.0);
  p = __fma_rn(p, r, 1.0 / 24.0);
  p = __fma_rn(p, r, 1.0 / 6.0);
  p = __fma_rn(p, r, 0.5);
  p = __fma_rn(p, r, 1.0);
  p = __fma_rn(p, r, 1.0);
  long long ki = (long long)k;
  double s = __longlong_as_double((ki + 1023) << 52);
  return (float)__dmul_rn(p, s);
}

// layout 0: NCHW (reference), layout 1: NHWC with channel strides c_score / c_delta.
struct DecodeArgs {
  const float* scores;   // fg score of anchor a = channel (A + a)
  const float* deltas;   // channels 4a..4a+3
  const float* im_info;  // [B,3] (h, w, scale)
  const float* valid_ranges;  // [B,2]
  int B, A, H, W, stride, layout;
  int score_cstride, delta_cstride;  // NHWC: number of channels per pixel in each tensor
  int variant;         // 0: MultiProposalTarget (multi_proposal_target.cu:263-331); 1: MultiProposal inference
                       //    (multi_proposal.cc:91-105,176: min-size test with +1 and ||, box grown by 1.5, area with +1,
                       //    no valid-range filter)
  int suppress_types;  // variant 1: anchor types (a+4)%7==0 || (a+2)%7==0 get score -1 (multi_proposal.cu:505-508)
  float4* boxes;
  float* score_out;
  float* area_out;
};

__global__ void __launch_bounds__(256) mpt_decode_kernel(DecodeArgs p, AnchorTable anchors) {
  const int HW = p.H * p.W;
  const int AHW = p.A * HW;
  const long total = (long)p.B * AHW;
  for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
    const int b = (int)(t / AHW);
    const int index = (int)(t - (long)b * AHW);
    const int a = index / HW;
    const int mat = index - a * HW;
    const int h = mat / p.W;
    const int w = mat - h * p.W;
    float score, dx, dy, dw, dh;
    if (p.layout == 0) {
      score = __ldg(p.scores + (size_t)b * AHW * 2 + (size_t)((p.A + a) * p.H + h) * p.W + w);
      const float* d = p.deltas + (size_t)b * AHW * 4 + (size_t)a * 4 * HW + h * p.W + w;
      dx = __ldg(d);
      dy = __ldg(d + HW);
      dw = __ldg(d + 2 * HW);
      dh = __ldg(d + 3 * HW);
    } else {
      const size_t pix = (size_t)b * HW + mat;
      score = __ldg(p.scores + pix * p.score_cstride + p.A + a);
      const float4 d4 = __ldg(reinterpret_cast<const float4*>(p.deltas + pix * p.delta_cstride + 4 * a));
      dx = d4.x; dy = d4.y; dw = d4.z; dh = d4.w;
    }
    float bx0 = __fadd_rn(anchors.v[4 * a + 0], (float)(w * p.stride));
    float by0 = __fadd_rn(anchors.v[4 * a + 1], (float)(h * p.stride));
    float bx1 = __fadd_rn(anchors.v[4 * a + 2], (float)(w * p.stride));
    float by1 = __fadd_rn(anchors.v[4 * a + 3], (float)(h * p.stride));
    const float width = (float)__dadd_rn((double)__fsub_rn(bx1, bx0), 1.0);
    const float height = (float)__dadd_rn((double)__fsub_rn(by1, by0), 1.0);
    const float ctr_x = (float)__dadd_rn((double)bx0, __dmul_rn(0.5, __dadd_rn((double)width, -1.0)));
    const float ctr_y = (float)__dadd_rn((double)by0, __dmul_rn(0.5, __dadd_rn((double)height, -1.0)));
    const float pred_ctr_x = __fadd_rn(__fmul_rn(dx, width), ctr_x);
    const float pred_ctr_y = __fadd_rn(__fmul_rn(dy, height), ctr_y);
    const float pred_w = __fmul_rn(sn_expf(dw), width);
    const float pred_h = __fmul_rn(sn_expf(dh), height);
    const double hw_ = __dmul_rn(0.5, __dadd_rn((double)pred_w, -1.0));
    const double hh_ = __dmul_rn(0.5, __dadd_rn((double)pred_h, -1.0));
    float x1 = (float)__dadd_rn((double)pred_ctr_x, -hw_);
    float y1 = (float)__dadd_rn((double)pred_ctr_y, -hh_);
    float x2 = (float)__dadd_rn((double)pred_ctr_x, hw_);
    float y2 = (float)__dadd_rn((double)pred_ctr_y, hh_);
    const float imw = __fsub_rn(__ldg(p.im_info + 3 * b + 1), 1.0f);
    const float imh = __fsub_rn(__ldg(p.im_info + 3 * b), 1.0f);
    x1 = fmaxf(fminf(x1, imw), 0.0f);
    y1 = fmaxf(fminf(y1, imh), 0.0f);
    x2 = fmaxf(fminf(x2, imw), 0.0f);
    y2 = fmaxf(fminf(y2, imh), 0.0f);
    float area;
    if (p.variant == 0) {
      if (__fsub_rn(y2, y1) < 3.0f && __fsub_rn(x2, x1) < 3.0f) {
        x1 = __fsub_rn(x1, 1.0f);
        y1 = __fsub_rn(y1, 1.0f);
        x2 = __fadd_rn(x2, 1.0f);
        y2 = __fadd_rn(y2, 1.0f);
        score = -1.0f;
      }
      area = __fmul_rn(__fsub_rn(x2, x1), __fsub_rn(y2, y1));
      const float vr0 = __ldg(p.valid_ranges + 2 * b), vr1 = __ldg(p.valid_ranges + 2 * b + 1);
      if (area >= __fmul_rn(vr1, vr1) || area < __fmul_rn(vr0, vr0)) score = -1.0f;
    } else {
      if (p.suppress_types && ((a + 4) % 7 == 0 || (a + 2) % 7 == 0)) score = -1.0f;
      const float iw = __fadd_rn(__fsub_rn(x2, x1), 1.0f), ih = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
      if (iw < 3.0f || ih < 3.0f) {
        x1 = __fsub_rn(x1, 1.5f);
        y1 = __fsub_rn(y1, 1.5f);
        x2 = __fadd_rn(x2, 1.5f);
        y2 = __fadd_rn(y2, 1.5f);
        score = -1.0f;
      }
      area = __fmul_rn(__fadd_rn(__fsub_rn(x2, x1), 1.0f), __fadd_rn(__fsub_rn(y2, y1), 1.0f));
    }
    p.boxes[t] = make_float4(x1, y1, x2, y2);
    p.score_out[t] = score;
    p.area_out[t] = area;
  }
}

__device__ __forceinline__ uint32_t ord_desc(float f) {
  // monotone map float -> uint32 such that larger float => smaller uint (for min-reduction)
  uint32_t u = __float_as_uint(f);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~u;
}
__device__ __forceinline__ float ord_desc_inv(uint32_t k) {
  uint32_t u = ~k;
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  return __uint_as_float(u);
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    unsigned long long o = __shfl_xor_sync(0xffffffffu, v, off);
    v = o < v ? o : v;
  }
  return v;
}

__device__ __forceinline__ float iou_ref(float ix1, float iy1, float ix2, float iy2, float iarea, float4 d,
                                         float darea) {
  // multi_proposal_target.cu:229-237: inter uses +1, areas do not
  const float xx1 = fmaxf(ix1, d.x), yy1 = fmaxf(iy1, d.y);
  const float xx2 = fminf(ix2, d.z), yy2 = fminf(iy2, d.w);
  const float w = fmaxf(0.0f, __fadd_rn(__fsub_rn(xx2, xx1), 1.0f));
  const float h = fmaxf(0.0f, __fadd_rn(__fsub_rn(yy2, yy1), 1.0f));
  const float inter = __fmul_rn(w, h);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(iarea, darea), inter));
}

// "FastNMS" of the reference's GPU-build inference operator (multi_proposal.cu:267-387, 511-575): a kept proposal only
// tests the anchors listed in a precomputed anchor-overlap map -- anchor type c2 at grid offset (row j, column k) is
// listed for c1 iff the IoU of the two UNDECODED anchors is >= roi_iou_thresh -- and the reference applies the stored
// (row, column) offsets as (dw, dh), i.e. swapped.  The map is a pure function of (c1, c2, |dw|, |dh|) and is evaluated
// on the fly here.  enabled = 0: every pair is tested (exact NMS).
struct OverlapMap {
  int enabled;
  int H, W, stride;
  float thresh;
  const int32_t* id_map;   // row of the (compacted) arrays -> original anchor index a*H*W + h*W + w; null = identity
  float anchors[4 * kMaxAnchors];
  float area[kMaxAnchors];
};

__device__ __forceinline__ bool overlap_listed(const OverlapMap& m, int id1, int id2) {
  const int hw = m.H * m.W;
  const int c1 = id1 / hw, r1 = id1 - c1 * hw, h1 = r1 / m.W, w1 = r1 - h1 * m.W;
  const int c2 = id2 / hw, r2 = id2 - c2 * hw, h2 = r2 / m.W, w2 = r2 - h2 * m.W;
  const int j = abs(w2 - w1), k = abs(h2 - h1);      // dx = +-j is a ROW offset of the map, dy = +-k a COLUMN offset
  if (j >= m.H || k >= m.W) return false;
  if (j == 0 && k == 0 && c2 == c1) return false;
  const float sx = (float)(k * m.stride), sy = (float)(j * m.stride);
  const float xx1 = fmaxf(m.anchors[4 * c1], __fadd_rn(m.anchors[4 * c2], sx));
  const float yy1 = fmaxf(m.anchors[4 * c1 + 1], __fadd_rn(m.anchors[4 * c2 + 1], sy));
  const float xx2 = fminf(m.anchors[4 * c1 + 2], __fadd_rn(m.anchors[4 * c2 + 2], sx));
  const float yy2 = fminf(m.anchors[4 * c1 + 3], __fadd_rn(m.anchors[4 * c2 + 3], sy));
  const float w = fmaxf(0.0f, __fadd_rn(__fsub_rn(xx2, xx1), 1.0f));
  const float h = fmaxf(0.0f, __fadd_rn(__fsub_rn(yy2, yy1), 1.0f));
  const float inter = __fmul_rn(w, h);
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(m.area[c1], m.area[c2]), inter));
  return ovr >= m.thresh;
}
__device__ __forceinline__ int orig_id(const OverlapMap& m, size_t chip_base, int row) {
  return m.id_map ? m.id_map[chip_base + row] : row;
}

struct NmsArgs {
  const float4* boxes;
  const float* scores;
  const float* areas;
  const float* gt_boxes;      // [B,max_gt,5]
  const float* valid_ranges;  // [B,2]
  int AHW, R, max_gt;
  float nms_thresh;
  float* rois;         // [B*R,5]
  float* label;        // [B*R]
  float* bbox_target;  // [B*R,4]
  float* bbox_weight;  // [B*R,4]
  int32_t* keep_idx;   // optional [B*R]
  int32_t* num_kept;   // optional [B]
  int do_assign;       // 0: proposals only (MultiProposal-style output), 1: full target assignment
  const int32_t* id_map;   // optional [B*AHW]: original anchor index of every (compacted) row, reported in keep_idx
  float* score_out;        // optional [B*R]: score of the kept rows, 0 for filler rows (do_assign = 0)
  long filler_stride;      // rows per chip used by the filler rule (cu:244-249); AHW unless the rows are compacted
  OverlapMap omap;         // FastNMS pair restriction (inference operator, GPU build); enabled = 0 otherwise
  const int32_t* fast_keep;      // optional results of mpt_nms_fast_kernel: [B,1024], [B], [B]
  const int32_t* fast_nkept;
  const int32_t* fast_fallback;
  int index_ties;          // 1: equal scores are kept in ascending row order (MultiProposal); 0: the reference's scan order
};

constexpr int kNmsThreads = 1024;

// ------------------------------------------------------------------------------------------------
// Fast path of the greedy NMS: two-level score histogram -> top <= 4096 candidates -> exact bitonic sort ->
// trips of <= 64 candidates resolved with IoU bit masks (ballot / shuffle reductions) by one thread.  Exact score
// ties: with index_ties (the inference operator) in ascending row order, i.e. the sorted order of the (score, row)
// keys; otherwise (MultiProposalTarget) the thread replays the reference's row swaps, so ties are broken in the
// reference's scan order (lexicographic (d%32, (d%1024)/32, d/1024) of the candidate's current row distance d to
// the front).  It falls back (flag) to the round-by-round emulation in mpt_nms_assign_kernel when a run of equal scores
// is longer than a trip, when more than 4096 candidates share the boundary sub-bin, or when the selection
// is exhausted before R boxes are kept while unselected valid candidates remain.
constexpr int kFastCap = 4096;          // candidates sorted per chip
constexpr int kFastBins = 4096;

struct FastArgs {
  const float4* boxes;
  const float* scores;
  const float* areas;
  int AHW, R;
  float nms_thresh;
  int32_t* keep_ids;   // [B,1024]
  int32_t* nkept;      // [B]
  int32_t* fallback;   // [B]
  OverlapMap omap;
  int index_ties;      // as NmsArgs::index_ties
};

__device__ __forceinline__ int score_bin(float s) {
  return (int)(fminf(fmaxf(s, 0.0f), 1.0f) * (float)(kFastBins - 1));
}
// position of s inside its coarse bin, again kFastBins levels; monotone in s for a fixed coarse bin
__device__ __forceinline__ int score_subbin(float s, int q) {
  const float f = fminf(fmaxf(s, 0.0f), 1.0f) * (float)(kFastBins - 1) - (float)q;   // in [0,1)
  const int r = (int)(f * (float)kFastBins);
  return r < 0 ? 0 : (r > kFastBins - 1 ? kFastBins - 1 : r);
}

// Scans s_hist from the top bin down (thread t owns 4 bins) and returns, in *out, the number D of leading
// bins whose cumulative count stays <= cap, and in *cum_out the count inside those D bins.
__device__ __forceinline__ void top_prefix(const int* s_hist, int cap, int t, int lane, int warp, int* s_wsum,
                                           int* out_D, int* out_cum) {
  int h[4];
  int mine = 0;
#pragma unroll
  for (int u = 0; u < 4; ++u) { h[u] = s_hist[kFastBins - 1 - (4 * t + u)]; mine += h[u]; }
  int incl = mine;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += v;
  }
  if (lane == 31) s_wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = s_wsum[lane];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, w, off);
      if (lane >= off) w += v;
    }
    s_wsum[lane] = w;
  }
  __syncthreads();
  int c = incl - mine + (warp ? s_wsum[warp - 1] : 0);
  int ok = 0, okc = 0;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    c += h[u];
    if (c <= cap) { ++ok; okc += h[u]; }
  }
  ok = __reduce_add_sync(0xffffffffu, ok);
  okc = __reduce_add_sync(0xffffffffu, okc);
  if (lane == 0 && ok) { atomicAdd(out_D, ok); atomicAdd(out_cum, okc); }
  __syncthreads();
}

__global__ void __launch_bounds__(kNmsThreads, 1) mpt_nms_fast_kernel(FastArgs p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* s_key = reinterpret_cast<unsigned long long*>(smem_raw);              // [kFastCap]
  float4* s_box = reinterpret_cast<float4*>(s_key + kFastCap);                              // [kFastCap]
  float* s_area = reinterpret_cast<float*>(s_box + kFastCap);                               // [kFastCap]
  int* s_hist = reinterpret_cast<int*>(s_area + kFastCap);                                  // [kFastBins]
  float4* s_kbox = reinterpret_cast<float4*>(s_hist + kFastBins);                           // [1024]
  float* s_karea = reinterpret_cast<float*>(s_kbox + 1024);                                 // [1024]
  unsigned long long* s_mask = reinterpret_cast<unsigned long long*>(s_karea + 1024);       // [64]
  int* s_alive = reinterpret_cast<int*>(s_mask + 64);                                       // [64]
  unsigned short* s_pos = reinterpret_cast<unsigned short*>(s_alive + 64);                  // [kFastCap] current row
  short* s_atpos = reinterpret_cast<short*>(s_pos + kFastCap);                              // [1024] row -> sorted idx
  __shared__ int s_D, s_cum, s_D2, s_cum2, s_nsel, s_nvalid, s_bad, s_nk, s_wsum[32];
  __shared__ int s_koid[1024];   // original anchor index of the kept boxes (FastNMS map)
  const int chip = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int AHW = p.AHW;
  const size_t chip_base = (size_t)chip * AHW;
  const float* sc = p.scores + (size_t)chip * AHW;
  const float4* boxes = p.boxes + (size_t)chip * AHW;
  const float* areas = p.areas + (size_t)chip * AHW;
  for (int i = t; i < kFastBins; i += kNmsThreads) s_hist[i] = 0;
  if (t == 0) { s_nsel = 0; s_nvalid = 0; s_bad = 0; s_nk = 0; s_D = 0; s_cum = 0; s_D2 = 0; s_cum2 = 0; }
  __syncthreads();
  // ---- 1. coarse histogram of the scores (bins are monotone in the score)
  int nv = 0;
  for (int i = t; i < AHW; i += kNmsThreads) {
    const float s = sc[i];
    if (s != -1.0f) {
      atomicAdd(&s_hist[score_bin(s)], 1);
      ++nv;
    }
  }
  nv = __reduce_add_sync(0xffffffffu, nv);
  if (lane == 0 && nv) atomicAdd(&s_nvalid, nv);
  __syncthreads();
  top_prefix(s_hist, kFastCap, t, lane, warp, s_wsum, &s_D, &s_cum);
  const int qb = kFastBins - 1 - s_D;   // boundary bin: taken only partially (or -1 if everything fits)
  const int above = s_cum;              // candidates in bins > qb
  // ---- 2. refine inside the boundary bin
  int sub_star = kFastBins;             // sub-bins >= sub_star of bin qb are selected
  if (qb >= 0) {
    for (int i = t; i < kFastBins; i += kNmsThreads) s_hist[i] = 0;
    __syncthreads();
    for (int i = t; i < AHW; i += kNmsThreads) {
      const float s = sc[i];
      if (s != -1.0f && score_bin(s) == qb) atomicAdd(&s_hist[score_subbin(s, qb)], 1);
    }
    __syncthreads();
    top_prefix(s_hist, kFastCap - above, t, lane, warp, s_wsum, &s_D2, &s_cum2);
    sub_star = kFastBins - s_D2;
  }
  // ---- 3. gather the selected candidates as 64-bit keys (score descending, then index)
  for (int i = t; i < kFastCap; i += kNmsThreads) s_key[i] = ~0ull;
  for (int i = t; i < 1024; i += kNmsThreads) s_atpos[i] = -1;
  __syncthreads();
  for (int i = t; i < AHW; i += kNmsThreads) {
    const float s = sc[i];
    if (s != -1.0f) {
      const int q = score_bin(s);
      if (q > qb || (q == qb && score_subbin(s, q) >= sub_star)) {
        const int slot = atomicAdd(&s_nsel, 1);
        if (slot < kFastCap) s_key[slot] = ((unsigned long long)ord_desc(s) << 32) | (unsigned)i;
      }
    }
  }
  __syncthreads();
  const int nsel = s_nsel;   // <= kFastCap by construction
  // ---- 4. bitonic sort (padding = ~0 sorts last)
  for (int k = 2; k <= kFastCap; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < kFastCap; i += kNmsThreads) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = s_key[i], b = s_key[l];
          const bool up = ((i & k) == 0);
          if ((a > b) == up) { s_key[i] = b; s_key[l] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = t; i < nsel; i += kNmsThreads) {
    const int id = (int)(unsigned)s_key[i];
    s_box[i] = boxes[id];
    s_area[i] = areas[id];
    s_pos[i] = (unsigned short)id;
    if (id < 1024) s_atpos[id] = (short)i;
  }
  __syncthreads();
  // ---- 5. greedy NMS over the sorted list, trips of <= 64 candidates that never split a run of equal scores
  const int grp = t >> 4, sub = t & 15;   // 64 groups of 16 threads: one candidate each
  int base = 0;
  while (base < nsel) {
    const int nk = s_nk;
    if (nk >= p.R || s_bad) break;
    int end = min(base + 64, nsel);
    if (end < nsel)
      while (end > base && (unsigned)(s_key[end - 1] >> 32) == (unsigned)(s_key[end] >> 32)) --end;
    if (end == base) {   // a run of equal scores longer than a trip
      if (t == 0) s_bad = 1;
      break;
    }
    const int len = end - base;
    const int ci = base + grp;
    const bool have = grp < len;
    float4 cb = make_float4(0.f, 0.f, 0.f, 0.f);
    float ca = 0.f;
    int coid = 0;
    if (have) {
      cb = s_box[ci]; ca = s_area[ci];
      if (p.omap.enabled) coid = orig_id(p.omap, chip_base, (int)(unsigned)s_key[ci]);
    }
    // (a) against everything kept so far
    int dead = 0;
    if (have)
      for (int k = sub; k < nk; k += 16) {
        if (p.omap.enabled && !overlap_listed(p.omap, s_koid[k], coid)) continue;
        dead |= (iou_ref(s_kbox[k].x, s_kbox[k].y, s_kbox[k].z, s_kbox[k].w, s_karea[k], cb, ca) > p.nms_thresh);
      }
    const unsigned dm = __ballot_sync(0xffffffffu, dead);
    const bool alive = have && (((dm >> (lane & 16)) & 0xffffu) == 0);
    // (b) against every other member of this trip (symmetric: inside a tie run the order is not known yet)
    unsigned long long m = 0;
    if (have) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = sub * 4 + u;
        if (j != grp && j < len) {
          const float4 ob = s_box[base + j];
          const float oa = s_area[base + j];
          // bit j of mask[grp]: candidate grp, once kept, suppresses candidate j
          if (p.omap.enabled &&
              !overlap_listed(p.omap, coid, orig_id(p.omap, chip_base, (int)(unsigned)s_key[base + j])))
            continue;
          // the reference evaluates IoU with the selected box first; float min/max/add are symmetric
          if (iou_ref(cb.x, cb.y, cb.z, cb.w, ca, ob, oa) > p.nms_thresh) m |= 1ull << j;
        }
      }
    }
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) m |= __shfl_xor_sync(0xffffffffu, m, off);
    if (sub == 0) { s_mask[grp] = m; s_alive[grp] = alive ? 1 : 0; }
    __syncthreads();
    // (c) sequential resolve by one thread; the swaps are replayed for the reference's tie order (index_ties = 0)
    if (t == 0) {
      unsigned long long removed = 0;   // suppressed or already selected
      int k = nk;
      int i = 0;
      while (i < len && k < p.R) {
        int e = i + 1;
        const unsigned sc_i = (unsigned)(s_key[base + i] >> 32);
        while (e < len && (unsigned)(s_key[base + e] >> 32) == sc_i) ++e;
        while (k < p.R) {
          int best = -1;
          unsigned bestkey = 0xffffffffu;
          for (int c = i; c < e; ++c) {
            if (!s_alive[c] || ((removed >> c) & 1ull)) continue;
            const unsigned d = (unsigned)((int)s_pos[base + c] - k);   // row distance to the front (row k)
            const unsigned key = p.index_ties ? (unsigned)c : ((d & 31u) << 10) | (((d >> 5) & 31u) << 5) | (d >> 10);
            if (key < bestkey) { bestkey = key; best = c; }
          }
          if (best < 0) break;
          const int ci2 = base + best;
          s_kbox[k] = s_box[ci2];
          s_karea[k] = s_area[ci2];
          if (p.omap.enabled) s_koid[k] = orig_id(p.omap, chip_base, (int)(unsigned)s_key[ci2]);
          p.keep_ids[(size_t)chip * 1024 + k] = (int)(unsigned)s_key[ci2];
          // swap rows k and pos(best) (multi_proposal_target.cu:178-199)
          const int pb = s_pos[ci2];
          const int f = s_atpos[k];      // k < R <= 1024
          if (f >= 0 && f != ci2) {
            s_pos[f] = (unsigned short)pb;
            if (pb < 1024) s_atpos[pb] = (short)f;
          } else if (f < 0 && pb < 1024) {
            s_atpos[pb] = -1;            // an unselected row moved there
          }
          s_atpos[k] = (short)ci2;
          s_pos[ci2] = (unsigned short)k;
          removed |= s_mask[best] | (1ull << best);
          ++k;
        }
        i = e;
      }
      s_nk = k;
    }
    __syncthreads();
    base = end;
  }
  __syncthreads();
  if (t == 0) {
    const int nk = s_nk;
    const bool bad = s_bad != 0;
    // not enough: there are valid candidates outside the selection that the reference would still visit
    const bool exhausted = !bad && nk < p.R && nsel < s_nvalid;
    p.nkept[chip] = nk;
    p.fallback[chip] = (bad || exhausted) ? 1 : 0;
  }
}

// One CTA per chip.  Positions 0..AHW-1 hold (score, id) in shared memory; the reference's row swap
// (cu:178-199) becomes a 6-byte swap here, the 16-byte boxes never move.  Tie order of the
// reference's three-level strided argmax (cu:139-176) == lexicographic (lane, warp, stride index)
// among equal scores, which is what the packed 64-bit key below encodes.  With index_ties the lowest
// row id wins a tie instead (the inference operator), and the low bits only carry the position.  kIndexTies ==
// p.index_ties, a template parameter so that the training operator's scan is not slowed by the tie test.
template <bool kIndexTies>
__global__ void __launch_bounds__(kNmsThreads, 1) mpt_nms_assign_kernel(NmsArgs p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s_score = reinterpret_cast<float*>(smem_raw);
  uint16_t* s_id = reinterpret_cast<uint16_t*>(s_score + p.AHW);
  __shared__ unsigned long long s_warpkey[32];
  __shared__ int s_keep[1024];
  __shared__ int s_numgt;
  const int chip = blockIdx.x;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int AHW = p.AHW;
  const float4* boxes = p.boxes + (size_t)chip * AHW;
  const float* areas = p.areas + (size_t)chip * AHW;
  const bool use_fast = p.fast_fallback != nullptr && p.fast_fallback[chip] == 0;
  int vct = 0;
  if (use_fast) {
    vct = p.fast_nkept[chip];
    for (int i = t; i < vct; i += kNmsThreads) s_keep[i] = p.fast_keep[(size_t)chip * 1024 + i];
  } else {
    for (int i = t; i < AHW; i += kNmsThreads) {
      s_score[i] = p.scores[(size_t)chip * AHW + i];
      s_id[i] = (uint16_t)i;
    }
  }
  if (t == 0) s_numgt = 0;
  __syncthreads();

  for (int j = 0; !use_fast && j < AHW && vct < p.R; ++j) {
    // ---- argmax over positions >= j (cu:139-176)
    float best = -2.0f;
    uint32_t besti = 0, bestid = 0;
    {
      int i = 0;
      for (int pos = j + t; pos < AHW; pos += kNmsThreads, ++i) {
        const float s = s_score[pos];
        if (s > best || (kIndexTies && s == best && s_id[pos] < bestid)) {
          best = s;
          besti = i;
          bestid = s_id[pos];
        }
      }
    }
    // index_ties: id (15 bits, AHW <= 32768) | stride index (5) | thread (10); else lane | warp | stride index | id
    const uint32_t lo_key = kIndexTies ? (bestid << 15) | (besti << 10) | (uint32_t)t
                                       : (lane << 26) | (warp << 21) | (besti << 16) | bestid;
    unsigned long long key = ((unsigned long long)ord_desc(best) << 32) | lo_key;
    key = warp_min_u64(key);
    if (lane == 0) s_warpkey[warp] = key;
    __syncthreads();
    key = warp_min_u64(s_warpkey[lane]);
    const uint32_t lo = (uint32_t)key;
    const float sel_score = ord_desc_inv((uint32_t)(key >> 32));
    const int sel_id = kIndexTies ? (int)(lo >> 15) : (int)(lo & 0xffff);
    const int m = j + (kIndexTies ? (int)(lo & 1023) + (int)((lo >> 10) & 31) * kNmsThreads
                                  : (int)(((lo >> 21) & 31) * 32 + (lo >> 26)) + (int)((lo >> 16) & 31) * kNmsThreads);
    if (sel_score == -1.0f) break;  // cu:214-216 (uniform across the block)
    if (t == 0) s_keep[vct] = sel_id;
    vct++;
    const float4 sb = __ldg(boxes + sel_id);
    const float sarea = __ldg(areas + sel_id);
    const int sel_oid = p.omap.enabled ? orig_id(p.omap, (size_t)chip * AHW, sel_id) : 0;
    // element displaced from position j by the swap lands on position m
    const float oldj_score = s_score[j];
    const uint16_t oldj_id = s_id[j];
    // ---- suppression over positions > j (cu:218-240)
    // four positions per thread per trip: the (L2-resident) box loads of a trip are independent and in flight
    // together, which is what bounds this latency-limited loop
    for (int base = j + 1 + t; base < AHW; base += 4 * kNmsThreads) {
      float s[4];
      int id[4];
      float4 d[4];
      float da[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int pos = base + u * kNmsThreads;
        s[u] = -1.0f;
        id[u] = 0;
        if (pos < AHW) {
          if (pos == m) {
            s[u] = oldj_score;
            id[u] = oldj_id;
            s_id[pos] = oldj_id;
          } else {
            s[u] = s_score[pos];
            id[u] = s_id[pos];
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (s[u] != -1.0f) {
          d[u] = __ldg(boxes + id[u]);
          da[u] = __ldg(areas + id[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int pos = base + u * kNmsThreads;
        if (pos >= AHW) continue;
        float sv = s[u];
        if (sv != -1.0f &&
            (!p.omap.enabled || overlap_listed(p.omap, sel_oid, orig_id(p.omap, (size_t)chip * AHW, id[u])))) {
          const float ovr = iou_ref(sb.x, sb.y, sb.z, sb.w, sarea, d[u], da[u]);
          if (ovr > p.nms_thresh) sv = -1.0f;
        }
        if (pos == m || sv == -1.0f) s_score[pos] = sv;
      }
    }
    __syncthreads();
  }
  __syncthreads();

  // ---- outputs: kept rows, filler rows (cu:244-258), then the host section (cu:435-588)
  const int R = p.R;
  if (p.num_kept && t == 0) p.num_kept[chip] = vct;
  if (!p.do_assign) {
    for (int r = t; r < R; r += kNmsThreads) {
      float4 bx;
      if (r < vct) {
        bx = __ldg(boxes + s_keep[r]);
      } else {
        const float f = (float)(int)(((long)chip * p.filler_stride + r) % 100);
        bx = make_float4(f, f, f + 200.0f, f + 200.0f);
      }
      float* o = p.rois + ((size_t)chip * R + r) * 5;
      o[0] = (float)chip; o[1] = bx.x; o[2] = bx.y; o[3] = bx.z; o[4] = bx.w;
      if (p.keep_idx)
        p.keep_idx[(size_t)chip * R + r] =
            r < vct ? (p.id_map ? p.id_map[(size_t)chip * AHW + s_keep[r]] : s_keep[r]) : -1;
      if (p.score_out) {
        float so = r < vct ? p.scores[(size_t)chip * AHW + s_keep[r]] : 0.0f;
        if (p.omap.enabled && r < vct) {
          // the map is not applied symmetrically: a box kept LATER may list this one and mark it (the reference reads
          // the scores after the NMS, multi_proposal.cu:592, so such a row is output with score -1)
          const int my = orig_id(p.omap, (size_t)chip * AHW, s_keep[r]);
          const float ma = __ldg(areas + s_keep[r]);
          for (int q = r + 1; q < vct; ++q) {
            const int qo = orig_id(p.omap, (size_t)chip * AHW, s_keep[q]);
            if (!overlap_listed(p.omap, qo, my)) continue;
            const float4 qb = __ldg(boxes + s_keep[q]);
            if (iou_ref(qb.x, qb.y, qb.z, qb.w, __ldg(areas + s_keep[q]), bx, ma) > p.nms_thresh) { so = -1.0f; break; }
          }
        }
        p.score_out[(size_t)chip * R + r] = so;
      }
    }
    return;
  }
  float* s_gt = s_score;  // reuse: [max_gt*5]
  const float* gt = p.gt_boxes + (size_t)chip * p.max_gt * 5;
  for (int i = t; i < p.max_gt * 5; i += kNmsThreads) s_gt[i] = gt[i];
  __syncthreads();
  {
    int c = 0;
    for (int g = t; g < p.max_gt; g += kNmsThreads) c += (s_gt[g * 5 + 4] != -1.0f);
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0 && c) atomicAdd(&s_numgt, c);
  }
  __syncthreads();
  const int numgt = s_numgt;
  const float vr0 = p.valid_ranges[2 * chip], vr1 = p.valid_ranges[2 * chip + 1];
  for (int r = t; r < R; r += kNmsThreads) {
    float4 bx;
    if (r < vct) {
      bx = __ldg(boxes + s_keep[r]);
    } else {
      const float f = (float)(int)(((long)chip * AHW + r) % 100);
      bx = make_float4(f, f, f + 200.0f, f + 200.0f);
    }
    if (r >= R - numgt) {  // GT append, cu:469-479
      const float* g = s_gt + (r - (R - numgt)) * 5;
      const float area = __fmul_rn(__fsub_rn(g[2], g[0]), __fsub_rn(g[3], g[1]));
      if (area >= __fmul_rn(vr0, vr0) && area <= __fmul_rn(vr1, vr1)) bx = make_float4(g[0], g[1], g[2], g[3]);
    }
    float lab = 0.0f, maxov = 0.0f;
    int arg = -1;
    const float a2 = __fmul_rn(__fsub_rn(bx.z, bx.x), __fsub_rn(bx.w, bx.y));
    for (int g = 0; g < numgt; ++g) {  // cu:503-531, first max wins ties (strict >)
      const float* gb = s_gt + g * 5;
      const float a1 = __fmul_rn(__fsub_rn(gb[2], gb[0]), __fsub_rn(gb[3], gb[1]));
      const float ovr = iou_ref(gb[0], gb[1], gb[2], gb[3], a1, bx, a2);
      if (ovr > maxov && ovr > 0.5f) {
        maxov = ovr;
        arg = g;
        lab = gb[4];
      }
    }
    float tg[4] = {1.0f, 1.0f, 1.0f, 1.0f};
    float wt = 0.0f;
    if (arg >= 0) {  // cu:537-573
      wt = 1.0f;
      const float* gb = s_gt + arg * 5;
      const float gw = __fadd_rn(__fsub_rn(gb[2], gb[0]), 1.0f);
      const float gh = __fadd_rn(__fsub_rn(gb[3], gb[1]), 1.0f);
      const float gcx = (float)__dadd_rn((double)gb[0], __dmul_rn((double)gw, 0.5));
      const float gcy = (float)__dadd_rn((double)gb[1], __dmul_rn((double)gh, 0.5));
      const float pw = __fadd_rn(__fsub_rn(bx.z, bx.x), 1.0f);
      const float ph = __fadd_rn(__fsub_rn(bx.w, bx.y), 1.0f);
      const float pcx = (float)__dadd_rn((double)bx.x, __dmul_rn((double)__fsub_rn(pw, 1.0f), 0.5));
      const float pcy = (float)__dadd_rn((double)bx.y, __dmul_rn((double)__fsub_rn(ph, 1.0f), 0.5));
      const double pwe = __dadd_rn((double)pw, 1e-7), phe = __dadd_rn((double)ph, 1e-7);
      tg[0] = (float)__ddiv_rn((double)__fmul_rn(10.0f, __fsub_rn(gcx, pcx)), pwe);
      tg[1] = (float)__ddiv_rn((double)__fmul_rn(10.0f, __fsub_rn(gcy, pcy)), phe);
      tg[2] = (float)__dmul_rn(5.0, log(__ddiv_rn((double)gw, pwe)));
      tg[3] = (float)__dmul_rn(5.0, log(__ddiv_rn((double)gh, phe)));
    }
    const size_t row = (size_t)chip * R + r;
    float* o = p.rois + row * 5;
    o[0] = (float)chip; o[1] = bx.x; o[2] = bx.y; o[3] = bx.z; o[4] = bx.w;
    p.label[row] = lab;
    reinterpret_cast<float4*>(p.bbox_target)[row] = make_float4(tg[0], tg[1], tg[2], tg[3]);
    reinterpret_cast<float4*>(p.bbox_weight)[row] = make_float4(wt, wt, wt, wt);
    if (p.keep_idx) p.keep_idx[row] = r < vct ? s_keep[r] : -1;
  }
}

// ------------------------------------------------------------------------------------------------
// Pre-NMS selection of the inference operator (multi_proposal.cc:176-199: only the pre_nms_top_n best-scoring
// anchors of an image enter the NMS).  One CTA per image: exact K-th key by a 3-pass MSB radix select over the
// order-preserving 32-bit score keys, then an index-ordered compaction of the K best rows (ties at the K-th score
// are taken in index order; the reference's std::sort leaves them unspecified).
struct SelectArgs {
  const float4* boxes;
  const float* scores;
  const float* areas;
  int AHW, K;
  float4* boxes_c;   // [B*K]
  float* scores_c;
  float* areas_c;
  int32_t* ids_c;    // original anchor index
};

__global__ void __launch_bounds__(1024, 1) mp_select_kernel(SelectArgs p) {
  __shared__ int s_hist[2048];
  __shared__ uint32_t s_prefix, s_mask;
  __shared__ int s_remaining;
  __shared__ int s_warp[32];
  __shared__ int s_base_lt, s_base_eq;
  const int img = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float* sc = p.scores + (size_t)img * p.AHW;
  if (t == 0) { s_prefix = 0; s_mask = 0; s_remaining = p.K; }
  __syncthreads();
  const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
  for (int pass = 0; pass < 3; ++pass) {
    for (int i = t; i < 2048; i += 1024) s_hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix, mask = s_mask;
    const int sh = shifts[pass];
    const uint32_t bm = (1u << bits[pass]) - 1u;
    for (int i = t; i < p.AHW; i += 1024) {
      const uint32_t k = ord_desc(sc[i]);
      if ((k & mask) == prefix) atomicAdd(&s_hist[(k >> sh) & bm], 1);
    }
    __syncthreads();
    if (t == 0) {
      int rem = s_remaining, b = 0;
      while (s_hist[b] < rem) { rem -= s_hist[b]; ++b; }     // terminates: the matching rows number >= rem
      s_remaining = rem;
      s_prefix = prefix | ((uint32_t)b << sh);
      s_mask = mask | (bm << sh);
    }
    __syncthreads();
  }
  const uint32_t kth = s_prefix;
  const int take_eq = s_remaining;   // rows equal to the K-th key that still fit
  if (t == 0) { s_base_lt = 0; s_base_eq = 0; }
  __syncthreads();
  for (int i0 = 0; i0 < p.AHW; i0 += 1024) {
    const int i = i0 + t;
    uint32_t k = 0xffffffffu;
    if (i < p.AHW) k = ord_desc(sc[i]);
    const int lt = (i < p.AHW && k < kth) ? 1 : 0, eq = (i < p.AHW && k == kth) ? 1 : 0;
    int v = lt | (eq << 16), incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += o;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, w, off);
        if (lane >= off) w += o;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int excl = incl - v + (warp ? s_warp[warp - 1] : 0);
    const int lt_before = s_base_lt + (excl & 0xffff), eq_before = s_base_eq + (excl >> 16);
    const int eq_taken_before = eq_before < take_eq ? eq_before : take_eq;
    const bool take = lt || (eq && eq_before < take_eq);
    if (take) {
      const size_t dst = (size_t)img * p.K + lt_before + eq_taken_before;
      const size_t src = (size_t)img * p.AHW + i;
      p.boxes_c[dst] = p.boxes[src];
      p.scores_c[dst] = sc[i];
      p.areas_c[dst] = p.areas[src];
      p.ids_c[dst] = i;
    }
    __syncthreads();
    if (t == 0) {
      const int total = s_warp[31];
      s_base_lt += total & 0xffff;
      s_base_eq += total >> 16;
    }
    __syncthreads();
  }
}

// host twin of multi_proposal_target.cu:75-114 (anchor table is 4*A floats, passed by value)
int make_anchors(int feat_stride, const float* scales, int ns, const float* ratios, int nr, AnchorTable* out) {
  const float base2 = (float)(feat_stride - 1.0);
  int n = 0;
  for (int j = 0; j < nr; ++j) {
    for (int k = 0; k < ns; ++k) {
      const float scale = scales[k], ratio = ratios[j];
      const float w = base2 - 0.0f + 1.0f, h = base2 - 0.0f + 1.0f;
      const float x_ctr = (float)(0.0f + 0.5 * (w - 1.0f));
      const float y_ctr = (float)(0.0f + 0.5 * (h - 1.0f));
      const float size = w * h;
      const float size_ratios = floorf(size / ratio);
      const float new_w = floorf(sqrtf(size_ratios) + 0.5f) * scale;
      const float new_h = floorf((new_w / scale * ratio) + 0.5f) * scale;
      out->v[4 * n + 0] = x_ctr - 0.5f * (new_w - 1.0f);
      out->v[4 * n + 1] = y_ctr - 0.5f * (new_h - 1.0f);
      out->v[4 * n + 2] = x_ctr + 0.5f * (new_w - 1.0f);
      out->v[4 * n + 3] = y_ctr + 0.5f * (new_h - 1.0f);
      ++n;
    }
  }
  return n;
}

size_t ws_bytes_impl(int B, int A, int H, int W) {
  const size_t total = (size_t)B * A * H * W;
  return total * (sizeof(float4) + 2 * sizeof(float)) + 256 + (size_t)B * (1024 + 2) * sizeof(int32_t) + 64;
}

}  // namespace

// SNIPER_NMS_FAST=0 forces the sequential emulation (used by the parity tests to exercise both paths)
bool nms_fast_enabled() {
  const char* e = getenv("SNIPER_NMS_FAST");
  return !(e && e[0] == '0');
}

extern "C" {

size_t sniper_multi_proposal_target_workspace_bytes(int B, int A, int H, int W) { return ws_bytes_impl(B, A, H, W); }

int sniper_generate_anchors(int feat_stride, const float* scales, int ns, const float* ratios, int nr, float* out) {
  SN_CHECK(ns * nr <= kMaxAnchors && ns > 0 && nr > 0, "generate_anchors: need 0 < ns*nr <= %d", kMaxAnchors);
  AnchorTable t;
  make_anchors(feat_stride, scales, ns, ratios, nr, &t);
  memcpy(out, t.v, sizeof(float) * 4 * ns * nr);
  return 0;
}

// Stage 1 only (K1): decode + clip + filters.  boxes/score/area are caller-owned device arrays.
int sniper_proposal_decode(const float* cls_prob, const float* bbox_pred, const float* im_info,
                           const float* valid_ranges, int B, int A, int H, int W, int feat_stride,
                           const float* scales, int ns, const float* ratios, int nr, int layout,
                           int score_cstride, int delta_cstride, float* boxes, float* score, float* area,
                           void* stream) {
  SN_CHECK(A == ns * nr, "proposal_decode: A (%d) != ns*nr (%d)", A, ns * nr);
  SN_CHECK(A <= kMaxAnchors, "proposal_decode: A (%d) > %d", A, kMaxAnchors);
  SN_CHECK(layout == 0 || layout == 1, "proposal_decode: layout must be 0 (NCHW) or 1 (NHWC)");
  SN_CHECK(layout == 0 || (delta_cstride % 4 == 0 && ((uintptr_t)bbox_pred & 15) == 0),
           "proposal_decode: NHWC deltas need 16-byte aligned pixels");
  AnchorTable t;
  make_anchors(feat_stride, scales, ns, ratios, nr, &t);
  DecodeArgs a;
  a.scores = cls_prob; a.deltas = bbox_pred; a.im_info = im_info; a.valid_ranges = valid_ranges;
  a.B = B; a.A = A; a.H = H; a.W = W; a.stride = feat_stride; a.layout = layout;
  a.score_cstride = score_cstride; a.delta_cstride = delta_cstride;
  a.variant = 0; a.suppress_types = 0;
  a.boxes = reinterpret_cast<float4*>(boxes); a.score_out = score; a.area_out = area;
  const long total = (long)B * A * H * W;
  int grid = sn::div_up(total, 256);
  if (grid > sn::kNumSMs * 8) grid = sn::kNumSMs * 8;
  mpt_decode_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, t);
  SN_LAUNCH_CHECK();
  return 0;
}

static int nms_assign_launch(const float* boxes, const float* score, const float* area, const float* gt_boxes,
                             const float* valid_ranges, int B, int AHW, int max_gt, int R, float nms_thresh,
                             float* rois, float* label, float* bbox_target, float* bbox_weight,
                             int32_t* keep_idx, int32_t* num_kept, int do_assign, int32_t* fast_scratch,
                             void* stream, const int32_t* id_map = nullptr, float* score_out = nullptr,
                             long filler_stride = 0, const OverlapMap* omap = nullptr, int index_ties = 0) {
  SN_CHECK(AHW >= R, "nms: anchors per chip (%d) < post_nms_top_n (%d)", AHW, R);
  SN_CHECK(AHW <= 32768, "nms: anchors per chip (%d) > 32768", AHW);
  SN_CHECK(R <= 1024, "nms: post_nms_top_n (%d) > 1024", R);
  SN_CHECK(!do_assign || (max_gt <= R && max_gt * 5 <= AHW), "nms: max_gt (%d) too large", max_gt);
  NmsArgs n;
  n.boxes = reinterpret_cast<const float4*>(boxes); n.scores = score; n.areas = area;
  n.gt_boxes = gt_boxes; n.valid_ranges = valid_ranges; n.AHW = AHW; n.R = R; n.max_gt = max_gt;
  n.nms_thresh = nms_thresh; n.rois = rois; n.label = label; n.bbox_target = bbox_target;
  n.bbox_weight = bbox_weight; n.keep_idx = keep_idx; n.num_kept = num_kept; n.do_assign = do_assign;
  n.id_map = id_map; n.score_out = score_out; n.filler_stride = filler_stride > 0 ? filler_stride : AHW;
  if (omap) n.omap = *omap; else { memset(&n.omap, 0, sizeof(n.omap)); }
  n.index_ties = index_ties;
  const size_t smem = (size_t)AHW * 6 + 16;
  static bool attr_set = false;
  const size_t fast_smem = (size_t)kFastCap * (8 + 16 + 4 + 2) + kFastBins * 4 + 1024 * (20 + 2) + 64 * 8 + 64 * 4 + 64;
  if (!attr_set) {
    SN_CUDA(cudaFuncSetAttribute(mpt_nms_assign_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SN_CUDA(cudaFuncSetAttribute(mpt_nms_assign_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SN_CUDA(cudaFuncSetAttribute(mpt_nms_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  n.fast_keep = nullptr; n.fast_nkept = nullptr; n.fast_fallback = nullptr;
  if (fast_scratch) {
    FastArgs f;
    f.boxes = n.boxes; f.scores = score; f.areas = area; f.AHW = AHW; f.R = R; f.nms_thresh = nms_thresh;
    f.keep_ids = fast_scratch; f.nkept = fast_scratch + (size_t)B * 1024; f.fallback = f.nkept + B;
    f.omap = n.omap;
    f.index_ties = index_ties;
    mpt_nms_fast_kernel<<<B, kNmsThreads, fast_smem, (cudaStream_t)stream>>>(f);
    SN_LAUNCH_CHECK();
    n.fast_keep = f.keep_ids; n.fast_nkept = f.nkept; n.fast_fallback = f.fallback;
  }
  if (index_ties)
    mpt_nms_assign_kernel<true><<<B, kNmsThreads, smem, (cudaStream_t)stream>>>(n);
  else
    mpt_nms_assign_kernel<false><<<B, kNmsThreads, smem, (cudaStream_t)stream>>>(n);
  SN_LAUNCH_CHECK();
  return 0;
}

// Drop-in for MultiProposalTargetGPUOp::Forward.  All pointers are device pointers owned by the
// caller; no allocation and no synchronisation happen inside.
int sniper_multi_proposal_target_fwd(const float* cls_prob, const float* bbox_pred, const float* im_info,
                                     const float* gt_boxes, const float* valid_ranges, int B, int A, int H, int W,
                                     int max_gt, int post_nms_top_n, int feat_stride, const float* scales, int ns,
                                     const float* ratios, int nr, float nms_thresh, int layout, int score_cstride,
                                     int delta_cstride, float* rois, float* label, float* bbox_target,
                                     float* bbox_weight, int32_t* keep_idx, int32_t* num_kept, void* workspace,
                                     size_t ws_bytes, void* stream) {
  SN_CHECK(ws_bytes >= ws_bytes_impl(B, A, H, W), "multi_proposal_target: workspace too small (%zu < %zu)", ws_bytes,
           ws_bytes_impl(B, A, H, W));
  SN_CHECK(((uintptr_t)workspace & 15) == 0, "multi_proposal_target: workspace must be 16-byte aligned");
  SN_CHECK(((uintptr_t)bbox_target & 15) == 0 && ((uintptr_t)bbox_weight & 15) == 0,
           "multi_proposal_target: bbox_target/bbox_weight must be 16-byte aligned");
  const size_t total = (size_t)B * A * H * W;
  float* boxes = reinterpret_cast<float*>(workspace);
  float* score = boxes + 4 * total;
  float* area = score + total;
  if (sniper_proposal_decode(cls_prob, bbox_pred, im_info, valid_ranges, B, A, H, W, feat_stride, scales, ns, ratios,
                             nr, layout, score_cstride, delta_cstride, boxes, score, area, stream))
    return -1;
  int32_t* fast_scratch = reinterpret_cast<int32_t*>(area + total + 16);
  return nms_assign_launch(boxes, score, area, gt_boxes, valid_ranges, B, A * H * W, max_gt, post_nms_top_n,
                           nms_thresh, rois, label, bbox_target, bbox_weight, keep_idx, num_kept, 1,
                           nms_fast_enabled() ? fast_scratch : nullptr, stream);
}

// Workspace of sniper_multi_proposal_fwd: decoded rows of every anchor + the compacted pre_nms_top_n rows per image.
size_t sniper_multi_proposal_workspace_bytes(int B, int A, int H, int W, int pre_nms_top_n) {
  const size_t total = (size_t)B * A * H * W;
  const size_t K = (size_t)(pre_nms_top_n < A * H * W ? pre_nms_top_n : A * H * W);
  return total * 24 + 64 + (size_t)B * K * 28 + 64 + (size_t)B * (1024 + 2) * sizeof(int32_t) + 256;
}

// Inference proposal operator: drop-in for MultiProposal (multi_proposal-inl.h:55-167; CPU op multi_proposal.cc:273-374,
// GPU-build op multi_proposal.cu:400-631) entirely on device -- decode, min-size filter, top pre_nms_top_n selection,
// greedy NMS (> 0.7 as the reference hard-codes; nms_thresh is passed through), rois [B*post,5] and scores [B*post].
// flags: 1 = anchor-type suppression of the GPU build (.cu:505-508); 2 = the GPU build's FastNMS (a kept box only tests
// the anchors of its precomputed anchor-overlap map, roi_iou_thresh; .cu:267-387) instead of the exact NMS of the CPU op.
// Rows after the kept ones are rand() boxes in the reference; here the deterministic filler of the training operator
// with score 0.  keep_idx / num_kept: optional parity outputs (original anchor indices).
// Equal scores are taken in ascending anchor index, by the selection and by both NMS kernels (the reference sorts with
// std::sort / nth_element, whose order of equal scores is unspecified; the compacted rows keep the index order).
int sniper_multi_proposal_fwd(const float* cls_prob, const float* bbox_pred, const float* im_info, int B, int A, int H,
                              int W, int pre_nms_top_n, int post_nms_top_n, int feat_stride, const float* scales, int ns,
                              const float* ratios, int nr, float nms_thresh, int flags, float roi_iou_thresh, int layout,
                              int score_cstride,
                              int delta_cstride, float* rois, float* scores, int32_t* keep_idx, int32_t* num_kept,
                              void* workspace, size_t ws_bytes, void* stream) {
  SN_CHECK(A == ns * nr && A <= kMaxAnchors, "multi_proposal: A (%d) must equal ns*nr and be <= %d", A, kMaxAnchors);
  SN_CHECK((flags & ~3) == 0, "multi_proposal: unsupported flags %d", flags);
  SN_CHECK(layout == 0 || layout == 1, "multi_proposal: layout must be 0 (NCHW) or 1 (NHWC)");
  SN_CHECK(layout == 0 || (delta_cstride % 4 == 0 && ((uintptr_t)bbox_pred & 15) == 0),
           "multi_proposal: NHWC deltas need 16-byte aligned pixels");
  SN_CHECK(ws_bytes >= sniper_multi_proposal_workspace_bytes(B, A, H, W, pre_nms_top_n),
           "multi_proposal: workspace too small");
  SN_CHECK(((uintptr_t)workspace & 15) == 0, "multi_proposal: workspace must be 16-byte aligned");
  const int AHW = A * H * W;
  const int K = pre_nms_top_n < AHW ? pre_nms_top_n : AHW;
  SN_CHECK(K >= post_nms_top_n && K <= 32768, "multi_proposal: need post_nms_top_n <= min(pre_nms_top_n, A*H*W) <= 32768");
  const size_t total = (size_t)B * AHW;
  // carve the workspace (every array 16-byte aligned)
  unsigned char* wp = static_cast<unsigned char*>(workspace);
  auto carve = [&wp](size_t bytes) { void* r = wp; wp += (bytes + 15) & ~(size_t)15; return r; };
  float* boxes = static_cast<float*>(carve(16 * total));
  float* score = static_cast<float*>(carve(4 * total));
  float* area = static_cast<float*>(carve(4 * total));
  float* boxes_c = static_cast<float*>(carve(16 * (size_t)B * K));
  float* score_c = static_cast<float*>(carve(4 * (size_t)B * K));
  float* area_c = static_cast<float*>(carve(4 * (size_t)B * K));
  int32_t* ids_c = static_cast<int32_t*>(carve(4 * (size_t)B * K));
  int32_t* fast_scratch = static_cast<int32_t*>(carve((size_t)B * (1024 + 2) * sizeof(int32_t)));
  AnchorTable t;
  make_anchors(feat_stride, scales, ns, ratios, nr, &t);
  DecodeArgs a;
  a.scores = cls_prob; a.deltas = bbox_pred; a.im_info = im_info; a.valid_ranges = nullptr;
  a.B = B; a.A = A; a.H = H; a.W = W; a.stride = feat_stride; a.layout = layout;
  a.score_cstride = score_cstride; a.delta_cstride = delta_cstride;
  a.variant = 1; a.suppress_types = flags & 1;
  a.boxes = reinterpret_cast<float4*>(boxes); a.score_out = score; a.area_out = area;
  int grid = sn::div_up((long)total, 256);
  if (grid > sn::kNumSMs * 8) grid = sn::kNumSMs * 8;
  mpt_decode_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, t);
  SN_LAUNCH_CHECK();
  const int32_t* id_map = nullptr;
  if (K < AHW) {
    SelectArgs sa;
    sa.boxes = reinterpret_cast<const float4*>(boxes); sa.scores = score; sa.areas = area; sa.AHW = AHW; sa.K = K;
    sa.boxes_c = reinterpret_cast<float4*>(boxes_c); sa.scores_c = score_c; sa.areas_c = area_c; sa.ids_c = ids_c;
    mp_select_kernel<<<B, 1024, 0, (cudaStream_t)stream>>>(sa);
    SN_LAUNCH_CHECK();
    boxes = boxes_c; score = score_c; area = area_c; id_map = ids_c;
  }
  OverlapMap om;
  memset(&om, 0, sizeof(om));
  if (flags & 2) {
    om.enabled = 1; om.H = H; om.W = W; om.stride = feat_stride; om.thresh = roi_iou_thresh; om.id_map = id_map;
    memcpy(om.anchors, t.v, sizeof(float) * 4 * A);
    for (int i = 0; i < A; ++i)   // multi_proposal.cu:489-496
      om.area[i] = (t.v[4 * i + 2] - t.v[4 * i] + 1) * (t.v[4 * i + 3] - t.v[4 * i + 1] + 1);
  }
  return nms_assign_launch(boxes, score, area, nullptr, nullptr, B, K, 0, post_nms_top_n, nms_thresh, rois, nullptr,
                           nullptr, nullptr, keep_idx, num_kept, 0, nms_fast_enabled() ? fast_scratch : nullptr, stream,
                           id_map, scores, (long)AHW, &om, 1);
}

}  // extern "C"
