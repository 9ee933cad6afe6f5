// Batched per-(image, class) soft-NMS / NMS on the device for the multi-scale inference aggregation.
//
// Replaces the `Pool(32)` of host processes running `cpu_soft_nms` (lib/nms/cpu_nms.pyx:17-110, Gaussian, sigma 0.55,
// score threshold 0.001; called per image and class by Tester.aggregate, lib/inference.py:152-200, through
// nms_worker.worker) -- the "per-scale NMS latency" of BASELINE config 5.  One CTA per problem; all problems of a scale
// (images x 80 classes) run in one launch.
//
// Semantics of the reference loop, restated order-free: repeat { take the highest-scoring remaining box (rows the
// reference has swapped to the front are exactly the boxes taken so far, in order); multiply the score of every other
// remaining box by w(IoU with it); drop boxes whose score falls below `threshold` }.  The output rows are the taken boxes
// in the order taken, each with the score it had when taken = the reference's returned array.  Arithmetic follows the
// Cythonized reference (float IoU with the `+ 1` sums evaluated in double and narrowed once, Gaussian weight =
// exp evaluated in double); this file is compiled with -fmad=false.  Exact score ties are broken by the lower input row
// (the reference breaks them by its current, swap-dependent order).
#include "common.cuh"
#include <math.h>

namespace {

constexpr int kNmsTPB = 256;

__global__ void __launch_bounds__(kNmsTPB) soft_nms_batched_kernel(float* __restrict__ dets, const int* __restrict__ offsets,
                                                                   float sigma, float Nt, float threshold,
                                                                   unsigned method, int* __restrict__ out_counts,
                                                                   float* __restrict__ scratch) {
  const int p = blockIdx.x;
  const int base = offsets[p], N = offsets[p + 1] - base;
  float* d = dets + (size_t)base * 5;
  float* work = scratch + (size_t)base * 5;     // the remaining boxes (score < 0 marks a removed / taken row)
  __shared__ float s_val[kNmsTPB / 32];
  __shared__ int s_idx[kNmsTPB / 32];
  __shared__ float s_t[5];
  __shared__ int s_stop;
  for (int i = threadIdx.x; i < N * 5; i += blockDim.x) work[i] = d[i];
  __syncthreads();
  int taken = 0;
  for (;;) {
    // ---- argmax over the remaining rows (scores are >= threshold > 0 or original; removed rows carry -1)
    float best = -1.f;
    int bi = -1;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      const float s = work[5 * j + 4];
      if (s > best) { best = s; bi = j; }          // strict >: the lowest row index wins a tie within a thread
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (ob > best || (ob == best && oi >= 0 && (bi < 0 || oi < bi))) { best = ob; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { s_val[threadIdx.x >> 5] = best; s_idx[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float b = s_val[0];
      int k = s_idx[0];
      for (int w = 1; w < kNmsTPB / 32; ++w)
        if (s_val[w] > b || (s_val[w] == b && s_idx[w] >= 0 && (k < 0 || s_idx[w] < k))) { b = s_val[w]; k = s_idx[w]; }
      s_stop = (k < 0 || b < 0.f) ? 1 : 0;
      if (!s_stop) {
#pragma unroll
        for (int c = 0; c < 5; ++c) s_t[c] = work[5 * k + c];
        work[5 * k + 4] = -1.f;                    // taken
#pragma unroll
        for (int c = 0; c < 5; ++c) d[5 * taken + c] = s_t[c];
      }
    }
    __syncthreads();
    if (s_stop) break;
    ++taken;
    const float tx1 = s_t[0], ty1 = s_t[1], tx2 = s_t[2], ty2 = s_t[3];
    // ---- decay / remove the others
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      const float s = work[5 * j + 4];
      if (s < 0.f) continue;
      const float x1 = work[5 * j], y1 = work[5 * j + 1], x2 = work[5 * j + 2], y2 = work[5 * j + 3];
      const float area = (float)(((double)(x2 - x1) + 1.0) * ((double)(y2 - y1) + 1.0));
      const float iw = (float)((double)(fminf(tx2, x2) - fmaxf(tx1, x1)) + 1.0);
      if (iw > 0) {
        const float ih = (float)((double)(fminf(ty2, y2) - fmaxf(ty1, y1)) + 1.0);
        if (ih > 0) {
          const float inter = iw * ih;
          const float ua = (float)(((((double)(tx2 - tx1) + 1.0) * ((double)(ty2 - ty1) + 1.0)) + (double)area) -
                                   (double)inter);
          const float ov = inter / ua;
          float weight;
          if (method == 1) weight = ov > Nt ? (float)(1.0 - (double)ov) : 1.f;
          else if (method == 2) weight = (float)exp((double)(-(ov * ov) / sigma));
          else weight = ov > Nt ? 0.f : 1.f;
          const float ns = weight * s;
          work[5 * j + 4] = ns < threshold ? -1.f : ns;
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out_counts[p] = taken;
}

// nmsp (lib/nms/nms.py:48-80, threshold 0.7) for one image per CTA: the proposal NMS that imdb.load_rpn_data runs on
// every training image before its proposals join the roidb.  The rows are sorted once by (score, row) descending -- the
// order of `scores.argsort()[::-1]` with a stable argsort, i.e. exact ties go to the higher row -- and then swept in
// that order: a row nobody suppressed is kept and suppresses every later row with IoU > 0.7.  Since the IoU is
// symmetric this is the reference's loop.  Arithmetic is nmsp's float32 expressions, each operation rounded (no FMA).
constexpr int kPropNmsTPB = 1024;
constexpr int kPropNmsCap = 4096;
constexpr int kPropNmsSlots = kPropNmsCap / kPropNmsTPB;

__global__ void __launch_bounds__(kPropNmsTPB) proposal_nms_batched_kernel(const float* __restrict__ dets,
                                                                          const int* __restrict__ offsets,
                                                                          int* __restrict__ out_counts,
                                                                          int* __restrict__ keep) {
  __shared__ unsigned long long s_key[kPropNmsCap];      // (score bits << 32 | row), sorted descending
  __shared__ unsigned char s_sup[kPropNmsCap];           // suppressed flag per sorted position
  __shared__ int s_bad;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int base = offsets[p], N = offsets[p + 1] - base;
  const float* d = dets + (size_t)base * 5;
  int P2 = 1;
  while (P2 < N) P2 <<= 1;
  if (tid == 0) s_bad = 0;
  __syncthreads();
  for (int i = tid; i < P2; i += kPropNmsTPB) {
    unsigned long long k = 0ull;                           // padding sorts last (a real key of 0 is indistinguishable)
    if (i < N) {
      const float s = d[5 * i + 4];
      if (!(s >= 0.f)) s_bad = 1;
      k = ((unsigned long long)__float_as_uint(s + 0.f) << 32) | (unsigned)i;     // + 0: -0 -> +0
    }
    s_key[i] = k;
    s_sup[i] = 0;
  }
  __syncthreads();
  if (s_bad) {
    if (tid == 0) out_counts[p] = -1;
    return;
  }
  // bitonic sort, descending
  for (int k = 2; k <= P2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P2; i += kPropNmsTPB) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = s_key[i], b = s_key[ixj];
          if (((i & k) == 0) ? (a < b) : (a > b)) { s_key[i] = b; s_key[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  // each thread holds the boxes of sorted positions tid + s * kPropNmsTPB
  float bx1[kPropNmsSlots], by1[kPropNmsSlots], bx2[kPropNmsSlots], by2[kPropNmsSlots], bar[kPropNmsSlots];
#pragma unroll
  for (int s = 0; s < kPropNmsSlots; ++s) {
    const int u = tid + s * kPropNmsTPB;
    bx1[s] = by1[s] = bx2[s] = by2[s] = bar[s] = 0.f;
    if (u < N) {
      const int r = (int)(s_key[u] & 0xffffffffu);
      bx1[s] = d[5 * r];
      by1[s] = d[5 * r + 1];
      bx2[s] = d[5 * r + 2];
      by2[s] = d[5 * r + 3];
      bar[s] = ((bx2[s] - bx1[s]) + 1.f) * ((by2[s] - by1[s]) + 1.f);
    }
  }
  const float thresh = 0.7f;
  int kept = 0;
  for (int t = 0; t < N; ++t) {
    if (s_sup[t]) continue;                                // written before the last barrier: uniform
    const int r = (int)(s_key[t] & 0xffffffffu);
    if (tid == 0) keep[base + kept] = r;
    ++kept;
    const float tx1 = d[5 * r], ty1 = d[5 * r + 1], tx2 = d[5 * r + 2], ty2 = d[5 * r + 3];
    const float tar = ((tx2 - tx1) + 1.f) * ((ty2 - ty1) + 1.f);
#pragma unroll
    for (int s = 0; s < kPropNmsSlots; ++s) {
      const int u = tid + s * kPropNmsTPB;
      if (u > t && u < N && !s_sup[u]) {
        const float xx1 = fmaxf(tx1, bx1[s]), yy1 = fmaxf(ty1, by1[s]);
        const float xx2 = fminf(tx2, bx2[s]), yy2 = fminf(ty2, by2[s]);
        const float w = fmaxf(0.f, (xx2 - xx1) + 1.f), h = fmaxf(0.f, (yy2 - yy1) + 1.f);
        const float inter = w * h;
        const float ovr = inter / ((tar + bar[s]) - inter);
        if (!(ovr <= thresh)) s_sup[u] = 1;                // np.where(ovr <= thresh) drops NaN as well
      }
    }
    __syncthreads();
  }
  if (tid == 0) out_counts[p] = kept;
}

}  // namespace

extern "C" {

// dets: [total, 5] (x1, y1, x2, y2, score) rows of all problems back to back, problem p = rows [offsets[p],
// offsets[p+1]); rewritten in place: the first out_counts[p] rows of each segment are the surviving detections in the
// order cpu_soft_nms returns them.  offsets: device int32 [P+1]; scratch: device float [total*5].  Scores must be >= 0.
// method 1 = linear, 2 = Gaussian (the reference's TEST default), 3 = hard NMS.
int sniper_soft_nms_batched(float* dets, const int* offsets, int P, float sigma, float Nt, float threshold,
                            unsigned method, int* out_counts, float* scratch, void* stream) {
  if (P <= 0) return 0;
  SN_CHECK(method >= 1 && method <= 3, "soft_nms_batched: method must be 1 (linear), 2 (gaussian) or 3 (hard)");
  SN_CHECK(threshold >= 0.f, "soft_nms_batched: threshold must be >= 0");
  soft_nms_batched_kernel<<<P, kNmsTPB, 0, (cudaStream_t)stream>>>(dets, offsets, sigma, Nt, threshold, method,
                                                                   out_counts, scratch);
  SN_LAUNCH_CHECK();
  return 0;
}

// nmsp (threshold 0.7) of every image p = rows [offsets[p], offsets[p+1]) of dets ([total, 5] x1, y1, x2, y2, score)
// in one launch.  keep: device int32 [total]; its first out_counts[p] entries from offsets[p] on are the kept rows of
// image p (indices local to the image) in keep order.  offsets: device int32 [P+1]; offsets_host: the same on the host,
// read to refuse an image of more than 4096 rows.  An image with a negative (or NaN) score gets out_counts[p] = -1.
int sniper_proposal_nms_batched(const float* dets, const int* offsets, const int* offsets_host, int P, int* out_counts,
                                int* keep, void* stream) {
  if (P <= 0) return 0;
  for (int p = 0; p < P; ++p) {
    const int n = offsets_host[p + 1] - offsets_host[p];
    SN_CHECK(n >= 0 && n <= kPropNmsCap, "proposal_nms_batched: image %d has %d rows (at most %d)", p, n, kPropNmsCap);
  }
  proposal_nms_batched_kernel<<<P, kPropNmsTPB, 0, (cudaStream_t)stream>>>(dets, offsets, out_counts, keep);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
