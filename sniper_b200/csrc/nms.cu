// Batched per-(image, class) soft-NMS / NMS on the device for the multi-scale inference aggregation.
//
// Replaces the `Pool(32)` of host processes running `cpu_soft_nms` (lib/nms/cpu_nms.pyx:17-110, Gaussian, sigma 0.55,
// score threshold 0.001; called per image and class by Tester.aggregate, lib/inference.py:152-200, through
// nms_worker.worker) -- the "per-scale NMS latency" of BASELINE config 5.  One CTA per problem; all problems of a scale
// (images x 80 classes) run in one launch.
//
// The kernel runs the reference loop on the reference's own row array, in parallel within each step.  Positions
// [i, live) of `work` hold the remaining rows, as boxes[i:N] do in the reference.  Take i: among them the highest
// score, the lowest position on exact ties (the reference's strict `<` scan from i); it swaps places with the row at
// position i.  Decay: every row at a position above i, each once against the taken box; a row whose score falls below
// `threshold` is removed.  Whether a row survives does not depend on its position, so the reference's swap-with-last
// compaction, which interleaves with its decay, can be replayed after the round: with M survivors at positions i+1 ..
// live-1, those below i+1+M stay, the h-th hole of [i+1, i+1+M) counting up receives the h-th survivor at >= i+1+M
// counting down from the end, and live becomes i+1+M.  So exact score ties go where the reference sends them, and
// positions [0, live) at the end are the reference's returned array.  Arithmetic follows the Cythonized reference
// (float IoU with the `+ 1` sums evaluated in double and narrowed once, Gaussian weight = exp evaluated in double);
// this file is compiled with -fmad=false.
#include "block_reduce.cuh"
#include "common.cuh"
#include <limits.h>
#include <math.h>

namespace {

constexpr int kNmsTPB = 256;
constexpr int kNmsWarps = kNmsTPB / 32;

__global__ void __launch_bounds__(kNmsTPB) soft_nms_batched_kernel(float* __restrict__ dets, const int* __restrict__ offsets,
                                                                   float sigma, float Nt, float threshold,
                                                                   unsigned method, int* __restrict__ out_counts,
                                                                   float* __restrict__ scratch) {
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int base = offsets[p], N = offsets[p + 1] - base;
  float* d = dets + (size_t)base * 5;
  float* work = scratch + (size_t)base * 6;     // [N,5] the rows by position (score -1: removed in this round)
  int* slot = reinterpret_cast<int*>(work + (size_t)N * 5);   // [N] compaction: hole positions up, movers down
  __shared__ float s_val[kNmsWarps];
  __shared__ int s_pos[kNmsWarps];
  __shared__ int s_cnt[kNmsWarps];
  __shared__ float s_t[5];
  __shared__ int s_moves, s_stop;
  for (int i = tid; i < N * 5; i += kNmsTPB) work[i] = d[i];
  __syncthreads();
  int live = N;
  for (int i = 0; i < live; ++i) {
    // ---- take: the highest score at positions [i, live), the lowest position on ties
    float best = -1.f;
    int bq = INT_MAX;
    for (int q = i + tid; q < live; q += kNmsTPB) {
      const float s = work[5 * q + 4];
      if (s > best) { best = s; bq = q; }          // strict >: the lowest position wins a tie within a thread
    }
    warp_argmax(best, bq);
    if (lane == 0) { s_val[warp] = best; s_pos[warp] = bq; }
    __syncthreads();
    if (tid == 0) {
      float b = s_val[0];
      int k = s_pos[0];
      for (int w = 1; w < kNmsWarps; ++w)
        if (argmax_beats(s_val[w], s_pos[w], b, k)) { b = s_val[w]; k = s_pos[w]; }
      s_stop = k == INT_MAX;                       // only scores the contract rules out (NaN, <= -1) remain
      if (!s_stop) {
#pragma unroll
        for (int c = 0; c < 5; ++c) {
          s_t[c] = work[5 * k + c];
          work[5 * k + c] = work[5 * i + c];
          work[5 * i + c] = s_t[c];
        }
      }
    }
    __syncthreads();
    if (s_stop) {
      live = i;
      break;
    }
    const float tx1 = s_t[0], ty1 = s_t[1], tx2 = s_t[2], ty2 = s_t[3];
    // ---- decay / remove the rows at positions (i, live)
    int removed = 0;
    for (int q = i + 1 + tid; q < live; q += kNmsTPB) {
      const float s = work[5 * q + 4];
      const float x1 = work[5 * q], y1 = work[5 * q + 1], x2 = work[5 * q + 2], y2 = work[5 * q + 3];
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
          removed |= ns < threshold;
          work[5 * q + 4] = ns < threshold ? -1.f : ns;
        }
      }
    }
    if (!__syncthreads_or(removed)) continue;
    // ---- compaction in the reference's swap-with-last order.  Thread t owns the contiguous positions [q0, q1) of
    // (i, live); a block-wide scan of the survivor counts gives each position its survivor rank.
    const int lo = i + 1, per = (live - lo + kNmsTPB - 1) / kNmsTPB;
    const int q0 = min(live, lo + tid * per), q1 = min(live, q0 + per);
    int mine = 0;
    for (int q = q0; q < q1; ++q) mine += work[5 * q + 4] >= 0.f;
    int incl = mine;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += v;
    }
    if (lane == 31) s_cnt[warp] = incl;
    __syncthreads();
    int before = incl - mine, M = 0;                // survivors before q0; survivors in all of (i, live)
#pragma unroll
    for (int w = 0; w < kNmsWarps; ++w) {
      before += w < warp ? s_cnt[w] : 0;
      M += s_cnt[w];
    }
    const int keep_end = lo + M;
    // hole h (counting up below keep_end) -> slot[h]; survivor g at >= keep_end (counting down) -> slot[N - 1 - g].
    // There are as many of one as of the other, at most (live - lo) / 2 each, so the two ends never meet.
    for (int q = q0, r = before; q < q1; ++q) {
      const bool alive = work[5 * q + 4] >= 0.f;
      if (q == keep_end) s_moves = M - r;         // the survivors from here on fill the holes
      if (q < keep_end && !alive) slot[q - lo - r] = q;
      if (q >= keep_end && alive) slot[N - 1 - (M - 1 - r)] = q;
      r += alive;
    }
    __syncthreads();
    // the movers' positions are >= keep_end, the holes' below it: no row is read here after it is written
    for (int h = tid; h < s_moves; h += kNmsTPB) {
      const int to = slot[h], from = slot[N - 1 - h];
#pragma unroll
      for (int c = 0; c < 5; ++c) work[5 * to + c] = work[5 * from + c];
    }
    live = keep_end;
    __syncthreads();
  }
  for (int j = tid; j < live * 5; j += kNmsTPB) d[j] = work[j];
  if (tid == 0) out_counts[p] = live;
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
// order cpu_soft_nms returns them, exact score ties included.  offsets: device int32 [P+1]; scratch: device, 24 bytes
// per row (total * 6 floats).  Scores must be >= 0.  method 1 = linear, 2 = Gaussian (the reference's TEST default),
// 3 = hard NMS.
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
