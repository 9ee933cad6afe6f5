// PASCAL VOC box evaluation on the device: the matching loop, the precision / recall and voc_ap of the reference's
// voc_eval (lib/dataset/pascal_voc_eval.py:39-181), bit-exact.
//
// Every quantity here is an IEEE double add, subtract, multiply, divide, max, min or compare, or an integer count, so
// the results equal the reference's byte for byte as long as nothing is contracted to an FMA (this file is built with
// -fmad=false and the products / sums are spelled out with __d*_rn).
//
// Detections are one class-major array in the host's order: class c owns positions det_off[c] .. det_off[c+1], in the
// order np.argsort(-confidence) gave on the host (the unstable sort's tie order is the host's, not recomputed here).
// GTs are a CSR over the (class, image) pairs, p = c * num_images + i: all objects of class c in image i in annotation
// order, `difficult` ones included.  pair_det_off / pair_det_pos list, for every pair, the sorted positions of its
// detections in increasing order.
#include <float.h>
#include <limits.h>
#include <math.h>

#include "block_reduce.cuh"
#include "common.cuh"
#include "np_pairwise.cuh"

namespace {

constexpr int kMaxT = 16;      // overlap thresholds in one launch
constexpr int kMax07 = 32;     // recall thresholds of the 11-point metric
constexpr int kMatchTPB = 128;
constexpr int kAccTPB = 256;
constexpr int kAccWarps = kAccTPB / 32;

struct MatchParams {
  double thr[kMaxT];
  int P, T;
  long N, G;
};

// The loop of voc_eval (pascal_voc_eval.py:137-171) for one (pair, threshold) per thread: the pair's detections in
// sorted order, each against all of the pair's GTs.  ovmax / jmax are np.max / np.argmax of the overlaps (a NaN wins
// and the first one is taken; otherwise the first maximum); `ovmax > thr` is strict; a difficult GT sets neither tp nor
// fp; a second hit on a taken GT is an fp.  taken[t * G + g] is the reference's r['det'].
// flags[t * N + pos]: 1 tp, 2 fp, 0 neither.
__global__ void voc_match_kernel(const double* __restrict__ det_box, const int* __restrict__ pair_det_off,
                                 const int* __restrict__ pair_det_pos, const double* __restrict__ gt_box,
                                 const unsigned char* __restrict__ gt_difficult, const int* __restrict__ gt_off,
                                 const MatchParams prm, unsigned char* __restrict__ flags,
                                 unsigned char* __restrict__ taken) {
  const long x = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (long)prm.P * prm.T) return;
  const int t = (int)(x % prm.T);
  const int p = (int)(x / prm.T);
  const int d0 = pair_det_off[p], d1 = pair_det_off[p + 1];
  if (d0 == d1) return;
  const int g0 = gt_off[p], G = gt_off[p + 1] - g0;
  const double thr = prm.thr[t];
  unsigned char* det = taken + (long)t * prm.G + g0;
  unsigned char* out = flags + (long)t * prm.N;
  for (int g = 0; g < G; ++g) det[g] = 0;
  for (int k = d0; k < d1; ++k) {
    const int pos = pair_det_pos[k];
    const double* bb = det_box + 4L * pos;
    const double b0 = bb[0], b1 = bb[1], b2 = bb[2], b3 = bb[3];
    // (bb[2] - bb[0] + 1.) * (bb[3] - bb[1] + 1.)
    const double barea = __dmul_rn(__dadd_rn(__dsub_rn(b2, b0), 1.0), __dadd_rn(__dsub_rn(b3, b1), 1.0));
    double ovmax = -INFINITY;
    int jmax = -1;
    for (int g = 0; g < G; ++g) {
      const double* q = gt_box + 4L * (g0 + g);
      const double ixmin = np_max(q[0], b0), iymin = np_max(q[1], b1);
      const double ixmax = np_min(q[2], b2), iymax = np_min(q[3], b3);
      const double iw = np_max(__dadd_rn(__dsub_rn(ixmax, ixmin), 1.0), 0.0);
      const double ih = np_max(__dadd_rn(__dsub_rn(iymax, iymin), 1.0), 0.0);
      const double inters = __dmul_rn(iw, ih);
      const double garea = __dmul_rn(__dadd_rn(__dsub_rn(q[2], q[0]), 1.0), __dadd_rn(__dsub_rn(q[3], q[1]), 1.0));
      const double uni = __dsub_rn(__dadd_rn(barea, garea), inters);
      const double ov = __ddiv_rn(inters, uni);
      if (g == 0 || (!isnan(ovmax) && (isnan(ov) || ov > ovmax))) {
        ovmax = ov;
        jmax = g;
      }
    }
    unsigned char f = 2;
    if (ovmax > thr) {
      if (gt_difficult[g0 + jmax]) {
        f = 0;
      } else if (!det[jmax]) {
        f = 1;
        det[jmax] = 1;
      }
    }
    out[pos] = f;
  }
}

struct AccParams {
  double thr07[kMax07];
  int n07, use07, C, T;
  long N;
};

// pascal_voc_eval.py:173-179 and voc_ap (:39-70) for one (class, threshold) per block.
// Pass 1 (forward): the integer scans of tp / fp, rec = tp / float(npos), prec = tp / max(tp + fp, eps), the 11-point
// maxima, and the count of positions where mrec = [0, rec, 1] changes.  Pass 2 (area metric, chunks from the end):
// the mpre envelope as a running suffix max, and each changed position's term (mrec[k+1] - mrec[k]) * mpre[k+1]
// written compacted to terms; then one thread adds them in numpy's pairwise order.
__global__ void __launch_bounds__(kAccTPB) voc_accumulate_kernel(const unsigned char* __restrict__ flags,
                                                                 const int* __restrict__ det_off,
                                                                 const int* __restrict__ npos, const AccParams prm,
                                                                 double* __restrict__ rec, double* __restrict__ prec,
                                                                 double* __restrict__ ap, double* __restrict__ terms) {
  __shared__ int2 sh2[kAccWarps];
  __shared__ int sh1[kAccWarps];
  __shared__ double shd[kAccWarps];
  __shared__ double s07[kAccWarps][kMax07];
  __shared__ int s_changed;
  const int c = blockIdx.x % prm.C, t = blockIdx.x / prm.C;
  const int i0 = det_off[c], n = det_off[c + 1] - i0;
  const double npd = (double)npos[c];
  const unsigned char* fl = flags + (long)t * prm.N + i0;
  double* rc = rec + (long)t * prm.N + i0;
  double* pc = prec + (long)t * prm.N + i0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double m07[kMax07];
  for (int j = 0; j < prm.n07; ++j) m07[j] = -1.0;
  if (threadIdx.x == 0) s_changed = 0;
  __syncthreads();
  const int nchunk = (n + kAccTPB - 1) / kAccTPB;
  int2 before = make_int2(0, 0);
  int changed = 0;
  for (int ch = 0; ch < nchunk; ++ch) {
    const int i = ch * kAccTPB + threadIdx.x;
    const unsigned char f = i < n ? fl[i] : 0;
    int2 chunk;
    const int2 incl = block_inclusive_scan<int2, kAccWarps>(make_int2(f == 1, f == 2), sh2, &chunk) + before;
    before = before + chunk;
    if (i < n) {
      const double tpd = (double)incl.x, fpd = (double)incl.y;
      const double r = __ddiv_rn(tpd, npd);
      const double pr = __ddiv_rn(tpd, fmax(__dadd_rn(tpd, fpd), DBL_EPSILON));
      rc[i] = r;
      pc[i] = pr;
      if (prm.use07) {
        for (int j = 0; j < prm.n07; ++j)
          if (r >= prm.thr07[j]) m07[j] = fmax(m07[j], pr);
      } else {
        const double r_prev = i == 0 ? 0.0 : __ddiv_rn((double)(incl.x - (f == 1)), npd);
        changed += r != r_prev;
      }
    }
  }
  if (prm.use07) {
    for (int j = 0; j < prm.n07; ++j) {
      double v = m07[j];
      for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(~0u, v, o));
      if (lane == 0) s07[warp][j] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      // ap = 0.; ap += p / 11. in threshold order, p = 0 where no recall reaches the threshold
      double a = 0.0;
      for (int j = 0; j < prm.n07; ++j) {
        double p = -1.0;
        for (int w = 0; w < kAccWarps; ++w) p = fmax(p, s07[w][j]);
        a = __dadd_rn(a, __ddiv_rn(p < 0.0 ? 0.0 : p, 11.0));
      }
      ap[(long)t * prm.C + c] = a;
    }
    return;
  }
  // the last step of mrec, rec[n-1] -> 1 (0 -> 1 when there is no detection)
  const double r_last = n == 0 ? 0.0 : __ddiv_rn((double)before.x, npd);
  for (int o = 16; o > 0; o >>= 1) changed += __shfl_xor_sync(~0u, changed, o);
  if (lane == 0) atomicAdd(&s_changed, changed);
  __syncthreads();
  const int m = s_changed + (r_last != 1.0);
  double* tm = terms + (long)t * (prm.N + prm.C) + i0 + c;
  if (threadIdx.x == 0 && r_last != 1.0) tm[m - 1] = __dmul_rn(__dsub_rn(1.0, r_last), 0.0);
  // pass 2: chunks from the end; `after` counts the changed positions past the chunk, carry is mpre past it
  int after = 0;
  double carry = 0.0;
  for (int ch = nchunk - 1; ch >= 0; --ch) {
    const int i = ch * kAccTPB + threadIdx.x;
    double r = 0.0, r_prev = 0.0, pr = -1.0;
    int ci = 0;
    if (i < n) {
      r = rc[i];
      pr = pc[i];
      r_prev = i == 0 ? 0.0 : rc[i - 1];
      ci = r != r_prev;
    }
    const double mp = fmax(block_suffix_max<kAccWarps>(pr, shd), carry);
    // changed positions at and after i within the chunk: an inclusive scan from the end
    int tot;
    const int incl = block_inclusive_scan<int, kAccWarps>(ci, sh1, &tot);
    const int at_or_after = tot - incl + ci;
    if (ci) tm[s_changed - after - at_or_after] = __dmul_rn(__dsub_rn(r, r_prev), mp);
    if (threadIdx.x == 0) shd[0] = mp;
    __syncthreads();
    carry = shd[0];
    after += tot;
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x == 0) ap[(long)t * prm.C + c] = np_sum(tm, m);
}

}  // namespace

extern "C" {

int sniper_voc_match(const double* det_box, const int* pair_det_off, const int* pair_det_pos, const double* gt_box,
                     const unsigned char* gt_difficult, const int* gt_off, const int* pair_det_off_host,
                     const int* gt_off_host, int P, const double* thresholds, int T, unsigned char* flags,
                     unsigned char* taken, void* stream) {
  SN_CHECK(P >= 0, "voc_match: P (%d) must not be negative", P);
  SN_CHECK(T >= 1 && T <= kMaxT, "voc_match: T (%d overlap thresholds) must be in [1, %d]", T, kMaxT);
  SN_CHECK(thresholds, "voc_match: thresholds (host) must not be null");
  if (P == 0) return 0;
  SN_CHECK(pair_det_off_host && gt_off_host, "voc_match: the host offsets must not be null");
  SN_CHECK(sn::offsets_ok(pair_det_off_host, P), "voc_match: pair_det_off must start at 0 and not decrease");
  SN_CHECK(sn::offsets_ok(gt_off_host, P), "voc_match: gt_off must start at 0 and not decrease");
  const long N = pair_det_off_host[P], G = gt_off_host[P];
  SN_CHECK(pair_det_off && gt_off, "voc_match: pair_det_off / gt_off must not be null");
  SN_CHECK(N == 0 || (det_box && pair_det_pos && flags), "voc_match: det_box / pair_det_pos / flags must not be null");
  SN_CHECK(G == 0 || (gt_box && gt_difficult && taken), "voc_match: gt_box / gt_difficult / taken must not be null");
  const long threads = (long)P * T;
  SN_CHECK(threads / kMatchTPB < INT_MAX, "voc_match: P x T (%ld) is too large for one launch", threads);
  if (N == 0) return 0;
  MatchParams prm;
  for (int t = 0; t < T; ++t) prm.thr[t] = thresholds[t];
  prm.P = P; prm.T = T; prm.N = N; prm.G = G;
  voc_match_kernel<<<(int)((threads + kMatchTPB - 1) / kMatchTPB), kMatchTPB, 0, (cudaStream_t)stream>>>(
      det_box, pair_det_off, pair_det_pos, gt_box, gt_difficult, gt_off, prm, flags, taken);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_voc_accumulate(const unsigned char* flags, const int* det_off, const int* npos, const int* det_off_host,
                          int C, int T, int use_07_metric, const double* thresholds_07, int n07, double* rec,
                          double* prec, double* ap, double* terms, void* stream) {
  SN_CHECK(C >= 0, "voc_accumulate: C (%d) must not be negative", C);
  SN_CHECK(T >= 1 && T <= kMaxT, "voc_accumulate: T (%d overlap thresholds) must be in [1, %d]", T, kMaxT);
  SN_CHECK(use_07_metric == 0 || use_07_metric == 1, "voc_accumulate: use_07_metric (%d) must be 0 or 1",
           use_07_metric);
  if (use_07_metric) {
    SN_CHECK(n07 >= 1 && n07 <= kMax07, "voc_accumulate: n07 (%d recall thresholds) must be in [1, %d]", n07, kMax07);
    SN_CHECK(thresholds_07, "voc_accumulate: thresholds_07 (host) must not be null");
  }
  if (C == 0) return 0;
  SN_CHECK(det_off_host, "voc_accumulate: the host offsets must not be null");
  SN_CHECK(sn::offsets_ok(det_off_host, C), "voc_accumulate: det_off must start at 0 and not decrease");
  const long N = det_off_host[C];
  SN_CHECK(det_off && npos && ap, "voc_accumulate: det_off / npos / ap must not be null");
  SN_CHECK(N == 0 || (flags && rec && prec), "voc_accumulate: flags / rec / prec must not be null");
  SN_CHECK(use_07_metric || terms, "voc_accumulate: terms must not be null for the area metric");
  const long blocks = (long)C * T;
  SN_CHECK(blocks < INT_MAX, "voc_accumulate: C x T (%ld) is too large for one launch", blocks);
  AccParams prm;
  for (int j = 0; use_07_metric && j < n07; ++j) prm.thr07[j] = thresholds_07[j];
  prm.n07 = use_07_metric ? n07 : 0; prm.use07 = use_07_metric; prm.C = C; prm.T = T; prm.N = N;
  voc_accumulate_kernel<<<(int)blocks, kAccTPB, 0, (cudaStream_t)stream>>>(flags, det_off, npos, prm, rec, prec, ap,
                                                                           terms);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
