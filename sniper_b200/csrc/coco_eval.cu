// COCO box evaluation on the device: the bbIou / evaluateImg / accumulate of the reference's pycocotools
// (lib/dataset/pycocotools/maskApi.c:98-109, cocoeval.py:189-374), bit-exact.
//
// Every quantity here is an IEEE double add, multiply, divide, min, max or compare, or an integer count, so the
// results equal the reference's byte for byte as long as nothing is contracted to an FMA (this file is built with
// -fmad=false and the products / sums are spelled out with __d*_rn).
//
// Input: a CSR over the non-empty (category, image) pairs, category-major, images in params.imgIds order.  Pair p owns
//   GT rows  gt_off[p] .. gt_off[p+1]  in annotation order: box xywh, area (the annotation's field), flags
//            (bit 0 iscrowd, bit 1 the `ignore` field), id;
//   DT rows  dt_off[p] .. dt_off[p+1]  sorted by descending score (stable) and cut to maxDets[-1]: box, area (w*h, as
//            loadRes computes it), id (results position + 1).
#include <float.h>
#include <limits.h>

#include "block_reduce.cuh"
#include "common.cuh"

namespace {

constexpr int kMaxT = 64;      // IoU thresholds
constexpr int kMaxA = 16;      // area ranges
constexpr int kMaxM = 16;      // maxDets settings
constexpr int kMaxR = 256;     // recall thresholds
constexpr int kIouTPB = 256;
constexpr int kMatchTPB = 128;
constexpr int kAccTPB = 256;
constexpr int kAccWarps = kAccTPB / 32;

// bbIou (maskApi.c:98-109) for one (dt, gt) pair.  crowd: the union is the detection's area.
__device__ __forceinline__ double bb_iou(const double* D, const double* G, bool crowd) {
  const double ga = __dmul_rn(G[2], G[3]);
  const double da = __dmul_rn(D[2], D[3]);
  const double w = __dsub_rn(fmin(__dadd_rn(D[2], D[0]), __dadd_rn(G[2], G[0])), fmax(D[0], G[0]));
  if (w <= 0) return 0.0;
  const double h = __dsub_rn(fmin(__dadd_rn(D[3], D[1]), __dadd_rn(G[3], G[1])), fmax(D[1], G[1]));
  if (h <= 0) return 0.0;
  const double i = __dmul_rn(w, h);
  const double u = crowd ? da : __dsub_rn(__dadd_rn(da, ga), i);
  return __ddiv_rn(i, u);
}

// one block per pair: the [D_p x G_p] matrix, row-major, at out + iou_off[p]
__global__ void coco_box_iou_kernel(const double* __restrict__ dt_box, const double* __restrict__ gt_box,
                                    const unsigned char* __restrict__ gt_flags, const int* __restrict__ dt_off,
                                    const int* __restrict__ gt_off, const long* __restrict__ iou_off,
                                    double* __restrict__ out) {
  const int p = blockIdx.x;
  const int d0 = dt_off[p], D = dt_off[p + 1] - d0;
  const int g0 = gt_off[p], G = gt_off[p + 1] - g0;
  double* o = out + iou_off[p];
  for (long e = threadIdx.x; e < (long)D * G; e += blockDim.x) {
    const int d = (int)(e / G), g = (int)(e % G);
    o[e] = bb_iou(dt_box + 4L * (d0 + d), gt_box + 4L * (g0 + g), gt_flags[g0 + g] & 1);
  }
}

struct MatchParams {
  double iou_thrs[kMaxT];
  double area_rng[2 * kMaxA];
  int P, T, A;
  long Dtot, Gtot;
};

// evaluateImg (cocoeval.py:189-272) for one (pair, area range, IoU threshold) per thread.  The GTs are visited in the
// reference's order -- non-ignored first, then ignored, each in annotation order (its stable sort on _ignore) -- by two
// passes over the pair's rows; `pos` is the visited GT's index in that order.  gt_match doubles as the reference's gtm:
// the matching dt id, 0 when unmatched, at [(a*T + t)*Gtot + gt_off[p] + pos].
__global__ void coco_match_kernel(const double* __restrict__ dt_box, const double* __restrict__ dt_area,
                                  const long* __restrict__ dt_id, const double* __restrict__ gt_box,
                                  const double* __restrict__ gt_area, const unsigned char* __restrict__ gt_flags,
                                  const long* __restrict__ gt_id, const int* __restrict__ dt_off,
                                  const int* __restrict__ gt_off, const MatchParams prm, unsigned char* dt_flags,
                                  int* npig, long* gt_match, long* dt_match, int* gt_order) {
  const long x = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (long)prm.P * prm.A * prm.T) return;
  const int t = (int)(x % prm.T);
  const int a = (int)((x / prm.T) % prm.A);
  const int p = (int)(x / ((long)prm.T * prm.A));
  const int d0 = dt_off[p], D = dt_off[p + 1] - d0;
  const int g0 = gt_off[p], G = gt_off[p + 1] - g0;
  const double lo = prm.area_rng[2 * a], hi = prm.area_rng[2 * a + 1];
  // _ignore: iscrowd == 1, the `ignore` field, or the area outside [lo, hi]
  auto ignored = [&](int g) -> int {
    const double ar = gt_area[g0 + g];
    return (gt_flags[g0 + g] & 3) || ar < lo || ar > hi;
  };
  long* gm = gt_match + ((long)a * prm.T + t) * prm.Gtot + g0;
  for (int i = 0; i < G; ++i) gm[i] = 0;
  if (t == 0) {
    int n = 0, pos = 0;
    for (int pass = 0; pass < 2; ++pass)
      for (int g = 0; g < G; ++g) {
        if (ignored(g) != pass) continue;
        if (gt_order) gt_order[(long)a * prm.Gtot + g0 + pos] = g;
        ++pos;
        n += pass == 0;
      }
    npig[(long)p * prm.A + a] = n;
  }
  const double thr = fmin(prm.iou_thrs[t], 1.0 - 1e-10);
  const long out0 = ((long)a * prm.T + t) * prm.Dtot + d0;
  for (int d = 0; d < D; ++d) {
    const double* db = dt_box + 4L * (d0 + d);
    double best = thr;
    int m = -1, mg = -1, mig = 0, pos = 0;
    bool stop = false;
    for (int pass = 0; pass < 2 && !stop; ++pass) {
      for (int g = 0; g < G; ++g) {
        if (ignored(g) != pass) continue;
        const int here = pos++;
        const bool crowd = gt_flags[g0 + g] & 1;
        // already matched, and not a crowd: skip
        if (gm[here] > 0 && !crowd) continue;
        // matched to a regular GT and reached the ignored ones: stop
        if (m > -1 && mig == 0 && pass == 1) { stop = true; break; }
        const double iou = bb_iou(db, gt_box + 4L * (g0 + g), crowd);
        // `<`, not `<=`: an IoU equal to the running best goes to the later GT
        if (iou < best) continue;
        best = iou;
        m = here;
        mg = g;
        mig = pass;
      }
    }
    long gid = 0;
    int dig = 0;
    if (m > -1) {
      gid = gt_id[g0 + mg];
      dig = mig;
      gm[m] = dt_id[d0 + d];
    }
    // "matched" is a non-zero stored GT id; unmatched detections outside the area range are ignored
    const double ar = dt_area[d0 + d];
    if (gid == 0 && (ar < lo || ar > hi)) dig = 1;
    dt_flags[out0 + d] = (unsigned char)((gid != 0) | (dig << 1));
    if (dt_match) dt_match[out0 + d] = gid;
  }
}

struct AccParams {
  double rec_thrs[kMaxR];
  int max_dets[kMaxM];
  int K, P, A, T, M, R;
};

// first r with rec_thrs[r] > v (rec_thrs sorted)
__device__ __forceinline__ int upper_bound(const double* thr, int R, double v) {
  int lo = 0, hi = R;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (thr[mid] > v) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// accumulate (cocoeval.py:274-374) for one (category, area range, maxDet, IoU threshold) per block.
// cat_order lists the category's detections sorted by (descending score, concatenation order): the restriction of
// that order to the detections of in-image rank < maxDet is the reference's mergesort of the maxDet-cut concatenation.
// Pass 1 counts tp / fp / kept over the segment; pass 2 walks the chunks from the end so that the running maximum of
// the precision (the reference's reverse loop) is carried along, and each kept detection i writes
// q[r] = max(pr[i:]) for the recall thresholds searchsorted assigns to it: rc[i-1] < rec_thrs[r] <= rc[i].
__global__ void __launch_bounds__(kAccTPB) coco_accumulate_kernel(
    const unsigned char* __restrict__ dt_flags, const int* __restrict__ dt_rank, const int* __restrict__ cat_order,
    const int* __restrict__ dt_off, const int* __restrict__ npig, const int* __restrict__ cat_pair_off,
    const AccParams prm, double* __restrict__ precision, double* __restrict__ recall) {
  __shared__ int3 sh3[kAccWarps];
  __shared__ double shd[kAccWarps];
  __shared__ double s_thr[kMaxR];
  __shared__ int s_npig;
  int b = blockIdx.x;
  const int t = b % prm.T; b /= prm.T;
  const int m = b % prm.M; b /= prm.M;
  const int a = b % prm.A;
  const int k = b / prm.A;
  const int K = prm.K, A = prm.A, M = prm.M, R = prm.R;
  const long rstride = (long)K * A * M;  // precision[t, r, k, a, m]: stride of r
  double* prec = precision + ((long)t * R * K + k) * A * M + (long)a * M + m;
  double* rec = recall + (((long)t * K + k) * A + a) * M + m;
  for (int r = threadIdx.x; r < R; r += blockDim.x) s_thr[r] = prm.rec_thrs[r];
  const int p0 = cat_pair_off[k], p1 = cat_pair_off[k + 1];
  int s = 0;
  for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) s += npig[(long)p * A + a];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(~0u, s, o);
  if (threadIdx.x == 0) s_npig = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_npig, s);
  __syncthreads();
  const int np = s_npig;
  if (p0 == p1 || np == 0) {  // E empty, or no non-ignored GT: the reference leaves -1
    for (int r = threadIdx.x; r < R; r += blockDim.x) prec[r * rstride] = -1.0;
    if (threadIdx.x == 0) *rec = -1.0;
    return;
  }
  const int i0 = dt_off[p0], i1 = dt_off[p1];
  const long Dtot = dt_off[prm.P];
  const unsigned char* fl = dt_flags + ((long)a * prm.T + t) * Dtot;
  const int max_det = prm.max_dets[m];
  const double npd = (double)np;
  auto entry = [&](int i) -> int3 {  // (tp, fp, kept) of sorted position i
    if (i >= i1) return make_int3(0, 0, 0);
    const int d = cat_order[i];
    if (dt_rank[d] >= max_det) return make_int3(0, 0, 0);
    const unsigned char f = fl[d];
    const int ign = (f >> 1) & 1, mt = f & 1;
    return make_int3(!ign && mt, !ign && !mt, 1);
  };
  // pass 1: totals
  int3 tot = make_int3(0, 0, 0);
  for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x) tot = tot + entry(i);
  int3 all;
  block_inclusive_scan<int3, kAccWarps>(tot, sh3, &all);
  if (threadIdx.x == 0) *rec = all.z ? __ddiv_rn((double)all.x, npd) : 0.0;
  for (int r = threadIdx.x; r < R; r += blockDim.x) prec[r * rstride] = 0.0;  // thresholds past the last recall
  __syncthreads();
  // pass 2: chunks from the end
  const int nchunk = (i1 - i0 + kAccTPB - 1) / kAccTPB;
  int3 after = make_int3(0, 0, 0);
  double carry_max = -1.0;
  for (int c = nchunk - 1; c >= 0; --c) {
    const int i = i0 + c * kAccTPB + threadIdx.x;
    const int3 e = entry(i);
    int3 chunk;
    const int3 incl = block_inclusive_scan<int3, kAccWarps>(e, sh3, &chunk);
    // counts up to and including i over the whole segment
    const int tp = all.x - after.x - chunk.x + incl.x;
    const int fp = all.y - after.y - chunk.y + incl.y;
    const int kept_before = all.z - after.z - chunk.z + incl.z - e.z;
    const double tpd = (double)tp;
    const double pr = e.z ? __ddiv_rn(tpd, __dadd_rn(__dadd_rn((double)fp, tpd), DBL_EPSILON)) : -1.0;
    const double suf = fmax(block_suffix_max<kAccWarps>(pr, shd), carry_max);
    if (e.z) {
      const double rc = __ddiv_rn(tpd, npd);
      const int lo = kept_before == 0 ? 0 : upper_bound(s_thr, R, __ddiv_rn((double)(tp - e.x), npd));
      const int hi = upper_bound(s_thr, R, rc);
      for (int r = lo; r < hi; ++r) prec[r * rstride] = suf;
    }
    // the chunk's first thread holds the suffix maximum of the whole chunk
    if (threadIdx.x == 0) shd[0] = suf;
    __syncthreads();
    carry_max = shd[0];
    after = after + chunk;
    __syncthreads();
  }
}

}  // namespace

extern "C" {

int sniper_coco_box_iou_batched(const double* dt_box, const double* gt_box, const unsigned char* gt_flags,
                                const int* dt_off, const int* gt_off, const long* iou_off, const int* dt_off_host,
                                const int* gt_off_host, const long* iou_off_host, int P, double* out, void* stream) {
  SN_CHECK(P >= 0, "coco_box_iou_batched: P (%d) must not be negative", P);
  if (P == 0) return 0;
  SN_CHECK(dt_off_host && gt_off_host && iou_off_host, "coco_box_iou_batched: the host offsets must not be null");
  SN_CHECK(sn::offsets_ok(dt_off_host, P), "coco_box_iou_batched: dt_off must start at 0 and not decrease");
  SN_CHECK(sn::offsets_ok(gt_off_host, P), "coco_box_iou_batched: gt_off must start at 0 and not decrease");
  SN_CHECK(iou_off_host[0] == 0, "coco_box_iou_batched: iou_off must start at 0");
  for (int p = 0; p < P; ++p) {
    const long n = (long)(dt_off_host[p + 1] - dt_off_host[p]) * (gt_off_host[p + 1] - gt_off_host[p]);
    SN_CHECK(iou_off_host[p + 1] - iou_off_host[p] == n,
             "coco_box_iou_batched: iou_off of pair %d spans %ld values, not D x G = %ld", p,
             iou_off_host[p + 1] - iou_off_host[p], n);
  }
  SN_CHECK(dt_off && gt_off && iou_off, "coco_box_iou_batched: dt_off / gt_off / iou_off must not be null");
  SN_CHECK((dt_box || dt_off_host[P] == 0) && (gt_box || gt_off_host[P] == 0) && (gt_flags || gt_off_host[P] == 0),
           "coco_box_iou_batched: dt_box / gt_box / gt_flags must not be null");
  SN_CHECK(out || iou_off_host[P] == 0, "coco_box_iou_batched: out must not be null");
  coco_box_iou_kernel<<<P, kIouTPB, 0, (cudaStream_t)stream>>>(dt_box, gt_box, gt_flags, dt_off, gt_off, iou_off, out);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_coco_match(const double* dt_box, const double* dt_area, const long* dt_id, const double* gt_box,
                      const double* gt_area, const unsigned char* gt_flags, const long* gt_id, const int* dt_off,
                      const int* gt_off, const int* dt_off_host, const int* gt_off_host, int P, const double* iou_thrs,
                      int T, const double* area_rng, int A, unsigned char* dt_flags, int* npig, long* gt_match,
                      long* dt_match, int* gt_order, void* stream) {
  SN_CHECK(P >= 0, "coco_match: P (%d) must not be negative", P);
  SN_CHECK(T >= 1 && T <= kMaxT, "coco_match: T (%d IoU thresholds) must be in [1, %d]", T, kMaxT);
  SN_CHECK(A >= 1 && A <= kMaxA, "coco_match: A (%d area ranges) must be in [1, %d]", A, kMaxA);
  SN_CHECK(iou_thrs && area_rng, "coco_match: iou_thrs / area_rng (host) must not be null");
  if (P == 0) return 0;
  SN_CHECK(dt_off_host && gt_off_host, "coco_match: the host offsets must not be null");
  SN_CHECK(sn::offsets_ok(dt_off_host, P), "coco_match: dt_off must start at 0 and not decrease");
  SN_CHECK(sn::offsets_ok(gt_off_host, P), "coco_match: gt_off must start at 0 and not decrease");
  const long Dtot = dt_off_host[P], Gtot = gt_off_host[P];
  SN_CHECK(dt_off && gt_off && npig, "coco_match: dt_off / gt_off / npig must not be null");
  SN_CHECK(Dtot == 0 || (dt_box && dt_area && dt_id && dt_flags),
           "coco_match: dt_box / dt_area / dt_id / dt_flags must not be null");
  SN_CHECK(Gtot == 0 || (gt_box && gt_area && gt_flags && gt_id && gt_match),
           "coco_match: gt_box / gt_area / gt_flags / gt_id / gt_match must not be null");
  const long threads = (long)P * A * T;
  SN_CHECK(threads / kMatchTPB < INT_MAX, "coco_match: P x A x T (%ld) is too large for one launch", threads);
  MatchParams prm;
  for (int t = 0; t < T; ++t) prm.iou_thrs[t] = iou_thrs[t];
  for (int i = 0; i < 2 * A; ++i) prm.area_rng[i] = area_rng[i];
  prm.P = P; prm.T = T; prm.A = A; prm.Dtot = Dtot; prm.Gtot = Gtot;
  coco_match_kernel<<<(int)((threads + kMatchTPB - 1) / kMatchTPB), kMatchTPB, 0, (cudaStream_t)stream>>>(
      dt_box, dt_area, dt_id, gt_box, gt_area, gt_flags, gt_id, dt_off, gt_off, prm, dt_flags, npig, gt_match,
      dt_match, gt_order);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_coco_accumulate(const unsigned char* dt_flags, const int* dt_rank, const int* cat_order, const int* dt_off,
                           const int* npig, const int* cat_pair_off, const int* dt_off_host,
                           const int* cat_pair_off_host, int K, int P, int A, int T, const int* max_dets, int M,
                           const double* rec_thrs, int R, double* precision, double* recall, void* stream) {
  SN_CHECK(K >= 0 && P >= 0, "coco_accumulate: K (%d) and P (%d) must not be negative", K, P);
  SN_CHECK(T >= 1 && T <= kMaxT, "coco_accumulate: T (%d IoU thresholds) must be in [1, %d]", T, kMaxT);
  SN_CHECK(A >= 1 && A <= kMaxA, "coco_accumulate: A (%d area ranges) must be in [1, %d]", A, kMaxA);
  SN_CHECK(M >= 1 && M <= kMaxM, "coco_accumulate: M (%d maxDets) must be in [1, %d]", M, kMaxM);
  SN_CHECK(R >= 1 && R <= kMaxR, "coco_accumulate: R (%d recall thresholds) must be in [1, %d]", R, kMaxR);
  SN_CHECK(max_dets && rec_thrs, "coco_accumulate: max_dets / rec_thrs (host) must not be null");
  for (int i = 0; i + 1 < M; ++i)
    SN_CHECK(max_dets[i] <= max_dets[i + 1], "coco_accumulate: maxDets must be sorted (%d > %d at %d)", max_dets[i],
             max_dets[i + 1], i);
  for (int i = 0; i + 1 < R; ++i)
    SN_CHECK(rec_thrs[i] <= rec_thrs[i + 1], "coco_accumulate: recThrs must be sorted (index %d)", i);
  if (K == 0) return 0;
  SN_CHECK(cat_pair_off_host && dt_off_host, "coco_accumulate: the host offsets must not be null");
  SN_CHECK(sn::offsets_ok(cat_pair_off_host, K) && cat_pair_off_host[K] == P,
           "coco_accumulate: cat_pair_off must start at 0, not decrease and end at P (%d)", P);
  SN_CHECK(sn::offsets_ok(dt_off_host, P), "coco_accumulate: dt_off must start at 0 and not decrease");
  SN_CHECK(cat_pair_off && dt_off && (npig || P == 0), "coco_accumulate: cat_pair_off / dt_off / npig must not be null");
  SN_CHECK(dt_off_host[P] == 0 || (dt_flags && dt_rank && cat_order),
           "coco_accumulate: dt_flags / dt_rank / cat_order must not be null");
  SN_CHECK(precision && recall, "coco_accumulate: precision / recall must not be null");
  const long blocks = (long)K * A * M * T;
  SN_CHECK(blocks < INT_MAX, "coco_accumulate: K x A x M x T (%ld) is too large for one launch", blocks);
  AccParams prm;
  for (int r = 0; r < R; ++r) prm.rec_thrs[r] = rec_thrs[r];
  for (int i = 0; i < M; ++i) prm.max_dets[i] = max_dets[i];
  prm.K = K; prm.P = P; prm.A = A; prm.T = T; prm.M = M; prm.R = R;
  coco_accumulate_kernel<<<(int)blocks, kAccTPB, 0, (cudaStream_t)stream>>>(dt_flags, dt_rank, cat_order, dt_off, npig,
                                                                           cat_pair_off, prm, precision, recall);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
