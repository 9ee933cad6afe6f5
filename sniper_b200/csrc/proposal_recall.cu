// Proposal recall on the device: the greedy matching, the recalls, the average recall and the proposal area histogram
// of the reference's IMDB.evaluate_recall (lib/dataset/imdb.py:291-397), bit-exact.
//
// Every quantity is an IEEE double add, subtract, multiply, divide or compare (the IoU of bbox_overlaps_cython,
// lib/bbox/bbox.pyx:17-57), a float32 / uint16 area in the box array's own dtype, or an integer count, so the results
// equal the reference's byte for byte as long as nothing is contracted to an FMA (this file is built with -fmad=false
// and the double operations are spelled out with __d*_rn).
//
// Inputs are CSRs over images: image i owns proposals prop_off[i] .. prop_off[i+1] (uint16, float32 or float64 as
// stored, widened to float64 in registers) and GTs gt_off[i] .. gt_off[i+1] (float64), the GTs the reference keeps
// (gt_classes > 0 and max gt_overlaps == 1) in roidb order.  gt_range[g] has bit r set when GT g's area, computed on
// the host in its own dtype, lies in area range r (0 = all, 1 .. 6 = 0-25 .. 300-inf).  A pair p = r * num_images + i
// is one (area range, image) of the reference's loop; its GTs are image i's with bit r, in order.
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include "block_reduce.cuh"
#include "common.cuh"
#include "np_pairwise.cuh"

namespace {

constexpr int kRanges = 7;
constexpr int kMatchTPB = 256;
constexpr int kMatchWarps = kMatchTPB / 32;
constexpr int kMaxCols = 1024;                  // GTs of one (image, range) pair
constexpr long kSmemCap = 110 * 1024;           // dynamic shared memory of a matching block: two blocks per SM
constexpr int kColBytes = 6 * 8 + 2 * 4;        // box[4], area, best value; best row, used
constexpr int kAccTPB = 256;
constexpr int kAccWarps = kAccTPB / 32;
constexpr int kAccChunk = 2048;                 // gt_overlaps values a counting block stages in shared memory

// matching status per pair: the reference's assert (a best overlap < 0 or NaN) and the ZeroDivisionError of
// bbox_overlaps_cython (a zero union)
constexpr unsigned char kStatusNegative = 1;
constexpr unsigned char kStatusZeroUnion = 2;

__host__ __device__ inline long meta_bytes(int m) { return (((long)m * kColBytes) + 15) / 16 * 16; }

// shared-memory bytes of a pair that keeps its IoU matrix in shared memory, or -1 when the matrix goes to the workspace
__host__ __device__ inline long smem_bytes(long n, int m) {
  const long all = meta_bytes(m) + n * m * 8;
  return all <= kSmemCap ? all : -1;
}

template <typename T>
__device__ __forceinline__ double widen(T v) { return (double)v; }

// cython's min / max of two C doubles: the second argument when it compares strictly less / greater
__device__ __forceinline__ double cy_min(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double cy_max(double a, double b) { return b > a ? b : a; }

struct MatchParams {
  int num_images, pair_begin;
  long long ws_base;
};

// One (area range, image) pair per block: the IoU matrix of the image's proposals x the range's GTs (column-major, in
// shared memory or in the pair's slice of the workspace), then the reference's rounds.  Each round takes, over the
// unused columns, the largest column maximum (lowest column on ties; each column's maximum is over the unused rows,
// lowest row on ties), records it, and retires its row and column.  Retiring a row sets it to -inf, so only the columns
// whose best row it was are rescanned.  out[pair_out_off[p] + k] is the k-th round's overlap, zeros after the last.
template <typename BoxT>
__global__ void __launch_bounds__(kMatchTPB, 2) recall_match_kernel(
    const BoxT* __restrict__ prop, const int* __restrict__ prop_off, const double* __restrict__ gt_box,
    const unsigned char* __restrict__ gt_range, const int* __restrict__ gt_off, const long long* __restrict__ pair_out_off,
    const long long* __restrict__ pair_ws_off, const MatchParams prm, double* __restrict__ ws,
    double* __restrict__ out, unsigned char* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char sm[];
  __shared__ int s_m, s_pick;
  const int p = prm.pair_begin + blockIdx.x;
  const int r = p / prm.num_images, i = p % prm.num_images;
  const int p0 = prop_off[i], n = prop_off[i + 1] - p0;
  if (n == 0) return;  // an image without proposals contributes nothing
  const int g0 = gt_off[i], G = gt_off[i + 1] - g0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // the range's GTs in roidb order: warp 0 compacts them with ballots
  if (threadIdx.x == 0) s_m = 0;
  __syncthreads();
  if (warp == 0) {
    int cnt = 0;
    for (int b = 0; b < G; b += 32) {
      const int g = b + lane;
      const bool in = g < G && ((gt_range[g0 + g] >> r) & 1);
      cnt += __popc(__ballot_sync(~0u, in));
    }
    if (lane == 0) s_m = cnt;
  }
  __syncthreads();
  const int m = s_m;
  if (m == 0) return;
  double* cbox = reinterpret_cast<double*>(sm);       // [4][m]
  double* carea = cbox + 4 * m;                        // [m]
  double* cbest = carea + m;                           // [m]
  int* crow = reinterpret_cast<int*>(cbest + m);       // [m]
  int* cused = crow + m;                               // [m]
  const long sb = smem_bytes(n, m);
  double* mat = sb >= 0 ? reinterpret_cast<double*>(sm + meta_bytes(m))
                        : ws + (pair_ws_off[p] - prm.ws_base) / 8;
  if (warp == 0) {
    int before = 0;
    for (int b = 0; b < G; b += 32) {
      const int g = b + lane;
      const bool in = g < G && ((gt_range[g0 + g] >> r) & 1);
      const unsigned bal = __ballot_sync(~0u, in);
      if (in) {
        const int j = before + __popc(bal & ((1u << lane) - 1));
        const double* q = gt_box + 4L * (g0 + g);
        const double q0 = q[0], q1 = q[1], q2 = q[2], q3 = q[3];
        cbox[j] = q0; cbox[m + j] = q1; cbox[2 * m + j] = q2; cbox[3 * m + j] = q3;
        // (query_boxes[k, 2] - query_boxes[k, 0] + 1) * (query_boxes[k, 3] - query_boxes[k, 1] + 1)
        carea[j] = __dmul_rn(__dadd_rn(__dsub_rn(q2, q0), 1.0), __dadd_rn(__dsub_rn(q3, q1), 1.0));
        cused[j] = 0;
      }
      before += __popc(bal);
    }
  }
  __syncthreads();
  // bbox_overlaps_cython(boxes.astype(np.float), gt_boxes.astype(np.float)), column-major
  const long cells = (long)n * m;
  bool zero_union = false;
  for (long c = threadIdx.x; c < cells; c += kMatchTPB) {
    const int j = (int)(c / n), row = (int)(c % n);
    const BoxT* b = prop + 4L * (p0 + row);
    const double b0 = widen(b[0]), b1 = widen(b[1]), b2 = widen(b[2]), b3 = widen(b[3]);
    const double q0 = cbox[j], q1 = cbox[m + j], q2 = cbox[2 * m + j], q3 = cbox[3 * m + j];
    double ov = 0.0;
    const double iw = __dadd_rn(__dsub_rn(cy_min(b2, q2), cy_max(b0, q0)), 1.0);
    if (iw > 0) {
      const double ih = __dadd_rn(__dsub_rn(cy_min(b3, q3), cy_max(b1, q1)), 1.0);
      if (ih > 0) {
        const double inter = __dmul_rn(iw, ih);
        const double barea = __dmul_rn(__dadd_rn(__dsub_rn(b2, b0), 1.0), __dadd_rn(__dsub_rn(b3, b1), 1.0));
        const double ua = __dsub_rn(__dadd_rn(barea, carea[j]), inter);
        if (ua == 0.0) zero_union = true;
        else ov = __ddiv_rn(inter, ua);
      }
    }
    mat[c] = ov;
  }
  if (__syncthreads_or(zero_union)) {
    if (threadIdx.x == 0) status[p] = kStatusZeroUnion;
    return;
  }
  // every column's best row (a NaN anywhere fails the first round's assert)
  bool nan_seen = false;
  for (int j = warp; j < m; j += kMatchWarps) {
    double bv = -INFINITY;
    int br = INT_MAX;
    for (int row = lane; row < n; row += 32) {
      const double v = mat[(long)j * n + row];
      nan_seen |= isnan(v);
      if (v > bv || br == INT_MAX) { bv = v; br = row; }
    }
    warp_argmax(bv, br);
    if (lane == 0) { cbest[j] = bv; crow[j] = br; }
  }
  if (__syncthreads_or(nan_seen)) {
    if (threadIdx.x == 0) status[p] = kStatusNegative;
    return;
  }
  const int R = min(n, m);
  double* o = out + pair_out_off[p];
  for (int k = 0; k < R; ++k) {
    if (warp == 0) {
      double bv = -INFINITY;
      int bj = INT_MAX;
      for (int j = lane; j < m; j += 32)
        if (!cused[j] && argmax_beats(cbest[j], j, bv, bj)) { bv = cbest[j]; bj = j; }
      warp_argmax(bv, bj);
      if (lane == 0) {
        // assert (gt_ovr >= 0)
        if (!(bv >= 0.0)) {
          status[p] = kStatusNegative;
          bj = -1;
        } else {
          o[k] = bv;
          cused[bj] = 1;
        }
        s_pick = bj;
      }
    }
    __syncthreads();
    const int jc = s_pick;
    if (jc < 0) return;
    if (k + 1 == R) break;
    const int used_row = crow[jc];
    for (int j = threadIdx.x; j < m; j += kMatchTPB) mat[(long)j * n + used_row] = -INFINITY;
    __syncthreads();
    for (int j = warp; j < m; j += kMatchWarps) {
      if (cused[j] || crow[j] != used_row) continue;
      double bv = -INFINITY;
      int br = INT_MAX;
      for (int row = lane; row < n; row += 32) {
        const double v = mat[(long)j * n + row];
        if (argmax_beats(v, row, bv, br)) { bv = v; br = row; }
      }
      warp_argmax(bv, br);
      if (lane == 0) { cbest[j] = bv; crow[j] = br; }
    }
    __syncthreads();
  }
  for (int k = R + threadIdx.x; k < m; k += kMatchTPB) o[k] = 0.0;
}

struct AccParams {
  long long range_off[kRanges + 1];  // each range's slice of gt_overlaps
  long long num_pos[kRanges];
  long long num_props;
  int T, prop_dtype, count_blocks, num_images;
};

// area_ranges[1:] of the reference as bounds in the box dtype: >= lo and < hi
__device__ int hist_bin_u16(const uint16_t* b) {
  // (boxes[:, 2] - boxes[:, 0] + 1) * (boxes[:, 3] - boxes[:, 1] + 1) in uint16, wrapping
  const uint16_t w = (uint16_t)((uint16_t)(b[2] - b[0]) + 1), h = (uint16_t)((uint16_t)(b[3] - b[1]) + 1);
  const long a = (uint16_t)((uint32_t)w * h);
  const long lo[6] = {0, 625, 2500, 10000, 40000, 90000}, hi[6] = {625, 2500, 10000, 40000, 90000, 10000000000L};
  for (int k = 0; k < 6; ++k)
    if (a >= lo[k] && a < hi[k]) return k;
  return -1;
}

__device__ int hist_bin_f32(const float* b) {
  const float a = __fmul_rn(__fadd_rn(__fsub_rn(b[2], b[0]), 1.0f), __fadd_rn(__fsub_rn(b[3], b[1]), 1.0f));
  const float lo[6] = {0.f, 625.f, 2500.f, 10000.f, 40000.f, 90000.f}, hi[6] = {625.f, 2500.f, 10000.f, 40000.f,
                                                                                 90000.f, 1e10f};
  for (int k = 0; k < 6; ++k)
    if (a >= lo[k] && a < hi[k]) return k;
  return -1;
}

__device__ int hist_bin_f64(const double* b) {
  const double a = __dmul_rn(__dadd_rn(__dsub_rn(b[2], b[0]), 1.0), __dadd_rn(__dsub_rn(b[3], b[1]), 1.0));
  const double lo[6] = {0., 625., 2500., 10000., 40000., 90000.}, hi[6] = {625., 2500., 10000., 40000., 90000., 1e10};
  for (int k = 0; k < 6; ++k)
    if (a >= lo[k] && a < hi[k]) return k;
  return -1;
}

// The counting blocks take a slice of one range's gt_overlaps each and count, per threshold, the values >= it; the
// histogram blocks count the proposals of each area range.  Counts are integer atomics (order-free).  The last block
// to finish computes recall[r, t] = count / float(num_pos), ar = recalls.mean() (numpy's pairwise sum, then / T), the
// fractions area_count / total_counts and total_counts / num_images.
__global__ void __launch_bounds__(kAccTPB) recall_accumulate_kernel(
    const double* __restrict__ gt_overlaps, const double* __restrict__ thr, const void* __restrict__ prop,
    const AccParams prm, unsigned long long* __restrict__ counts, unsigned int* __restrict__ done,
    double* __restrict__ recalls, double* __restrict__ ar, double* __restrict__ hist) {
  __shared__ double sv[kAccChunk];
  __shared__ unsigned long long sh[kAccWarps];
  __shared__ bool s_last;
  const int T = prm.T;
  if ((int)blockIdx.x < prm.count_blocks) {
    // block b: chunk c of range r, ranges' chunks in order
    int b = blockIdx.x, r = 0;
    long long lo = 0, hi = 0;
    for (r = 0; r < kRanges; ++r) {
      const long long len = prm.range_off[r + 1] - prm.range_off[r];
      const int nb = (int)((len + kAccChunk - 1) / kAccChunk);
      if (b < nb) {
        lo = prm.range_off[r] + (long long)b * kAccChunk;
        hi = min(lo + kAccChunk, prm.range_off[r + 1]);
        break;
      }
      b -= nb;
    }
    const int len = (int)(hi - lo);
    for (int k = threadIdx.x; k < len; k += kAccTPB) sv[k] = gt_overlaps[lo + k];
    __syncthreads();
    for (int t = 0; t < T; ++t) {
      const double th = thr[t];
      unsigned long long c = 0;
      for (int k = threadIdx.x; k < len; k += kAccTPB) c += sv[k] >= th;
      c = block_sum<unsigned long long, kAccWarps>(c, sh);
      if (threadIdx.x == 0 && c) atomicAdd(&counts[(long)r * T + t], c);
    }
  } else {
    unsigned long long c[6] = {0, 0, 0, 0, 0, 0};
    const long long nblk = gridDim.x - prm.count_blocks;
    for (long long q = (long long)(blockIdx.x - prm.count_blocks) * kAccTPB + threadIdx.x; q < prm.num_props;
         q += nblk * kAccTPB) {
      int k;
      if (prm.prop_dtype == 0) k = hist_bin_u16(static_cast<const uint16_t*>(prop) + 4 * q);
      else if (prm.prop_dtype == 1) k = hist_bin_f32(static_cast<const float*>(prop) + 4 * q);
      else k = hist_bin_f64(static_cast<const double*>(prop) + 4 * q);
      for (int j = 0; j < 6; ++j) c[j] += k == j;
    }
    for (int j = 0; j < 6; ++j) {
      const unsigned long long s = block_sum<unsigned long long, kAccWarps>(c[j], sh);
      if (threadIdx.x == 0 && s) atomicAdd(&counts[(long)kRanges * T + j], s);
    }
  }
  // the last block to arrive finishes
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const volatile unsigned long long* vc = counts;
  for (int x = threadIdx.x; x < kRanges * T; x += kAccTPB) {
    const int r = x / T;
    recalls[x] = __ddiv_rn((double)vc[x], (double)prm.num_pos[r]);
  }
  __syncthreads();
  if (threadIdx.x < kRanges) ar[threadIdx.x] = __ddiv_rn(np_sum(recalls + (long)threadIdx.x * T, T), (double)T);
  if (threadIdx.x == 0) {
    unsigned long long total = 0;
    for (int j = 0; j < 6; ++j) total += vc[(long)kRanges * T + j];
    const double tc = (double)total;
    for (int j = 0; j < 6; ++j) hist[j] = __ddiv_rn((double)vc[(long)kRanges * T + j], tc);
    hist[6] = __ddiv_rn(tc, (double)prm.num_images);
  }
}

// per pair: n, m; -1 with the message set when the inputs are refused
int pair_sizes(const int* prop_off_host, const int* gt_off_host, const unsigned char* gt_range_host, int num_images,
               int* pair_n, int* pair_m) {
  for (int i = 0; i < num_images; ++i) {
    int cnt[kRanges] = {0, 0, 0, 0, 0, 0, 0};
    for (int g = gt_off_host[i]; g < gt_off_host[i + 1]; ++g)
      for (int r = 0; r < kRanges; ++r) cnt[r] += (gt_range_host[g] >> r) & 1;
    for (int r = 0; r < kRanges; ++r) {
      SN_CHECK(cnt[r] <= kMaxCols, "proposal_recall: image %d has %d GTs in area range %d (at most %d)", i, cnt[r], r,
               kMaxCols);
      pair_n[(long)r * num_images + i] = prop_off_host[i + 1] - prop_off_host[i];
      pair_m[(long)r * num_images + i] = cnt[r];
    }
  }
  return 0;
}

int check_csr(const int* prop_off_host, const int* gt_off_host, const unsigned char* gt_range_host, int num_images) {
  SN_CHECK(num_images >= 0, "proposal_recall: num_images (%d) must not be negative", num_images);
  SN_CHECK((long)num_images * kRanges < INT_MAX, "proposal_recall: num_images (%d) is too large", num_images);
  SN_CHECK(prop_off_host && gt_off_host, "proposal_recall: the host offsets must not be null");
  SN_CHECK(sn::offsets_ok(prop_off_host, num_images), "proposal_recall: prop_off must start at 0 and not decrease");
  SN_CHECK(sn::offsets_ok(gt_off_host, num_images), "proposal_recall: gt_off must start at 0 and not decrease");
  SN_CHECK(gt_off_host[num_images] == 0 || gt_range_host, "proposal_recall: gt_range (host) must not be null");
  for (int g = 0; g < gt_off_host[num_images]; ++g)
    SN_CHECK(gt_range_host[g] < (1u << kRanges), "proposal_recall: gt_range[%d] (%d) has bits above the %d ranges", g,
             gt_range_host[g], kRanges);
  return 0;
}

}  // namespace

extern "C" {

int sniper_proposal_recall_workspace_bytes(const int* prop_off_host, const int* gt_off_host,
                                           const unsigned char* gt_range_host, int num_images,
                                           long long* pair_ws_off_host) {
  if (check_csr(prop_off_host, gt_off_host, gt_range_host, num_images)) return -1;
  SN_CHECK(pair_ws_off_host, "proposal_recall_workspace_bytes: pair_ws_off (host) must not be null");
  const long P = (long)num_images * kRanges;
  int* pn = new int[P + 1];
  int* pm = new int[P + 1];
  const int rc = pair_sizes(prop_off_host, gt_off_host, gt_range_host, num_images, pn, pm);
  if (rc == 0) {
    long long off = 0;
    for (long p = 0; p < P; ++p) {
      pair_ws_off_host[p] = off;
      if (pn[p] > 0 && pm[p] > 0 && smem_bytes(pn[p], pm[p]) < 0) off += (long long)pn[p] * pm[p] * 8;
    }
    pair_ws_off_host[P] = off;
  }
  delete[] pn;
  delete[] pm;
  return rc;
}

int sniper_proposal_recall_match(const void* prop_box, int prop_dtype, const int* prop_off, const double* gt_box,
                                 const unsigned char* gt_range, const int* gt_off, const long long* pair_out_off,
                                 const long long* pair_ws_off, const int* prop_off_host, const int* gt_off_host,
                                 const unsigned char* gt_range_host, const long long* pair_ws_off_host, int num_images,
                                 int pair_begin, int pair_end, void* workspace, double* gt_overlaps,
                                 unsigned char* status, void* stream) {
  SN_CHECK(prop_dtype >= 0 && prop_dtype <= 2, "proposal_recall_match: prop_dtype (%d) must be 0 (uint16), 1 (float32) "
           "or 2 (float64)", prop_dtype);
  if (check_csr(prop_off_host, gt_off_host, gt_range_host, num_images)) return -1;
  const long P = (long)num_images * kRanges;
  SN_CHECK(pair_begin >= 0 && pair_begin <= pair_end && pair_end <= P,
           "proposal_recall_match: pairs [%d, %d) must lie in [0, %ld)", pair_begin, pair_end, P);
  if (pair_begin == pair_end) return 0;
  SN_CHECK(pair_ws_off_host, "proposal_recall_match: pair_ws_off (host) must not be null");
  SN_CHECK(prop_off && gt_off && pair_out_off && pair_ws_off && status,
           "proposal_recall_match: prop_off / gt_off / pair_out_off / pair_ws_off / status must not be null");
  SN_CHECK(prop_off_host[num_images] == 0 || prop_box, "proposal_recall_match: prop_box must not be null");
  SN_CHECK(gt_off_host[num_images] == 0 || (gt_box && gt_range && gt_overlaps),
           "proposal_recall_match: gt_box / gt_range / gt_overlaps must not be null");
  int* pn = new int[P + 1];
  int* pm = new int[P + 1];
  long smem = 0;
  bool ws_ok = true;
  int rc = pair_sizes(prop_off_host, gt_off_host, gt_range_host, num_images, pn, pm);
  for (long p = pair_begin; rc == 0 && p < pair_end; ++p) {
    if (pn[p] == 0 || pm[p] == 0) continue;
    const long sb = smem_bytes(pn[p], pm[p]);
    if (sb >= 0) {
      smem = sb > smem ? sb : smem;
    } else {
      smem = meta_bytes(pm[p]) > smem ? meta_bytes(pm[p]) : smem;
      ws_ok &= pair_ws_off_host[p + 1] - pair_ws_off_host[p] == (long long)pn[p] * pm[p] * 8;
    }
  }
  delete[] pn;
  delete[] pm;
  if (rc) return rc;
  SN_CHECK(ws_ok, "proposal_recall_match: pair_ws_off does not match sniper_proposal_recall_workspace_bytes");
  SN_CHECK(pair_ws_off_host[pair_end] == pair_ws_off_host[pair_begin] || workspace,
           "proposal_recall_match: these pairs need a workspace of %lld bytes",
           pair_ws_off_host[pair_end] - pair_ws_off_host[pair_begin]);
  MatchParams prm;
  prm.num_images = num_images;
  prm.pair_begin = pair_begin;
  prm.ws_base = pair_ws_off_host[pair_begin];
  const int grid = pair_end - pair_begin;
  cudaStream_t st = (cudaStream_t)stream;
  double* ws = static_cast<double*>(workspace);
#define SN_RECALL_LAUNCH(T)                                                                                          \
  do {                                                                                                               \
    SN_CUDA(cudaFuncSetAttribute(recall_match_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCap)); \
    recall_match_kernel<T><<<grid, kMatchTPB, smem, st>>>(static_cast<const T*>(prop_box), prop_off, gt_box,         \
                                                          gt_range, gt_off, pair_out_off, pair_ws_off, prm, ws,      \
                                                          gt_overlaps, status);                                      \
  } while (0)
  if (prop_dtype == 0) SN_RECALL_LAUNCH(uint16_t);
  else if (prop_dtype == 1) SN_RECALL_LAUNCH(float);
  else SN_RECALL_LAUNCH(double);
#undef SN_RECALL_LAUNCH
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_proposal_recall_accumulate(const double* gt_overlaps, const long long* range_off_host,
                                      const long long* num_pos_host, const double* thresholds, int T,
                                      const void* prop_box, int prop_dtype, long num_props, int num_images,
                                      unsigned long long* counts, unsigned int* done, double* recalls, double* ar,
                                      double* hist, void* stream) {
  SN_CHECK(T >= 0, "proposal_recall_accumulate: T (%d thresholds) must not be negative", T);
  SN_CHECK(prop_dtype >= 0 && prop_dtype <= 2, "proposal_recall_accumulate: prop_dtype (%d) must be 0 (uint16), "
           "1 (float32) or 2 (float64)", prop_dtype);
  SN_CHECK(num_props >= 0 && num_images >= 0, "proposal_recall_accumulate: num_props (%ld) and num_images (%d) must "
           "not be negative", num_props, num_images);
  SN_CHECK(range_off_host && num_pos_host, "proposal_recall_accumulate: range_off / num_pos (host) must not be null");
  SN_CHECK(range_off_host[0] == 0, "proposal_recall_accumulate: range_off must start at 0");
  SN_CHECK(sn::offsets_ok(range_off_host, kRanges), "proposal_recall_accumulate: range_off must not decrease");
  for (int r = 0; r < kRanges; ++r)
    SN_CHECK(num_pos_host[r] >= 0, "proposal_recall_accumulate: num_pos[%d] must not be negative", r);
  SN_CHECK(counts && done && ar && hist, "proposal_recall_accumulate: counts / done / ar / hist must not be null");
  SN_CHECK(T == 0 || (thresholds && recalls), "proposal_recall_accumulate: thresholds / recalls must not be null");
  SN_CHECK(range_off_host[kRanges] == 0 || gt_overlaps, "proposal_recall_accumulate: gt_overlaps must not be null");
  SN_CHECK(num_props == 0 || prop_box, "proposal_recall_accumulate: prop_box must not be null");
  AccParams prm;
  long long cb = 0;
  for (int r = 0; r <= kRanges; ++r) prm.range_off[r] = range_off_host[r];
  for (int r = 0; r < kRanges; ++r) {
    prm.num_pos[r] = num_pos_host[r];
    cb += (range_off_host[r + 1] - range_off_host[r] + kAccChunk - 1) / kAccChunk;
  }
  const long long hb = (num_props + kAccTPB - 1) / kAccTPB;
  const long long hist_blocks = hb < 1 ? 1 : (hb > 1024 ? 1024 : hb);
  SN_CHECK(cb + hist_blocks < INT_MAX, "proposal_recall_accumulate: %lld values are too many for one launch", cb);
  prm.num_props = num_props;
  prm.T = T;
  prm.prop_dtype = prop_dtype;
  prm.count_blocks = (int)cb;
  prm.num_images = num_images;
  cudaStream_t st = (cudaStream_t)stream;
  SN_CUDA(cudaMemsetAsync(counts, 0, sizeof(unsigned long long) * ((size_t)kRanges * T + 6), st));
  SN_CUDA(cudaMemsetAsync(done, 0, sizeof(unsigned int), st));
  recall_accumulate_kernel<<<(int)(cb + hist_blocks), kAccTPB, 0, st>>>(gt_overlaps, thresholds, prop_box, prm,
                                                                       counts, done, recalls, ar, hist);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
