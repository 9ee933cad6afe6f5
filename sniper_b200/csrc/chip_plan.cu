// The SNIPER training epoch plan on the device: chip_worker.chip_extractor and chip_worker.box_assigner
// (sniper_b200/chip_worker.py, the reference's data_workers.py:394-594) for every roidb entry of an epoch in a few
// launches, byte-equal to the host path.
//
// A "call" is one (entry, scale) problem of the host: one chips_generate greedy cover and one _assign.  Every launch
// takes a table with one int64 row of kCols per call (see the column names below) and runs one block per call.
//   sniper_chip_plan_count   the GT boxes chip_extractor selects per call (the host draws a call's candidate shuffle only
//                            when it has boxes, as sniper_chips_generate does);
//   sniper_chip_plan_cover   the greedy cover of sniper_chips_generate over the call's boxes, with the candidate order
//                            drawn on the host (sniper_chips_shuffle): mode 0 the positive chips (chip_extractor's
//                            boxes), mode 1 the negative chips (the boxes no positive chip kept);
//   sniper_chip_plan_assign  _assign: each selected box's owner chip (first arg-max of the float64 ignore_overlaps) and
//                            whether that chip keeps it; mode 0 over the positive chips (box_assigner's boxes,
//                            `<= hi`), mode 1 over the negative chips (the uncovered boxes, `< hi`).
// The per-box integer sizes (w, h of _int_sizes, computed on the host in the roidb's own dtype) and the boxes (float32:
// uint16 and float32 roidbs are exact in it) are read from the caller's arrays; box b of the call's entry e is row
// box_off[e] + b.  Owners are written per (box, scale) as int16: >= 0 the owning chip, -1 selected but not kept, -2 not
// selected.  A cover's scratch (boxes, candidate counts, containment bitsets) lives in shared memory up to kSmemCap and
// otherwise in its slice of a caller-owned workspace (sniper_chip_plan_layout).  Built with -fmad=false.
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "block_reduce.cuh"
#include "common.cuh"
#include "np_pairwise.cuh"

namespace {

constexpr int kCols = 16;
// table columns
constexpr int cEntry = 0, cScale = 1, cKind = 2, cW = 3, cH = 4, cNCand = 5, cNBox = 6, cPermOff = 7, cOutOff = 8,
              cOutCap = 9, cWsOff = 10, cF = 11, cThr = 12, cLo = 13, cHi = 14, cF32 = 15;
constexpr int kFirst = 0, kLast = 2;                     // cKind (1: a middle scale); with one scale it is kLast
constexpr int kTPB = 256, kWarps = kTPB / 32;
constexpr int kAssignTPB = 128;
constexpr long kSmemCap = 64 * 1024;
constexpr int kMaxExtent = 1 << 24;                      // W, H, chip size: every coordinate is exact in float32
constexpr int kHostCap = 4096;                           // host.chips_generate keeps the first 4096 chips of a call

__host__ __device__ inline long cover_bytes(long nb, long n_cand) {
  const long words = (nb + 63) / 64;
  return 16 * nb + (4 * n_cand + 15) / 16 * 16 + 8 * n_cand * words + 8 * words;
}

__host__ __device__ inline void grid_dims(long W, long H, long cs, long s, long* nx, long* ny) {
  *nx = W - cs > 0 ? (W - cs + s - 1) / s : 0;
  *ny = H - cs > 0 ? (H - cs + s - 1) / s : 0;
}

__host__ __device__ inline long n_candidates(long W, long H, long cs, long s) {
  long nx, ny;
  grid_dims(W, H, cs, s, &nx, &ny);
  return 3 + nx * ny + ny + nx;
}

__device__ __forceinline__ double bits(long long v) { return __longlong_as_double(v); }

// std::min / std::max as the host code calls them: min(a, b) = b < a ? b : a, max(a, b) = a < b ? b : a
template <typename T>
__device__ __forceinline__ T std_min(T a, T b) { return b < a ? b : a; }
template <typename T>
__device__ __forceinline__ T std_max(T a, T b) { return a < b ? b : a; }

// the k-th candidate of sniper_chips_generate's push order
__device__ float4 candidate(int k, int W, int H, int cs, int s, int nx, int ny) {
  if (k == 0) return make_float4((float)max(W - cs, 0), 0.f, (float)(W - 1), (float)min(cs, H - 1));
  if (k == 1) return make_float4(0.f, (float)max(H - cs, 0), (float)min(cs, W - 1), (float)(H - 1));
  if (k == 2) return make_float4((float)max(W - cs, 0), (float)max(H - cs, 0), (float)(W - 1), (float)(H - 1));
  k -= 3;
  if (k < nx * ny) {
    const int i = k / ny * s, j = k % ny * s;
    return make_float4((float)i, (float)j, (float)(i + cs - 1), (float)(j + cs - 1));
  }
  k -= nx * ny;
  if (k < ny) return make_float4((float)max(W - cs - 1, 0), (float)(k * s), (float)(W - 1), (float)(k * s + cs - 1));
  k -= ny;
  return make_float4((float)(k * s), (float)max(H - cs - 1, 0), (float)(k * s + cs - 1), (float)(H - 1));
}

struct Rule {
  int kind;
  double thr, lo, hi;
};

__device__ __forceinline__ Rule rule_of(const long long* t) {
  return Rule{(int)t[cKind], bits(t[cThr]), bits(t[cLo]), bits(t[cHi])};
}

// size = np.sqrt(w * h) with numpy's wrapping int32 product, longest = np.maximum(w, h)
__device__ __forceinline__ double int_size(int w, int h) { return sqrt((double)(int)((unsigned)w * (unsigned)h)); }

// chip_extractor's selection of GT boxes
__device__ __forceinline__ bool pos_selected(int2 wh, const Rule& r) {
  const double size = int_size(wh.x, wh.y);
  if (r.kind == kLast) return size >= r.lo;
  const bool fits = (double)max(wh.x, wh.y) < r.thr;
  if (r.kind == kFirst) return size < r.hi && fits && wh.x >= 2 && wh.y >= 2;
  return size >= r.lo && size < r.hi && fits;
}

// box_assigner's selection of all boxes
__device__ __forceinline__ bool asg_selected(int2 wh, const Rule& r) {
  const double size = int_size(wh.x, wh.y);
  if (r.kind == kLast) return size >= r.lo;
  return size < r.hi && (double)max(wh.x, wh.y) < r.thr && wh.x >= 2 && wh.y >= 2;
}

__global__ void __launch_bounds__(kAssignTPB) chip_plan_count_kernel(const long long* __restrict__ table,
                                                                     const long long* __restrict__ box_off,
                                                                     const int2* __restrict__ wh,
                                                                     const unsigned char* __restrict__ gt,
                                                                     int* __restrict__ counts) {
  __shared__ int s_red[kAssignTPB / 32];
  const long long* t = table + (long)blockIdx.x * kCols;
  const Rule r = rule_of(t);
  const long b0 = box_off[t[cEntry]], b1 = box_off[t[cEntry] + 1];
  int n = 0;
  for (long b = b0 + threadIdx.x; b < b1; b += kAssignTPB) n += gt[b] && pos_selected(wh[b], r);
  n = block_sum<int, kAssignTPB / 32>(n, s_red);
  if (threadIdx.x == 0) counts[blockIdx.x] = n;
}

__global__ void __launch_bounds__(kTPB) chip_plan_cover_kernel(
    const long long* __restrict__ table, int mode, int S, const long long* __restrict__ box_off,
    const float4* __restrict__ boxes, const int2* __restrict__ wh, const unsigned char* __restrict__ gt,
    const short* __restrict__ pos_owner, const int* __restrict__ perm, int cs, int stride,
    unsigned char* __restrict__ ws, float4* __restrict__ chips32, double4* __restrict__ chips64,
    int* __restrict__ nchips) {
  extern __shared__ __align__(16) unsigned char sm[];
  __shared__ int s_n;
  __shared__ int s_v[kWarps], s_i[kWarps];
  const int call = blockIdx.x;
  const long long* t = table + (long)call * kCols;
  const int nb = (int)t[cNBox];
  if (nb == 0) {
    if (threadIdx.x == 0) nchips[call] = 0;
    return;
  }
  const int W = (int)t[cW], H = (int)t[cH], n = (int)t[cNCand], s = (int)t[cScale];
  long nx, ny;
  grid_dims(W, H, cs, stride, &nx, &ny);
  if (n != 3 + nx * ny + ny + nx) {
    if (threadIdx.x == 0) nchips[call] = -2;
    return;
  }
  const int words = (nb + 63) / 64;
  unsigned char* base = t[cWsOff] < 0 ? sm : ws + t[cWsOff];
  float4* bx = reinterpret_cast<float4*>(base);
  int* cnt = reinterpret_cast<int*>(base + 16L * nb);
  uint64_t* match = reinterpret_cast<uint64_t*>(base + 16L * nb + (4L * n + 15) / 16 * 16);
  uint64_t* taken = match + (long)n * words;
  const Rule r = rule_of(t);
  const double f = bits(t[cF]);
  const float ff = __double2float_rn(f);
  const bool f32 = mode == 0 && t[cF32] != 0;
  const double wm2 = (double)(W - 2), hm2 = (double)(H - 2);
  if (threadIdx.x == 0) s_n = 0;
  for (int i = threadIdx.x; i < n; i += kTPB) cnt[i] = 0;
  __syncthreads();
  // the call's boxes, scaled by f (positives of a float32 roidb in float32, as numpy multiplies them, otherwise in
  // float64), clipped to [0, W - 2] x [0, H - 2] in float64 and narrowed to float32; their order does not matter
  const long b0 = box_off[t[cEntry]], b1 = box_off[t[cEntry] + 1];
  for (long b = b0 + threadIdx.x; b < b1; b += kTPB) {
    const bool sel = mode == 0 ? gt[b] && pos_selected(wh[b], r) : pos_owner[b * S + s] == -1;
    if (!sel) continue;
    const int k = atomicAdd(&s_n, 1);
    if (k >= nb) continue;
    const float4 v = boxes[b];
    double x1, y1, x2, y2;
    if (f32) {
      x1 = __fmul_rn(v.x, ff); y1 = __fmul_rn(v.y, ff); x2 = __fmul_rn(v.z, ff); y2 = __fmul_rn(v.w, ff);
    } else {
      x1 = __dmul_rn(v.x, f); y1 = __dmul_rn(v.y, f); x2 = __dmul_rn(v.z, f); y2 = __dmul_rn(v.w, f);
    }
    bx[k] = make_float4(__double2float_rn(np_max(np_min(x1, wm2), 0.0)), __double2float_rn(np_max(np_min(y1, hm2), 0.0)),
                        __double2float_rn(np_max(np_min(x2, wm2), 0.0)), __double2float_rn(np_max(np_min(y2, hm2), 0.0)));
  }
  __syncthreads();
  if (s_n != nb) {                                 // the table's box count is not this call's
    if (threadIdx.x == 0) nchips[call] = -2;
    return;
  }
  // containment bitsets: candidate at shuffled position i, 64 boxes per word; the float32 test iw * ih / area2 == 1
  const int* pm = perm + t[cPermOff];
  for (long p = threadIdx.x; p < (long)n * words; p += kTPB) {
    const int i = (int)(p / words), w = (int)(p - (long)i * words);
    const float4 c = candidate(pm[i], W, H, cs, stride, (int)nx, (int)ny);
    uint64_t m = 0;
    const int j1 = min(nb, 64 * w + 64);
    for (int j = 64 * w; j < j1; ++j) {
      const float4 q = bx[j];
      const float area2 = __fmul_rn(__fadd_rn(__fsub_rn(q.z, q.x), 1.f), __fadd_rn(__fsub_rn(q.w, q.y), 1.f));
      const float iw = __fadd_rn(__fsub_rn(std_min(c.z, q.z), std_max(c.x, q.x)), 1.f);
      if (iw > 0) {
        const float ih = __fadd_rn(__fsub_rn(std_min(c.w, q.w), std_max(c.y, q.y)), 1.f);
        if (ih > 0 && __fdiv_rn(__fmul_rn(iw, ih), area2) == 1.f) m |= (uint64_t)1 << (j - 64 * w);
      }
    }
    match[p] = m;
    if (m) atomicAdd(cnt + i, __popcll(m));
  }
  __syncthreads();
  // the greedy cover: the first maximum count in shuffled order, then its boxes leave every other candidate
  const long long out_off = t[cOutOff], out_cap = t[cOutCap];
  int nout = 0;
  while (true) {
    int bv = -1, bi = INT_MAX;
    for (int i = threadIdx.x; i < n; i += kTPB)
      if (argmax_beats(cnt[i], i, bv, bi)) { bv = cnt[i]; bi = i; }
    warp_argmax(bv, bi);
    if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = bv; s_i[threadIdx.x >> 5] = bi; }
    __syncthreads();
    bv = s_v[0]; bi = s_i[0];
    for (int w = 1; w < kWarps; ++w)
      if (argmax_beats(s_v[w], s_i[w], bv, bi)) { bv = s_v[w]; bi = s_i[w]; }
    if (bv <= 0) break;
    if (threadIdx.x == 0 && nout < out_cap) {
      const float4 c = candidate(pm[bi], W, H, cs, stride, (int)nx, (int)ny);
      chips32[out_off + nout] = c;
      chips64[out_off + nout] = make_double4(__ddiv_rn(c.x, f), __ddiv_rn(c.y, f), __ddiv_rn(c.z, f), __ddiv_rn(c.w, f));
    }
    ++nout;
    for (int w = threadIdx.x; w < words; w += kTPB) taken[w] = match[(long)bi * words + w];
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kTPB) {
      if (cnt[i] == 0) continue;
      uint64_t* m = match + (long)i * words;
      int c = 0;
      for (int w = 0; w < words; ++w) {
        m[w] &= ~taken[w];
        c += __popcll(m[w]);
      }
      cnt[i] = c;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) nchips[call] = nout;
}

__global__ void __launch_bounds__(kAssignTPB) chip_plan_assign_kernel(
    const long long* __restrict__ table, int mode, int S, const long long* __restrict__ box_off,
    const float4* __restrict__ boxes, const int2* __restrict__ wh, const short* __restrict__ pos_owner,
    const double4* __restrict__ chips64, const int* __restrict__ nchips, short* __restrict__ owner_out,
    int* __restrict__ left_count) {
  __shared__ int s_red[kAssignTPB / 32];
  const long long* t = table + (long)blockIdx.x * kCols;
  const Rule r = rule_of(t);
  const int s = (int)t[cScale];
  const int nch = min(max(nchips[blockIdx.x], 0), kHostCap);
  const double4* ch = chips64 + t[cOutOff];
  const long b0 = box_off[t[cEntry]], b1 = box_off[t[cEntry] + 1];
  int left = 0;
  for (long b = b0 + threadIdx.x; b < b1; b += kAssignTPB) {
    const bool sel = mode == 0 ? asg_selected(wh[b], r) : pos_owner[b * S + s] == -1;
    if (!sel) {
      owner_out[b * S + s] = -2;
      continue;
    }
    short own = -1;
    if (nch > 0) {
      const float4 v = boxes[b];
      const double q0 = v.x, q1 = v.y, q2 = v.z, q3 = v.w;
      const double qa = __dmul_rn(__dadd_rn(__dsub_rn(q2, q0), 1.0), __dadd_rn(__dsub_rn(q3, q1), 1.0));
      // ignore_overlaps(chips, boxes).argmax(axis=0): the first maximum, a NaN wins as in numpy
      double best = 0.0;
      int k_best = 0;
      for (int k = 0; k < nch; ++k) {
        const double4 c = ch[k];
        double ov = 0.0;
        const double iw = __dadd_rn(__dsub_rn(std_min(c.z, q2), std_max(c.x, q0)), 1.0);
        if (iw > 0) {
          const double ih = __dadd_rn(__dsub_rn(std_min(c.w, q3), std_max(c.y, q1)), 1.0);
          if (ih > 0) ov = __ddiv_rn(__dmul_rn(iw, ih), qa);
        }
        if (k == 0 || (best == best && (ov != ov || ov > best))) {
          best = ov;
          k_best = k;
        }
      }
      const double4 c = ch[k_best];
      const double x1 = np_max(c.x, q0), x2 = np_min(c.z, q2), y1 = np_max(c.y, q1), y2 = np_min(c.w, q3);
      const double dx = __dsub_rn(x2, x1), dy = __dsub_rn(y2, y1);
      const double side = sqrt(fabs(__dmul_rn(dx, dy)));
      const bool in_range = r.kind == kLast ? side >= r.lo : (mode == 1 ? side < r.hi : side <= r.hi);
      if (dx >= 1 && dy >= 1 && in_range) own = (short)k_best;
    }
    owner_out[b * S + s] = own;
    left += own == -1;
  }
  left = block_sum<int, kAssignTPB / 32>(left, s_red);
  if (threadIdx.x == 0 && left_count) left_count[blockIdx.x] = left;
}

// the host-side checks every entry point shares; *smem gets the dynamic shared memory of a cover launch
int check_table(const long long* th, int n_calls, int S, int cs, int stride, bool cover, long* smem, long long* ws_total,
                const char* who) {
  SN_CHECK(n_calls >= 0, "%s: n_calls (%d) must not be negative", who, n_calls);
  SN_CHECK(n_calls == 0 || th, "%s: table (host) must not be null", who);
  SN_CHECK(S >= 1, "%s: the scale count S (%d) must be at least 1", who, S);
  SN_CHECK(cs > 0 && cs < kMaxExtent && stride > 0, "%s: bad chip size (%d) / stride (%d)", who, cs, stride);
  long sm = 0;
  long long off = 0;
  for (int c = 0; c < n_calls; ++c) {
    const long long* t = th + (long)c * kCols;
    SN_CHECK(t[cEntry] >= 0 && t[cScale] >= 0 && t[cScale] < S && t[cKind] >= kFirst && t[cKind] <= kLast,
             "%s: call %d: bad entry / scale / kind", who, c);
    SN_CHECK(t[cW] >= 0 && t[cH] >= 0 && t[cW] < kMaxExtent && t[cH] < kMaxExtent,
             "%s: call %d: the scaled image %lld x %lld must lie in [0, %d)", who, c, t[cW], t[cH], kMaxExtent);
    if (!cover) continue;
    const long n = n_candidates(t[cW], t[cH], cs, stride);
    SN_CHECK(t[cNCand] == n, "%s: call %d: n_cand %lld, the geometry gives %ld", who, c, t[cNCand], n);
    SN_CHECK(t[cNBox] >= 0 && t[cNBox] < (1 << 30), "%s: call %d: bad box count %lld", who, c, t[cNBox]);
    SN_CHECK(t[cNBox] == 0 || (t[cPermOff] >= 0 && t[cOutOff] >= 0 && t[cOutCap] >= std::min((long long)n, t[cNBox])),
             "%s: call %d: perm / output offsets, or fewer output slots than min(n_cand, n_box)", who, c);
    if (t[cNBox] == 0) continue;
    const long need = cover_bytes(t[cNBox], n);
    if (need <= kSmemCap) {
      SN_CHECK(t[cWsOff] == -1, "%s: call %d: the table's workspace offsets are not sniper_chip_plan_layout's", who, c);
      sm = std::max(sm, need);
    } else {
      SN_CHECK(t[cWsOff] == off, "%s: call %d: the table's workspace offsets are not sniper_chip_plan_layout's", who, c);
      off += (need + 15) / 16 * 16;
    }
  }
  if (smem) *smem = sm;
  if (ws_total) *ws_total = off;
  return 0;
}

}  // namespace

extern "C" {

int sniper_chip_plan_layout(long long* table_host, int n_calls, int chip_size, int stride, long long* ws_bytes) {
  SN_CHECK(n_calls >= 0 && (n_calls == 0 || table_host) && ws_bytes, "chip_plan_layout: null table / ws_bytes");
  SN_CHECK(chip_size > 0 && chip_size < kMaxExtent && stride > 0, "chip_plan_layout: bad chip size / stride");
  long long off = 0;
  for (int c = 0; c < n_calls; ++c) {
    long long* t = table_host + (long)c * kCols;
    SN_CHECK(t[cNBox] >= 0 && t[cW] >= 0 && t[cH] >= 0 && t[cW] < kMaxExtent && t[cH] < kMaxExtent,
             "chip_plan_layout: call %d: bad geometry or box count", c);
    const long need = t[cNBox] == 0 ? 0 : cover_bytes(t[cNBox], n_candidates(t[cW], t[cH], chip_size, stride));
    if (need > kSmemCap) {
      t[cWsOff] = off;
      off += (need + 15) / 16 * 16;
    } else {
      t[cWsOff] = -1;
    }
  }
  *ws_bytes = off;
  return 0;
}

int sniper_chip_plan_count(const long long* table, const long long* table_host, int n_calls, int S, int chip_size,
                           int stride, const long long* box_off, const int* wh, const unsigned char* gt, int* counts,
                           void* stream) {
  if (check_table(table_host, n_calls, S, chip_size, stride, false, nullptr, nullptr, "chip_plan_count")) return -1;
  if (n_calls == 0) return 0;
  SN_CHECK(table && box_off && wh && gt && counts, "chip_plan_count: table / box_off / wh / gt / counts must not be null");
  chip_plan_count_kernel<<<n_calls, kAssignTPB, 0, (cudaStream_t)stream>>>(table, box_off,
                                                                            reinterpret_cast<const int2*>(wh), gt, counts);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_chip_plan_cover(const long long* table, const long long* table_host, int n_calls, int mode, int S,
                           int chip_size, int stride, const long long* box_off, const float* boxes, const int* wh,
                           const unsigned char* gt, const short* pos_owner, const int* perm, void* workspace,
                           long ws_bytes, float* chips32, double* chips64, int* nchips, void* stream) {
  long smem = 0;
  long long need = 0;
  if (check_table(table_host, n_calls, S, chip_size, stride, true, &smem, &need, "chip_plan_cover")) return -1;
  if (n_calls == 0) return 0;
  SN_CHECK(mode == 0 || mode == 1, "chip_plan_cover: mode (%d) must be 0 (positive) or 1 (negative)", mode);
  SN_CHECK(table && box_off && boxes && wh && perm && chips32 && chips64 && nchips,
           "chip_plan_cover: table / box_off / boxes / wh / perm / chips32 / chips64 / nchips must not be null");
  SN_CHECK(mode == 1 || gt, "chip_plan_cover: the positive cover needs gt");
  SN_CHECK(mode == 0 || pos_owner, "chip_plan_cover: the negative cover needs pos_owner");
  SN_CHECK(need == 0 || (workspace && ws_bytes >= need), "chip_plan_cover: these calls need a workspace of %lld bytes",
           need);
  SN_CHECK(((uintptr_t)boxes & 15) == 0 && ((uintptr_t)wh & 7) == 0 && ((uintptr_t)chips32 & 15) == 0 &&
               ((uintptr_t)chips64 & 31) == 0 && ((uintptr_t)workspace & 15) == 0,
           "chip_plan_cover: boxes / chips32 / workspace must be 16-byte, wh 8-byte and chips64 32-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  SN_CUDA(cudaFuncSetAttribute(chip_plan_cover_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCap));
  chip_plan_cover_kernel<<<n_calls, kTPB, smem, st>>>(
      table, mode, S, box_off, reinterpret_cast<const float4*>(boxes), reinterpret_cast<const int2*>(wh), gt, pos_owner,
      perm, chip_size, stride, static_cast<unsigned char*>(workspace), reinterpret_cast<float4*>(chips32),
      reinterpret_cast<double4*>(chips64), nchips);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_chip_plan_assign(const long long* table, const long long* table_host, int n_calls, int mode, int S,
                            const long long* box_off, const float* boxes, const int* wh, const short* pos_owner,
                            const double* chips64, const int* nchips, short* owner_out, int* left_count,
                            void* stream) {
  if (check_table(table_host, n_calls, S, 1, 1, false, nullptr, nullptr, "chip_plan_assign")) return -1;
  if (n_calls == 0) return 0;
  SN_CHECK(mode == 0 || mode == 1, "chip_plan_assign: mode (%d) must be 0 (positive) or 1 (negative)", mode);
  SN_CHECK(table && box_off && boxes && wh && chips64 && nchips && owner_out,
           "chip_plan_assign: table / box_off / boxes / wh / chips64 / nchips / owner_out must not be null");
  SN_CHECK(mode == 0 || pos_owner, "chip_plan_assign: the negative assignment needs pos_owner");
  SN_CHECK(((uintptr_t)boxes & 15) == 0 && ((uintptr_t)wh & 7) == 0 && ((uintptr_t)chips64 & 31) == 0,
           "chip_plan_assign: boxes must be 16-byte, wh 8-byte and chips64 32-byte aligned");
  chip_plan_assign_kernel<<<n_calls, kAssignTPB, 0, (cudaStream_t)stream>>>(
      table, mode, S, box_off, reinterpret_cast<const float4*>(boxes), reinterpret_cast<const int2*>(wh), pos_owner,
      reinterpret_cast<const double4*>(chips64), nchips, owner_out, left_count);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
