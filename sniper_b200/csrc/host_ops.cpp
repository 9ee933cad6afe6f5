// Host-side (CPU) members of the path: chip sampling, hard / soft NMS, box overlaps.  north_star keeps
// lib/chips and lib/iterators on the host feeding pinned chip batches; these are fresh implementations
// behind the C-ABI with results identical to the reference's Cython/C++:
//   chips::cgenerate            lib/chips/cchips.cpp:54-177   (greedy cover; same std::random_shuffle/rand() stream)
//   cpu_nms / cpu_soft_nms      lib/nms/cpu_nms.pyx:112-163 / :17-110
//   bbox_overlaps / ignore_...  lib/bbox/bbox.pyx:17-57 / :59-95
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "common.cuh"

namespace {

struct Box4 {
  float x1, y1, x2, y2;
};

// 0 .. n-1 in the order std::random_shuffle of libstdc++ (bits/stl_algo.h) leaves them: for i in 1..n-1:
// swap(ids[i], ids[rand() % (i+1)]); n - 1 draws from rand()
void shuffled_ids(int* ids, int n) {
  std::iota(ids, ids + n, 0);
  for (int i = 1; i < n; ++i) {
    const int j = rand() % (i + 1);
    if (i != j) std::swap(ids[i], ids[j]);
  }
}

}  // namespace

extern "C" {

// boxes: host float[num_boxes,4] (already scaled and clipped, chip_generator.py:23-27).  Writes up to
// max_out chips (x1,y1,x2,y2) in pick order and returns their number (or -1).  The candidate order, the
// libstdc++ random_shuffle loop (j = rand() % (i+1)), the float32 containment test (iw*ih/area2 == 1) and
// the first-max greedy cover are the reference's; containment sets are bitsets instead of std::set<int>.
int sniper_chips_generate(const float* boxes, int num_boxes, int width, int height, int chipsize, int stride,
                          float* out_chips, int max_out) {
  SN_CHECK(stride > 0 && chipsize > 0, "chips_generate: bad chipsize/stride");
  if (num_boxes <= 0) return 0;
  std::vector<Box4> cand;
  auto push = [&](float a, float b, float c, float d) { cand.push_back(Box4{a, b, c, d}); };
  push((float)std::max(width - chipsize, 0), 0.f, (float)(width - 1), (float)std::min(chipsize, height - 1));
  push(0.f, (float)std::max(height - chipsize, 0), (float)std::min(chipsize, width - 1), (float)(height - 1));
  push((float)std::max(width - chipsize, 0), (float)std::max(height - chipsize, 0), (float)(width - 1), (float)(height - 1));
  for (int i = 0; i < width - chipsize; i += stride)
    for (int j = 0; j < height - chipsize; j += stride)
      push((float)i, (float)j, (float)(i + chipsize - 1), (float)(j + chipsize - 1));
  for (int i = 0; i < height - chipsize; i += stride)
    push((float)std::max(width - chipsize - 1, 0), (float)i, (float)(width - 1), (float)(i + chipsize - 1));
  for (int i = 0; i < width - chipsize; i += stride)
    push((float)i, (float)std::max(height - chipsize - 1, 0), (float)(i + chipsize - 1), (float)(height - 1));
  const int n = (int)cand.size();
  std::vector<int> ids(n);
  shuffled_ids(ids.data(), n);
  const int words = (num_boxes + 63) / 64;
  std::vector<uint64_t> match((size_t)n * words, 0);
  std::vector<int> count(n, 0);
  for (int i = 0; i < n; ++i) {
    const Box4 c = cand[ids[i]];
    for (int j = 0; j < num_boxes; ++j) {
      const float xx1 = boxes[4 * j], yy1 = boxes[4 * j + 1], xx2 = boxes[4 * j + 2], yy2 = boxes[4 * j + 3];
      const float area2 = (xx2 - xx1 + 1) * (yy2 - yy1 + 1);
      const float iw = std::min(c.x2, xx2) - std::max(c.x1, xx1) + 1;
      if (iw > 0) {
        const float ih = std::min(c.y2, yy2) - std::max(c.y1, yy1) + 1;
        if (ih > 0) {
          const float ov = iw * ih / area2;
          if (ov == 1) {
            match[(size_t)i * words + (j >> 6)] |= (uint64_t)1 << (j & 63);
            count[i]++;
          }
        }
      }
    }
  }
  int nout = 0;
  while (true) {
    int best = 0, mid = 0;
    for (int i = 0; i < n; ++i)
      if (count[i] > best) {
        best = count[i];
        mid = i;
      }
    if (best == 0) break;
    if (nout < max_out) {
      const Box4 c = cand[ids[mid]];
      out_chips[4 * nout] = c.x1; out_chips[4 * nout + 1] = c.y1; out_chips[4 * nout + 2] = c.x2; out_chips[4 * nout + 3] = c.y2;
    }
    ++nout;
    std::vector<uint64_t> taken(match.begin() + (size_t)mid * words, match.begin() + (size_t)(mid + 1) * words);
    for (int i = 0; i < n; ++i) {
      if (count[i] == 0) continue;
      int c = 0;
      uint64_t* m = &match[(size_t)i * words];
      for (int w = 0; w < words; ++w) {
        m[w] &= ~taken[w];
        c += __builtin_popcountll(m[w]);
      }
      count[i] = c;
    }
  }
  return nout;
}

// The candidate orders of a sequence of sniper_chips_generate calls, drawn from rand() as those calls draw them: call c
// has n_cand[c] candidates (0: a call without boxes, which draws nothing) and its order goes to
// perm_out[sum(n_cand[:c]) ...].  rand() ends where it would after the calls.  Refuses before drawing anything.
int sniper_chips_shuffle(const int* n_cand, int n_calls, int* perm_out) {
  SN_CHECK(n_calls >= 0, "chips_shuffle: n_calls (%d) must not be negative", n_calls);
  SN_CHECK(n_calls == 0 || n_cand, "chips_shuffle: n_cand must not be null");
  long total = 0;
  for (int c = 0; c < n_calls; ++c) {
    SN_CHECK(n_cand[c] >= 0, "chips_shuffle: call %d has %d candidates", c, n_cand[c]);
    total += n_cand[c];
  }
  SN_CHECK(total == 0 || perm_out, "chips_shuffle: perm_out must not be null");
  long off = 0;
  for (int c = 0; c < n_calls; ++c) {
    shuffled_ids(perm_out + off, n_cand[c]);
    off += n_cand[c];
  }
  return 0;
}

// dets: host float[n,5]; order: host int64[n] = scores.argsort()[::-1] (or NULL: stable descending order is
// computed here, ties -> higher index first, i.e. argsort(kind='stable')[::-1]).  keep: int32[n].  Returns #kept.
int sniper_cpu_nms(const float* dets, const int64_t* order_in, int n, double thresh, int32_t* keep) {
  if (n <= 0) return 0;
  std::vector<int64_t> order(n);
  if (order_in) {
    memcpy(order.data(), order_in, sizeof(int64_t) * n);
  } else {
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return dets[5 * a + 4] < dets[5 * b + 4]; });
    std::reverse(order.begin(), order.end());
  }
  std::vector<float> areas(n);
  for (int i = 0; i < n; ++i) areas[i] = (dets[5 * i + 2] - dets[5 * i] + 1) * (dets[5 * i + 3] - dets[5 * i + 1] + 1);
  std::vector<char> sup(n, 0);
  int nk = 0;
  for (int a = 0; a < n; ++a) {
    const int i = (int)order[a];
    if (sup[i]) continue;
    keep[nk++] = i;
    const float ix1 = dets[5 * i], iy1 = dets[5 * i + 1], ix2 = dets[5 * i + 2], iy2 = dets[5 * i + 3], ia = areas[i];
    for (int b = a + 1; b < n; ++b) {
      const int j = (int)order[b];
      if (sup[j]) continue;
      const float xx1 = std::max(ix1, dets[5 * j]), yy1 = std::max(iy1, dets[5 * j + 1]);
      const float xx2 = std::min(ix2, dets[5 * j + 2]), yy2 = std::min(iy2, dets[5 * j + 3]);
      const float w = (float)std::max(0.0, (double)(xx2 - xx1 + 1));
      const float h = (float)std::max(0.0, (double)(yy2 - yy1 + 1));
      const float inter = w * h;
      const float ovr = inter / (ia + areas[j] - inter);
      if ((double)ovr >= thresh) sup[j] = 1;
    }
  }
  return nk;
}

// boxes: host float[n,5], modified in place exactly as the reference does; returns the surviving count.
int sniper_cpu_soft_nms(float* b, int N, float sigma, float Nt, float threshold, unsigned method) {
  for (int i = 0; i < N; ++i) {
    float maxscore = b[5 * i + 4];
    int maxpos = i;
    float t[5];
    memcpy(t, b + 5 * i, sizeof(t));
    for (int pos = i + 1; pos < N; ++pos)
      if (maxscore < b[5 * pos + 4]) {
        maxscore = b[5 * pos + 4];
        maxpos = pos;
      }
    memcpy(b + 5 * i, b + 5 * maxpos, sizeof(t));
    memcpy(b + 5 * maxpos, t, sizeof(t));
    memcpy(t, b + 5 * i, sizeof(t));
    int pos = i + 1;
    while (pos < N) {
      const float x1 = b[5 * pos], y1 = b[5 * pos + 1], x2 = b[5 * pos + 2], y2 = b[5 * pos + 3];
      // the reference's Cython turns the int literal of `x2 - x1 + 1` into the double 1.0: sums / products in double,
      // narrowed to float on assignment (lib/nms/cpu_nms.pyx:73-80 as cythonized)
      const float area = (float)(((double)(x2 - x1) + 1.0) * ((double)(y2 - y1) + 1.0));
      const float iw = (float)((double)(std::min(t[2], x2) - std::max(t[0], x1)) + 1.0);
      if (iw > 0) {
        const float ih = (float)((double)(std::min(t[3], y2) - std::max(t[1], y1)) + 1.0);
        if (ih > 0) {
          const float inter = iw * ih;
          const float ua = (float)(((((double)(t[2] - t[0]) + 1.0) * ((double)(t[3] - t[1]) + 1.0)) + (double)area) -
                                   (double)inter);
          const float ov = inter / ua;
          float weight;
          if (method == 1) weight = ov > Nt ? (float)(1.0 - (double)ov) : 1;
          else if (method == 2) weight = (float)exp((double)(-(ov * ov) / sigma));
          else weight = ov > Nt ? 0 : 1;
          b[5 * pos + 4] = weight * b[5 * pos + 4];
          if (b[5 * pos + 4] < threshold) {
            memcpy(b + 5 * pos, b + 5 * (N - 1), sizeof(t));
            --N;
            --pos;
          }
        }
      }
      ++pos;
    }
  }
  return N;
}

// boxes [N,4], query [K,4] host float64 -> overlaps [N,K].  ignore=1: intersection / query area (ignore_overlaps).
int sniper_bbox_overlaps(const double* boxes, int N, const double* query, int K, double* overlaps, int ignore) {
  for (long i = 0; i < (long)N * K; ++i) overlaps[i] = 0;
  // small problems stay on the calling thread: waking a 128-thread team costs more than the 100 x 300 IoUs of one chip
  // (the iterator calls this ~6 times per chip; on a 128-core host the fork/join made a batch 3x slower)
#pragma omp parallel for schedule(static) if ((long)N * K > 200000) num_threads(8)
  for (int k = 0; k < K; ++k) {
    const double qa = (query[4 * k + 2] - query[4 * k] + 1) * (query[4 * k + 3] - query[4 * k + 1] + 1);
    for (int n = 0; n < N; ++n) {
      const double iw = std::min(boxes[4 * n + 2], query[4 * k + 2]) - std::max(boxes[4 * n], query[4 * k]) + 1;
      if (iw <= 0) continue;
      const double ih = std::min(boxes[4 * n + 3], query[4 * k + 3]) - std::max(boxes[4 * n + 1], query[4 * k + 1]) + 1;
      if (ih <= 0) continue;
      const double ua = ignore ? qa
                               : (boxes[4 * n + 2] - boxes[4 * n] + 1) * (boxes[4 * n + 3] - boxes[4 * n + 1] + 1) + qa - iw * ih;
      overlaps[(size_t)n * K + k] = iw * ih / ua;
    }
  }
  return 0;
}

}  // extern "C"
