// AutoFocus FocusChips on the device: gmask of the reference's chips_inference (lib/chips/chips_inference.py:12-89) for
// every FocusPixel map of a test scale in ONE launch, byte-equal to the host restatement (sniper_b200/chips_inference.py
// `gmask`, whose OpenCV primitives it restates).
//
// One block per map.  The map is read in place (any element strides: the `focus_map` output is the strided view
// softmax(z)[..., 1]), thresholded in float32, dilated, and then the merge loop runs on a byte mask:
//   * contours: one union-find over all cells, foreground cells joined to their 8 neighbours, background cells to their
//     4 neighbours.  A join links the higher root to the lower index, so every component's root is its raster-first
//     cell.  A foreground root starts an outer border (rect = the component's box); a background root whose box touches
//     no frame row or column starts a hole border (rect = the hole's box grown by one cell, clamped to the map; its
//     start pixel is one left of the root, which keeps the start pixels in the roots' order).  The host lists contours
//     by start pixel, descending, which is descending root index.
//   * each pass paints every placed rect (`_place`, Python floor division on non-negative ints, clamped against
//     iw / ih) into the mask, clipped to the map's own extents, and relabels; the loop stops when the contour count
//     equals the previous pass's.  The mask only grows, so more than H * W + 2 passes is an error, not a hang.
//   * the last pass's rects, placed, scaled by 16, clamped to im_width / im_height, divided by cscale and shifted by
//     the crop origin in double (no FMA: this file is built with -fmad=false), are written in contour order.
// A map's scratch (mask bytes, then label, x-min, x-max and y-max per cell) lives in shared memory when it fits under
// kSmemCap and otherwise in its slice of a caller-owned workspace (sniper_focus_chips_workspace_bytes).
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include "block_reduce.cuh"
#include "common.cuh"

namespace {

constexpr int kTPB = 256;
constexpr int kWarps = kTPB / 32;
constexpr long kSmemCap = 100 * 1024;           // two blocks per SM at the largest shared-memory map
constexpr int kCols = 12;                       // table columns, see sniper_focus_chips
constexpr long kMaxCells = 1L << 26;
constexpr int kMaxExtent = 1 << 26;             // ms, iw, ih: (x + w) * 16 stays an int

// per-map scratch bytes: the mask (16-byte padded), then four int32 arrays
__host__ __device__ inline long map_bytes(long cells) { return (cells + 15) / 16 * 16 + 16 * cells; }

__device__ __forceinline__ int find_root(volatile int* lab, int a) {
  while (lab[a] != a) a = lab[a];
  return a;
}

// Playne & Hawick's lock-free union: the higher of the two roots is linked to the lower with atomicMin, retried when
// another thread linked it first
__device__ void unite(int* lab, int a, int b) {
  volatile int* vl = lab;
  bool done;
  do {
    a = find_root(vl, a);
    b = find_root(vl, b);
    if (b < a) {
      const int old = atomicMin(lab + a, b);
      done = old == a;
      a = old;
    } else if (a < b) {
      const int old = atomicMin(lab + b, a);
      done = old == b;
      b = old;
    } else {
      done = true;
    }
  } while (!done);
}

struct Scratch {
  unsigned char* mask;
  int *lab, *x0, *x1, *y1;
  int H, W;
};

// contour_rects(mask): labels the components, takes their boxes and tags every contour's root in lab (-1 outer border,
// -2 hole border); returns the contour count (block-uniform)
__device__ int label_pass(const Scratch& s, int* s_red) {
  const int H = s.H, W = s.W, HW = H * W;
  for (int c = threadIdx.x; c < HW; c += kTPB) {
    s.lab[c] = c;
    s.x0[c] = INT_MAX;
    s.x1[c] = -1;
    s.y1[c] = -1;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < HW; c += kTPB) {
    const int y = c / W, x = c - y * W;
    const bool fg = s.mask[c] != 0;
    if (x > 0 && (s.mask[c - 1] != 0) == fg) unite(s.lab, c, c - 1);
    if (y > 0) {
      if ((s.mask[c - W] != 0) == fg) unite(s.lab, c, c - W);
      if (fg && x > 0 && s.mask[c - W - 1]) unite(s.lab, c, c - W - 1);
      if (fg && x + 1 < W && s.mask[c - W + 1]) unite(s.lab, c, c - W + 1);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < HW; c += kTPB) s.lab[c] = find_root(s.lab, c);
  __syncthreads();
  for (int c = threadIdx.x; c < HW; c += kTPB) {
    const int r = s.lab[c], y = c / W, x = c - y * W;
    atomicMin(s.x0 + r, x);
    atomicMax(s.x1 + r, x);
    atomicMax(s.y1 + r, y);
  }
  __syncthreads();
  int cnt = 0;
  for (int c = threadIdx.x; c < HW; c += kTPB) {
    if (s.lab[c] != c) continue;
    const bool fg = s.mask[c] != 0;
    const bool frame = s.x0[c] == 0 || c < W || s.x1[c] == W - 1 || s.y1[c] == H - 1;
    if (fg || !frame) {
      s.lab[c] = fg ? -1 : -2;
      ++cnt;
    }
  }
  return block_sum<int, kWarps>(cnt, s_red);
}

struct Rect {
  int x, y, w, h;
};

// the boundingRect of the contour rooted at c
__device__ Rect contour_rect(const Scratch& s, int c) {
  const int y0 = c / s.W, x0 = s.x0[c], x1 = s.x1[c], y1 = s.y1[c];
  if (s.lab[c] == -1) return Rect{x0, y0, x1 - x0 + 1, y1 - y0 + 1};
  const int X0 = max(x0 - 1, 0), Y0 = max(y0 - 1, 0), X1 = min(x1 + 2, s.W), Y1 = min(y1 + 2, s.H);
  return Rect{X0, Y0, X1 - X0, Y1 - Y0};
}

// _place: every operand is a non-negative int, so C division is Python's floor division
__device__ Rect place(Rect r, int ms, int iw, int ih) {
  const int cx = (r.x + r.x + r.w) / 2, cy = (r.y + r.y + r.h) / 2;
  const int w = max(ms, r.w), h = max(ms, r.h);
  int x, y;
  if (cx + w / 2 >= iw) x = iw - w >= 0 ? iw - w : 0;
  else if (cx - w / 2 < 0) x = 0;
  else x = cx - w / 2;
  if (cy + h / 2 >= ih) y = ih - h >= 0 ? ih - h : 0;
  else if (cy - h / 2 < 0) y = 0;
  else y = cy - h / 2;
  return Rect{x, y, w, h};
}

// mask[y:y+h, x:x+w] = 255 for every placed rect: each warp takes its lanes' rects one at a time and paints them
// together (all writes store the same value, so overlapping rects need no order)
__device__ void paint(const Scratch& s, int ms, int iw, int ih) {
  const int HW = s.H * s.W, lane = threadIdx.x & 31;
  const int rounds = (HW + kTPB - 1) / kTPB;
  for (int k = 0; k < rounds; ++k) {
    const int c = k * kTPB + threadIdx.x;
    bool pend = false;
    int px = 0, py = 0, pw = 0, ph = 0;
    if (c < HW && s.lab[c] < 0) {
      const Rect p = place(contour_rect(s, c), ms, iw, ih);
      px = p.x;
      py = p.y;
      pw = min(p.x + p.w, s.W) - p.x;
      ph = min(p.y + p.h, s.H) - p.y;
      pend = pw > 0 && ph > 0;
    }
    unsigned bal;
    while ((bal = __ballot_sync(~0u, pend)) != 0) {
      const int src = __ffs(bal) - 1;
      const int rx = __shfl_sync(~0u, px, src), ry = __shfl_sync(~0u, py, src);
      const int rw = __shfl_sync(~0u, pw, src), rh = __shfl_sync(~0u, ph, src);
      for (int q = lane; q < rw * rh; q += 32) {
        const int yy = q / rw;
        s.mask[(ry + yy) * s.W + rx + (q - yy * rw)] = 255;
      }
      if (lane == src) pend = false;
    }
  }
}

__device__ __forceinline__ double as_double(long long v) { return __longlong_as_double(v); }

// The final scaling of gmask (:80-88) and the crop shift of add_chips (:158-162) for one chip
__device__ void write_chip(double* o, Rect p, int ms, double imw, double imh, double cscale, double ox, double oy) {
  double x1 = (double)(p.x * 16), y1 = (double)(p.y * 16);
  double x2 = (double)((p.x + p.w) * 16), y2 = (double)((p.y + p.h) * 16);
  const double m16 = (double)ms * 16.0;
  if (x2 > imw) {
    x2 = imw;
    const double t = __dsub_rn(x2, m16);
    const double mn = t < x1 ? t : x1;           // Python min(x1, x2 - ms * 16)
    x1 = 0.0 > mn ? 0.0 : mn;                    // max(., 0)
  }
  if (y2 > imh) {
    y2 = imh;
    const double t = __dsub_rn(y2, m16);
    const double mn = t < y1 ? t : y1;
    y1 = 0.0 > mn ? 0.0 : mn;
  }
  o[0] = __dadd_rn(__ddiv_rn(x1, cscale), ox);
  o[1] = __dadd_rn(__ddiv_rn(y1, cscale), oy);
  o[2] = __dadd_rn(__ddiv_rn(x2, cscale), ox);
  o[3] = __dadd_rn(__ddiv_rn(y2, cscale), oy);
}

__global__ void __launch_bounds__(kTPB) focus_chips_kernel(const long long* __restrict__ table,
                                                           const long long* __restrict__ ws_off,
                                                           unsigned char* __restrict__ ws, int d, float thresh, int ms,
                                                           int cap, long smem_avail, double* __restrict__ chips,
                                                           int* __restrict__ counts) {
  extern __shared__ __align__(16) unsigned char sm[];
  __shared__ int s_red[kWarps];
  const int m = blockIdx.x;
  const long long* t = table + (long)m * kCols;
  const int H = (int)t[3], W = (int)t[4], HW = H * W;
  if (HW == 0) {                                 // an empty map has no contour
    if (threadIdx.x == 0) counts[m] = 0;
    return;
  }
  const long need = map_bytes(HW), slice = (long)(ws_off[m + 1] - ws_off[m]);
  if ((slice == 0 && need > smem_avail) || (slice != 0 && slice != need)) {
    if (threadIdx.x == 0) counts[m] = -2;        // the table disagrees with the sizes the launch was given
    return;
  }
  unsigned char* base = slice == 0 ? sm : ws + ws_off[m];
  Scratch s;
  s.mask = base;
  s.lab = reinterpret_cast<int*>(base + (HW + 15) / 16 * 16);
  s.x0 = s.lab + HW;
  s.x1 = s.x0 + HW;
  s.y1 = s.x1 + HW;
  s.H = H;
  s.W = W;
  const float* src = reinterpret_cast<const float*>(t[0]);
  const long long sy = t[1], sx = t[2];
  const int iw = (int)t[5], ih = (int)t[6];
  // mask >= thresh_value in float32, then cv2.dilate with a d x d window anchored at d // 2: a max over rows (into lab),
  // then over columns
  for (int c = threadIdx.x; c < HW; c += kTPB) {
    const int y = c / W, x = c - y * W;
    s.mask[c] = src[y * sy + x * sx] >= thresh;
  }
  __syncthreads();
  const int a = d / 2;
  for (int c = threadIdx.x; c < HW; c += kTPB) {
    const int y = c / W, x = c - y * W;
    const int lo = max(x - a, 0), hi = min(x - a + d - 1, W - 1);
    int v = 0;
    for (int i = lo; i <= hi && !v; ++i) v = s.mask[y * W + i];
    s.lab[c] = v;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < HW; c += kTPB) {
    const int y = c / W, x = c - y * W;
    const int lo = max(y - a, 0), hi = min(y - a + d - 1, H - 1);
    int v = 0;
    for (int j = lo; j <= hi && !v; ++j) v = s.lab[j * W + x];
    s.mask[c] = v ? 255 : 0;
  }
  __syncthreads();
  // the merge loop: nchips starts at 0 after the first pass, and the loop ends when a pass finds as many contours as
  // the one before
  label_pass(s, s_red);
  int prev = 0, n;
  for (long pass = 1;; ++pass) {
    if (pass > (long)HW + 2) {
      if (threadIdx.x == 0) counts[m] = -1;
      return;
    }
    __syncthreads();
    paint(s, ms, iw, ih);
    __syncthreads();
    n = label_pass(s, s_red);
    if (n == prev) break;
    prev = n;
  }
  // contours in descending root order: thread t owns the cells [t * C, t * C + C) and writes its roots from the last
  // one down, after the roots of every higher thread
  const int C = (HW + kTPB - 1) / kTPB;
  const int lo = min((int)threadIdx.x * C, HW), hi = min(lo + C, HW);
  int cnt = 0;
  for (int c = lo; c < hi; ++c) cnt += s.lab[c] < 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int v = cnt;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_down_sync(~0u, v, o);
    if (lane + o < 32) v += u;
  }
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  int k = v - cnt;
  for (int w = warp + 1; w < kWarps; ++w) k += s_red[w];
  const double imw = as_double(t[7]), imh = as_double(t[8]), cscale = as_double(t[9]);
  const double ox = as_double(t[10]), oy = as_double(t[11]);
  for (int c = hi - 1; c >= lo; --c) {
    if (s.lab[c] >= 0) continue;
    if (k < cap) write_chip(chips + ((long)m * cap + k) * 4, place(contour_rect(s, c), ms, iw, ih), ms, imw, imh, cscale,
                            ox, oy);
    ++k;
  }
  if (threadIdx.x == 0) counts[m] = n;
}

double as_double_host(long long v) {
  double d;
  memcpy(&d, &v, sizeof(d));
  return d;
}

int check_table(const long long* table_host, int n_maps, const char* who) {
  SN_CHECK(n_maps >= 0, "%s: n_maps (%d) must not be negative", who, n_maps);
  SN_CHECK(n_maps == 0 || table_host, "%s: table (host) must not be null", who);
  for (int m = 0; m < n_maps; ++m) {
    const long long* t = table_host + (long)m * kCols;
    SN_CHECK(t[3] >= 0 && t[4] >= 0 && t[3] * t[4] <= kMaxCells, "%s: map %d is %lld x %lld cells (at most %ld)", who, m,
             t[3], t[4], kMaxCells);
    SN_CHECK(t[3] * t[4] == 0 || t[0], "%s: map %d has a null address", who, m);
    SN_CHECK(t[5] >= 0 && t[6] >= 0 && t[5] < kMaxExtent && t[6] < kMaxExtent,
             "%s: map %d: iw / ih (%lld, %lld) must lie in [0, %d)", who, m, t[5], t[6], kMaxExtent);
    SN_CHECK(as_double_host(t[9]) > 0, "%s: map %d: cscale must be positive", who, m);
  }
  return 0;
}

}  // namespace

extern "C" {

int sniper_focus_chips_workspace_bytes(const long long* table_host, int n_maps, long long* ws_off_host) {
  if (check_table(table_host, n_maps, "focus_chips_workspace_bytes")) return -1;
  SN_CHECK(ws_off_host, "focus_chips_workspace_bytes: ws_off (host) must not be null");
  long long off = 0;
  for (int m = 0; m < n_maps; ++m) {
    ws_off_host[m] = off;
    const long cells = (long)(table_host[(long)m * kCols + 3] * table_host[(long)m * kCols + 4]);
    if (cells > 0 && map_bytes(cells) > kSmemCap) off += map_bytes(cells);
  }
  ws_off_host[n_maps] = off;
  return 0;
}

int sniper_focus_chips(const long long* table, const long long* ws_off, const long long* table_host,
                       const long long* ws_off_host, int n_maps, int d, float thresh, int ms, void* workspace, int cap,
                       double* chips, int* counts, void* stream) {
  if (check_table(table_host, n_maps, "focus_chips")) return -1;
  if (n_maps == 0) return 0;
  SN_CHECK(d >= 1, "focus_chips: the dilation size d (%d) must be at least 1", d);
  SN_CHECK(ms >= 0 && ms < kMaxExtent, "focus_chips: the minimum chip size ms (%d) must lie in [0, %d)", ms, kMaxExtent);
  SN_CHECK(cap >= 0, "focus_chips: cap (%d chips per map) must not be negative", cap);
  SN_CHECK(table && ws_off && counts, "focus_chips: table / ws_off / counts must not be null");
  SN_CHECK(cap == 0 || chips, "focus_chips: chips must not be null");
  SN_CHECK(ws_off_host, "focus_chips: ws_off (host) must not be null");
  long smem = 0;
  long long off = 0;
  for (int m = 0; m < n_maps; ++m) {
    const long cells = (long)(table_host[(long)m * kCols + 3] * table_host[(long)m * kCols + 4]);
    const bool in_smem = cells == 0 || map_bytes(cells) <= kSmemCap;
    if (in_smem && cells > 0 && map_bytes(cells) > smem) smem = map_bytes(cells);
    SN_CHECK(ws_off_host[m] == off, "focus_chips: ws_off does not match sniper_focus_chips_workspace_bytes");
    if (!in_smem) off += map_bytes(cells);
  }
  SN_CHECK(ws_off_host[n_maps] == off, "focus_chips: ws_off does not match sniper_focus_chips_workspace_bytes");
  SN_CHECK(off == 0 || workspace, "focus_chips: these maps need a workspace of %lld bytes", off);
  cudaStream_t st = (cudaStream_t)stream;
  SN_CUDA(cudaFuncSetAttribute(focus_chips_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCap));
  focus_chips_kernel<<<n_maps, kTPB, smem, st>>>(table, ws_off, static_cast<unsigned char*>(workspace), d, thresh, ms,
                                                 cap, smem, chips, counts);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
