// Detection post-processing of the multi-scale inference path on the device: everything between the R-FCN head and
// the cross-scale soft-NMS, for one batch of chips in one launch.
//
// Replaces, per batch, four blocking D2H copies and the numpy code of Tester.detect (lib/inference.py:100-139:
// bbox_pred = nonlinear_pred of lib/bbox/bbox_transform.py:93-133, clip_boxes, division by the chip's scale), the score
// threshold and chip-border pruning of Tester.get_detections (:291-301, check_valid :235-258, projection :335-351) and
// the valid-range filter of Tester.aggregate (:176-186).  Surviving (x1, y1, x2, y2, score) rows are appended to a
// caller-owned run buffer at a device-side cursor, each with a 64-bit order key (image, class, scale, chip, roi): one
// sort by key over a whole run puts every (image, class) problem's rows in the order the reference stacks them.
//
// Arithmetic: float64 from the float32 rois / deltas on (sizes with the +1, exp in double), the clip bound is the
// float32 `im_info - 1`, rows are rounded to float32 where `inference.threshold_detections` stores them, widened
// again for the projection to image coordinates and the border test, rounded once more as `inference.aggregate`
// does, and the valid-range areas are float32 products without the +1.  This file is compiled with -fmad=false.
//
// Determinism: the launch is cooperative.  Every warp owns a contiguous range of roi rows; the grid counts, meets at
// one grid-wide barrier, and writes at offsets given by the exclusive scan of the counts, so the buffer holds the
// rows in (chip, roi, class) order whatever the block schedule.
#include "common.cuh"
#include "np_pairwise.cuh"
#include <cooperative_groups.h>
#include <math.h>

namespace cg = cooperative_groups;

namespace {

constexpr int kDpTPB = 256;
constexpr int kDpWarps = kDpTPB / 32;
constexpr int kDpMaxBlocks = 2 * sn::kNumSMs;
constexpr int kChipCols = 12;   // image, chip id, chip x1 y1 x2 y2, image width, height, prune, valid lo, hi, unused

// key = image:19 | class:10 | scale:4 | chip:14 | roi:16 (63 bits: sorts the same signed or unsigned)
constexpr int kRoiBits = 16, kChipBits = 14, kScaleBits = 4, kClassBits = 10;

struct Args {
  const float* rois;
  const float* cls_prob;
  const float* bbox_pred;
  long bbox_ld;
  const float* im_info;
  const double* chips;
  int B, R, K;
  float cls_thresh;
  int scale;
  float* out_rows;
  long* out_keys;
  long capacity;
  long* state;         // [0] cursor (rows in the buffer), [1] rows a refused launch needed (0 = none refused)
  int* block_counts;   // [gridDim.x]
};

// The class-independent part of one roi row: the float32 box the host path would hand to the NMS, and whether the
// chip-border pruning and the valid range keep it.
__device__ __forceinline__ bool decode_row(const Args& a, int row, int b, const double* __restrict__ c, float box[4]) {
  const float* r = a.rois + (size_t)row * 5;
  const double x1 = r[1], y1 = r[2], x2 = r[3], y2 = r[4];
  const float* dl = a.bbox_pred + (size_t)row * a.bbox_ld;
  const double d0 = dl[0], d1 = dl[1], d2 = dl[2], d3 = dl[3];
  const double w = x2 - x1 + 1.0, h = y2 - y1 + 1.0;
  const double cx = x1 + 0.5 * (w - 1.0), cy = y1 + 0.5 * (h - 1.0);
  const double pcx = d0 * w + cx, pcy = d1 * h + cy;
  const double pw = exp(d2) * w, ph = exp(d3) * h;
  double o[4] = {pcx - 0.5 * (pw - 1.0), pcy - 0.5 * (ph - 1.0), pcx + 0.5 * (pw - 1.0), pcy + 0.5 * (ph - 1.0)};
  const float* info = a.im_info + 3 * b;
  const double xmax = (double)(info[1] - 1.f), ymax = (double)(info[0] - 1.f), s = (double)info[2];
#pragma unroll
  for (int k = 0; k < 4; ++k) box[k] = (float)(np_max(np_min(o[k], (k & 1) ? ymax : xmax), 0.0) / s);
  bool ok = true;
  if (c[8] != 0.0) {
    const double delta = 10.0;
    double p[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) p[k] = (double)box[k] + c[2 + (k & 1)];
    if (c[2] >= 0.5 && fabs(p[0] - c[2]) < delta) ok = false;
    if (c[3] >= 0.5 && fabs(p[1] - c[3]) < delta) ok = false;
    if (c[4] < c[6] - 0.5 && fabs(p[2] - c[4]) < delta) ok = false;
    if (c[5] < c[7] - 0.5 && fabs(p[3] - c[5]) < delta) ok = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) box[k] = (float)p[k];
  }
  const float area = (box[3] - box[1]) * (box[2] - box[0]);
  if (c[9] > 0.0 && !(area > (float)(c[9] * c[9]))) ok = false;
  if (c[10] > 0.0 && !(area <= (float)(c[10] * c[10]))) ok = false;
  return ok;
}

__global__ void __launch_bounds__(kDpTPB) detect_post_kernel(const Args a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ int s_warp[kDpWarps];
  __shared__ long s_base;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int N = a.B * a.R;
  const int warps = gridDim.x * kDpWarps;
  const int per = (N + warps - 1) / warps;
  const int row0 = min(N, (blockIdx.x * kDpWarps + wib) * per), row1 = min(N, row0 + per);
  const long cursor = a.state[0];            // read by every block before the barrier, rewritten after it

  // ---- count
  int cnt = 0;
  for (int row = row0; row < row1; ++row) {
    const int b = row / a.R;
    const double* c = a.chips + (size_t)b * kChipCols;
    float box[4];
    if (c[0] < 0.0 || !decode_row(a, row, b, c, box)) continue;
    const float* p = a.cls_prob + (size_t)row * a.K;
    for (int j0 = 1; j0 < a.K; j0 += 32) {
      const int j = j0 + lane;
      cnt += __popc(__ballot_sync(0xffffffffu, j < a.K && p[j] > a.cls_thresh));
    }
  }
  if (lane == 0) s_warp[wib] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kDpWarps; ++w) t += s_warp[w];
    a.block_counts[blockIdx.x] = t;
  }
  grid.sync();

  // ---- scan: rows of the blocks before this one, rows of the whole launch
  if (wib == 0) {
    long before = 0, total = 0;
    for (int g = lane; g < (int)gridDim.x; g += 32) {
      const int v = a.block_counts[g];
      total += v;
      if (g < (int)blockIdx.x) before += v;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      before += __shfl_xor_sync(0xffffffffu, before, off);
      total += __shfl_xor_sync(0xffffffffu, total, off);
    }
    if (lane == 0) {
      const bool fits = cursor + total <= a.capacity;
      s_base = fits ? cursor + before : -1;
      if (blockIdx.x == 0) {
        if (fits) a.state[0] = cursor + total;
        else a.state[1] = cursor + total;    // nothing is written: the run is refused as a whole, never truncated
      }
    }
  }
  __syncthreads();
  if (s_base < 0) return;
  long at = s_base;
  for (int w = 0; w < wib; ++w) at += s_warp[w];

  // ---- write
  for (int row = row0; row < row1; ++row) {
    const int b = row / a.R;
    const double* c = a.chips + (size_t)b * kChipCols;
    float box[4];
    if (c[0] < 0.0 || !decode_row(a, row, b, c, box)) continue;
    const long khi = ((long)c[0] << kClassBits);
    const long klo = ((((long)a.scale << kChipBits) | (long)c[1]) << kRoiBits) | (long)(row - b * a.R);
    const float* p = a.cls_prob + (size_t)row * a.K;
    for (int j0 = 1; j0 < a.K; j0 += 32) {
      const int j = j0 + lane;
      const float sc = j < a.K ? p[j] : 0.f;
      const bool pass = j < a.K && sc > a.cls_thresh;
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (pass) {
        const long o = at + __popc(m & ((1u << lane) - 1u));
        float* dst = a.out_rows + o * 5;
        dst[0] = box[0]; dst[1] = box[1]; dst[2] = box[2]; dst[3] = box[3]; dst[4] = sc;
        a.out_keys[o] = ((khi | (long)j) << (kScaleBits + kChipBits + kRoiBits)) | klo;
      }
      at += __popc(m);
    }
  }
}

}  // namespace

extern "C" {

// Bytes of the caller-owned scratch of sniper_detect_post (one int per block of the largest grid).
size_t sniper_detect_post_workspace_bytes(void) { return sizeof(int) * kDpMaxBlocks; }

// One batch of B chips with R rois each, as MultiProposal and the R-FCN head write them: rois [B*R, 5] (rows b*R ..
// b*R + R - 1 belong to chip b), cls_prob [B*R, K], bbox_pred [B*R, 4] with a row stride of bbox_ld floats, im_info
// [B, 3] (resized height, width, scale).  chips: float64 [B, 12] = image id (negative: the chip emits nothing), chip
// id within its image, chip x1 y1 x2 y2 in image coordinates, image width, height, prune flag, valid range lo, hi
// (<= 0: no bound), one unused column.  Rows with cls_prob[:, j] > cls_thresh, j >= 1, that survive the pruning and
// the valid range are appended to out_rows [capacity, 5] / out_keys [capacity] at state[0], which advances; key =
// image << 44 | class << 34 | scale << 30 | chip << 16 | roi.  rows_bound: the caller's upper bound on state[0] at
// launch; the call is refused when rows_bound + B*R*(K-1) exceeds capacity.  Should the rows of a launch not fit after
// all, the launch writes none of them and stores the row count it needed in state[1].  workspace: device,
// sniper_detect_post_workspace_bytes().
int sniper_detect_post(const float* rois, const float* cls_prob, const float* bbox_pred, long bbox_ld,
                       const float* im_info, const double* chips, int B, int R, int K, float cls_thresh, int scale,
                       float* out_rows, long* out_keys, long capacity, long rows_bound, long* state, int* workspace,
                       void* stream) {
  if (B <= 0 || R <= 0) return 0;
  SN_CHECK(K >= 2 && K <= (1 << kClassBits), "detect_post: K = %d classes (2 .. %d)", K, 1 << kClassBits);
  SN_CHECK(R <= (1 << kRoiBits), "detect_post: %d rois per chip (at most %d)", R, 1 << kRoiBits);
  SN_CHECK(scale >= 0 && scale < (1 << kScaleBits), "detect_post: scale index %d (0 .. %d)", scale, (1 << kScaleBits) - 1);
  SN_CHECK(bbox_ld >= 4, "detect_post: bbox_pred row stride %ld < 4", bbox_ld);
  SN_CHECK((long)B * R < (1l << 31) / K, "detect_post: batch of %d x %d rois x %d classes is too large", B, R, K);
  const long worst = (long)B * R * (K - 1);
  SN_CHECK(rows_bound >= 0 && rows_bound + worst <= capacity,
           "detect_post: run buffer of %ld rows cannot take this batch (up to %ld rows held + up to %ld new)", capacity,
           rows_bound, worst);
  static int per_sm = -1;
  if (per_sm < 0) {
    int n = 0;
    SN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, detect_post_kernel, kDpTPB, 0));
    per_sm = n;
  }
  int dev = 0, sms = 0;
  SN_CUDA(cudaGetDevice(&dev));
  SN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int resident = per_sm * sms < kDpMaxBlocks ? per_sm * sms : kDpMaxBlocks;
  SN_CHECK(resident >= 1, "detect_post: the kernel does not fit on this device");
  const int want = sn::div_up((long)B * R, kDpWarps);
  Args a{rois, cls_prob, bbox_pred, bbox_ld, im_info, chips, B, R, K, cls_thresh, scale,
         out_rows, out_keys, capacity, state, workspace};
  void* params[] = {&a};
  SN_CUDA(cudaLaunchCooperativeKernel((const void*)detect_post_kernel, dim3(want < resident ? want : resident),
                                      dim3(kDpTPB), params, 0, (cudaStream_t)stream));
  return 0;
}

}  // extern "C"
