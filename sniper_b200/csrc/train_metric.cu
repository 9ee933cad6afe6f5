// The reference's training metrics (lib/train_utils/metric.py:50-95, 104-300) on the device, one launch per step.
//
// Replaces the per-step `asnumpy()` of RPNAccMetric, RPNLogLossMetric, RPNL1LossMetric, RCNNAccMetric,
// RCNNLogLossMetric, RCNNL1LossCRCNNMetric and (TRAIN.AUTO_FOCUS) AutoFocusAccMetric / AutoFocusLogLossMetric.  The
// step's terms are ADDED into a caller-owned accumulator that the kernel never resets:
//
//   int64  num_inst[8]   the metric's instance count (label != -1), from the step's count_valid results
//   int64  hits[8]       accuracy numerators: #(argmax == label) over rows with label != -1
//   double sum[8]        log-loss sums -sum log(p[label] + 1e-14) and the two L1 loss sums
//
// slots: 0 RPNAcc, 1 RPNLogLoss, 2 RPNL1Loss, 3 RCNNAcc, 4 RCNNLogLoss, 5 RCNNL1LossCRCNN, 6 AutoFocusAcc,
// 7 AutoFocusLogLoss.  Argmax ties go to the first maximum (argmax_channel / np.argmax: background for the 2-way
// problems).  p + 1e-14 is formed in float32 as the reference's `cls += 1e-14` does; the log and the sums are float64.
//
// Determinism: the grid size depends only on the shapes, each block's share of the rows is fixed by its index, and the
// block partials are summed in block order by the last block to finish (atomic ticket, reset by that block, so a
// captured graph can be replayed).  Two runs give byte-identical accumulators.  The L1 sums are read from the loss
// buffer the smooth-L1 loss kernels filled with float atomics and inherit their last-bit run-to-run variation.
// This file is compiled with -fmad=false.
#include "block_reduce.cuh"
#include "common.cuh"
#include <math.h>

namespace {

constexpr int kTmTPB = 256;
constexpr int kTmWarps = kTmTPB / 32;
constexpr int kTmBlocksPerSM = 8;              // the launch bound keeps the registers low enough for 8 to fit
constexpr int kTmMaxBlocks = kTmBlocksPerSM * sn::kNumSMs;   // one full wave: the anchor loop is latency-bound
constexpr int kSlots = 8;

struct Partial {
  double loss[3];     // RPN, R-CNN, AutoFocus log-loss
  long long hits[3];
};

struct Workspace {
  unsigned int ticket;
  unsigned int pad[3];
  Partial part[kTmMaxBlocks];
};

struct Args {
  const float* rpn_prob;
  int ld_rpn;
  const float* rpn_label;
  int B, H, W, A;
  const float* cls_prob;
  int ld_cls;
  const float* cls_label;
  int N, K;
  const float* af_prob;
  int ld_af;
  const float* af_label;
  int Haf, Waf;
  const int* counts;
  const float* loss_buf;
  long long* acc;
  Workspace* ws;
};

__device__ __forceinline__ double log_term(float p) { return -log((double)(p + 1e-14f)); }

// One 2-way problem in rpn_softmax_kernel's layout: prob NHWC [B,H,W,ld] with bg = channel a, fg = channel A+a; labels
// [B, A*H*W] in (a,h,w) order.
__device__ __forceinline__ void two_way(const float* __restrict__ prob, int ld, const float* __restrict__ label, int B,
                                        int H, int W, int A, long long& hits, double& loss) {
  const int total = B * H * W * A;     // < 2^31, checked by the entry point: 32-bit index arithmetic
  const int HW = H * W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int pix = i / A, a = i - pix * A;
    const int b = pix / HW, hw = pix - b * HW;
    const int l = (int)label[(long)(b * A + a) * HW + hw];
    if (l == -1) continue;
    const float p0 = prob[(long)pix * ld + a], p1 = prob[(long)pix * ld + A + a];
    hits += ((p1 > p0 ? 1 : 0) == l);
    loss += log_term(l == 1 ? p1 : p0);
  }
}

__global__ void __launch_bounds__(kTmTPB, kTmBlocksPerSM) train_metric_kernel(Args a) {
  __shared__ double shd[kTmWarps];
  __shared__ long long shl[kTmWarps];
  __shared__ bool last;
  long long hits[3] = {0, 0, 0};
  double loss[3] = {0.0, 0.0, 0.0};
  two_way(a.rpn_prob, a.ld_rpn, a.rpn_label, a.B, a.H, a.W, a.A, hits[0], loss[0]);
  if (a.af_prob) two_way(a.af_prob, a.ld_af, a.af_label, a.B, a.Haf, a.Waf, 1, hits[2], loss[2]);
  // R-CNN: one warp per row of cls_prob [N, ld]
  const int lane = threadIdx.x & 31;
  const long gwarp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long r = gwarp; r < a.N; r += nwarps) {
    const int l = (int)a.cls_label[r];
    if (l == -1) continue;                   // warp-uniform
    const float* row = a.cls_prob + r * a.ld_cls;
    float m = -INFINITY;
    int mi = a.K;
    for (int k = lane; k < a.K; k += 32) {
      const float v = row[k];
      if (v > m) m = v, mi = k;              // strictly greater: the lane keeps its first maximum
    }
    warp_argmax(m, mi);
    if (lane == 0) {
      hits[1] += (mi == l);
      loss[1] += log_term(row[l]);
    }
  }
  Partial* mine = &a.ws->part[blockIdx.x];
  for (int j = 0; j < 3; ++j) {
    const long long h = block_sum<long long, kTmWarps>(hits[j], shl);
    const double s = block_sum<double, kTmWarps>(loss[j], shd);
    if (threadIdx.x == 0) mine->hits[j] = h, mine->loss[j] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&a.ws->ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // the last block: partials in block order (lane-strided, then a fixed tree), then the fold into the accumulator
  if (threadIdx.x >= 32) return;
  long long* num_inst = a.acc;
  long long* acc_hits = a.acc + kSlots;
  double* acc_sum = reinterpret_cast<double*>(a.acc + 2 * kSlots);
  for (int j = 0; j < 3; ++j) {
    long long h = 0;
    double s = 0.0;
    for (int b = lane; b < (int)gridDim.x; b += 32) {
      const volatile Partial* p = &a.ws->part[b];
      h += p->hits[j];
      s += p->loss[j];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      h += __shfl_down_sync(0xffffffffu, h, off);
      s += __shfl_down_sync(0xffffffffu, s, off);
    }
    if (lane == 0 && (j < 2 || a.af_prob)) {
      acc_hits[3 * j] += h;
      acc_sum[3 * j + 1] += s;
      const long long n = a.counts[j];
      num_inst[3 * j] += n;
      num_inst[3 * j + 1] += n;
      if (j < 2) num_inst[3 * j + 2] += n;
    }
  }
  if (lane == 0) {
    acc_sum[2] += (double)a.loss_buf[1];
    acc_sum[5] += (double)a.loss_buf[3];
    a.ws->ticket = 0;
  }
}

}  // namespace

extern "C" {

size_t sniper_train_metric_workspace_bytes(void) { return sizeof(Workspace); }

// acc: int64 num_inst[8] | int64 hits[8] | float64 sum[8] (slots in the comment at the top), accumulated into.
// counts: the step's count_valid results (int32 [2], [3] with the AutoFocus problem); loss_buf: the step's loss sums,
// [1] RPN and [3] R-CNN smooth-L1.  workspace: sniper_train_metric_workspace_bytes() bytes, zero-filled once by the
// caller.  af_prob = NULL: no AutoFocus problem (slots 6 / 7 untouched).
int sniper_train_metric_accum(const float* rpn_prob, int ld_rpn, const float* rpn_label, int B, int H, int W, int A,
                              const float* cls_prob, int ld_cls, const float* cls_label, int N, int K,
                              const float* af_prob, int ld_af, const float* af_label, int Haf, int Waf,
                              const int* counts, const float* loss_buf, long long* acc, void* workspace,
                              void* stream) {
  SN_CHECK(B >= 0, "train_metric_accum: B (%d) must not be negative", B);
  SN_CHECK(N >= 0, "train_metric_accum: N (%d) must not be negative", N);
  SN_CHECK(H > 0 && W > 0, "train_metric_accum: H (%d) and W (%d) must be positive", H, W);
  SN_CHECK(A >= 1, "train_metric_accum: A (%d) must be at least 1", A);
  SN_CHECK(K >= 1, "train_metric_accum: K (%d) must be at least 1", K);
  SN_CHECK(ld_rpn >= 2 * A, "train_metric_accum: ld of rpn_prob (%d) is smaller than 2A (%d)", ld_rpn, 2 * A);
  SN_CHECK(ld_cls >= K, "train_metric_accum: ld of cls_prob (%d) is smaller than K (%d)", ld_cls, K);
  SN_CHECK(rpn_prob != nullptr, "train_metric_accum: rpn_prob must not be null");
  SN_CHECK(rpn_label != nullptr, "train_metric_accum: rpn_label must not be null");
  SN_CHECK(cls_prob != nullptr, "train_metric_accum: cls_prob must not be null");
  SN_CHECK(cls_label != nullptr, "train_metric_accum: cls_label must not be null");
  SN_CHECK(counts != nullptr, "train_metric_accum: counts must not be null");
  SN_CHECK(loss_buf != nullptr, "train_metric_accum: loss_buf must not be null");
  SN_CHECK(acc != nullptr, "train_metric_accum: acc must not be null");
  SN_CHECK(workspace != nullptr, "train_metric_accum: workspace must not be null");
  if (af_prob != nullptr) {
    SN_CHECK(af_label != nullptr, "train_metric_accum: af_label must not be null when af_prob is given");
    SN_CHECK(Haf > 0 && Waf > 0, "train_metric_accum: Haf (%d) and Waf (%d) must be positive", Haf, Waf);
    SN_CHECK(ld_af >= 2, "train_metric_accum: ld of af_prob (%d) is smaller than 2", ld_af);
  }
  SN_CHECK((long)B * H * W * A < (1L << 31), "train_metric_accum: B*H*W*A (%ld) must be below 2^31",
           (long)B * H * W * A);
  SN_CHECK(af_prob == nullptr || (long)B * Haf * Waf < (1L << 31),
           "train_metric_accum: B*Haf*Waf (%ld) must be below 2^31", (long)B * Haf * Waf);
  if (B == 0 || N == 0) return 0;    // an empty step (the R-CNN rows come from the chips): nothing to add
  Args a;
  a.rpn_prob = rpn_prob; a.ld_rpn = ld_rpn; a.rpn_label = rpn_label; a.B = B; a.H = H; a.W = W; a.A = A;
  a.cls_prob = cls_prob; a.ld_cls = ld_cls; a.cls_label = cls_label; a.N = N; a.K = K;
  a.af_prob = af_prob; a.ld_af = ld_af; a.af_label = af_label; a.Haf = Haf; a.Waf = Waf;
  a.counts = counts; a.loss_buf = loss_buf; a.acc = acc; a.ws = static_cast<Workspace*>(workspace);
  const long work = (long)B * H * W * A + (long)N * 32 + (af_prob ? (long)B * Haf * Waf : 0);
  long g = (work + kTmTPB - 1) / kTmTPB;
  if (g > kTmMaxBlocks) g = kTmMaxBlocks;
  train_metric_kernel<<<(int)g, kTmTPB, 0, (cudaStream_t)stream>>>(a);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
