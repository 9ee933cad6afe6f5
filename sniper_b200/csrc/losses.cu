// Loss layers of the SNIPER graph, forward + gradient in one pass, valid-count kept on the device.
//
// Replaces SoftmaxOutput (SNIPER-mxnet/src/operator/softmax_output-inl.h:108-132 fwd, :162-206
// multi_output bwd, :207-263 flat bwd; the reference copies the labels to the host every backward to
// count non-ignored entries, :184-195 / :243-253), smooth_l1 (mshadow_op.h:642-678) and MakeLoss as used by
// symbols/faster/resnet_mx_101_e2e.py:279-281, 310-319, 330-334.
#include "common.cuh"
#include <math.h>

namespace {

__global__ void count_valid_kernel(const float* __restrict__ label, long n, int ignore, int* __restrict__ out) {
  int c = 0;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    c += ((int)label[i] != ignore);
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

// RPN 2-way softmax over (bg = channel a, fg = channel A+a) of NHWC scores [B,H,W,ld]; labels [B,A*H*W] in
// (a,h,w) order with -1 = ignore.  Writes prob (same layout as scores) and dscore = (p - onehot)*gs/valid.
__global__ void __launch_bounds__(256) rpn_softmax_kernel(const float* __restrict__ score, int ld,
                                                           const float* __restrict__ label, int B, int H, int W, int A,
                                                           float grad_scale, const int* __restrict__ valid_cnt,
                                                           float* __restrict__ prob, int ldp,
                                                           float* __restrict__ dscore, int ldg,
                                                           float* __restrict__ loss_sum) {
  const long total = (long)B * H * W * A;
  const int HW = H * W;
  float norm = 1.0f;
  if (valid_cnt) {
    const int v = *valid_cnt;
    norm = grad_scale / (float)(v == 0 ? 1 : v);
  }
  float lsum = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int a = (int)(i % A);
    const long pix = i / A;  // b*HW + hw
    const int b = (int)(pix / HW), hw = (int)(pix - (long)b * HW);
    const float s0 = score[pix * ld + a], s1 = score[pix * ld + A + a];
    const float m = fmaxf(s0, s1);
    const float e0 = expf(s0 - m), e1 = expf(s1 - m);
    const float inv = 1.0f / (e0 + e1);
    const float p0 = e0 * inv, p1 = e1 * inv;
    prob[pix * ldp + a] = p0;
    prob[pix * ldp + A + a] = p1;
    if (dscore) {
      const int l = (int)label[(long)b * A * HW + (long)a * HW + hw];
      float g0 = 0.f, g1 = 0.f;
      if (l != -1) {
        g0 = (p0 - (l == 0 ? 1.f : 0.f)) * norm;
        g1 = (p1 - (l == 1 ? 1.f : 0.f)) * norm;
        lsum -= logf(fmaxf(l == 1 ? p1 : p0, 1e-14f));
      }
      dscore[pix * ldg + a] = g0;
      dscore[pix * ldg + A + a] = g1;
    }
  }
  if (loss_sum) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, off);
    if ((threadIdx.x & 31) == 0 && lsum != 0.f) atomicAdd(loss_sum, lsum);
  }
}

__device__ __forceinline__ float smooth_l1(float d) { return fabsf(d) < 1.f ? 0.5f * d * d : fabsf(d) - 0.5f; }
__device__ __forceinline__ float smooth_l1_grad(float d) { return fabsf(d) < 1.f ? d : (d > 0.f ? 1.f : -1.f); }

// RPN box loss: pred NHWC [B,H,W,ld] channel 4a+j; target/weight NCHW [B,4A,H,W] (the iterator's layout)
__global__ void __launch_bounds__(256) rpn_smooth_l1_kernel(const float* __restrict__ pred, int ld,
                                                             const float* __restrict__ target,
                                                             const float* __restrict__ weight, int B, int H, int W,
                                                             int C4, float grad_scale, float* __restrict__ dpred,
                                                             int ldg, float* __restrict__ loss_sum) {
  const long total = (long)B * H * W * C4;
  const int HW = H * W;
  float lsum = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    const long pix = i / C4;
    const int b = (int)(pix / HW), hw = (int)(pix - (long)b * HW);
    const long t = ((long)b * C4 + c) * HW + hw;
    const float w = weight[t];
    const float d = pred[pix * ld + c] - target[t];
    dpred[pix * ldg + c] = w * smooth_l1_grad(d) * grad_scale;
    lsum += w * smooth_l1(d);
  }
  if (loss_sum) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, off);
    if ((threadIdx.x & 31) == 0 && lsum != 0.f) atomicAdd(loss_sum, lsum);
  }
}

// flat softmax + CE gradient, one warp per row of [N,K] (K <= 1024)
__global__ void __launch_bounds__(256) softmax_ce_kernel(const float* __restrict__ logits, int ld,
                                                          const float* __restrict__ label, int N, int K, int ignore,
                                                          float grad_scale, const int* __restrict__ valid_cnt,
                                                          float* __restrict__ prob, int ldp, float* __restrict__ grad,
                                                          int ldg, float* __restrict__ loss_sum) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  float norm = grad_scale;
  if (valid_cnt) {
    const int v = *valid_cnt;
    norm = grad_scale / (float)(v == 0 ? 1 : v);
  }
  const float* row = logits + (long)warp * ld;
  float m = -INFINITY;
  for (int k = lane; k < K; k += 32) m = fmaxf(m, row[k]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s += expf(row[k] - m);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  const float inv = 1.0f / s;
  const int l = (int)label[warp];
  for (int k = lane; k < K; k += 32) {
    const float p = expf(row[k] - m) * inv;
    if (prob) prob[(long)warp * ldp + k] = p;
    if (grad) grad[(long)warp * ldg + k] = l == ignore ? 0.f : (p - (k == l ? 1.f : 0.f)) * norm;
    if (loss_sum && k == l && l != ignore) atomicAdd(loss_sum, -logf(fmaxf(p, 1e-14f)));
  }
}

// R-CNN box loss on [N,C]: grad = weight * smooth_l1'(pred - target) * grad_scale
__global__ void __launch_bounds__(256) smooth_l1_kernel(const float* __restrict__ pred, int ld,
                                                         const float* __restrict__ target,
                                                         const float* __restrict__ weight, long N, int C,
                                                         float grad_scale, float* __restrict__ grad, int ldg,
                                                         float* __restrict__ loss_sum) {
  const long total = N * C;
  float lsum = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C;
    const int c = (int)(i - r * C);
    const float w = weight[i];
    const float d = pred[r * ld + c] - target[i];
    grad[r * ldg + c] = w * smooth_l1_grad(d) * grad_scale;
    lsum += w * smooth_l1(d);
  }
  if (loss_sum) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, off);
    if ((threadIdx.x & 31) == 0 && lsum != 0.f) atomicAdd(loss_sum, lsum);
  }
}

int lgrid(long n) {
  long g = (n + 255) / 256;
  const long cap = (long)sn::kNumSMs * 8;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace

extern "C" {

// out_count must be zeroed by the caller (device int)
int sniper_count_valid(const float* label, long n, int ignore_label, int* out_count, void* stream) {
  SN_CHECK(n >= 0, "count_valid: n (%ld) must not be negative", n);
  SN_CHECK(label != nullptr && out_count != nullptr, "count_valid: label / out_count must not be null");
  if (n == 0) return 0;
  count_valid_kernel<<<lgrid(n), 256, 0, (cudaStream_t)stream>>>(label, n, ignore_label, out_count);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_rpn_softmax_loss(const float* score, int ld, const float* label, int B, int H, int W, int A,
                            float grad_scale, const int* valid_cnt, float* prob, int ldp, float* dscore, int ldg,
                            float* loss_sum, void* stream) {
  SN_CHECK(B >= 0 && H > 0 && W > 0 && A >= 1, "rpn_softmax_loss: need B >= 0, H, W > 0 and A >= 1");
  SN_CHECK(score != nullptr && prob != nullptr, "rpn_softmax_loss: score / prob must not be null");
  SN_CHECK(ld >= 2 * A, "rpn_softmax_loss: ld of score (%d) is smaller than 2A (%d)", ld, 2 * A);
  SN_CHECK(ldp >= 2 * A, "rpn_softmax_loss: ld of prob (%d) is smaller than 2A (%d)", ldp, 2 * A);
  SN_CHECK(dscore == nullptr || ldg >= 2 * A, "rpn_softmax_loss: ld of dscore (%d) is smaller than 2A (%d)", ldg, 2 * A);
  SN_CHECK(dscore == nullptr || label != nullptr, "rpn_softmax_loss: label is null (the gradient needs it)");
  if (B == 0) return 0;
  rpn_softmax_kernel<<<lgrid((long)B * H * W * A), 256, 0, (cudaStream_t)stream>>>(
      score, ld, label, B, H, W, A, grad_scale, valid_cnt, prob, ldp, dscore, ldg, loss_sum);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_rpn_smooth_l1_loss(const float* pred, int ld, const float* target, const float* weight, int B, int H, int W,
                              int C4, float grad_scale, float* dpred, int ldg, float* loss_sum, void* stream) {
  SN_CHECK(B >= 0 && H > 0 && W > 0 && C4 >= 1, "rpn_smooth_l1_loss: need B >= 0, H, W > 0 and C4 >= 1");
  SN_CHECK(pred && target && weight && dpred, "rpn_smooth_l1_loss: pred / target / weight / dpred must not be null");
  SN_CHECK(ld >= C4, "rpn_smooth_l1_loss: ld of pred (%d) is smaller than C4 (%d)", ld, C4);
  SN_CHECK(ldg >= C4, "rpn_smooth_l1_loss: ld of dpred (%d) is smaller than C4 (%d)", ldg, C4);
  if (B == 0) return 0;
  rpn_smooth_l1_kernel<<<lgrid((long)B * H * W * C4), 256, 0, (cudaStream_t)stream>>>(
      pred, ld, target, weight, B, H, W, C4, grad_scale, dpred, ldg, loss_sum);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_softmax_ce(const float* logits, int ld, const float* label, int N, int K, int ignore_label,
                      float grad_scale, const int* valid_cnt, float* prob, int ldp, float* grad, int ldg,
                      float* loss_sum, void* stream) {
  SN_CHECK(K >= 1 && K <= 4096, "softmax_ce: K (%d) must be in [1, 4096]", K);
  SN_CHECK(N >= 0, "softmax_ce: N (%d) must not be negative", N);
  SN_CHECK(logits != nullptr && label != nullptr, "softmax_ce: logits / label must not be null");
  SN_CHECK(ld >= K, "softmax_ce: ld of logits (%d) is smaller than K (%d)", ld, K);
  SN_CHECK(prob == nullptr || ldp >= K, "softmax_ce: ld of prob (%d) is smaller than K (%d)", ldp, K);
  SN_CHECK(grad == nullptr || ldg >= K, "softmax_ce: ld of grad (%d) is smaller than K (%d)", ldg, K);
  if (N == 0) return 0;
  softmax_ce_kernel<<<sn::div_up((long)N * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      logits, ld, label, N, K, ignore_label, grad_scale, valid_cnt, prob, ldp, grad, ldg, loss_sum);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_smooth_l1_loss(const float* pred, int ld, const float* target, const float* weight, long N, int C,
                          float grad_scale, float* grad, int ldg, float* loss_sum, void* stream) {
  SN_CHECK(N >= 0 && C >= 1, "smooth_l1_loss: need N >= 0 and C >= 1");
  SN_CHECK(pred && target && weight && grad, "smooth_l1_loss: pred / target / weight / grad must not be null");
  SN_CHECK(ld >= C, "smooth_l1_loss: ld of pred (%d) is smaller than C (%d)", ld, C);
  SN_CHECK(ldg >= C, "smooth_l1_loss: ld of grad (%d) is smaller than C (%d)", ldg, C);
  if (N == 0) return 0;
  smooth_l1_kernel<<<lgrid(N * C), 256, 0, (cudaStream_t)stream>>>(pred, ld, target, weight, N, C, grad_scale, grad,
                                                                 ldg, loss_sum);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
