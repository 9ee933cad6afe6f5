// HBM-bound layers of the SNIPER training path on NHWC activations viewed as [M rows, C channels]
// with a row stride `ld` (so that layers can read/write slices of the c4|c5 concat buffer in place).
//
// Replaces (reference): BatchNorm train/frozen (src/operator/nn/batch_norm.cu:658-700, cuDNN BN),
// Activation relu, Pooling max 3x3/2 (nn/pool.cuh), elemwise add, Concat, SoftmaxOutput
// (softmax_output-inl.h:108-132 fwd, :162-263 bwd incl. the host-side valid count :184-195),
// smooth_l1 + MakeLoss (mshadow_op.h:642-678), SGD momentum (optimizer_op-inl.h:279-300).
// All kernels: 128-bit vectorised loads/stores along C, grids sized in multiples of the SM count.
#include "common.cuh"
#include <cuda_bf16.h>
#include <math.h>

namespace {

constexpr int kTPB = 256;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
typedef __nv_bfloat16 bf16;
// 4 consecutive channels as float4, from fp32 (16 bytes) or bf16 (8 bytes) storage: the mixed-precision path keeps
// activations in bf16 and does all arithmetic in fp32 registers (dtype codes of the C-ABI: 0 = fp32, 1 = bf16)
__device__ __forceinline__ float4 ld4(const bf16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

// i -> (row, 4*col) for rows of c4 float4 groups; shift path when c4 is a power of two (all BN widths are),
// 32-bit division otherwise -- never 64-bit division in the inner loop.
struct RowSplit {
  unsigned c4;
  int shift;   // log2(c4) or -1
  __device__ __forceinline__ void split(long i, long& r, int& c) const {
    if (shift >= 0) {
      r = i >> shift;
      c = (int)(i & (c4 - 1)) << 2;
    } else {
      const unsigned u = (unsigned)i;
      const unsigned q = u / c4;
      r = q;
      c = (int)(u - q * c4) << 2;
    }
  }
};
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(bf16* p, float4 v) {
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&lo);
  u.y = *reinterpret_cast<const uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = u;
}

// ------------------------------------------------------------------ row-blocked [M, C] kernels
// A block of 256 threads covers LX*4 channels (LX = 32 lanes, 16 when C == 64) x RY = 256/LX row lanes.  Each
// thread keeps the per-channel constants of its 4 channels in registers (the flat grid-stride versions re-loaded
// 2-6 float4 of constants per float4 of data) and streams rows r0 + ry, + RY, ... with kUnroll independent
// 16-byte loads per operand in flight (HBM latency x bandwidth needs ~6 MB outstanding across the SMs).
constexpr int kUnroll = 4;

struct RowBlock {
  int lx_shift;         // log2(LX)
  int rows_per_block;   // multiple of RY
  dim3 grid;
};

// Vector width per thread: 16 bytes of storage either way = 4 fp32 or 8 bf16 channels.
template <typename T> struct VT;
// U = independent 16-byte loads per operand in flight per thread.  The loads are kept RAW (packed, 4 registers each)
// until they are consumed: with bf16 unpacked at load time (8 floats per load) only U = 2 fitted the register budget
// and the bf16 kernels, at 2 resident blocks per SM, had ~32 KB in flight per SM -- below the ~47 KB that HBM latency x
// bandwidth needs -- and ran at 2-3 TB/s (tools/ew_time.py).
template <> struct VT<float> { static constexpr int N = 4, U = 4; typedef float4 Raw; };
template <> struct VT<bf16> { static constexpr int N = 8, U = 4; typedef uint4 Raw; };

template <int N>
__device__ __forceinline__ void ldc(const float* p, float (&v)[N]) {   // N per-channel constants (fp32)
#pragma unroll
  for (int k = 0; k < N; k += 4) {
    const float4 t = ld4(p + k);
    v[k] = t.x; v[k + 1] = t.y; v[k + 2] = t.z; v[k + 3] = t.w;
  }
}
__device__ __forceinline__ void ldv(const float* p, float (&v)[4]) {
  const float4 t = ld4(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ldv(const bf16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[k]));
    v[2 * k] = f.x;
    v[2 * k + 1] = f.y;
  }
}
__device__ __forceinline__ void stv(float* p, const float (&v)[4]) { st4(p, make_float4(v[0], v[1], v[2], v[3])); }
__device__ __forceinline__ void stv(bf16* p, const float (&v)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
    w[k] = *reinterpret_cast<const uint32_t*>(&h);
  }
  *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ float4 ldraw(const float* p) { return ld4(p); }
__device__ __forceinline__ uint4 ldraw(const bf16* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ void unpack(const float4& t, float (&v)[4]) { v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
__device__ __forceinline__ void unpack(const uint4& u, float (&v)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {      // bf16 -> fp32 is a 16-bit shift: low half = element 2k, high half = 2k + 1
    v[2 * k] = __uint_as_float(w[k] << 16);
    v[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u);
  }
}

template <int VEC>
__device__ __forceinline__ bool rb_setup(int lx_shift, int C, int rows_per_block, long M, int& c, int& ry, int& RY,
                                         long& r0, long& r1) {
  const int lx = 1 << lx_shift;
  c = ((int)blockIdx.y * lx + ((int)threadIdx.x & (lx - 1))) * VEC;
  ry = (int)threadIdx.x >> lx_shift;
  RY = 256 >> lx_shift;
  r0 = (long)blockIdx.x * rows_per_block;
  r1 = min(M, r0 + rows_per_block);
  return c < C;
}

// y = relu?(x*scale[c] + shift[c])
template <typename T>
__global__ void __launch_bounds__(256) affine_act_kernel(const T* __restrict__ x, long ldx,
                                                          const float* __restrict__ scale,
                                                          const float* __restrict__ shift, T* __restrict__ y,
                                                          long ldy, long M, int C, int relu, int lx_shift,
                                                          int rows_per_block) {
  constexpr int N = VT<T>::N, KU = VT<T>::U;
  int c, ry, RY;
  long r0, r1;
  if (!rb_setup<N>(lx_shift, C, rows_per_block, M, c, ry, RY, r0, r1)) return;
  const float act_hi = relu == 2 ? 6.f : __int_as_float(0x7f800000);     // relu 2 = clip(y, 0, 6) (mobilenetv2_e2e.py:18-19)
  float s[N], t[N];
  ldc<N>(scale + c, s);
  ldc<N>(shift + c, t);
  for (long r = r0 + ry; r < r1; r += (long)KU * RY) {
    typename VT<T>::Raw raw[KU];
#pragma unroll
    for (int u = 0; u < KU; ++u)
      if (r + (long)u * RY < r1) raw[u] = ldraw(x + (r + (long)u * RY) * ldx + c);
#pragma unroll
    for (int u = 0; u < KU; ++u) {
      const long rr = r + (long)u * RY;
      if (rr >= r1) break;
      float v[N], o[N];
      unpack(raw[u], v);
#pragma unroll
      for (int k = 0; k < N; ++k) {
        o[k] = fmaf(v[k], s[k], t[k]);
        if (relu) o[k] = fminf(fmaxf(o[k], 0.f), act_hi);
      }
      stv(y + rr * ldy + c, o);
    }
  }
}

// Train-mode BatchNorm apply with the finalisation folded in: the producing conv's epilogue left (sum, sum of squares)
// of the input in `sums`; every thread derives scale / shift of its own channels from them (a handful of double ops),
// the first row-block of each channel slab also publishes mean / invstd / scale / shift (the backward pass reads them)
// and updates the moving statistics.  Same arithmetic as bn_finalize_kernel.  `sums` is NOT cleared here (other blocks
// are still reading it): the caller clears it at the end of the step (sniper_bn_param_grad_batched).  Saves one tiny
// launch per BatchNorm layer (90 per training step).
template <typename T>
__global__ void __launch_bounds__(256) bn_apply_train_kernel(const T* __restrict__ x, long ldx,
                                                              const double* __restrict__ sums,
                                                              const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, float eps, float momentum,
                                                              int fix_gamma, float* __restrict__ moving_mean,
                                                              float* __restrict__ moving_var, float* __restrict__ mean,
                                                              float* __restrict__ invstd, float* __restrict__ scale,
                                                              float* __restrict__ shift, T* __restrict__ y, long ldy,
                                                              long M, int C, int relu, int lx_shift, int rows_per_block) {
  constexpr int N = VT<T>::N, KU = VT<T>::U;
  int c, ry, RY;
  long r0, r1;
  if (!rb_setup<N>(lx_shift, C, rows_per_block, M, c, ry, RY, r0, r1)) return;
  const float act_hi = relu == 2 ? 6.f : __int_as_float(0x7f800000);     // relu 2 = clip(y, 0, 6)
  float s[N], t[N];
  const bool publish = blockIdx.x == 0 && ry == 0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const double m = sums[c + k] / (double)M;
    double var = sums[C + c + k] / (double)M - m * m;
    if (var < 0) var = 0;
    const float is = (float)(1.0 / sqrt(var + (double)eps));
    const float g = fix_gamma ? 1.0f : gamma[c + k];
    s[k] = g * is;
    t[k] = beta[c + k] - (float)m * g * is;
    if (publish) {
      mean[c + k] = (float)m;
      invstd[c + k] = is;
      scale[c + k] = s[k];
      shift[c + k] = t[k];
      if (moving_mean) {
        const double unbiased = M > 1 ? var * (double)M / (double)(M - 1) : var;
        moving_mean[c + k] = moving_mean[c + k] * momentum + (float)m * (1.0f - momentum);
        moving_var[c + k] = moving_var[c + k] * momentum + (float)unbiased * (1.0f - momentum);
      }
    }
  }
  for (long r = r0 + ry; r < r1; r += (long)KU * RY) {
    typename VT<T>::Raw raw[KU];
#pragma unroll
    for (int u = 0; u < KU; ++u)
      if (r + (long)u * RY < r1) raw[u] = ldraw(x + (r + (long)u * RY) * ldx + c);
#pragma unroll
    for (int u = 0; u < KU; ++u) {
      const long rr = r + (long)u * RY;
      if (rr >= r1) break;
      float v[N], o[N];
      unpack(raw[u], v);
#pragma unroll
      for (int k = 0; k < N; ++k) {
        o[k] = fmaf(v[k], s[k], t[k]);
        if (relu) o[k] = fminf(fmaxf(o[k], 0.f), act_hi);
      }
      stv(y + rr * ldy + c, o);
    }
  }
}

// ------------------------------------------------------------------ per-channel sums over rows
// MODE 0: sums[c] += x, sums[C+c] += x*x                              (BN forward statistics)
// MODE 1: g = dy * (x*scale+shift > 0); sums[c] += g; sums[C+c] += g * (x-mean)*invstd   (BN+ReLU backward)
// MODE 2: the same with the clip(y, 0, 6) mask 0 <= y <= 6 (clip_grad, tensor/matrix_op-inl.h:1319-1332); MODE 3: no
//         activation (g = dy): the BatchNorm of MobileNetV2's linear bottleneck (mobilenetv2_e2e.py:68-77)
template <int MODE, typename T>
__global__ void __launch_bounds__(256) colsum_kernel(const T* __restrict__ x, long ldx,
                                                      const T* __restrict__ dy, long lddy,
                                                      const float* __restrict__ scale, const float* __restrict__ shift,
                                                      const float* __restrict__ mean, const float* __restrict__ invstd,
                                                      long M, int C, int lx_shift, int rows_per_block,
                                                      double* __restrict__ sums) {
  constexpr int N = VT<T>::N, KU = VT<T>::U;
  int c, ry, RY;
  long r0, r1;
  const bool cok = rb_setup<N>(lx_shift, C, rows_per_block, M, c, ry, RY, r0, r1);
  float a[N], b[N];
#pragma unroll
  for (int k = 0; k < N; ++k) { a[k] = 0.f; b[k] = 0.f; }
  if (cok) {
    float sc[N], sh[N], mu[N], is[N];
    if (MODE >= 1) { ldc<N>(scale + c, sc); ldc<N>(shift + c, sh); ldc<N>(mean + c, mu); ldc<N>(invstd + c, is); }
    for (long r = r0 + ry; r < r1; r += (long)KU * RY) {
      typename VT<T>::Raw rx[KU], rg[KU];
#pragma unroll
      for (int u = 0; u < KU; ++u) {
        const long rr = r + (long)u * RY;
        if (rr < r1) {
          rx[u] = ldraw(x + rr * ldx + c);
          if (MODE >= 1) rg[u] = ldraw(dy + rr * lddy + c);
        }
      }
#pragma unroll
      for (int u = 0; u < KU; ++u) {
        if (r + (long)u * RY >= r1) break;
        float v[N], g[N];
        unpack(rx[u], v);
        if (MODE >= 1) unpack(rg[u], g);
#pragma unroll
        for (int k = 0; k < N; ++k) {
          if (MODE == 0) {
            a[k] += v[k];
            b[k] = fmaf(v[k], v[k], b[k]);
          } else {
            const float yv = fmaf(v[k], sc[k], sh[k]);
            const float gg = MODE == 3 ? g[k] : MODE == 2 ? ((yv >= 0.f && yv <= 6.f) ? g[k] : 0.f) : (yv > 0.f ? g[k] : 0.f);
            a[k] += gg;
            b[k] = fmaf(gg, (v[k] - mu[k]) * is[k], b[k]);
          }
        }
      }
    }
  }
  // Block partials, summed in a fixed thread order -> one double atomic per (block, channel, sum).  Same-address double
  // atomics serialise in L2 and can set the kernel time (it grows with the block count), so row_block keeps the grid to
  // one wave.
  __shared__ float sa[256][N + 1], sb[256][N + 1];
  __shared__ double part[2][32 * N];
#pragma unroll
  for (int k = 0; k < N; ++k) { sa[threadIdx.x][k] = a[k]; sb[threadIdx.x][k] = b[k]; }
  __syncthreads();
  const int lx = 1 << lx_shift;
  if (ry == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      double ax = 0, bx = 0;
      for (int j = 0; j < RY; ++j) {
        ax += sa[j * lx + threadIdx.x][k];
        bx += sb[j * lx + threadIdx.x][k];
      }
      part[0][threadIdx.x * N + k] = ax;     // threadIdx.x < lx here; channel = slab base + threadIdx.x * N + k
      part[1][threadIdx.x * N + k] = bx;
    }
  }
  __syncthreads();
  const int per = lx * N;                    // channels of this slab
  const int cbase = (int)blockIdx.y * per;
  for (int i = threadIdx.x; i < 2 * per; i += 256) {
    const int which = i >= per ? 1 : 0, j = i - which * per;
    if (cbase + j >= C) continue;
    const double t = part[which][j];
    if (t != 0.0) atomicAdd(sums + which * C + cbase + j, t);
  }
}

RowBlock row_block(long M, int C, int vec, int occ);
template <typename K> int resident_blocks(K kernel);

template <int MODE, typename T>
int launch_colsum(cudaStream_t st, const T* x, long ldx, const T* dy, long lddy, const float* scale,
                  const float* shift, const float* mean, const float* invstd, long M, int C, double* sums) {
  const RowBlock rb = row_block(M, C, VT<T>::N, resident_blocks(colsum_kernel<MODE, T>));
  colsum_kernel<MODE, T><<<rb.grid, 256, 0, st>>>(x, ldx, dy, lddy, scale, shift, mean, invstd, M, C, rb.lx_shift,
                                                  rb.rows_per_block, sums);
  SN_LAUNCH_CHECK();
  return 0;
}

// sums -> mean/invstd/scale/shift (+ moving statistics, cuDNN convention: running var unbiased); zeroes sums
__global__ void bn_finalize_kernel(double* __restrict__ sums, long M, int C, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float momentum, int fix_gamma,
                                   float* __restrict__ moving_mean, float* __restrict__ moving_var,
                                   float* __restrict__ mean, float* __restrict__ invstd, float* __restrict__ scale,
                                   float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double m = sums[c] / (double)M;
  double var = sums[C + c] / (double)M - m * m;
  if (var < 0) var = 0;
  sums[c] = 0.0;
  sums[C + c] = 0.0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  const float g = fix_gamma ? 1.0f : gamma[c];
  mean[c] = (float)m;
  invstd[c] = is;
  scale[c] = g * is;
  shift[c] = beta[c] - (float)m * g * is;
  if (moving_mean) {
    const double unbiased = M > 1 ? var * (double)M / (double)(M - 1) : var;
    moving_mean[c] = moving_mean[c] * momentum + (float)m * (1.0f - momentum);
    moving_var[c] = moving_var[c] * momentum + (float)unbiased * (1.0f - momentum);
  }
}

// frozen BN (use_global_stats): scale/shift from the moving statistics
__global__ void bn_frozen_kernel(int C, const float* gamma, const float* beta, const float* moving_mean,
                                 const float* moving_var, float eps, int fix_gamma, float* scale, float* shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float is = 1.0f / sqrtf(moving_var[c] + eps);
  const float g = fix_gamma ? 1.0f : gamma[c];
  scale[c] = g * is;
  shift[c] = beta[c] - moving_mean[c] * g * is;
}

// dx = scale * (g - s1/M - xhat * s2/M) (+add), g = dy * (x*scale+shift > 0), xhat = (x-mean)*invstd; sums = (s1, s2)
template <typename T, int ACT = 1>      // ACT 1: ReLU, 2: clip(0, 6), 3: none -- the masks of colsum_kernel MODE 1 / 2 / 3
__global__ void __launch_bounds__(256) bn_relu_bwd_apply_kernel(const T* __restrict__ x, long ldx,
                                                                 const T* __restrict__ dy, long lddy,
                                                                 const float* __restrict__ scale,
                                                                 const float* __restrict__ shift,
                                                                 const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd,
                                                                 const double* __restrict__ sums,
                                                                 const T* __restrict__ add, long ldadd,
                                                                 T* __restrict__ dx, long lddx, long M, int C,
                                                                 int lx_shift, int rows_per_block) {
  constexpr int N = VT<T>::N, KU = VT<T>::U;
  int c, ry, RY;
  long r0, r1;
  if (!rb_setup<N>(lx_shift, C, rows_per_block, M, c, ry, RY, r0, r1)) return;
  const float invM = 1.0f / (float)M;
  float scv[N], shv[N], muv[N], isv[N], s1[N], s2[N];
  ldc<N>(scale + c, scv); ldc<N>(shift + c, shv); ldc<N>(mean + c, muv); ldc<N>(invstd + c, isv);
#pragma unroll
  for (int k = 0; k < N; ++k) {
    s1[k] = (float)sums[c + k] * invM;
    s2[k] = (float)sums[C + c + k] * invM;
  }
  for (long r = r0 + ry; r < r1; r += (long)KU * RY) {
    typename VT<T>::Raw rx[KU], rg[KU], ra[KU];
#pragma unroll
    for (int u = 0; u < KU; ++u) {
      const long rr = r + (long)u * RY;
      if (rr < r1) {
        rx[u] = ldraw(x + rr * ldx + c);
        rg[u] = ldraw(dy + rr * lddy + c);
        if (add) ra[u] = ldraw(add + rr * ldadd + c);
      }
    }
#pragma unroll
    for (int u = 0; u < KU; ++u) {
      const long rr = r + (long)u * RY;
      if (rr >= r1) break;
      float v[N], g[N], ad[N], o[N];
      unpack(rx[u], v);
      unpack(rg[u], g);
      if (add) unpack(ra[u], ad);
#pragma unroll
      for (int k = 0; k < N; ++k) {
        const float yv = fmaf(v[k], scv[k], shv[k]);
        const float gk = ACT == 3 ? g[k] : ACT == 2 ? ((yv >= 0.f && yv <= 6.f) ? g[k] : 0.f) : (yv > 0.f ? g[k] : 0.f);
        const float xhat = (v[k] - muv[k]) * isv[k];
        o[k] = scv[k] * (gk - s1[k] - xhat * s2[k]);
        if (add) o[k] += ad[k];
      }
      stv(dx + rr * lddx + c, o);
    }
  }
}

// dgamma[c] = s2, dbeta[c] = s1 (accumulate), then zero the sums for reuse
__global__ void bn_param_grad_kernel(double* sums, int C, float* dgamma, float* dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (dbeta) dbeta[c] += (float)sums[c];
  if (dgamma) dgamma[c] += (float)sums[C + c];
  sums[c] = 0.0;
  sums[C + c] = 0.0;
}

// frozen BN + ReLU backward: dx = scale * dy * (x*scale+shift > 0) (+add)   [not needed below stage 2, kept for fix_bn]
__global__ void __launch_bounds__(kTPB) affine_relu_bwd_kernel(const float* __restrict__ x, long ldx,
                                                                const float* __restrict__ dy, long lddy,
                                                                const float* __restrict__ scale,
                                                                const float* __restrict__ shift,
                                                                const float* __restrict__ add, long ldadd,
                                                                float* __restrict__ dx, long lddx, long M, int C,
                                                                int relu) {
  const int c4 = C >> 2;
  const long total = M * c4;
  RowSplit rs;
  rs.c4 = (unsigned)c4;
  rs.shift = (c4 & (c4 - 1)) == 0 ? __ffs(c4) - 1 : -1;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    long r;
    int c;
    rs.split(i, r, c);
    const float4 v = ld4(x + r * ldx + c);
    const float4 g = ld4(dy + r * lddy + c);
    const float4 sc = ld4(scale + c), sh = ld4(shift + c);
    float4 o;
    o.x = (!relu || fmaf(v.x, sc.x, sh.x) > 0.f) ? g.x * sc.x : 0.f;
    o.y = (!relu || fmaf(v.y, sc.y, sh.y) > 0.f) ? g.y * sc.y : 0.f;
    o.z = (!relu || fmaf(v.z, sc.z, sh.z) > 0.f) ? g.z * sc.z : 0.f;
    o.w = (!relu || fmaf(v.w, sc.w, sh.w) > 0.f) ? g.w * sc.w : 0.f;
    if (add) {
      const float4 ad = ld4(add + r * ldadd + c);
      o.x += ad.x; o.y += ad.y; o.z += ad.z; o.w += ad.w;
    }
    st4(dx + r * lddx + c, o);
  }
}

// relu backward through a stored activation: dx = dy * (y > 0); optional per-column bias gradient
template <typename T>
__global__ void __launch_bounds__(kTPB) relu_bwd_kernel(const T* __restrict__ y, long ldy,
                                                         const T* __restrict__ dy, long lddy,
                                                         T* __restrict__ dx, long lddx, long M, int C) {
  const int c4 = C >> 2;
  const long total = M * c4;
  RowSplit rs;
  rs.c4 = (unsigned)c4;
  rs.shift = (c4 & (c4 - 1)) == 0 ? __ffs(c4) - 1 : -1;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    long r;
    int c;
    rs.split(i, r, c);
    const float4 v = ld4(y + r * ldy + c);
    float4 g = ld4(dy + r * lddy + c);
    g.x = v.x > 0.f ? g.x : 0.f; g.y = v.y > 0.f ? g.y : 0.f; g.z = v.z > 0.f ? g.z : 0.f; g.w = v.w > 0.f ? g.w : 0.f;
    st4(dx + r * lddx + c, g);
  }
}

// ------------------------------------------------------------------ max pool 3x3 stride 2 pad 1, NHWC
template <typename T>
__global__ void __launch_bounds__(kTPB) maxpool3x3s2_kernel(const T* __restrict__ x, T* __restrict__ y, int NB,
                                                             int H, int W, int C, int Ho, int Wo) {
  const int c4 = C >> 2;
  const long total = (long)NB * Ho * Wo * c4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4) << 2;
    long p = i / c4;
    const int ow = (int)(p % Wo); p /= Wo;
    const int oh = (int)(p % Ho);
    const int n = (int)(p / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = oh * 2 - 1 + kh;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int iw = ow * 2 - 1 + kw;
        if (iw < 0 || iw >= W) continue;
        const float4 v = ld4(x + (((size_t)n * H + ih) * W + iw) * C + c);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    st4(y + (((size_t)n * Ho + oh) * Wo + ow) * C + c, m);
  }
}

// ------------------------------------------------------------------ stem as a tensor-core contraction: im2col of
// bn_data(x) for conv0 (7x7, stride 2, pad 3, 3 channels; resnet_mx_101_e2e.py:402-404).  col[(n, oy, ox)][k], k =
// (kh * 7 + kw) * 3 + c for k < 147 and 0 up to Kp (the MMA's K granularity: 160 for fp32/TF32 rows, 192 for bf16);
// padding pixels are zero AFTER bn_data, as in the reference graph.  One block = 64 consecutive output pixels of one
// output row: the 7 x 133 x 3 input patch is staged (normalised) in shared memory, the 64 x Kp block of col is
// written fully coalesced, 16 bytes per thread.  The 7x7 conv itself then runs on the wgmma kernel (M = NB*Ho*Wo,
// N = 64, K = Kp) with bn0 + ReLU in its epilogue; the FP32-FMA kernel below took 1.0 ms for 24.6 GFLOP.
constexpr int kStemCols = 64;
template <typename T>
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ x, const float* __restrict__ in_scale,
                                                           const float* __restrict__ in_shift, T* __restrict__ col,
                                                           int H, int W, int Ho, int Wo, int Kp) {
  constexpr int PW = kStemCols * 2 + 5;            // 133 input columns
  __shared__ float patch[3][7][PW + 1];
  const int n = blockIdx.z, oy = blockIdx.y, ox0 = blockIdx.x * kStemCols;
  const int iy0 = oy * 2 - 3, ix0 = ox0 * 2 - 3;
  for (int i = threadIdx.x; i < 3 * 7 * PW; i += blockDim.x) {
    const int c = i / (7 * PW), r = (i / PW) % 7, q = i % PW;
    const int iy = iy0 + r, ix = ix0 + q;
    float v = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W)
      v = fmaf(__ldg(x + (((size_t)n * 3 + c) * H + iy) * W + ix), in_scale[c], in_shift[c]);
    patch[c][r][q] = v;
  }
  __syncthreads();
  constexpr int V = 16 / (int)sizeof(T);           // elements per 16-byte store: 4 fp32 / 8 bf16
  const int vecs = Kp / V;
  const int cols = min(kStemCols, Wo - ox0);
  T* dst = col + (((size_t)n * Ho + oy) * Wo + ox0) * Kp;
  for (int e = threadIdx.x; e < cols * vecs; e += blockDim.x) {
    const int row = e / vecs, k = (e - row * vecs) * V;
    float v[V];
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const int kk = k + j;
      if (kk < 147) {
        const int tap = kk / 3, c = kk - tap * 3, kh = tap / 7, kw = tap - kh * 7;
        v[j] = patch[c][kh][row * 2 + kw];
      } else {
        v[j] = 0.f;
      }
    }
    T* o = dst + (size_t)row * Kp + k;
    if (sizeof(T) == 4) {
      *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
      uint32_t w[V / 2];
#pragma unroll
      for (int j = 0; j < V / 2; ++j) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
        w[j] = *reinterpret_cast<const uint32_t*>(&h);
      }
      *reinterpret_cast<uint4*>(o) = make_uint4(w[0], w[1], w[2 % (V / 2)], w[3 % (V / 2)]);
    }
  }
}

// ------------------------------------------------------------------ stem: bn_data -> conv0 7x7/2 -> bn0 -> relu
// (resnet_mx_101_e2e.py:402-408).  Input NCHW fp32 [NB,3,H,W] (the iterator's layout), output NHWC
// [NB,H/2,W/2,64].  One block = 8x16 output pixels x 64 channels; weights [64][7][7][3] and the input
// patch live in shared memory; bn_data is applied to in-bounds pixels only (padding is zero AFTER bn_data).
constexpr int kStemTH = 8, kStemTW = 16;
template <typename T>
__global__ void __launch_bounds__(128) stem_conv_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                         const float* __restrict__ in_scale,
                                                         const float* __restrict__ in_shift,
                                                         const float* __restrict__ out_scale,
                                                         const float* __restrict__ out_shift, T* __restrict__ y,
                                                         int NB, int H, int W, int Ho, int Wo) {
  constexpr int PH = kStemTH * 2 + 5, PW = kStemTW * 2 + 5;  // 21 x 37
  __shared__ __align__(16) float s_w[147][64];  // [(kh,kw,c)][co]
  __shared__ float s_in[3][PH][PW + 1];  // [(kh,kw,c)][co]
  const int n = blockIdx.z;
  const int oh0 = blockIdx.y * kStemTH, ow0 = blockIdx.x * kStemTW;
  for (int i = threadIdx.x; i < 147 * 64; i += 128) {
    const int co = i & 63, k = i >> 6;
    s_w[k][co] = w[co * 147 + k];
  }
  for (int i = threadIdx.x; i < 3 * PH * PW; i += 128) {
    const int c = i / (PH * PW);
    const int r = (i / PW) % PH, q = i % PW;
    const int ih = oh0 * 2 - 3 + r, iw = ow0 * 2 - 3 + q;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W)
      v = fmaf(x[(((size_t)n * 3 + c) * H + ih) * W + iw], in_scale[c], in_shift[c]);
    s_in[c][r][q] = v;
  }
  __syncthreads();
  const int ty = threadIdx.x / kStemTW, tx = threadIdx.x % kStemTW;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int kh = 0; kh < 7; ++kh) {
    for (int kw = 0; kw < 7; ++kw) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = s_in[c][ty * 2 + kh][tx * 2 + kw];
        const float4* wr = reinterpret_cast<const float4*>(&s_w[(kh * 7 + kw) * 3 + c][0]);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float4 ww = wr[j];
          acc[4 * j] = fmaf(v, ww.x, acc[4 * j]);
          acc[4 * j + 1] = fmaf(v, ww.y, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(v, ww.z, acc[4 * j + 2]);
          acc[4 * j + 3] = fmaf(v, ww.w, acc[4 * j + 3]);
        }
      }
    }
  }
  const int oh = oh0 + ty, ow = ow0 + tx;
  if (oh < Ho && ow < Wo) {
    T* o = y + (((size_t)n * Ho + oh) * Wo + ow) * 64;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float4 s = ld4(out_scale + 4 * j), t = ld4(out_shift + 4 * j);
      float4 v;
      v.x = fmaxf(fmaf(acc[4 * j], s.x, t.x), 0.f);
      v.y = fmaxf(fmaf(acc[4 * j + 1], s.y, t.y), 0.f);
      v.z = fmaxf(fmaf(acc[4 * j + 2], s.z, t.z), 0.f);
      v.w = fmaxf(fmaf(acc[4 * j + 3], s.w, t.w), 0.f);
      st4(o + 4 * j, v);
    }
  }
}

// ------------------------------------------------------------------ weight re-layout for data gradients
// w [Cout, T, Cin] -> wt [Cin, Tsel, Cout] with wt[ci, j, co] = w[co, sel[j], ci]
__global__ void weight_transpose_kernel(const float* __restrict__ w, float* __restrict__ wt, int Cout, int T, int Cin,
                                        int Tsel, const int* __restrict__ sel) {
  __shared__ float tile[32][33];
  const int j = blockIdx.z;
  const int t = sel[j];
  const int ci0 = blockIdx.x * 32, co0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int co = co0 + r, ci = ci0 + threadIdx.x;
    tile[r][threadIdx.x] = (co < Cout && ci < Cin) ? w[((size_t)co * T + t) * Cin + ci] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int ci = ci0 + r, co = co0 + threadIdx.x;
    if (ci < Cin && co < Cout) wt[((size_t)ci * Tsel + j) * Cout + co] = tile[threadIdx.x][r];
  }
}

// All re-layouts of a training step in ONE launch.  jobs: njobs x 9 int64 = {w, wt, sel, Cout, T, Cin, Tsel, block0,
// wt_is_bf16} (block0 = first block of the job, ascending); the block finds its job by bisection.  The source is
// always the fp32 (master) weight; the data-gradient operand is written in fp32 or bf16.
__global__ void weight_transpose_batched_kernel(const long long* __restrict__ jobs, int njobs) {
  __shared__ float tile[32][33];
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid * 9 + 7] <= (long long)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const long long* jb = jobs + lo * 9;
  const float* __restrict__ w = reinterpret_cast<const float*>(jb[0]);
  float* __restrict__ wt = reinterpret_cast<float*>(jb[1]);
  const int* __restrict__ sel = reinterpret_cast<const int*>(jb[2]);
  const int Cout = (int)jb[3], T = (int)jb[4], Cin = (int)jb[5], Tsel = (int)jb[6];
  const int local = (int)((long long)blockIdx.x - jb[7]);
  const int nbx = (Cin + 31) >> 5, nby = (Cout + 31) >> 5;
  const int bx = local % nbx, by = (local / nbx) % nby, j = local / (nbx * nby);
  const int t = sel[j];
  const int ci0 = bx * 32, co0 = by * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int co = co0 + r, ci = ci0 + threadIdx.x;
    tile[r][threadIdx.x] = (co < Cout && ci < Cin) ? w[((size_t)co * T + t) * Cin + ci] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int ci = ci0 + r, co = co0 + threadIdx.x;
    if (ci < Cin && co < Cout) {
      const size_t o = ((size_t)ci * Tsel + j) * Cout + co;
      if (jb[8]) reinterpret_cast<bf16*>(wt)[o] = __float2bfloat16(tile[threadIdx.x][r]);
      else wt[o] = tile[threadIdx.x][r];
    }
  }
}

// dgamma / dbeta of every BatchNorm of the network in ONE launch.  jobs: njobs x 5 int64 = {sums, dgamma, dbeta, C,
// fwd_sums}; block = job, threads stride over the channels; accumulates and zeroes the sums (as bn_param_grad_kernel)
// and clears the layer's forward-statistics accumulator (fwd_sums, may be 0) for the next step.
__global__ void bn_param_grad_batched_kernel(const long long* __restrict__ jobs) {
  const long long* jb = jobs + (size_t)blockIdx.x * 5;
  double* fwd = reinterpret_cast<double*>(jb[4]);
  double* sums = reinterpret_cast<double*>(jb[0]);
  float* dgamma = reinterpret_cast<float*>(jb[1]);
  float* dbeta = reinterpret_cast<float*>(jb[2]);
  const int C = (int)jb[3];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    if (dbeta) dbeta[c] += (float)sums[c];
    if (dgamma) dgamma[c] += (float)sums[C + c];
    sums[c] = 0.0;
    sums[C + c] = 0.0;
    if (fwd) {
      fwd[c] = 0.0;
      fwd[C + c] = 0.0;
    }
  }
}

// ------------------------------------------------------------------ column sums of [M,C] (bias gradients)
// One block per 32 columns walks all M rows (32 row lanes, each in row order) and reduces the 32 partials in a fixed
// order: the sum does not depend on scheduling, so bias gradients are bit-reproducible run to run.
__global__ void __launch_bounds__(1024) colsum_plain_kernel(const float* __restrict__ x, long ldx, long M, int C,
                                                             float* __restrict__ out) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (c < C) {
    long r = threadIdx.y;
    for (; r + 96 < M; r += 128) {
      a0 += x[r * ldx + c];
      a1 += x[(r + 32) * ldx + c];
      a2 += x[(r + 64) * ldx + c];
      a3 += x[(r + 96) * ldx + c];
    }
    for (; r < M; r += 32) a0 += x[r * ldx + c];
  }
  __shared__ float sa[32][33];
  sa[threadIdx.y][threadIdx.x] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) s += sa[k][threadIdx.x];
    out[c] += s;
  }
}

// ------------------------------------------------------------------ SGD momentum, multi-tensor in one flat buffer
// optimizer_op-inl.h:279-300: mom = momentum*mom - lr*wd*w - lr*rescale*g ; w += mom.  lr/wd per segment.
struct SgdSeg { long begin, end; float lr, wd; };
__global__ void __launch_bounds__(kTPB) sgd_mom_kernel(float* __restrict__ w, float* __restrict__ mom,
                                                        const float* __restrict__ g, long n, float lr, float wd,
                                                        float momentum, float rescale) {
  const long n4 = n >> 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    float4 ww = ld4(w + 4 * i), mm = ld4(mom + 4 * i);
    const float4 gg = ld4(g + 4 * i);
    mm.x = momentum * mm.x - lr * wd * ww.x - lr * rescale * gg.x;
    mm.y = momentum * mm.y - lr * wd * ww.y - lr * rescale * gg.y;
    mm.z = momentum * mm.z - lr * wd * ww.z - lr * rescale * gg.z;
    mm.w = momentum * mm.w - lr * wd * ww.w - lr * rescale * gg.w;
    ww.x += mm.x; ww.y += mm.y; ww.z += mm.z; ww.w += mm.w;
    st4(w + 4 * i, ww);
    st4(mom + 4 * i, mm);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long i = (n4 << 2) + threadIdx.x;
    const float m = momentum * mom[i] - lr * wd * w[i] - lr * rescale * g[i];
    mom[i] = m;
    w[i] += m;
  }
}

// Same update with the learning rate and weight decay read from DEVICE memory (hyper[0] = lr, hyper[1] = wd), so a
// CUDA graph that captured the launch follows a learning-rate schedule (WarmupMultiBatchScheduler,
// lib/train_utils/lr_scheduler.py:43-66) by a 8-byte H2D copy before each replay.  lr_mult / wd_mult are the
// per-group multipliers MXNet derives from the symbol attributes (optimizer.py _get_lr/_get_wd).  w16 (optional):
// bf16 copy of the updated weights = the multi_precision path (MP_SGDMomKernel, optimizer_op-inl.h:377-404: fp32
// master weights + momentum, low-precision weights rewritten every step).
__global__ void __launch_bounds__(kTPB) sgd_mom_dev_kernel(float* __restrict__ w, float* __restrict__ mom,
                                                            const float* __restrict__ g, long n,
                                                            const float* __restrict__ hyper, float lr_mult,
                                                            float wd_mult, float momentum, float rescale,
                                                            __nv_bfloat16* __restrict__ w16) {
  const float lr = hyper[0] * lr_mult, wd = hyper[1] * wd_mult;
  const long n4 = n >> 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    float4 ww = ld4(w + 4 * i), mm = ld4(mom + 4 * i);
    const float4 gg = ld4(g + 4 * i);
    mm.x = momentum * mm.x - lr * wd * ww.x - lr * rescale * gg.x;
    mm.y = momentum * mm.y - lr * wd * ww.y - lr * rescale * gg.y;
    mm.z = momentum * mm.z - lr * wd * ww.z - lr * rescale * gg.z;
    mm.w = momentum * mm.w - lr * wd * ww.w - lr * rescale * gg.w;
    ww.x += mm.x; ww.y += mm.y; ww.z += mm.z; ww.w += mm.w;
    st4(w + 4 * i, ww);
    st4(mom + 4 * i, mm);
    if (w16) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(ww.x, ww.y), hi = __floats2bfloat162_rn(ww.z, ww.w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&lo);
      pk.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(w16 + 4 * i) = pk;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long i = (n4 << 2) + threadIdx.x;
    const float m = momentum * mom[i] - lr * wd * w[i] - lr * rescale * g[i];
    mom[i] = m;
    w[i] += m;
    if (w16) w16[i] = __float2bfloat16(w[i]);
  }
}

// Cast of Concat's output / its gradient between the bf16 backbone and the fp32 heads (resnet_mx_101_e2e.py:250-252
// `mx.sym.Cast` after the concat): rows of C channels with independent strides (channel slices of the concat buffer).
template <typename TI, typename TO>
__global__ void __launch_bounds__(kTPB) cast_rows_kernel(const TI* __restrict__ x, long ldx, TO* __restrict__ y, long ldy,
                                                          long M, int C) {
  const int c4 = C >> 2;
  const long total = M * c4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / c4;
    const int c = (int)(i - r * c4) << 2;
    st4(y + r * ldy + c, ld4(x + r * ldx + c));
  }
}

int ew_grid(long work) {
  long g = (work + kTPB - 1) / kTPB;
  const long cap = (long)sn::kNumSMs * 8;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}


// Grid of a row-blocked kernel: ONE wave of resident blocks.  `occ` = blocks of that kernel an SM can hold (occupancy
// API, cached per kernel); the rows are cut so that every slab's row blocks together fill <= kNumSMs * occ slots.  Sizing the
// grid independently of the kernel's occupancy cost up to 2x: e.g. 640 blocks of the bf16 reduction kernel (2 resident
// blocks per SM = 296 slots) ran as three waves of latency-bound blocks (tools/ew_time.py: 20480 x 256 bf16 backward
// 47 us for 52 MB).
RowBlock row_block(long M, int C, int vec, int occ) {
  RowBlock rb;
  const int cv = C / vec;                       // vectors per row
  rb.lx_shift = cv >= 32 ? 5 : (cv >= 16 ? 4 : 3);
  const int lx = 1 << rb.lx_shift, RY = 256 >> rb.lx_shift;
  const int by = sn::div_up(cv, lx);
  if (occ < 1) occ = 1;
  long slots = (long)sn::kNumSMs * occ - by;    // ceil() of the row split can add one block per slab
  if (slots < by) slots = by;
  long rpb = sn::div_up(M * by, slots);
  rpb = (rpb + RY - 1) / RY * RY;               // whole thread rows; the kernels guard the unrolled tail
  if (rpb < RY) rpb = RY;
  rb.rows_per_block = (int)rpb;
  rb.grid = dim3((unsigned)sn::div_up(M, rpb), (unsigned)by, 1);
  return rb;
}

template <typename K>
int resident_blocks(K kernel) {
  // keyed on (kernel address, device): a process may drive several GPUs.  Benign race: worst case two threads query twice.
  struct Entry { const void* fn; int dev, n; };
  static Entry table[64];
  static int used = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  const void* key = reinterpret_cast<const void*>(kernel);
  for (int i = 0; i < used; ++i)
    if (table[i].fn == key && table[i].dev == dev) return table[i].n;
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, 256, 0) != cudaSuccess || n < 1) n = 4;
  if (used < 64) { table[used].fn = key; table[used].dev = dev; table[used].n = n; ++used; }
  return n;
}

}  // namespace

namespace {
// Argument checks of the entry points, made BEFORE any CUDA call: the kernels read and write whole 16-byte (row-blocked
// kernels, fp32 flat kernels) or 8-byte (bf16 in the flat ld4 / st4 kernels) vectors, so a base pointer or a row
// stride that is not a whole number of vectors would be a misaligned-address fault on the device, not an error code.
// `what` names the argument in the message.
int check_rows(const char* fn, const char* what, const void* p, long ld, int C, int vec, int bytes) {
  SN_CHECK(p != nullptr, "%s: %s is null", fn, what);
  SN_CHECK(((uintptr_t)p & (uintptr_t)(bytes - 1)) == 0, "%s: %s must be %d-byte aligned", fn, what, bytes);
  SN_CHECK(ld % vec == 0, "%s: row stride of %s (%ld) must be a multiple of %d", fn, what, ld, vec);
  SN_CHECK(ld >= C, "%s: row stride of %s (%ld) is smaller than C (%d)", fn, what, ld, C);
  return 0;
}
// per-channel fp32 vector read with float4 loads
int check_chan(const char* fn, const char* what, const void* p) {
  SN_CHECK(p != nullptr, "%s: %s is null", fn, what);
  SN_CHECK(((uintptr_t)p & 15) == 0, "%s: %s must be 16-byte aligned", fn, what);
  return 0;
}
int check_shape(const char* fn, long M, int C, int vec) {
  SN_CHECK(M >= 0, "%s: M (%ld) must not be negative", fn, M);
  SN_CHECK(C > 0 && C % vec == 0, "%s: C (%d) must be a positive multiple of %d", fn, C, vec);
  return 0;
}
int check_dtype(const char* fn, int dtype) {
  SN_CHECK(dtype == 0 || dtype == 1, "%s: dtype must be 0 (fp32) or 1 (bf16)", fn);
  return 0;
}
#define SN_TRY(call) do { if (call) return -1; } while (0)

template <typename T, int ACT>
int bn_act_bwd_launch(const void* x, long ldx, const void* dy, long lddy, const float* scale, const float* shift,
                      const float* mean, const float* invstd, double* sums, const void* add, long ldadd, void* dx,
                      long lddx, long M, int C, cudaStream_t st) {
  const RowBlock rb = row_block(M, C, VT<T>::N, resident_blocks(bn_relu_bwd_apply_kernel<T, ACT>));
  if (launch_colsum<ACT, T>(st, static_cast<const T*>(x), ldx, static_cast<const T*>(dy), lddy, scale, shift, mean,
                            invstd, M, C, sums))
    return -1;
  SN_LAUNCH_CHECK();
  bn_relu_bwd_apply_kernel<T, ACT><<<rb.grid, 256, 0, st>>>(
      static_cast<const T*>(x), ldx, static_cast<const T*>(dy), lddy, scale, shift, mean, invstd, sums,
      static_cast<const T*>(add), ldadd, static_cast<T*>(dx), lddx, M, C, rb.lx_shift, rb.rows_per_block);
  SN_LAUNCH_CHECK();
  return 0;
}
}  // namespace

extern "C" {

// dtype (here and below): storage type of the activation tensors, 0 = fp32, 1 = bf16 (arithmetic is fp32 either way)
int sniper_affine_act(const void* x, long ldx, const float* scale, const float* shift, void* y, long ldy, long M,
                      int C, int relu, int dtype, void* stream) {
  SN_TRY(check_dtype("affine_act", dtype));
  const int vec = dtype == 0 ? 4 : 8;
  SN_TRY(check_shape("affine_act", M, C, vec));
  SN_TRY(check_rows("affine_act", "x", x, ldx, C, vec, 16));
  SN_TRY(check_rows("affine_act", "y", y, ldy, C, vec, 16));
  SN_TRY(check_chan("affine_act", "scale", scale));
  SN_TRY(check_chan("affine_act", "shift", shift));
  if (M == 0) return 0;
  const RowBlock rb = dtype == 0 ? row_block(M, C, 4, resident_blocks(affine_act_kernel<float>))
                                 : row_block(M, C, 8, resident_blocks(affine_act_kernel<bf16>));
  if (dtype == 0)
    affine_act_kernel<float><<<rb.grid, 256, 0, (cudaStream_t)stream>>>(
        static_cast<const float*>(x), ldx, scale, shift, static_cast<float*>(y), ldy, M, C, relu, rb.lx_shift,
        rb.rows_per_block);
  else
    affine_act_kernel<bf16><<<rb.grid, 256, 0, (cudaStream_t)stream>>>(
        static_cast<const bf16*>(x), ldx, scale, shift, static_cast<bf16*>(y), ldy, M, C, relu, rb.lx_shift,
        rb.rows_per_block);
  SN_LAUNCH_CHECK();
  return 0;
}

// Train-mode BN statistics of x[M,C] -> (mean, invstd, scale, shift) + moving stats.  `sums` is a
// caller-owned, zero-initialised double[2*C] scratch that is left zeroed.
int sniper_bn_stats(const void* x, long ldx, long M, int C, const float* gamma, const float* beta, float eps,
                    float momentum, int fix_gamma, float* moving_mean, float* moving_var, double* sums, float* mean,
                    float* invstd, float* scale, float* shift, int dtype, void* stream) {
  SN_TRY(check_dtype("bn_stats", dtype));
  const int vec = dtype == 0 ? 4 : 8;
  SN_TRY(check_shape("bn_stats", M, C, vec));
  SN_TRY(check_rows("bn_stats", "x", x, ldx, C, vec, 16));
  SN_CHECK(sums != nullptr && ((uintptr_t)sums & 7) == 0, "bn_stats: sums must be a non-null, 8-byte aligned double[2C]");
  SN_CHECK((moving_mean == nullptr) == (moving_var == nullptr), "bn_stats: moving_mean and moving_var go together");
  SN_CHECK(M >= 1, "bn_stats: M (%ld) must be at least 1 (statistics of no rows are undefined)", M);
  int rc;
  if (dtype == 0)
    rc = launch_colsum<0, float>((cudaStream_t)stream, static_cast<const float*>(x), ldx, nullptr, 0, nullptr, nullptr,
                                 nullptr, nullptr, M, C, sums);
  else
    rc = launch_colsum<0, bf16>((cudaStream_t)stream, static_cast<const bf16*>(x), ldx, nullptr, 0, nullptr, nullptr,
                                nullptr, nullptr, M, C, sums);
  if (rc) return rc;
  SN_LAUNCH_CHECK();
  bn_finalize_kernel<<<sn::div_up(C, 128), 128, 0, (cudaStream_t)stream>>>(sums, M, C, gamma, beta, eps, momentum,
                                                                          fix_gamma, moving_mean, moving_var, mean,
                                                                          invstd, scale, shift);
  SN_LAUNCH_CHECK();
  return 0;
}

// Second half of sniper_bn_stats for producers that already accumulated the column sums (wgmma epilogue).
int sniper_bn_finalize(double* sums, long M, int C, const float* gamma, const float* beta, float eps, float momentum,
                       int fix_gamma, float* moving_mean, float* moving_var, float* mean, float* invstd, float* scale,
                       float* shift, void* stream) {
  SN_CHECK(C > 0, "bn_finalize: C (%d) must be positive", C);
  SN_CHECK(M >= 0, "bn_finalize: M (%ld) must not be negative", M);
  SN_CHECK(sums != nullptr && ((uintptr_t)sums & 7) == 0, "bn_finalize: sums must be a non-null, 8-byte aligned double[2C]");
  SN_CHECK(mean && invstd && scale && shift, "bn_finalize: mean / invstd / scale / shift must not be null");
  SN_CHECK((moving_mean == nullptr) == (moving_var == nullptr), "bn_finalize: moving_mean and moving_var go together");
  SN_CHECK(M >= 1, "bn_finalize: M (%ld) must be at least 1 (statistics of no rows are undefined)", M);
  bn_finalize_kernel<<<sn::div_up(C, 128), 128, 0, (cudaStream_t)stream>>>(sums, M, C, gamma, beta, eps, momentum,
                                                                          fix_gamma, moving_mean, moving_var, mean,
                                                                          invstd, scale, shift);
  SN_LAUNCH_CHECK();
  return 0;
}

// sniper_bn_finalize + sniper_affine_act in one launch: y = relu?(bn_train(x)) with the statistics of x already in `sums`
// (double[2C], left untouched: clear it with sniper_bn_param_grad_batched's fwd_sums column before the next accumulation).
int sniper_bn_apply_train(const void* x, long ldx, const double* sums, long M, int C, const float* gamma,
                          const float* beta, float eps, float momentum, int fix_gamma, float* moving_mean,
                          float* moving_var, float* mean, float* invstd, float* scale, float* shift, void* y, long ldy,
                          int relu, int dtype, void* stream) {
  SN_TRY(check_dtype("bn_apply_train", dtype));
  const int vec = dtype == 0 ? 4 : 8;
  SN_TRY(check_shape("bn_apply_train", M, C, vec));
  SN_TRY(check_rows("bn_apply_train", "x", x, ldx, C, vec, 16));
  SN_TRY(check_rows("bn_apply_train", "y", y, ldy, C, vec, 16));
  SN_CHECK(sums != nullptr && ((uintptr_t)sums & 7) == 0,
           "bn_apply_train: sums must be a non-null, 8-byte aligned double[2C]");
  SN_CHECK(mean && invstd && scale && shift, "bn_apply_train: mean / invstd / scale / shift must not be null");
  SN_CHECK((moving_mean == nullptr) == (moving_var == nullptr), "bn_apply_train: moving_mean and moving_var go together");
  SN_CHECK(M >= 1, "bn_apply_train: M (%ld) must be at least 1 (statistics of no rows are undefined)", M);
  const RowBlock rb = dtype == 0 ? row_block(M, C, 4, resident_blocks(bn_apply_train_kernel<float>))
                                 : row_block(M, C, 8, resident_blocks(bn_apply_train_kernel<bf16>));
  if (dtype == 0)
    bn_apply_train_kernel<float><<<rb.grid, 256, 0, (cudaStream_t)stream>>>(
        static_cast<const float*>(x), ldx, sums, gamma, beta, eps, momentum, fix_gamma, moving_mean, moving_var, mean,
        invstd, scale, shift, static_cast<float*>(y), ldy, M, C, relu, rb.lx_shift, rb.rows_per_block);
  else
    bn_apply_train_kernel<bf16><<<rb.grid, 256, 0, (cudaStream_t)stream>>>(
        static_cast<const bf16*>(x), ldx, sums, gamma, beta, eps, momentum, fix_gamma, moving_mean, moving_var, mean,
        invstd, scale, shift, static_cast<bf16*>(y), ldy, M, C, relu, rb.lx_shift, rb.rows_per_block);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_bn_frozen(int C, const float* gamma, const float* beta, const float* moving_mean, const float* moving_var,
                     float eps, int fix_gamma, float* scale, float* shift, void* stream) {
  SN_CHECK(C > 0, "bn_frozen: C (%d) must be positive", C);
  SN_CHECK(beta && moving_mean && moving_var && scale && shift && (fix_gamma || gamma),
           "bn_frozen: gamma / beta / moving_mean / moving_var / scale / shift must not be null");
  bn_frozen_kernel<<<sn::div_up(C, 128), 128, 0, (cudaStream_t)stream>>>(C, gamma, beta, moving_mean, moving_var, eps,
                                                                        fix_gamma, scale, shift);
  SN_LAUNCH_CHECK();
  return 0;
}

// Backward of y = act(bn_train(x)):  dx (+add), dgamma += , dbeta += .  sums: zeroed double[2C], left zeroed.
// act 1: ReLU (Activation, y > 0), 2: clip(y, 0, 6) (mobilenetv2_e2e.py:18-19; gradient where 0 <= y <= 6,
// tensor/matrix_op-inl.h:1319-1332), 3: no activation (linear bottleneck).
int sniper_bn_act_bwd(const void* x, long ldx, const void* dy, long lddy, const float* scale, const float* shift,
                      const float* mean, const float* invstd, double* sums, const void* add, long ldadd, void* dx,
                      long lddx, float* dgamma, float* dbeta, long M, int C, int act, int dtype, void* stream) {
  SN_TRY(check_dtype("bn_act_bwd", dtype));
  SN_CHECK(act >= 1 && act <= 3, "bn_act_bwd: act must be 1 (relu), 2 (relu6) or 3 (none)");
  const int vec = dtype == 0 ? 4 : 8;
  SN_TRY(check_shape("bn_act_bwd", M, C, vec));
  SN_TRY(check_rows("bn_act_bwd", "x", x, ldx, C, vec, 16));
  SN_TRY(check_rows("bn_act_bwd", "dy", dy, lddy, C, vec, 16));
  SN_TRY(check_rows("bn_act_bwd", "dx", dx, lddx, C, vec, 16));
  if (add) SN_TRY(check_rows("bn_act_bwd", "add", add, ldadd, C, vec, 16));
  SN_TRY(check_chan("bn_act_bwd", "scale", scale));
  SN_TRY(check_chan("bn_act_bwd", "shift", shift));
  SN_TRY(check_chan("bn_act_bwd", "mean", mean));
  SN_TRY(check_chan("bn_act_bwd", "invstd", invstd));
  SN_CHECK(sums != nullptr && ((uintptr_t)sums & 7) == 0, "bn_act_bwd: sums must be a non-null, 8-byte aligned double[2C]");
  if (M == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
#define SN_BN_BWD(T, A) rc = bn_act_bwd_launch<T, A>(x, ldx, dy, lddy, scale, shift, mean, invstd, sums, add, ldadd, dx, lddx, M, C, st)
  if (dtype == 0) {
    if (act == 1) SN_BN_BWD(float, 1); else if (act == 2) SN_BN_BWD(float, 2); else SN_BN_BWD(float, 3);
  } else {
    if (act == 1) SN_BN_BWD(bf16, 1); else if (act == 2) SN_BN_BWD(bf16, 2); else SN_BN_BWD(bf16, 3);
  }
#undef SN_BN_BWD
  if (rc) return -1;
  if (dgamma || dbeta) {   // both null: the caller finishes with sniper_bn_param_grad_batched (sums stay live)
    bn_param_grad_kernel<<<sn::div_up(C, 128), 128, 0, (cudaStream_t)stream>>>(sums, C, dgamma, dbeta);
    SN_LAUNCH_CHECK();
  }
  return 0;
}

// Backward of y = relu(bn_train(x)) (residual_unit, resnet_mx_101_e2e.py:36-69): sniper_bn_act_bwd with act = 1.
int sniper_bn_relu_bwd(const void* x, long ldx, const void* dy, long lddy, const float* scale, const float* shift,
                       const float* mean, const float* invstd, double* sums, const void* add, long ldadd, void* dx,
                       long lddx, float* dgamma, float* dbeta, long M, int C, int dtype, void* stream) {
  return sniper_bn_act_bwd(x, ldx, dy, lddy, scale, shift, mean, invstd, sums, add, ldadd, dx, lddx, dgamma, dbeta, M, C,
                           1, dtype, stream);
}

int sniper_affine_relu_bwd(const float* x, long ldx, const float* dy, long lddy, const float* scale,
                           const float* shift, const float* add, long ldadd, float* dx, long lddx, long M, int C,
                           int relu, void* stream) {
  SN_TRY(check_shape("affine_relu_bwd", M, C, 4));
  SN_TRY(check_rows("affine_relu_bwd", "x", x, ldx, C, 4, 16));
  SN_TRY(check_rows("affine_relu_bwd", "dy", dy, lddy, C, 4, 16));
  SN_TRY(check_rows("affine_relu_bwd", "dx", dx, lddx, C, 4, 16));
  if (add) SN_TRY(check_rows("affine_relu_bwd", "add", add, ldadd, C, 4, 16));
  SN_TRY(check_chan("affine_relu_bwd", "scale", scale));
  SN_TRY(check_chan("affine_relu_bwd", "shift", shift));
  // RowSplit's division path (C/4 not a power of two) splits the flat vector index in 32 bits
  SN_CHECK(M * (C / 4) < (1L << 32), "affine_relu_bwd: M * C/4 must be below 2^32");
  if (M == 0) return 0;
  affine_relu_bwd_kernel<<<ew_grid(M * (C / 4)), kTPB, 0, (cudaStream_t)stream>>>(x, ldx, dy, lddy, scale, shift, add,
                                                                                 ldadd, dx, lddx, M, C, relu);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_relu_bwd(const void* y, long ldy, const void* dy, long lddy, void* dx, long lddx, long M, int C, int dtype,
                    void* stream) {
  SN_TRY(check_dtype("relu_bwd", dtype));
  SN_TRY(check_shape("relu_bwd", M, C, 4));
  const int bytes = dtype == 0 ? 16 : 8;      // 4 channels per access in either storage type
  SN_TRY(check_rows("relu_bwd", "y", y, ldy, C, 4, bytes));
  SN_TRY(check_rows("relu_bwd", "dy", dy, lddy, C, 4, bytes));
  SN_TRY(check_rows("relu_bwd", "dx", dx, lddx, C, 4, bytes));
  // RowSplit's division path (C/4 not a power of two) splits the flat vector index in 32 bits
  SN_CHECK(M * (C / 4) < (1L << 32), "relu_bwd: M * C/4 must be below 2^32");
  if (M == 0) return 0;
  if (dtype == 0)
    relu_bwd_kernel<float><<<ew_grid(M * (C / 4)), kTPB, 0, (cudaStream_t)stream>>>(
        static_cast<const float*>(y), ldy, static_cast<const float*>(dy), lddy, static_cast<float*>(dx), lddx, M, C);
  else
    relu_bwd_kernel<bf16><<<ew_grid(M * (C / 4)), kTPB, 0, (cudaStream_t)stream>>>(
        static_cast<const bf16*>(y), ldy, static_cast<const bf16*>(dy), lddy, static_cast<bf16*>(dx), lddx, M, C);
  SN_LAUNCH_CHECK();
  return 0;
}

// y[M,C] (ldy) = cast(x[M,C] (ldx)); dtypes 0 = fp32, 1 = bf16.
int sniper_cast_rows(const void* x, long ldx, int x_dtype, void* y, long ldy, int y_dtype, long M, int C, void* stream) {
  SN_CHECK((x_dtype | y_dtype | 1) == 1, "cast_rows: dtypes must be 0 (fp32) or 1 (bf16)");
  SN_TRY(check_shape("cast_rows", M, C, 4));
  SN_TRY(check_rows("cast_rows", "x", x, ldx, C, 4, x_dtype == 0 ? 16 : 8));
  SN_TRY(check_rows("cast_rows", "y", y, ldy, C, 4, y_dtype == 0 ? 16 : 8));
  if (M == 0) return 0;
  const int g = ew_grid(M * (C / 4));
  cudaStream_t st = (cudaStream_t)stream;
  if (x_dtype == 0 && y_dtype == 0)
    cast_rows_kernel<float, float><<<g, kTPB, 0, st>>>(static_cast<const float*>(x), ldx, static_cast<float*>(y), ldy, M, C);
  else if (x_dtype == 0)
    cast_rows_kernel<float, bf16><<<g, kTPB, 0, st>>>(static_cast<const float*>(x), ldx, static_cast<bf16*>(y), ldy, M, C);
  else if (y_dtype == 0)
    cast_rows_kernel<bf16, float><<<g, kTPB, 0, st>>>(static_cast<const bf16*>(x), ldx, static_cast<float*>(y), ldy, M, C);
  else
    cast_rows_kernel<bf16, bf16><<<g, kTPB, 0, st>>>(static_cast<const bf16*>(x), ldx, static_cast<bf16*>(y), ldy, M, C);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_maxpool3x3s2_nhwc(const void* x, void* y, int NB, int H, int W, int C, int dtype, void* stream) {
  SN_TRY(check_dtype("maxpool", dtype));
  SN_CHECK(NB >= 0 && H > 0 && W > 0, "maxpool: NB (%d) must not be negative, H (%d) and W (%d) must be positive", NB, H, W);
  SN_TRY(check_shape("maxpool", NB, C, 4));
  SN_TRY(check_rows("maxpool", "x", x, C, C, 4, dtype == 0 ? 16 : 8));
  SN_TRY(check_rows("maxpool", "y", y, C, C, 4, dtype == 0 ? 16 : 8));
  if (NB == 0) return 0;
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const int g = ew_grid((long)NB * Ho * Wo * (C / 4));
  if (dtype == 0)
    maxpool3x3s2_kernel<float><<<g, kTPB, 0, (cudaStream_t)stream>>>(static_cast<const float*>(x), static_cast<float*>(y),
                                                                      NB, H, W, C, Ho, Wo);
  else
    maxpool3x3s2_kernel<bf16><<<g, kTPB, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(x), static_cast<bf16*>(y),
                                                                     NB, H, W, C, Ho, Wo);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_stem_conv(const float* x_nchw, const float* w /*[64,7,7,3]*/, const float* in_scale, const float* in_shift,
                     const float* out_scale, const float* out_shift, void* y_nhwc, int NB, int H, int W,
                     int out_dtype, void* stream) {
  SN_CHECK(out_dtype == 0 || out_dtype == 1, "stem_conv: out_dtype must be 0 (fp32) or 1 (bf16)");
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  dim3 grid(sn::div_up(Wo, kStemTW), sn::div_up(Ho, kStemTH), NB);
  if (out_dtype == 0)
    stem_conv_kernel<float><<<grid, 128, 0, (cudaStream_t)stream>>>(x_nchw, w, in_scale, in_shift, out_scale, out_shift,
                                                                    static_cast<float*>(y_nhwc), NB, H, W, Ho, Wo);
  else   // the reference casts to fp16 right after conv0 (resnet_mx_101_e2e.py:405-406); bn0 + relu ride in the same pass
    stem_conv_kernel<bf16><<<grid, 128, 0, (cudaStream_t)stream>>>(x_nchw, w, in_scale, in_shift, out_scale, out_shift,
                                                                   static_cast<bf16*>(y_nhwc), NB, H, W, Ho, Wo);
  SN_LAUNCH_CHECK();
  return 0;
}

// col [NB*Ho*Wo, Kp] (fp32: Kp a multiple of 32 >= 147; bf16: a multiple of 64) = im2col of bn_data(x) for conv0;
// feed it to sniper_gemm_nt with the [64, Kp] weight rows ((kh, kw, c)-major, zero-padded) and bn0 + ReLU as epilogue.
int sniper_stem_im2col(const float* x_nchw, const float* in_scale, const float* in_shift, void* col, int NB, int H,
                       int W, int Kp, int dtype, void* stream) {
  SN_CHECK(dtype == 0 || dtype == 1, "stem_im2col: dtype must be 0 (fp32) or 1 (bf16)");
  SN_CHECK(Kp >= 148 && Kp % (dtype == 0 ? 4 : 8) == 0 && ((uintptr_t)col & 15) == 0,
           "stem_im2col: Kp must be >= 148 and a multiple of 4 (fp32) / 8 (bf16), col 16-byte aligned");
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  dim3 grid(sn::div_up(Wo, kStemCols), Ho, NB);
  if (dtype == 0)
    stem_im2col_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(x_nchw, in_scale, in_shift,
                                                                      static_cast<float*>(col), H, W, Ho, Wo, Kp);
  else
    stem_im2col_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>(x_nchw, in_scale, in_shift,
                                                                     static_cast<bf16*>(col), H, W, Ho, Wo, Kp);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_weight_transpose(const float* w, float* wt, int Cout, int T, int Cin, int Tsel, const int* sel_dev,
                            void* stream) {
  dim3 grid(sn::div_up(Cin, 32), sn::div_up(Cout, 32), Tsel), block(32, 8);
  weight_transpose_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(w, wt, Cout, T, Cin, Tsel, sel_dev);
  SN_LAUNCH_CHECK();
  return 0;
}

// jobs_dev: device array of njobs x 9 int64 {w, wt, sel_dev, Cout, T, Cin, Tsel, block0, wt_is_bf16} with block0 the
// running sum of ceil(Cin/32) * ceil(Cout/32) * Tsel; total_blocks = that sum over all jobs.
int sniper_weight_transpose_batched(const void* jobs_dev, int njobs, int total_blocks, void* stream) {
  if (njobs <= 0 || total_blocks <= 0) return 0;
  weight_transpose_batched_kernel<<<total_blocks, dim3(32, 8), 0, (cudaStream_t)stream>>>(
      static_cast<const long long*>(jobs_dev), njobs);
  SN_LAUNCH_CHECK();
  return 0;
}

// Second half of sniper_bn_relu_bwd for callers that defer it (defer_param_grad != 0 there): jobs_dev = njobs x 5
// int64 {sums, dgamma, dbeta, C, fwd_sums}.  dgamma += s2, dbeta += s1, sums zeroed, fwd_sums (if not 0) zeroed.
int sniper_bn_param_grad_batched(const void* jobs_dev, int njobs, void* stream) {
  if (njobs <= 0) return 0;
  bn_param_grad_batched_kernel<<<njobs, 256, 0, (cudaStream_t)stream>>>(static_cast<const long long*>(jobs_dev));
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_colsum(const float* x, long ldx, long M, int C, float* out_accum, void* stream) {
  dim3 grid(sn::div_up(C, 32)), block(32, 32);
  colsum_plain_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, ldx, M, C, out_accum);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_sgd_mom(float* w, float* mom, const float* g, long n, float lr, float wd, float momentum, float rescale,
                   void* stream) {
  SN_CHECK(n >= 0, "sgd_mom: n (%ld) must not be negative", n);
  SN_CHECK(w && mom && g, "sgd_mom: w / mom / g must not be null");
  SN_CHECK((((uintptr_t)w | (uintptr_t)mom | (uintptr_t)g) & 15) == 0, "sgd_mom: w / mom / g must be 16-byte aligned");
  if (n == 0) return 0;
  sgd_mom_kernel<<<ew_grid(n / 4 + 1), kTPB, 0, (cudaStream_t)stream>>>(w, mom, g, n, lr, wd, momentum, rescale);
  SN_LAUNCH_CHECK();
  return 0;
}

// hyper: device float[2] = {lr, wd}.  w_bf16: optional bf16 copy of the updated weights (8-byte aligned).
int sniper_sgd_mom_dev(float* w, float* mom, const float* g, long n, const float* hyper, float lr_mult, float wd_mult,
                       float momentum, float rescale, void* w_bf16, void* stream) {
  SN_CHECK(n >= 0, "sgd_mom_dev: n (%ld) must not be negative", n);
  SN_CHECK(w && mom && g, "sgd_mom_dev: w / mom / g must not be null");
  SN_CHECK((((uintptr_t)w | (uintptr_t)mom | (uintptr_t)g) & 15) == 0, "sgd_mom_dev: w / mom / g must be 16-byte aligned");
  SN_CHECK(hyper != nullptr && ((uintptr_t)hyper & 3) == 0, "sgd_mom_dev: hyper (device {lr, wd}) is required");
  SN_CHECK(((uintptr_t)w_bf16 & 7) == 0, "sgd_mom_dev: w_bf16 must be 8-byte aligned");
  if (n == 0) return 0;
  sgd_mom_dev_kernel<<<ew_grid(n / 4 + 1), kTPB, 0, (cudaStream_t)stream>>>(
      w, mom, g, n, hyper, lr_mult, wd_mult, momentum, rescale, static_cast<__nv_bfloat16*>(w_bf16));
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
