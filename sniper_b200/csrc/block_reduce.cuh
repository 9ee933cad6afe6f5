// Warp and block collectives shared by the bit-exact evaluation kernels.  They only add, compare and take maxima, so
// they add no multiply-add to the -fmad=false translation units that include them.
//
// The block helpers take the block's warp count kWarps (blockDim.x == 32 * kWarps), must be reached by every thread of
// the block, and give every thread the result.  Each one puts a barrier between the last read of its shared scratch
// `sh` (kWarps elements) and the next write, so consecutive calls can share one scratch array.
#pragma once
#include <cuda_runtime.h>

namespace {

__device__ __forceinline__ int2 operator+(int2 a, int2 b) { return make_int2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ int3 operator+(int3 a, int3 b) { return make_int3(a.x + b.x, a.y + b.y, a.z + b.z); }

__device__ __forceinline__ int shfl_up(int v, int o) { return __shfl_up_sync(~0u, v, o); }
__device__ __forceinline__ int2 shfl_up(int2 v, int o) {
  return make_int2(__shfl_up_sync(~0u, v.x, o), __shfl_up_sync(~0u, v.y, o));
}
__device__ __forceinline__ int3 shfl_up(int3 v, int o) {
  return make_int3(__shfl_up_sync(~0u, v.x, o), __shfl_up_sync(~0u, v.y, o), __shfl_up_sync(~0u, v.z, o));
}

// The block's sum: a shfl_down tree inside each warp, then the warp partials added in warp order from T(0).  For a
// floating-point T that order is part of the result.
template <typename T, int kWarps>
__device__ __forceinline__ T block_sum(T v, T* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(~0u, v, o);
  __syncthreads();                               // sh of an earlier call has been read
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  T s = 0;
  for (int w = 0; w < kWarps; ++w) s += sh[w];
  return s;
}

// Inclusive block scan of int / int2 / int3 counts; *total gets the block's sum.
template <typename V, int kWarps>
__device__ V block_inclusive_scan(V v, V* sh, V* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const V n = shfl_up(v, o);
    if (lane >= o) v = v + n;
  }
  if (lane == 31) sh[warp] = v;
  __syncthreads();
  V before{}, all{};
  for (int w = 0; w < kWarps; ++w) {
    if (w < warp) before = before + sh[w];
    all = all + sh[w];
  }
  __syncthreads();
  *total = all;
  return v + before;
}

// Inclusive suffix max over the block: the maximum of v over this thread and every later one (fmax: a NaN is skipped).
template <int kWarps>
__device__ double block_suffix_max(double v, double* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const double n = __shfl_down_sync(~0u, v, o);
    if (lane + o < 32) v = fmax(v, n);
  }
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  for (int w = warp + 1; w < kWarps; ++w) v = fmax(v, sh[w]);
  __syncthreads();
  return v;
}

// The arg-max order: (v, i) beats (bv, bi) when its value is larger, or equal with a lower index.
template <typename T>
__device__ __forceinline__ bool argmax_beats(T v, int i, T bv, int bi) {
  return v > bv || (v == bv && i < bi);
}

// (v, idx) of every lane becomes the warp's best pair in argmax_beats order.
template <typename T>
__device__ __forceinline__ void warp_argmax(T& v, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const T ov = __shfl_xor_sync(~0u, v, o);
    const int oi = __shfl_xor_sync(~0u, idx, o);
    if (argmax_beats(ov, oi, v, idx)) { v = ov; idx = oi; }
  }
}

}  // namespace
