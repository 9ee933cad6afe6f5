// Depthwise 3x3 convolution (forward, data gradient, weight gradient), the first-layer im2col and the shortcut add of
// the MobileNetV2 SNIPER backbone (BASELINE config 4; symbols/faster/mobilenetv2_e2e.py:27-91, 204-212).
//
// These layers carry 9 MACs per loaded element: they are HBM / L1 bound, not tensor-core work, so they are plain
// coalesced NHWC kernels (4 channels per thread, consecutive threads on consecutive channel vectors of a pixel, fp32
// accumulation); the 1x1 expand / project convolutions around them run on the wgmma kernel (gemm_tc.cu).  The
// per-thread bodies live in depthwise_core.cuh so that the CPU test can execute the same index arithmetic.
// Reference kernels replaced: src/operator/nn/depthwise_convolution-inl.h (DepthwiseConvolutionOp::Forward / Backward,
// depthwise_convolution_tf.cuh), elemwise_add, im2col of nn/convolution-inl.h for the 3-channel first layer.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "depthwise_core.cuh"

namespace {

typedef __nv_bfloat16 bf16;
constexpr int kTPB = 256;

template <typename T, int S, int PW, bool FLIP>
__global__ void __launch_bounds__(kTPB) dw_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w,
                                                       T* __restrict__ y, dwc::Params p, long nthreads) {
  const long tid = (long)blockIdx.x * kTPB + threadIdx.x;
  if (tid < nthreads) dwc::fwd<T, S, PW, FLIP>(tid, x, w, y, p);
}

// shared-memory tiled forward (bf16, C % 64 == 0); grid = (tiles, C / 64)
template <int S, bool FLIP>
__global__ void __launch_bounds__(kTPB) dw_fwd_tiled_kernel(const bf16* __restrict__ x, const float* __restrict__ w,
                                                             bf16* __restrict__ y, dwc::Params p) {
  __shared__ __align__(16) bf16 tile[dwc::Tile<S>::ELEMS];
  const dwc::TileId t = dwc::tile_id<S>((long)blockIdx.x, (int)blockIdx.y, p);
  dwc::tile_stage<S>((int)threadIdx.x, kTPB, t, x, tile, p);
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  dwc::tile_compute<S, FLIP>((int)threadIdx.x, kTPB, t, tile, w, y, p);
}

template <int S, bool FLIP>
int launch_fwd_tiled(const void* x, const float* w, void* y, const dwc::Params& p, cudaStream_t st) {
  const long blocks = dwc::tile_blocks<S>(p);
  SN_CHECK(blocks < (1L << 31), "depthwise3x3: too many tiles");
  dw_fwd_tiled_kernel<S, FLIP><<<dim3((unsigned)blocks, (unsigned)(p.C / 64), 1), kTPB, 0, st>>>(
      static_cast<const bf16*>(x), w, static_cast<bf16*>(y), p);
  return 0;
}

// the tiled kernel takes bf16 with whole 64-channel groups; fp32 and other shapes run the register-window kernels.
// cp.async copies 16 bytes from x + pixel * ld_in + 64k + 8j: the base and the pixel rows must both be 16-byte aligned
// (a channel slice such as big[..., 4:68] of a bf16 map is only 8-byte aligned; it runs the register kernel, same bits)
bool use_tiled(int dtype, int C, long ld_in, const void* in) {
  return dtype == 1 && C % 64 == 0 && ld_in % 8 == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0;
}

template <typename T>
__global__ void __launch_bounds__(kTPB) dw_dgrad_s2_kernel(const T* __restrict__ dy, const float* __restrict__ w,
                                                            T* __restrict__ dx, dwc::Params p, long nthreads) {
  const long tid = (long)blockIdx.x * kTPB + threadIdx.x;
  if (tid < nthreads) dwc::dgrad_s2<T>(tid, dy, w, dx, p);
}

// block = 32 x 8 threads; a warp row covers LC channel vectors x 32/LC strips (depthwise_core.cuh).  Partial sums of
// the strip lanes are combined in shared memory, then each block stores its [9 x its channels] partial to row blockIdx.x
// of a slab part[gridDim.x][9][C] in the caller's workspace; dw_wgrad_reduce_kernel adds the rows in a fixed order.  No
// atomics: the result does not depend on the order in which blocks run, so two launches give the same bits.  The grid
// is ONE wave of resident blocks (occupancy API), capped so that the slab fits the workspace; each thread loops over
// its strips.
constexpr int kWgTY = 8;
template <typename T, int S, int PW>
__global__ void __launch_bounds__(32 * kWgTY) dw_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                               float* __restrict__ part, dwc::Params p) {
  __shared__ float red[kWgTY][32][37];
  const int tx = threadIdx.x, ty = threadIdx.y;
  float acc[9][4];
  dwc::wgrad_partial<T, S, PW>((int)blockIdx.x, (int)blockIdx.y, tx, ty, kWgTY, (int)gridDim.x, x, dy, p, acc);
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int k = 0; k < 4; ++k) red[ty][tx][t * 4 + k] = acc[t][k];
  __syncthreads();
  const int LC = dwc::wgrad_lc(p.C), PPW = 32 / LC;
  float* row = part + (long)blockIdx.x * 9 * p.C;
  for (int i = ty * 32 + tx; i < LC * 36; i += 32 * kWgTY) {
    const int lane = i / 36, e = i - lane * 36;
    float s = 0.f;
    for (int ps = 0; ps < PPW; ++ps)
#pragma unroll
      for (int j = 0; j < kWgTY; ++j) s += red[j][ps * LC + lane][e];
    const int c = (((int)blockIdx.y * LC + lane) << 2) + (e & 3);
    if (c < p.C) row[(e >> 2) * p.C + c] = s;
  }
}

// dw[o] += sum over b of part[b][o], o < n = 9 C, in a fixed order: thread row ty sums the contiguous block range
// [gx*ty/8, gx*(ty+1)/8) in increasing b, then row 0 adds the 8 row sums in increasing ty and adds the total to dw
// once.  Block = 32 outputs x 8 rows; the 32 lanes of a warp read 32 consecutive floats of a slab row.
constexpr int kRdTY = 8;
__global__ void __launch_bounds__(32 * kRdTY) dw_wgrad_reduce_kernel(const float* __restrict__ part, int gx, int n,
                                                                      float* __restrict__ dw) {
  __shared__ float red[kRdTY][32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int o = (int)blockIdx.x * 32 + tx;
  float s = 0.f;
  if (o < n) {
    const int b0 = gx * ty / kRdTY, b1 = gx * (ty + 1) / kRdTY;
#pragma unroll 8
    for (int b = b0; b < b1; ++b) s += part[(long)b * n + o];
  }
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && o < n) {
    float t = red[0][tx];
#pragma unroll
    for (int j = 1; j < kRdTY; ++j) t += red[j][tx];
    dw[o] += t;
  }
}

template <typename K>
int wgrad_blocks_per_sm(K kernel) {
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, 32 * kWgTY, 0) != cudaSuccess || n < 1) n = 2;
  return n;
}

template <typename T>
__global__ void __launch_bounds__(kTPB) im2col3x3s2_kernel(const float* __restrict__ x, T* __restrict__ col, int NB,
                                                            int H, int W, int Ho, int Wo, int Kp, long nthreads) {
  const long tid = (long)blockIdx.x * kTPB + threadIdx.x;
  if (tid < nthreads) dwc::im2col3x3s2<T, 3>(tid, x, col, NB, H, W, Ho, Wo, Kp);
}

template <typename T>
__global__ void __launch_bounds__(kTPB) add_rows_kernel(const T* a, long lda, const T* b,
                                                         long ldb, T* o, long ldo, long M, int C,
                                                         long nthreads) {
  const long tid = (long)blockIdx.x * kTPB + threadIdx.x;
  if (tid < nthreads) dwc::add_rows<T>(tid, a, lda, b, ldb, o, ldo, M, C);
}

int fill_params(dwc::Params& p, int NB, int H, int W, int C, int stride, long ld_in, long ld_out, int dtype,
                const char* who) {
  SN_CHECK(dtype == 0 || dtype == 1, "%s: dtype must be 0 (fp32) or 1 (bf16)", who);
  SN_CHECK(stride == 1 || stride == 2, "%s: stride must be 1 or 2", who);
  SN_CHECK(NB > 0 && H > 0 && W > 0, "%s: NB (%d), H (%d) and W (%d) must be positive", who, NB, H, W);
  SN_CHECK(C > 0 && C % 4 == 0, "%s: C (%d) must be a positive multiple of 4", who, C);
  SN_CHECK(ld_in >= C && ld_out >= C && ld_in % 4 == 0 && ld_out % 4 == 0, "%s: pixel strides must be multiples of 4 and >= C",
           who);
  p.NB = NB; p.H = H; p.W = W; p.C = C; p.stride = stride;
  p.Ho = (H - 1) / stride + 1;          // (H + 2*1 - 3) / stride + 1
  p.Wo = (W - 1) / stride + 1;
  p.ldx = ld_in; p.ldy = ld_out;
  return 0;
}

// The pointers of a forward / data-gradient launch: the map operands are read and written as 4-channel vectors (float4
// in fp32, 8 bytes in bf16) and the weights as float4, so each must be non-null and aligned to its vector.
int check_ptrs(const void* in, const char* in_name, const float* w, const void* out, const char* out_name, int dtype,
               const char* who) {
  const uintptr_t vec = dtype == 0 ? 16 : 8;
  SN_CHECK(in != nullptr, "%s: %s must not be null", who, in_name);
  SN_CHECK(reinterpret_cast<uintptr_t>(in) % vec == 0, "%s: %s must be %d-byte aligned", who, in_name, (int)vec);
  SN_CHECK(w != nullptr, "%s: w must not be null", who);
  SN_CHECK((reinterpret_cast<uintptr_t>(w) & 15) == 0, "%s: w must be 16-byte aligned", who);
  SN_CHECK(out != nullptr, "%s: %s must not be null", who, out_name);
  SN_CHECK(reinterpret_cast<uintptr_t>(out) % vec == 0, "%s: %s must be %d-byte aligned", who, out_name, (int)vec);
  return 0;
}

inline unsigned blocks_for(long nthreads) { return (unsigned)((nthreads + kTPB - 1) / kTPB); }

}  // namespace

extern "C" {

// y[NB,Ho,Wo,C] = depthwise3x3(x[NB,H,W,C], w[9,C]), pad 1, stride 1 | 2.  ldx / ldy: elements between pixels.
// Alignment: x and y 16-byte (fp32) / 8-byte (bf16) aligned, w [9,C] fp32 16-byte aligned; refused otherwise.  bf16
// with C % 64 == 0, ldx % 8 == 0 and a 16-byte aligned x runs the shared-memory tiled kernel, anything else the
// register kernel; both give the same bits.
int sniper_depthwise3x3_fwd(const void* x, long ldx, const float* w, void* y, long ldy, int NB, int H, int W, int C,
                            int stride, int dtype, void* stream) {
  dwc::Params p;
  if (fill_params(p, NB, H, W, C, stride, ldx, ldy, dtype, "depthwise3x3_fwd")) return -1;
  if (check_ptrs(x, "x", w, y, "y", dtype, "depthwise3x3_fwd")) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tiled(dtype, C, ldx, x)) {
    if (stride == 1 ? launch_fwd_tiled<1, false>(x, w, y, p, st) : launch_fwd_tiled<2, false>(x, w, y, p, st)) return -1;
    SN_LAUNCH_CHECK();
    return 0;
  }
#define DW_FWD(T, S, PW)                                                                                       \
  do {                                                                                                         \
    const long nt = dwc::fwd_threads<S, PW>(p);                                                                \
    dw_fwd_kernel<T, S, PW, false><<<blocks_for(nt), kTPB, 0, st>>>(static_cast<const T*>(x), w, static_cast<T*>(y), p, nt); \
  } while (0)
  if (dtype == 0) { if (stride == 1) DW_FWD(float, 1, 4); else DW_FWD(float, 2, 2); }
  else            { if (stride == 1) DW_FWD(bf16, 1, 4);  else DW_FWD(bf16, 2, 2); }
#undef DW_FWD
  SN_LAUNCH_CHECK();
  return 0;
}

// dx[NB,H,W,C] = depthwise3x3^T(dy[NB,Ho,Wo,C], w[9,C]); H, W, stride describe the FORWARD convolution.
// stride 1: the forward kernel on dy with the flipped filter; stride 2: one thread per dy pixel -> 2 x 2 block of dx.
// Alignment as for the forward (dy in the place of x, dx in the place of y); the stride-1 gradient picks the tiled
// kernel by the forward's rule applied to dy.
int sniper_depthwise3x3_dgrad(const void* dy, long lddy, const float* w, void* dx, long lddx, int NB, int H, int W,
                              int C, int stride, int dtype, void* stream) {
  dwc::Params p;
  cudaStream_t st = (cudaStream_t)stream;
  if (stride == 1) {
    if (fill_params(p, NB, H, W, C, 1, lddy, lddx, dtype, "depthwise3x3_dgrad")) return -1;   // "input" = dy, "output" = dx
    if (check_ptrs(dy, "dy", w, dx, "dx", dtype, "depthwise3x3_dgrad")) return -1;
    if (use_tiled(dtype, C, lddy, dy)) {
      if (launch_fwd_tiled<1, true>(dy, w, dx, p, st)) return -1;
      SN_LAUNCH_CHECK();
      return 0;
    }
    const long nt = dwc::fwd_threads<1, 4>(p);
    if (dtype == 0)
      dw_fwd_kernel<float, 1, 4, true><<<blocks_for(nt), kTPB, 0, st>>>(static_cast<const float*>(dy), w, static_cast<float*>(dx), p, nt);
    else
      dw_fwd_kernel<bf16, 1, 4, true><<<blocks_for(nt), kTPB, 0, st>>>(static_cast<const bf16*>(dy), w, static_cast<bf16*>(dx), p, nt);
  } else {
    if (fill_params(p, NB, H, W, C, stride, lddx, lddy, dtype, "depthwise3x3_dgrad")) return -1;
    if (check_ptrs(dy, "dy", w, dx, "dx", dtype, "depthwise3x3_dgrad")) return -1;
    const long nt = dwc::dgrad_s2_threads(p);
    if (dtype == 0)
      dw_dgrad_s2_kernel<float><<<blocks_for(nt), kTPB, 0, st>>>(static_cast<const float*>(dy), w, static_cast<float*>(dx), p, nt);
    else
      dw_dgrad_s2_kernel<bf16><<<blocks_for(nt), kTPB, 0, st>>>(static_cast<const bf16*>(dy), w, static_cast<bf16*>(dx), p, nt);
  }
  SN_LAUNCH_CHECK();
  return 0;
}

// dw[9,C] += sum over pixels of dy * shifted x (fp32; one addition into the existing value: zero dw for kWriteTo).
// The block partials go through the workspace registered for (current device, stream) and are added in a fixed
// order, so every launch gives the same bits.
int sniper_depthwise3x3_wgrad(const void* x, long ldx, const void* dy, long lddy, float* dw, int NB, int H, int W,
                              int C, int stride, int dtype, void* stream) {
  SN_CHECK(dtype == 0 || dtype == 1, "depthwise3x3_wgrad: dtype (%d) must be 0 (fp32) or 1 (bf16)", dtype);
  SN_CHECK(stride == 1 || stride == 2, "depthwise3x3_wgrad: stride (%d) must be 1 or 2", stride);
  SN_CHECK(NB > 0 && H > 0 && W > 0, "depthwise3x3_wgrad: NB (%d), H (%d) and W (%d) must be positive", NB, H, W);
  SN_CHECK(C > 0 && C % 4 == 0, "depthwise3x3_wgrad: C (%d) must be a positive multiple of 4", C);
  SN_CHECK(ldx >= C && ldx % 4 == 0, "depthwise3x3_wgrad: ldx (%ld) must be a multiple of 4 and >= C (%d)", ldx, C);
  SN_CHECK(lddy >= C && lddy % 4 == 0, "depthwise3x3_wgrad: lddy (%ld) must be a multiple of 4 and >= C (%d)", lddy, C);
  dwc::Params p;
  if (fill_params(p, NB, H, W, C, stride, ldx, lddy, dtype, "depthwise3x3_wgrad")) return -1;
  SN_CHECK(x != nullptr, "depthwise3x3_wgrad: x must not be null");
  SN_CHECK(dy != nullptr, "depthwise3x3_wgrad: dy must not be null");
  const uintptr_t vec = dtype == 0 ? 16 : 8;          // x and dy are read as 4-channel vectors
  SN_CHECK(reinterpret_cast<uintptr_t>(x) % vec == 0, "depthwise3x3_wgrad: x must be %d-byte aligned", (int)vec);
  SN_CHECK(reinterpret_cast<uintptr_t>(dy) % vec == 0, "depthwise3x3_wgrad: dy must be %d-byte aligned", (int)vec);
  SN_CHECK(dw != nullptr, "depthwise3x3_wgrad: dw must not be null");
  SN_CHECK((reinterpret_cast<uintptr_t>(dw) & 3) == 0, "depthwise3x3_wgrad: dw must be 4-byte aligned");
  SN_CHECK(9L * C <= sn::kWgSlabFloats, "depthwise3x3_wgrad: C (%d) exceeds the workspace's %ld channels", C,
           sn::kWgSlabFloats / 9);
  sn::StreamWs ws;
  if (sn::stream_workspace(stream, &ws, "depthwise3x3_wgrad")) return -1;
  float* part = ws.slab;
  cudaStream_t st = (cudaStream_t)stream;
  const int LC = dwc::wgrad_lc(C), PL = kWgTY * (32 / LC);
  const int gy = sn::div_up(C >> 2, LC);
  const dim3 block(32, kWgTY, 1);
  long gx = 1;
#define DW_WG(T, S, PW)                                                                                              \
  do {                                                                                                               \
    const long strips = (long)NB * p.Ho * ((p.Wo + PW - 1) / PW);                                                    \
    gx = ((long)sn::kNumSMs * wgrad_blocks_per_sm(dw_wgrad_kernel<T, S, PW>) + gy - 1) / gy;   /* one wave */         \
    const long gx_max = (strips + PL - 1) / PL;                                                                      \
    if (gx > gx_max) gx = gx_max;                                                                                    \
    if (gx > sn::kWgSlabFloats / (9L * C)) gx = sn::kWgSlabFloats / (9L * C);                                        \
    if (gx < 1) gx = 1;                                                                                              \
    dw_wgrad_kernel<T, S, PW><<<dim3((unsigned)gx, (unsigned)gy, 1), block, 0, st>>>(                                \
        static_cast<const T*>(x), static_cast<const T*>(dy), part, p);                                              \
  } while (0)
  if (dtype == 0) { if (stride == 1) DW_WG(float, 1, 4); else DW_WG(float, 2, 2); }
  else            { if (stride == 1) DW_WG(bf16, 1, 4);  else DW_WG(bf16, 2, 2); }
#undef DW_WG
  const int n = 9 * C;
  dw_wgrad_reduce_kernel<<<(unsigned)sn::div_up(n, 32), dim3(32, kRdTY, 1), 0, st>>>(part, (int)gx, n, dw);
  SN_LAUNCH_CHECK();
  return 0;
}

// col[NB*Ho*Wo, Kp] = im2col of a 3x3 / stride 2 / pad 1 convolution over an fp32 NCHW image with 3 channels, K order
// (kh, kw, ci), zero-padded to Kp (a multiple of the wgmma kernel's K atom: 32 fp32 / 64 bf16 elements).  col must be
// 16-byte (fp32) / 8-byte (bf16) aligned: each thread stores 4 consecutive columns.
int sniper_im2col3x3s2_nchw(const float* x, void* col, int NB, int H, int W, int Cin, int Kp, int dtype, void* stream) {
  SN_CHECK(dtype == 0 || dtype == 1, "im2col3x3s2: dtype must be 0 (fp32) or 1 (bf16)");
  SN_CHECK(Cin == 3, "im2col3x3s2: built for the 3-channel first layer (Cin = %d)", Cin);
  SN_CHECK(Kp >= 27 && Kp % 4 == 0, "im2col3x3s2: Kp (%d) must be a multiple of 4 and >= 27", Kp);
  SN_CHECK(NB > 0 && H > 0 && W > 0, "im2col3x3s2: empty input");
  SN_CHECK(x != nullptr, "im2col3x3s2: x must not be null");
  SN_CHECK((reinterpret_cast<uintptr_t>(x) & 3) == 0, "im2col3x3s2: x must be 4-byte aligned");
  SN_CHECK(col != nullptr, "im2col3x3s2: col must not be null");
  const uintptr_t vec = dtype == 0 ? 16 : 8;          // col is written as 4-column vectors
  SN_CHECK(reinterpret_cast<uintptr_t>(col) % vec == 0, "im2col3x3s2: col must be %d-byte aligned", (int)vec);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long nt = (long)NB * Ho * Wo * (Kp >> 2);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0)
    im2col3x3s2_kernel<float><<<blocks_for(nt), kTPB, 0, st>>>(x, static_cast<float*>(col), NB, H, W, Ho, Wo, Kp, nt);
  else
    im2col3x3s2_kernel<bf16><<<blocks_for(nt), kTPB, 0, st>>>(x, static_cast<bf16*>(col), NB, H, W, Ho, Wo, Kp, nt);
  SN_LAUNCH_CHECK();
  return 0;
}

// out[M,C] = a[M,C] + b[M,C] (row strides in elements; out may alias a or b).
int sniper_add_rows(const void* a, long lda, const void* b, long ldb, void* out, long ldo, long M, int C, int dtype,
                    void* stream) {
  SN_CHECK(dtype == 0 || dtype == 1, "add_rows: dtype must be 0 (fp32) or 1 (bf16)");
  SN_CHECK(M > 0 && C > 0 && C % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && ldo % 4 == 0,
           "add_rows: C and the row strides must be multiples of 4");
  const long nt = M * (C >> 2);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0)
    add_rows_kernel<float><<<blocks_for(nt), kTPB, 0, st>>>(static_cast<const float*>(a), lda, static_cast<const float*>(b),
                                                            ldb, static_cast<float*>(out), ldo, M, C, nt);
  else
    add_rows_kernel<bf16><<<blocks_for(nt), kTPB, 0, st>>>(static_cast<const bf16*>(a), lda, static_cast<const bf16*>(b),
                                                           ldb, static_cast<bf16*>(out), ldo, M, C, nt);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
