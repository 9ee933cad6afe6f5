// Deformable convolution (NHWC): bilinear-sampled im2col and its transposes; the contractions run on
// the wgmma GEMM (gemm_tc.cu), batched over the whole mini-batch instead of the reference's per-image loop.
//
// Replaces SNIPER-mxnet/src/operator/contrib/nn/deformable_im2col.cuh: deformable_im2col_gpu_kernel
// (:216-263, bilinear :78-113), deformable_col2im_gpu_kernel (:317-360, get_gradient_weight :117-158) and
// deformable_col2im_coord_gpu_kernel (:419-480, get_coordinate_weight :161-213), as driven by
// DeformableConvolutionOp::Forward/Backward (contrib/deformable_convolution-inl.h:111-168, 170-265).
//
// Layouts: x [NB,H,W,C]; offset [NB,Ho,Wo,OC] with channel dg*2*KK + 2*tap + {0:dh, 1:dw} (same channel
// meaning as the reference's NCHW offset tensor); col [NB*Ho*Wo, KK*C] tap-major, channel-minor, i.e. the
// K order of weights stored as [Cout, kh, kw, Cin].
// One warp = one (pixel, tap, 128-channel block): 32 lanes x float4.
#include "common.cuh"
#include <cuda_bf16.h>
#include <math.h>

namespace {

typedef __nv_bfloat16 bf16;

// x and col are fp32 or bf16 (template parameter T of the kernel; the mixed-precision backbone keeps activations and
// the im2col buffer in bf16); offsets, their gradient and the accumulated dx are always fp32.
struct DcArgs {
  const void* x;
  const float* offset;
  int NB, H, W, C, Ho, Wo, KH, KW, stride, dil, pad, dgroups, off_ld;
  void* col;         // fwd out / bwd in (dcol)
  float* dx;         // bwd out (accumulated into)
  float* doffset;    // bwd out [NB,Ho,Wo,off_ld] (written, each element owned by one warp)
  double* acc;       // bwd: zero-filled fp64 scratch shaped like dx (sniper_deform_col2im_fp64acc), or null
};

// acc -> dx: dx += (float)acc
__global__ void __launch_bounds__(256) add_f64_kernel(float* __restrict__ dst, const double* __restrict__ acc, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    dst[i] += (float)acc[i];
}

struct Sample {
  bool valid;
  int h_low, h_high, w_low, w_high;  // absolute
  float lh, lw;
};

// deformable_im2col.cuh:237-247 + :78-100: same arithmetic, relative coordinates as in the reference
__device__ __forceinline__ Sample make_sample(const DcArgs& p, int h_in, int w_in, int i, int j, float off_h, float off_w) {
  Sample s;
  const float h_im = (float)(h_in + i * p.dil) + off_h;
  const float w_im = (float)(w_in + j * p.dil) + off_w;
  s.valid = (h_im >= 0 && w_im >= 0 && h_im < p.H && w_im < p.W);
  float map_h = (float)(i * p.dil) + off_h;
  float map_w = (float)(j * p.dil) + off_w;
  const int cur_height = p.H - h_in, cur_width = p.W - w_in;
  int h_low = (int)floorf(map_h), w_low = (int)floorf(map_w), h_high, w_high;
  if (h_low >= cur_height - 1) { h_high = h_low = cur_height - 1; map_h = (float)h_low; } else { h_high = h_low + 1; }
  if (w_low >= cur_width - 1) { w_high = w_low = cur_width - 1; map_w = (float)w_low; } else { w_high = w_low + 1; }
  s.lh = map_h - h_low;
  s.lw = map_w - w_low;
  s.h_low = h_in + h_low; s.h_high = h_in + h_high; s.w_low = w_in + w_low; s.w_high = w_in + w_high;
  return s;
}

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld4(const bf16* p) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(bf16* p, float4 v) {
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&lo);
  u.y = *reinterpret_cast<const uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = u;
}

template <bool BWD, typename T>
__global__ void __launch_bounds__(256) deform_im2col_kernel(DcArgs p) {
  const int lane = threadIdx.x & 31;
  const int KK = p.KH * p.KW;
  const int cblocks = p.C / 128;
  const long nwarps_total = (long)p.NB * p.Ho * p.Wo * KK * cblocks;
  const int cpg = p.C / p.dgroups;  // channels per deformable group
  for (long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; wid < nwarps_total;
       wid += ((long)gridDim.x * blockDim.x) >> 5) {
    const int cb = (int)(wid % cblocks);
    long r = wid / cblocks;
    const int tap = (int)(r % KK);
    const long m = r / KK;
    const int wo = (int)(m % p.Wo);
    const int ho = (int)((m / p.Wo) % p.Ho);
    const int n = (int)(m / ((long)p.Wo * p.Ho));
    const int c = cb * 128 + lane * 4;
    const int dg = c / cpg;
    const int i = tap / p.KW, j = tap - i * p.KW;
    const float* offp = p.offset + m * p.off_ld + dg * 2 * KK + 2 * tap;
    const float off_h = __ldg(offp), off_w = __ldg(offp + 1);
    const int h_in = ho * p.stride - p.pad, w_in = wo * p.stride - p.pad;
    const Sample s = make_sample(p, h_in, w_in, i, j, off_h, off_w);
    T* colp = static_cast<T*>(p.col) + m * (long)KK * p.C + (long)tap * p.C + c;
    const T* xb = static_cast<const T*>(p.x) + (size_t)n * p.H * p.W * p.C + c;
    if (!BWD) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (s.valid) {
        const float hh = 1 - s.lh, hw = 1 - s.lw;
        const float w1 = hh * hw, w2 = hh * s.lw, w3 = s.lh * hw, w4 = s.lh * s.lw;
        const float4 v1 = ld4(xb + ((size_t)s.h_low * p.W + s.w_low) * p.C);
        const float4 v2 = ld4(xb + ((size_t)s.h_low * p.W + s.w_high) * p.C);
        const float4 v3 = ld4(xb + ((size_t)s.h_high * p.W + s.w_low) * p.C);
        const float4 v4 = ld4(xb + ((size_t)s.h_high * p.W + s.w_high) * p.C);
        v.x = w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
        v.y = w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
        v.z = w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
        v.w = w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
      }
      st4(colp, v);
    } else {
      float gh = 0.f, gw = 0.f;
      if (s.valid) {
        const float4 g = ld4(colp);
        const float hh = 1 - s.lh, hw = 1 - s.lw;
        const size_t o1 = ((size_t)s.h_low * p.W + s.w_low) * p.C, o2 = ((size_t)s.h_low * p.W + s.w_high) * p.C;
        const size_t o3 = ((size_t)s.h_high * p.W + s.w_low) * p.C, o4 = ((size_t)s.h_high * p.W + s.w_high) * p.C;
        float* db = p.dx + (size_t)n * p.H * p.W * p.C + c;
        const float w1 = hh * hw, w2 = hh * s.lw, w3 = s.lh * hw, w4 = s.lh * s.lw;
        if (p.acc) {
          // fp64 sums of exact fp64 products: practically independent of the order the warps arrive in
          double* ab = p.acc + (size_t)n * p.H * p.W * p.C + c;
          const size_t oo[4] = {o1, o2, o3, o4};
          const float ww[4] = {w1, w2, w3, w4};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (ww[q] == 0.f) continue;
            const double wq = (double)ww[q];
            atomicAdd(ab + oo[q], wq * g.x);
            atomicAdd(ab + oo[q] + 1, wq * g.y);
            atomicAdd(ab + oo[q] + 2, wq * g.z);
            atomicAdd(ab + oo[q] + 3, wq * g.w);
          }
        } else {
          atomicAdd(reinterpret_cast<float4*>(db + o1), make_float4(w1 * g.x, w1 * g.y, w1 * g.z, w1 * g.w));
          atomicAdd(reinterpret_cast<float4*>(db + o2), make_float4(w2 * g.x, w2 * g.y, w2 * g.z, w2 * g.w));
          atomicAdd(reinterpret_cast<float4*>(db + o3), make_float4(w3 * g.x, w3 * g.y, w3 * g.z, w3 * g.w));
          atomicAdd(reinterpret_cast<float4*>(db + o4), make_float4(w4 * g.x, w4 * g.y, w4 * g.z, w4 * g.w));
        }
        const float4 v1 = ld4(xb + o1), v2 = ld4(xb + o2), v3 = ld4(xb + o3), v4 = ld4(xb + o4);
        // d val / d h = hw*(v3 - v1) + lw*(v4 - v2);  d val / d w = hh*(v2 - v1) + lh*(v4 - v3)   (cuh:196-207)
        gh = g.x * (hw * (v3.x - v1.x) + s.lw * (v4.x - v2.x)) + g.y * (hw * (v3.y - v1.y) + s.lw * (v4.y - v2.y)) +
             g.z * (hw * (v3.z - v1.z) + s.lw * (v4.z - v2.z)) + g.w * (hw * (v3.w - v1.w) + s.lw * (v4.w - v2.w));
        gw = g.x * (hh * (v2.x - v1.x) + s.lh * (v4.x - v3.x)) + g.y * (hh * (v2.y - v1.y) + s.lh * (v4.y - v3.y)) +
             g.z * (hh * (v2.z - v1.z) + s.lh * (v4.z - v3.z)) + g.w * (hh * (v2.w - v1.w) + s.lh * (v4.w - v3.w));
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        gh += __shfl_xor_sync(0xffffffffu, gh, off);
        gw += __shfl_xor_sync(0xffffffffu, gw, off);
      }
      if (lane == 0) {
        float* dop = p.doffset + m * p.off_ld + dg * 2 * KK + 2 * tap;
        if (cpg == 128) {  // this warp is the only contributor
          dop[0] = gh;
          dop[1] = gw;
        } else {
          atomicAdd(dop, gh);
          atomicAdd(dop + 1, gw);
        }
      }
    }
  }
}

// floor((extent + 2 pad - dil (k - 1) - 1) / stride) + 1, or 0 when the dilated kernel does not fit once
long out_extent(int extent, int k, int stride, int dil, int pad) {
  const long span = (long)extent + 2L * pad - (long)dil * (k - 1) - 1;
  return span < 0 ? 0 : span / stride + 1;
}

// Every rule the kernels rely on, checked before any CUDA call: the warps read x and write col as whole 16-byte (fp32)
// or 8-byte (bf16) vectors of 4 channels, and the offsets as single floats.  `who` names the entry point.
int fill(DcArgs& a, const char* who, const void* x, const float* offset, int NB, int H, int W, int C, int KH, int KW,
         int stride, int dil, int pad, int dgroups, int off_ld, const void* col, int dtype) {
  SN_CHECK(dtype == 0 || dtype == 1, "%s: dtype must be 0 (fp32) or 1 (bf16)", who);
  SN_CHECK(NB >= 0 && H >= 0 && W >= 0, "%s: NB (%d), H (%d) and W (%d) must not be negative", who, NB, H, W);
  SN_CHECK(KH >= 1 && KW >= 1, "%s: KH (%d) and KW (%d) must be at least 1", who, KH, KW);
  SN_CHECK(stride >= 1, "%s: stride (%d) must be at least 1", who, stride);
  SN_CHECK(dil >= 1, "%s: dil (%d) must be at least 1", who, dil);
  SN_CHECK(pad >= 0, "%s: pad (%d) must not be negative", who, pad);
  SN_CHECK(C > 0 && C % 128 == 0, "%s: C (%d) must be a positive multiple of 128", who, C);
  SN_CHECK(dgroups > 0 && C % dgroups == 0 && (C / dgroups) % 128 == 0,
           "%s: channels per deformable group (C %d / dgroups %d) must be a multiple of 128", who, C, dgroups);
  SN_CHECK(off_ld >= dgroups * 2 * KH * KW, "%s: offset row stride off_ld (%d) is smaller than 2*dgroups*KH*KW (%d)",
           who, off_ld, dgroups * 2 * KH * KW);
  // a batch of empty maps would size the fp64-scratch reduction to nothing: only NB == 0 is an empty call
  SN_CHECK(NB == 0 || (H >= 1 && W >= 1), "%s: H (%d) and W (%d) must be at least 1 when NB (%d) > 0", who, H, W, NB);
  const long Ho = out_extent(H, KH, stride, dil, pad), Wo = out_extent(W, KW, stride, dil, pad);
  SN_CHECK(NB == 0 || (Ho >= 1 && Wo >= 1), "%s: the output map is empty (Ho %ld, Wo %ld)", who, Ho, Wo);
  SN_CHECK(x != nullptr && offset != nullptr && col != nullptr, "%s: x / offset / col must not be null", who);
  const uintptr_t vec = dtype == 0 ? 16 : 8;
  SN_CHECK(((uintptr_t)x & (vec - 1)) == 0, "%s: x must be %d-byte aligned", who, (int)vec);
  SN_CHECK(((uintptr_t)col & (vec - 1)) == 0, "%s: col must be %d-byte aligned", who, (int)vec);
  SN_CHECK(((uintptr_t)offset & 3) == 0, "%s: offset must be 4-byte aligned", who);
  a.x = x; a.offset = offset; a.NB = NB; a.H = H; a.W = W; a.C = C; a.KH = KH; a.KW = KW; a.stride = stride;
  a.dil = dil; a.pad = pad; a.dgroups = dgroups; a.off_ld = off_ld;
  a.Ho = (int)Ho;
  a.Wo = (int)Wo;
  a.col = nullptr; a.dx = nullptr; a.doffset = nullptr; a.acc = nullptr;
  return 0;
}

// the backward's outputs: dx is 4-byte aligned for the fp64-scratch entry (scalar adds) and 16-byte aligned for the
// float4 atomics of the float-atomic entry; doffset takes single-float stores / atomics
int check_bwd_out(const char* who, const float* dx, const float* doffset, uintptr_t dx_align) {
  SN_CHECK(dx != nullptr && doffset != nullptr, "%s: dx / doffset must not be null", who);
  SN_CHECK(((uintptr_t)dx & (dx_align - 1)) == 0, "%s: dx must be %d-byte aligned", who, (int)dx_align);
  SN_CHECK(((uintptr_t)doffset & 3) == 0, "%s: doffset must be 4-byte aligned", who);
  return 0;
}

int dc_grid(const DcArgs& a) {
  const long warps = (long)a.NB * a.Ho * a.Wo * a.KH * a.KW * (a.C / 128);
  long g = (warps + 7) / 8;
  const long cap = (long)sn::kNumSMs * 16;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace

extern "C" {

// dtype: storage of x and col, 0 = fp32, 1 = bf16 (offset is fp32)
int sniper_deform_im2col(const void* x, const float* offset, int NB, int H, int W, int C, int KH, int KW, int stride,
                         int dil, int pad, int dgroups, int off_ld, void* col, int dtype, void* stream) {
  DcArgs a;
  if (fill(a, "deform_im2col", x, offset, NB, H, W, C, KH, KW, stride, dil, pad, dgroups, off_ld, col, dtype)) return -1;
  if (NB == 0) return 0;
  a.col = col;
  if (dtype == 0) deform_im2col_kernel<false, float><<<dc_grid(a), 256, 0, (cudaStream_t)stream>>>(a);
  else deform_im2col_kernel<false, bf16><<<dc_grid(a), 256, 0, (cudaStream_t)stream>>>(a);
  SN_LAUNCH_CHECK();
  return 0;
}

// dx is accumulated into (zero it first); doffset rows are fully overwritten when C/dgroups == 128,
// accumulated otherwise (zero it first in that case).
// dtype: storage of dcol and x (0 = fp32, 1 = bf16); dx and doffset are fp32 (accumulated with float atomics).
int sniper_deform_col2im(const void* dcol, const void* x, const float* offset, int NB, int H, int W, int C, int KH,
                         int KW, int stride, int dil, int pad, int dgroups, int off_ld, float* dx, float* doffset,
                         int dtype, void* stream) {
  DcArgs a;
  if (fill(a, "deform_col2im", x, offset, NB, H, W, C, KH, KW, stride, dil, pad, dgroups, off_ld, dcol, dtype))
    return -1;
  if (check_bwd_out("deform_col2im", dx, doffset, 16)) return -1;
  if (NB == 0) return 0;
  a.col = const_cast<void*>(dcol); a.dx = dx; a.doffset = doffset;
  if (dtype == 0) deform_im2col_kernel<true, float><<<dc_grid(a), 256, 0, (cudaStream_t)stream>>>(a);
  else deform_im2col_kernel<true, bf16><<<dc_grid(a), 256, 0, (cudaStream_t)stream>>>(a);
  SN_LAUNCH_CHECK();
  return 0;
}

// sniper_deform_col2im with reproducible dx: the scattered dx contributions (exact fp64 products) are summed with fp64
// atomics in `acc`, a caller-owned, zero-filled fp64 buffer of acc_elems >= NB*H*W*C elements, and a second kernel
// then adds the sums to dx.  fp64 additions still round, so a different arrival order could in principle change a
// sum, but only in its last fp64 bits: the fp32 dx is practically always the same from run to run (float atomics
// straight into dx differ in the last fp32 bits).  Same arguments and semantics as sniper_deform_col2im otherwise.
int sniper_deform_col2im_fp64acc(const void* dcol, const void* x, const float* offset, int NB, int H, int W, int C,
                                 int KH, int KW, int stride, int dil, int pad, int dgroups, int off_ld, float* dx,
                                 float* doffset, int dtype, double* acc, long acc_elems, void* stream) {
  DcArgs a;
  if (fill(a, "deform_col2im_fp64acc", x, offset, NB, H, W, C, KH, KW, stride, dil, pad, dgroups, off_ld, dcol, dtype))
    return -1;
  if (check_bwd_out("deform_col2im_fp64acc", dx, doffset, 4)) return -1;
  const long n = (long)NB * H * W * C;
  SN_CHECK(acc != nullptr && acc_elems >= n, "deform_col2im_fp64acc: acc needs %ld elements, %ld given", n, acc_elems);
  SN_CHECK(((uintptr_t)acc & 7) == 0, "deform_col2im_fp64acc: acc must be 8-byte aligned");
  if (NB == 0) return 0;
  a.col = const_cast<void*>(dcol); a.dx = dx; a.doffset = doffset; a.acc = acc;
  if (dtype == 0) deform_im2col_kernel<true, float><<<dc_grid(a), 256, 0, (cudaStream_t)stream>>>(a);
  else deform_im2col_kernel<true, bf16><<<dc_grid(a), 256, 0, (cudaStream_t)stream>>>(a);
  SN_LAUNCH_CHECK();
  long g = (n + 255) / 256;
  if (g > (long)sn::kNumSMs * 16) g = (long)sn::kNumSMs * 16;
  add_f64_kernel<<<(int)g, 256, 0, (cudaStream_t)stream>>>(dx, acc, n);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
