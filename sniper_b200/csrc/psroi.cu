// DeformablePSROIPooling / PSROIPooling forward + backward.
//
// Replaces SNIPER-mxnet/src/operator/contrib/deformable_psroi_pooling.cu (fwd :71-161, bwd :203-330,
// bilinear_interp :49-68) and psroi_pooling.cu (fwd :51-118, bwd :146-210).  Bin / sample geometry is
// evaluated with explicit round-to-nearest intrinsics in the order of the reference source so that
// every floor/ceil/clamp index equals oracle/psroi.c bit for bit.
//
// Two layouts: 0 = NCHW data, (n,c,ph,pw) output (the reference's, used by the drop-in operator);
// 1 = NHWC data [B,H,W,C], (n,ph,pw,c) output (the native layout of this framework: a warp owns 32
// consecutive channels of one bin, so every bilinear corner is one coalesced 128-byte gather and the
// backward scatter is a coalesced RED).
#include <stdlib.h>
#include "common.cuh"
#include <math.h>

namespace {

struct PsArgs {
  const float* data;
  const float* rois;
  const float* trans;
  int num_rois, channels, height, width;
  float spatial_scale;
  int output_dim, group_size, pooled, part_size, sample_per_part;
  float trans_std;
  int no_trans, num_classes, channels_each_class;
  int layout;
  float* top_data;
  float* top_count;      // optional
  int32_t* sample_idx;   // optional debug/parity output, oracle order
  // backward
  const float* top_diff;
  float* data_diff;
  float* trans_diff;
  double* acc;           // optional fp64 scratch: [data_elems] sums for data_diff, then the trans_diff sums
  long data_elems;
};

// fp64 sums -> fp32 gradients: dst += (float)acc
__global__ void __launch_bounds__(256) ps_add_f64_kernel(float* __restrict__ dst, const double* __restrict__ acc, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    dst[i] += (float)acc[i];
}

struct Geom {
  int roi_batch_ind, part_h, part_w, class_id, c;
  float roi_width, roi_height, wstart, hstart, sub_w, sub_h;
};

__device__ __forceinline__ void decompose(const PsArgs& p, long index, int& n, int& ctop, int& ph, int& pw) {
  if (p.layout == 0) {
    pw = (int)(index % p.pooled);
    ph = (int)((index / p.pooled) % p.pooled);
    ctop = (int)((index / p.pooled / p.pooled) % p.output_dim);
    n = (int)(index / p.pooled / p.pooled / p.output_dim);
  } else {
    ctop = (int)(index % p.output_dim);
    pw = (int)((index / p.output_dim) % p.pooled);
    ph = (int)((index / p.output_dim / p.pooled) % p.pooled);
    n = (int)(index / p.output_dim / p.pooled / p.pooled);
  }
}

__device__ __forceinline__ long ref_index(const PsArgs& p, int n, int ctop, int ph, int pw) {
  return (((long)n * p.output_dim + ctop) * p.pooled + ph) * p.pooled + pw;
}

__device__ __forceinline__ size_t data_off(const PsArgs& p, int b, int c, int y, int x) {
  return p.layout == 0 ? (((size_t)b * p.channels + c) * p.height + y) * p.width + x
                       : (((size_t)b * p.height + y) * p.width + x) * p.channels + c;
}

__device__ __forceinline__ void deform_geom(const PsArgs& p, int n, int ctop, int ph, int pw, Geom& g) {
  const float* r = p.rois + (size_t)n * 5;
  g.roi_batch_ind = (int)r[0];
  const float roi_start_w = (float)__dadd_rn((double)__fmul_rn(roundf(r[1]), p.spatial_scale), -0.5);
  const float roi_start_h = (float)__dadd_rn((double)__fmul_rn(roundf(r[2]), p.spatial_scale), -0.5);
  const float roi_end_w =
      (float)__dadd_rn((double)__fmul_rn((float)__dadd_rn((double)roundf(r[3]), 1.0), p.spatial_scale), -0.5);
  const float roi_end_h =
      (float)__dadd_rn((double)__fmul_rn((float)__dadd_rn((double)roundf(r[4]), 1.0), p.spatial_scale), -0.5);
  g.roi_width = (float)fmax((double)__fsub_rn(roi_end_w, roi_start_w), 0.1);
  g.roi_height = (float)fmax((double)__fsub_rn(roi_end_h, roi_start_h), 0.1);
  const float bin_size_h = __fdiv_rn(g.roi_height, (float)p.pooled);
  const float bin_size_w = __fdiv_rn(g.roi_width, (float)p.pooled);
  g.sub_h = __fdiv_rn(bin_size_h, (float)p.sample_per_part);
  g.sub_w = __fdiv_rn(bin_size_w, (float)p.sample_per_part);
  g.part_h = (int)floorf(__fmul_rn(__fdiv_rn((float)ph, (float)p.pooled), (float)p.part_size));
  g.part_w = (int)floorf(__fmul_rn(__fdiv_rn((float)pw, (float)p.pooled), (float)p.part_size));
  g.class_id = ctop / p.channels_each_class;
  float trans_x = 0.0f, trans_y = 0.0f;
  if (!p.no_trans) {
    const size_t tb = (((size_t)(n * p.num_classes + g.class_id) * 2) * p.part_size + g.part_h) * p.part_size + g.part_w;
    trans_x = __fmul_rn(p.trans[tb], p.trans_std);
    trans_y = __fmul_rn(p.trans[tb + (size_t)p.part_size * p.part_size], p.trans_std);
  }
  float wstart = __fadd_rn(__fmul_rn((float)pw, bin_size_w), roi_start_w);
  wstart = __fadd_rn(wstart, __fmul_rn(trans_x, g.roi_width));
  float hstart = __fadd_rn(__fmul_rn((float)ph, bin_size_h), roi_start_h);
  hstart = __fadd_rn(hstart, __fmul_rn(trans_y, g.roi_height));
  g.wstart = wstart;
  g.hstart = hstart;
  int gw = (int)floorf(__fdiv_rn(__fmul_rn((float)pw, (float)p.group_size), (float)p.pooled));
  int gh = (int)floorf(__fdiv_rn(__fmul_rn((float)ph, (float)p.group_size), (float)p.pooled));
  gw = min(max(gw, 0), p.group_size - 1);
  gh = min(max(gh, 0), p.group_size - 1);
  g.c = (ctop * p.group_size + gh) * p.group_size + gw;
}

// returns false if the sample is skipped (deformable_psroi_pooling.cu:147-149)
__device__ __forceinline__ bool sample_pos(const PsArgs& p, const Geom& g, int ih, int iw, float& w, float& h) {
  w = __fadd_rn(g.wstart, __fmul_rn((float)iw, g.sub_w));
  h = __fadd_rn(g.hstart, __fmul_rn((float)ih, g.sub_h));
  if ((double)w < -0.5 || (double)w > (double)p.width - 0.5 || (double)h < -0.5 || (double)h > (double)p.height - 0.5)
    return false;
  w = (float)fmin(fmax((double)w, 0.), (double)p.width - 1.);
  h = (float)fmin(fmax((double)h, 0.), (double)p.height - 1.);
  return true;
}

__global__ void __launch_bounds__(256) deform_psroi_fwd_kernel(PsArgs p, long count) {
  for (long index = (long)blockIdx.x * blockDim.x + threadIdx.x; index < count; index += (long)gridDim.x * blockDim.x) {
    int n, ctop, ph, pw;
    decompose(p, index, n, ctop, ph, pw);
    Geom g;
    deform_geom(p, n, ctop, ph, pw, g);
    float sum = 0.0f;
    int cnt = 0;
    const int S = p.sample_per_part;
    const long ridx = ref_index(p, n, ctop, ph, pw);
    for (int ih = 0; ih < S; ++ih) {
      for (int iw = 0; iw < S; ++iw) {
        float w, h;
        int32_t* si = p.sample_idx ? p.sample_idx + ((size_t)ridx * S * S + ih * S + iw) * 4 : nullptr;
        if (!sample_pos(p, g, ih, iw, w, h)) {
          if (si) si[0] = si[1] = si[2] = si[3] = -1;
          continue;
        }
        const int x1 = (int)floorf(w), x2 = (int)ceilf(w), y1 = (int)floorf(h), y2 = (int)ceilf(h);
        const float dist_x = __fsub_rn(w, (float)x1), dist_y = __fsub_rn(h, (float)y1);
        const float v11 = __ldg(p.data + data_off(p, g.roi_batch_ind, g.c, y1, x1));
        const float v12 = __ldg(p.data + data_off(p, g.roi_batch_ind, g.c, y2, x1));
        const float v21 = __ldg(p.data + data_off(p, g.roi_batch_ind, g.c, y1, x2));
        const float v22 = __ldg(p.data + data_off(p, g.roi_batch_ind, g.c, y2, x2));
        const float omx = __fsub_rn(1.0f, dist_x), omy = __fsub_rn(1.0f, dist_y);
        float val = __fmul_rn(__fmul_rn(omx, omy), v11);
        val = __fadd_rn(val, __fmul_rn(__fmul_rn(omx, dist_y), v12));
        val = __fadd_rn(val, __fmul_rn(__fmul_rn(dist_x, omy), v21));
        val = __fadd_rn(val, __fmul_rn(__fmul_rn(dist_x, dist_y), v22));
        sum = __fadd_rn(sum, val);
        cnt++;
        if (si) {
          si[0] = y1 * p.width + x1; si[1] = y2 * p.width + x1;
          si[2] = y1 * p.width + x2; si[3] = y2 * p.width + x2;
        }
      }
    }
    p.top_data[index] = cnt == 0 ? 0.0f : __fdiv_rn(sum, (float)cnt);
    if (p.top_count) p.top_count[index] = (float)cnt;
  }
}

__global__ void __launch_bounds__(256) deform_psroi_bwd_kernel(PsArgs p, long count) {
  const int lane = threadIdx.x & 31;
  for (long base = (long)blockIdx.x * blockDim.x + threadIdx.x - lane; base < count;
       base += (long)gridDim.x * blockDim.x) {
    const long index = base + lane;
    const bool active = index < count;
    int n = 0, ctop = 0, ph = 0, pw = 0;
    Geom g;
    float diff_val = 0.0f;
    int cnt = 0;
    const int S = p.sample_per_part;
    if (active) {
      decompose(p, index, n, ctop, ph, pw);
      deform_geom(p, n, ctop, ph, pw, g);
      for (int ih = 0; ih < S; ++ih)
        for (int iw = 0; iw < S; ++iw) {
          float w, h;
          cnt += sample_pos(p, g, ih, iw, w, h) ? 1 : 0;
        }
      if (cnt > 0) diff_val = __fdiv_rn(p.top_diff[index], (float)cnt);
    }
    float tdx = 0.0f, tdy = 0.0f;
    if (active && cnt > 0) {
      for (int ih = 0; ih < S; ++ih) {
        for (int iw = 0; iw < S; ++iw) {
          float w, h;
          if (!sample_pos(p, g, ih, iw, w, h)) continue;
          const int x0 = (int)floorf(w), x1 = (int)ceilf(w), y0 = (int)floorf(h), y1 = (int)ceilf(h);
          const float dist_x = w - x0, dist_y = h - y0;
          const float q00 = (1 - dist_x) * (1 - dist_y), q01 = (1 - dist_x) * dist_y;
          const float q10 = dist_x * (1 - dist_y), q11 = dist_x * dist_y;
          const size_t o00 = data_off(p, g.roi_batch_ind, g.c, y0, x0), o01 = data_off(p, g.roi_batch_ind, g.c, y1, x0);
          const size_t o10 = data_off(p, g.roi_batch_ind, g.c, y0, x1), o11 = data_off(p, g.roi_batch_ind, g.c, y1, x1);
          atomicAdd(p.data_diff + o00, q00 * diff_val);
          atomicAdd(p.data_diff + o01, q01 * diff_val);
          atomicAdd(p.data_diff + o10, q10 * diff_val);
          atomicAdd(p.data_diff + o11, q11 * diff_val);
          if (p.no_trans) continue;
          const float U00 = __ldg(p.data + o00), U01 = __ldg(p.data + o01);
          const float U10 = __ldg(p.data + o10), U11 = __ldg(p.data + o11);
          float dx = (U11 * dist_y + U10 * (1 - dist_y) - U01 * dist_y - U00 * (1 - dist_y)) * p.trans_std * diff_val;
          float dy = (U11 * dist_x + U01 * (1 - dist_x) - U10 * dist_x - U00 * (1 - dist_x)) * p.trans_std * diff_val;
          tdx += dx * g.roi_width;
          tdy += dy * g.roi_height;
        }
      }
    }
    if (!p.no_trans) {
      // NHWC order: the 32 lanes of a warp are 32 channels of one bin -> one atomic per warp when
      // they share (n, class, part); otherwise fall back to per-lane atomics.
      const size_t tb = active ? (((size_t)(n * p.num_classes + g.class_id) * 2) * p.part_size + g.part_h) * p.part_size + g.part_w
                               : (size_t)-1;
      const size_t tb0 = __shfl_sync(0xffffffffu, tb, 0);
      const bool uniform = __all_sync(0xffffffffu, tb == tb0 || !active);
      if (uniform && tb0 != (size_t)-1) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          tdx += __shfl_xor_sync(0xffffffffu, tdx, off);
          tdy += __shfl_xor_sync(0xffffffffu, tdy, off);
        }
        if (lane == 0) {
          atomicAdd(p.trans_diff + tb0, tdx);
          atomicAdd(p.trans_diff + tb0 + (size_t)p.part_size * p.part_size, tdy);
        }
      } else if (active && cnt > 0) {
        atomicAdd(p.trans_diff + tb, tdx);
        atomicAdd(p.trans_diff + tb + (size_t)p.part_size * p.part_size, tdy);
      }
    }
  }
}

// ---------------------------------------------------------------- NHWC fast path (group_size 1, one class)
// One warp = one bin (n, ph, pw): the bin / sample geometry is evaluated once per warp instead of once per
// channel, every bilinear corner is a coalesced float4 gather over 128 channels, and the pooled values keep
// the oracle's per-channel operation order (so they stay bit-identical to the generic kernel).
template <int CC>  // CC = channels / 128
__global__ void __launch_bounds__(256) deform_psroi_fwd_nhwc_kernel(PsArgs p, long nbins) {
  const int lane = threadIdx.x & 31;
  const int S = p.sample_per_part;
  for (long bin = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; bin < nbins;
       bin += ((long)gridDim.x * blockDim.x) >> 5) {
    const int pw = (int)(bin % p.pooled);
    const int ph = (int)((bin / p.pooled) % p.pooled);
    const int n = (int)(bin / ((long)p.pooled * p.pooled));
    Geom g;
    deform_geom(p, n, 0, ph, pw, g);
    float4 sum[CC];
#pragma unroll
    for (int k = 0; k < CC; ++k) sum[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    int cnt = 0;
    const float* img = p.data + (size_t)g.roi_batch_ind * p.height * p.width * p.channels + lane * 4;
    for (int ih = 0; ih < S; ++ih) {
      for (int iw = 0; iw < S; ++iw) {
        float w, h;
        if (!sample_pos(p, g, ih, iw, w, h)) continue;
        const int x1 = (int)floorf(w), x2 = (int)ceilf(w), y1 = (int)floorf(h), y2 = (int)ceilf(h);
        const float dist_x = __fsub_rn(w, (float)x1), dist_y = __fsub_rn(h, (float)y1);
        const float omx = __fsub_rn(1.0f, dist_x), omy = __fsub_rn(1.0f, dist_y);
        const float w11 = __fmul_rn(omx, omy), w12 = __fmul_rn(omx, dist_y), w21 = __fmul_rn(dist_x, omy),
                    w22 = __fmul_rn(dist_x, dist_y);
        const float* p11 = img + ((size_t)y1 * p.width + x1) * p.channels;
        const float* p12 = img + ((size_t)y2 * p.width + x1) * p.channels;
        const float* p21 = img + ((size_t)y1 * p.width + x2) * p.channels;
        const float* p22 = img + ((size_t)y2 * p.width + x2) * p.channels;
#pragma unroll
        for (int k = 0; k < CC; ++k) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(p11 + k * 128));
          const float4 b = __ldg(reinterpret_cast<const float4*>(p12 + k * 128));
          const float4 c = __ldg(reinterpret_cast<const float4*>(p21 + k * 128));
          const float4 d = __ldg(reinterpret_cast<const float4*>(p22 + k * 128));
          float4 v;
          v.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w11, a.x), __fmul_rn(w12, b.x)), __fmul_rn(w21, c.x)), __fmul_rn(w22, d.x));
          v.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w11, a.y), __fmul_rn(w12, b.y)), __fmul_rn(w21, c.y)), __fmul_rn(w22, d.y));
          v.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w11, a.z), __fmul_rn(w12, b.z)), __fmul_rn(w21, c.z)), __fmul_rn(w22, d.z));
          v.w = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w11, a.w), __fmul_rn(w12, b.w)), __fmul_rn(w21, c.w)), __fmul_rn(w22, d.w));
          sum[k].x = __fadd_rn(sum[k].x, v.x); sum[k].y = __fadd_rn(sum[k].y, v.y);
          sum[k].z = __fadd_rn(sum[k].z, v.z); sum[k].w = __fadd_rn(sum[k].w, v.w);
        }
        cnt++;
      }
    }
    const float fc = (float)cnt;
    float* o = p.top_data + bin * p.channels + lane * 4;
#pragma unroll
    for (int k = 0; k < CC; ++k) {
      float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
      if (cnt) {
        r.x = __fdiv_rn(sum[k].x, fc); r.y = __fdiv_rn(sum[k].y, fc);
        r.z = __fdiv_rn(sum[k].z, fc); r.w = __fdiv_rn(sum[k].w, fc);
      }
      *reinterpret_cast<float4*>(o + k * 128) = r;
      if (p.top_count) *reinterpret_cast<float4*>(p.top_count + bin * p.channels + lane * 4 + k * 128) = make_float4(fc, fc, fc, fc);
    }
  }
}

// One axis of the sample grid of a bin: the S samples contribute bilinear weights to at most 2S distinct
// rows (columns); duplicates are merged so that the scatter touches each feature pixel once per bin.
struct AxisTab {
  int idx[8];
  float w[8];   // summed interpolation weight
  float d[8];   // summed d(weight)/d(coordinate)
  int n, nvalid;
};

__device__ __forceinline__ void axis_add(AxisTab& t, int i, float w, float d) {
  for (int k = 0; k < t.n; ++k)
    if (t.idx[k] == i) {
      t.w[k] += w;
      t.d[k] += d;
      return;
    }
  t.idx[t.n] = i; t.w[t.n] = w; t.d[t.n] = d;
  ++t.n;
}

__device__ __forceinline__ void axis_build(AxisTab& t, float start, float sub, int S, int extent) {
  t.n = 0;
  t.nvalid = 0;
  for (int i = 0; i < S && i < 4; ++i) {
    float c = __fadd_rn(start, __fmul_rn((float)i, sub));
    if ((double)c < -0.5 || (double)c > (double)extent - 0.5) continue;
    c = (float)fmin(fmax((double)c, 0.), (double)extent - 1.);
    const int lo = (int)floorf(c), hi = (int)ceilf(c);
    const float dist = c - lo;
    axis_add(t, lo, 1.0f - dist, -1.0f);
    axis_add(t, hi, dist, 1.0f);
    ++t.nvalid;
  }
}

// Backward of the pooling, separable form: the 16 samples of a bin form a 4x4 grid whose bilinear weights
// factor into (row weights) x (column weights), so dX[y][x] += dv * Wy[y] * Wx[x] over the few distinct
// (y,x) the bin touches -- ~8x fewer float4 REDs than scattering every sample's four corners
// (deformable_psroi_pooling.cu:203-330 semantics; summation order differs, results agree to rounding).
template <int CC>
__global__ void __launch_bounds__(256) deform_psroi_bwd_nhwc_kernel(PsArgs p, long nbins) {
  const int lane = threadIdx.x & 31;
  const int S = p.sample_per_part;
  for (long bin = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; bin < nbins;
       bin += ((long)gridDim.x * blockDim.x) >> 5) {
    const int pw = (int)(bin % p.pooled);
    const int ph = (int)((bin / p.pooled) % p.pooled);
    const int n = (int)(bin / ((long)p.pooled * p.pooled));
    Geom g;
    deform_geom(p, n, 0, ph, pw, g);
    AxisTab ax, ay;
    axis_build(ax, g.wstart, g.sub_w, S, p.width);
    axis_build(ay, g.hstart, g.sub_h, S, p.height);
    const int cnt = ax.nvalid * ay.nvalid;
    if (cnt == 0) continue;
    const float fc = (float)cnt;
    float4 dv[CC];
    const float* td = p.top_diff + bin * p.channels + lane * 4;
#pragma unroll
    for (int k = 0; k < CC; ++k) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(td + k * 128));
      dv[k] = make_float4(__fdiv_rn(t.x, fc), __fdiv_rn(t.y, fc), __fdiv_rn(t.z, fc), __fdiv_rn(t.w, fc));
    }
    const size_t ibase = (size_t)g.roi_batch_ind * p.height * p.width * p.channels + lane * 4;
    float tdx = 0.f, tdy = 0.f;
    for (int a = 0; a < ay.n; ++a) {
      for (int b = 0; b < ax.n; ++b) {
        const float wgt = ay.w[a] * ax.w[b];
        const size_t o = ibase + ((size_t)ay.idx[a] * p.width + ax.idx[b]) * p.channels;
#pragma unroll
        for (int k = 0; k < CC; ++k) {
          const float4 d = dv[k];
          if (wgt != 0.f) {
            if (p.acc) {
              // fp64 sums of exact fp64 products: practically independent of the order the warps arrive in
              double* ab = p.acc + o + k * 128;
              const double w = (double)wgt;
              atomicAdd(ab, w * d.x);
              atomicAdd(ab + 1, w * d.y);
              atomicAdd(ab + 2, w * d.z);
              atomicAdd(ab + 3, w * d.w);
            } else {
              atomicAdd(reinterpret_cast<float4*>(p.data_diff + o + k * 128),
                        make_float4(wgt * d.x, wgt * d.y, wgt * d.z, wgt * d.w));
            }
          }
          if (!p.no_trans) {
            const float4 U = __ldg(reinterpret_cast<const float4*>(p.data + o + k * 128));
            const float dot = U.x * d.x + U.y * d.y + U.z * d.z + U.w * d.w;
            tdx += ay.w[a] * ax.d[b] * dot;
            tdy += ay.d[a] * ax.w[b] * dot;
          }
        }
      }
    }
    if (!p.no_trans) {
      tdx *= p.trans_std * g.roi_width;
      tdy *= p.trans_std * g.roi_height;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        tdx += __shfl_xor_sync(0xffffffffu, tdx, off);
        tdy += __shfl_xor_sync(0xffffffffu, tdy, off);
      }
      if (lane == 0) {
        const size_t tb = (((size_t)n * 2) * p.part_size + g.part_h) * p.part_size + g.part_w;
        if (p.acc) {
          atomicAdd(p.acc + p.data_elems + tb, (double)tdx);
          atomicAdd(p.acc + p.data_elems + tb + (size_t)p.part_size * p.part_size, (double)tdy);
        } else {
          atomicAdd(p.trans_diff + tb, tdx);
          atomicAdd(p.trans_diff + tb + (size_t)p.part_size * p.part_size, tdy);
        }
      }
    }
  }
}

// Forward in the same separable form (default on the product path; SNIPER_PSROI_EXACT=1 selects the kernel above,
// which keeps the oracle's per-sample operation order and is bit-identical to it).  A bin's 4 x 4 sample grid
// touches only ~3 x 3 distinct feature pixels, so gathering each pixel once with the summed weight Wy[y] * Wx[x]
// replaces 64 float4 corner loads per 128 channels by ~9-16 (the exact kernel ran at ~50 % of the L1 bandwidth).
// Results agree with the per-sample order to fp32 rounding (|rel| ~ 1e-6); count = valid samples, as the reference.
template <int CC>
__global__ void __launch_bounds__(256) deform_psroi_fwd_sep_nhwc_kernel(PsArgs p, long nbins) {
  const int lane = threadIdx.x & 31;
  const int S = p.sample_per_part;
  for (long bin = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; bin < nbins;
       bin += ((long)gridDim.x * blockDim.x) >> 5) {
    const int pw = (int)(bin % p.pooled);
    const int ph = (int)((bin / p.pooled) % p.pooled);
    const int n = (int)(bin / ((long)p.pooled * p.pooled));
    Geom g;
    deform_geom(p, n, 0, ph, pw, g);
    AxisTab ax, ay;
    axis_build(ax, g.wstart, g.sub_w, S, p.width);
    axis_build(ay, g.hstart, g.sub_h, S, p.height);
    const int cnt = ax.nvalid * ay.nvalid;
    float4 sum[CC];
#pragma unroll
    for (int k = 0; k < CC; ++k) sum[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float* img = p.data + (size_t)g.roi_batch_ind * p.height * p.width * p.channels + lane * 4;
    if (cnt) {
      for (int a = 0; a < ay.n; ++a) {
        const float* rowp = img + (size_t)ay.idx[a] * p.width * p.channels;
        for (int b = 0; b < ax.n; ++b) {
          const float wgt = ay.w[a] * ax.w[b];
          if (wgt == 0.f) continue;
          const float* px = rowp + (size_t)ax.idx[b] * p.channels;
#pragma unroll
          for (int k = 0; k < CC; ++k) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(px + k * 128));
            sum[k].x = fmaf(wgt, v.x, sum[k].x); sum[k].y = fmaf(wgt, v.y, sum[k].y);
            sum[k].z = fmaf(wgt, v.z, sum[k].z); sum[k].w = fmaf(wgt, v.w, sum[k].w);
          }
        }
      }
    }
    const float fc = (float)cnt;
    const float inv = cnt ? 1.0f / fc : 0.f;
    float* o = p.top_data + bin * p.channels + lane * 4;
#pragma unroll
    for (int k = 0; k < CC; ++k) {
      *reinterpret_cast<float4*>(o + k * 128) = make_float4(sum[k].x * inv, sum[k].y * inv, sum[k].z * inv, sum[k].w * inv);
      if (p.top_count) *reinterpret_cast<float4*>(p.top_count + bin * p.channels + lane * 4 + k * 128) = make_float4(fc, fc, fc, fc);
    }
  }
}

// The warp-per-bin kernels read data and write top_data / top_count as float4: every such buffer must be 16-byte
// aligned, otherwise the call takes the generic per-output kernel.
bool fast_nhwc_ok(const PsArgs& a) {
  return a.layout == 1 && a.group_size == 1 && a.num_classes == 1 && a.sample_idx == nullptr &&
         a.sample_per_part <= 4 &&
         (a.channels == 128 || a.channels == 256 || a.channels == 512) &&
         ((uintptr_t)a.data & 15) == 0 && ((uintptr_t)a.top_data & 15) == 0 && ((uintptr_t)a.top_count & 15) == 0;
}

int fast_grid(long nbins) {
  long g = (nbins + 7) / 8;
  const long cap = (long)sn::kNumSMs * 16;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

__device__ __forceinline__ void psroi_bin(const PsArgs& p, int n, int ph, int pw, int& b, int& hstart, int& hend,
                                          int& wstart, int& wend) {
  const float* r = p.rois + (size_t)n * 5;
  b = (int)r[0];
  const float roi_start_w = __fmul_rn(roundf(r[1]), p.spatial_scale);
  const float roi_start_h = __fmul_rn(roundf(r[2]), p.spatial_scale);
  const float roi_end_w = __fmul_rn((float)__dadd_rn((double)roundf(r[3]), 1.0), p.spatial_scale);
  const float roi_end_h = __fmul_rn((float)__dadd_rn((double)roundf(r[4]), 1.0), p.spatial_scale);
  const float roi_width = (float)fmax((double)__fsub_rn(roi_end_w, roi_start_w), 0.1);
  const float roi_height = (float)fmax((double)__fsub_rn(roi_end_h, roi_start_h), 0.1);
  const float bin_size_h = __fdiv_rn(roi_height, (float)p.pooled);
  const float bin_size_w = __fdiv_rn(roi_width, (float)p.pooled);
  hstart = (int)floorf(__fadd_rn(__fmul_rn((float)ph, bin_size_h), roi_start_h));
  wstart = (int)floorf(__fadd_rn(__fmul_rn((float)pw, bin_size_w), roi_start_w));
  hend = (int)ceilf(__fadd_rn(__fmul_rn((float)(ph + 1), bin_size_h), roi_start_h));
  wend = (int)ceilf(__fadd_rn(__fmul_rn((float)(pw + 1), bin_size_w), roi_start_w));
  hstart = min(max(hstart, 0), p.height);
  hend = min(max(hend, 0), p.height);
  wstart = min(max(wstart, 0), p.width);
  wend = min(max(wend, 0), p.width);
}

__device__ __forceinline__ int psroi_channel(const PsArgs& p, int ctop, int ph, int pw) {
  int gw = (int)floorf(__fdiv_rn(__fmul_rn((float)pw, (float)p.group_size), (float)p.pooled));
  int gh = (int)floorf(__fdiv_rn(__fmul_rn((float)ph, (float)p.group_size), (float)p.pooled));
  gw = min(max(gw, 0), p.group_size - 1);
  gh = min(max(gh, 0), p.group_size - 1);
  return (ctop * p.group_size + gh) * p.group_size + gw;
}

__global__ void __launch_bounds__(256) psroi_fwd_kernel(PsArgs p, long count) {
  for (long index = (long)blockIdx.x * blockDim.x + threadIdx.x; index < count; index += (long)gridDim.x * blockDim.x) {
    int n, ctop, ph, pw, b, hstart, hend, wstart, wend;
    decompose(p, index, n, ctop, ph, pw);
    psroi_bin(p, n, ph, pw, b, hstart, hend, wstart, wend);
    const bool is_empty = (hend <= hstart) || (wend <= wstart);
    const int c = psroi_channel(p, ctop, ph, pw);
    float out_sum = 0.0f;
    for (int h = hstart; h < hend; ++h)
      for (int w = wstart; w < wend; ++w) out_sum = __fadd_rn(out_sum, __ldg(p.data + data_off(p, b, c, h, w)));
    const float bin_area = (float)((hend - hstart) * (wend - wstart));
    p.top_data[index] = is_empty ? 0.0f : __fdiv_rn(out_sum, bin_area);
    if (p.sample_idx) {
      int32_t* o = p.sample_idx + ref_index(p, n, ctop, ph, pw) * 4;
      o[0] = hstart; o[1] = hend; o[2] = wstart; o[3] = wend;
    }
  }
}

__global__ void __launch_bounds__(256) psroi_bwd_kernel(PsArgs p, long count) {
  for (long index = (long)blockIdx.x * blockDim.x + threadIdx.x; index < count; index += (long)gridDim.x * blockDim.x) {
    int n, ctop, ph, pw, b, hstart, hend, wstart, wend;
    decompose(p, index, n, ctop, ph, pw);
    psroi_bin(p, n, ph, pw, b, hstart, hend, wstart, wend);
    const bool is_empty = (hend <= hstart) || (wend <= wstart);
    if (is_empty) continue;
    const int c = psroi_channel(p, ctop, ph, pw);
    const float bin_area = (float)((hend - hstart) * (wend - wstart));
    const float diff_val = __fdiv_rn(p.top_diff[index], bin_area);
    for (int h = hstart; h < hend; ++h)
      for (int w = wstart; w < wend; ++w) atomicAdd(p.data_diff + data_off(p, b, c, h, w), diff_val);
  }
}

int grid_for(long count) {
  long g = (count + 255) / 256;
  const long cap = (long)sn::kNumSMs * 16;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

int fill_common(PsArgs& a, const float* data, const float* rois, const float* trans, int num_rois, int channels,
                int height, int width, float spatial_scale, int output_dim, int group_size, int pooled_size,
                int part_size, int sample_per_part, float trans_std, int no_trans, int num_classes, int layout) {
  SN_CHECK(layout == 0 || layout == 1, "psroi: layout must be 0 (NCHW) or 1 (NHWC)");
  SN_CHECK(num_rois >= 0, "psroi: num_rois (%d) must not be negative", num_rois);
  SN_CHECK(height >= 1 && width >= 1, "psroi: height (%d) and width (%d) must be at least 1", height, width);
  SN_CHECK(output_dim >= 1, "psroi: output_dim (%d) must be at least 1", output_dim);
  SN_CHECK(group_size >= 1, "psroi: group_size (%d) must be at least 1", group_size);
  SN_CHECK(pooled_size >= 1, "psroi: pooled_size (%d) must be at least 1", pooled_size);
  SN_CHECK(part_size >= 0, "psroi: part_size (%d) must not be negative", part_size);
  SN_CHECK(sample_per_part >= 1, "psroi: sample_per_part (%d) must be at least 1", sample_per_part);
  SN_CHECK(rois != nullptr, "psroi: rois must not be null");
  SN_CHECK(channels == output_dim * group_size * group_size, "psroi: channels (%d) != output_dim*group_size^2 (%d)",
           channels, output_dim * group_size * group_size);
  SN_CHECK(no_trans || (trans != nullptr && num_classes > 0 && output_dim % num_classes == 0),
           "deformable psroi: bad trans / num_classes");
  memset(&a, 0, sizeof(a));
  a.data = data; a.rois = rois; a.trans = no_trans ? nullptr : trans;
  a.num_rois = num_rois; a.channels = channels; a.height = height; a.width = width;
  a.spatial_scale = spatial_scale; a.output_dim = output_dim; a.group_size = group_size; a.pooled = pooled_size;
  a.part_size = part_size == 0 ? pooled_size : part_size; a.sample_per_part = sample_per_part;
  a.trans_std = trans_std; a.no_trans = no_trans; a.num_classes = no_trans ? 1 : num_classes;
  a.channels_each_class = no_trans ? output_dim : output_dim / num_classes;
  a.layout = layout;
  return 0;
}

}  // namespace

extern "C" {

int sniper_deform_psroi_fwd(const float* data, const float* rois, const float* trans, int num_rois, int channels,
                            int height, int width, float spatial_scale, int output_dim, int group_size,
                            int pooled_size, int part_size, int sample_per_part, float trans_std, int no_trans,
                            int num_classes, int layout, float* top_data, float* top_count, int32_t* sample_idx,
                            void* stream) {
  PsArgs a;
  if (fill_common(a, data, rois, trans, num_rois, channels, height, width, spatial_scale, output_dim, group_size,
                  pooled_size, part_size, sample_per_part, trans_std, no_trans, num_classes, layout))
    return -1;
  SN_CHECK(data != nullptr && top_data != nullptr, "deform_psroi_fwd: data / top_data must not be null");
  a.top_data = top_data; a.top_count = top_count; a.sample_idx = sample_idx;
  const long count = (long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return 0;
  if (fast_nhwc_ok(a)) {
    const long nbins = (long)num_rois * pooled_size * pooled_size;
    const int g = fast_grid(nbins);
    const char* ex = getenv("SNIPER_PSROI_EXACT");
    if (ex && ex[0] == '1') {
      if (channels == 128) deform_psroi_fwd_nhwc_kernel<1><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
      else if (channels == 256) deform_psroi_fwd_nhwc_kernel<2><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
      else deform_psroi_fwd_nhwc_kernel<4><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
    } else {
      if (channels == 128) deform_psroi_fwd_sep_nhwc_kernel<1><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
      else if (channels == 256) deform_psroi_fwd_sep_nhwc_kernel<2><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
      else deform_psroi_fwd_sep_nhwc_kernel<4><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
    }
    SN_LAUNCH_CHECK();
    return 0;
  }
  deform_psroi_fwd_kernel<<<grid_for(count), 256, 0, (cudaStream_t)stream>>>(a, count);
  SN_LAUNCH_CHECK();
  return 0;
}

// data_diff / trans_diff are ACCUMULATED into (req = kAddTo); zero them first for kWriteTo.
int sniper_deform_psroi_bwd(const float* top_diff, const float* data, const float* rois, const float* trans,
                            int num_rois, int channels, int height, int width, float spatial_scale, int output_dim,
                            int group_size, int pooled_size, int part_size, int sample_per_part, float trans_std,
                            int no_trans, int num_classes, int layout, float* data_diff, float* trans_diff,
                            void* stream) {
  PsArgs a;
  if (fill_common(a, data, rois, trans, num_rois, channels, height, width, spatial_scale, output_dim, group_size,
                  pooled_size, part_size, sample_per_part, trans_std, no_trans, num_classes, layout))
    return -1;
  SN_CHECK(no_trans || trans_diff != nullptr, "deformable psroi bwd: trans_diff is null");
  SN_CHECK(top_diff != nullptr && data != nullptr && data_diff != nullptr,
           "deform_psroi_bwd: top_diff / data / data_diff must not be null");
  a.top_diff = top_diff; a.data_diff = data_diff; a.trans_diff = trans_diff;
  a.acc = nullptr; a.data_elems = 0;
  const long count = (long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return 0;
  if (fast_nhwc_ok(a) && ((uintptr_t)data_diff & 15) == 0 && ((uintptr_t)top_diff & 15) == 0) {
    const long nbins = (long)num_rois * pooled_size * pooled_size;
    const int g = fast_grid(nbins);
    if (channels == 128) deform_psroi_bwd_nhwc_kernel<1><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
    else if (channels == 256) deform_psroi_bwd_nhwc_kernel<2><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
    else deform_psroi_bwd_nhwc_kernel<4><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
    SN_LAUNCH_CHECK();
    return 0;
  }
  deform_psroi_bwd_kernel<<<grid_for(count), 256, 0, (cudaStream_t)stream>>>(a, count);
  SN_LAUNCH_CHECK();
  return 0;
}

// sniper_deform_psroi_bwd for NHWC data of `batch` chips on the warp-per-bin kernels, with reproducible gradients:
// the scattered contributions (exact fp64 products) are summed with fp64 atomics in `acc`, a caller-owned, zero-filled
// fp64 buffer of batch*height*width*channels (+ num_rois*2*part_size^2 unless no_trans) elements, and second kernels
// add the sums to data_diff / trans_diff.  fp64 additions still round, so a different arrival order could in principle
// change a sum in its last fp64 bits; the fp32 gradients are practically always the same from run to run.  Returns -2
// (error string set) when the shape does not qualify for the NHWC kernels (layout, group_size 1, one class, <= 4
// samples per part, 128 / 256 / 512 channels, 16-byte aligned data, data_diff and top_diff): the caller then uses
// sniper_deform_psroi_bwd.
int sniper_deform_psroi_bwd_fp64acc(const float* top_diff, const float* data, const float* rois, const float* trans,
                                    int num_rois, int batch, int channels, int height, int width, float spatial_scale,
                                    int output_dim, int group_size, int pooled_size, int part_size,
                                    int sample_per_part, float trans_std, int no_trans, int num_classes,
                                    float* data_diff, float* trans_diff, double* acc, long acc_elems, void* stream) {
  PsArgs a;
  if (fill_common(a, data, rois, trans, num_rois, channels, height, width, spatial_scale, output_dim, group_size,
                  pooled_size, part_size, sample_per_part, trans_std, no_trans, num_classes, 1))
    return -1;
  SN_CHECK(no_trans || trans_diff != nullptr, "deformable psroi bwd: trans_diff is null");
  SN_CHECK(top_diff != nullptr && data != nullptr && data_diff != nullptr,
           "deform_psroi_bwd_fp64acc: top_diff / data / data_diff must not be null");
  SN_CHECK(batch >= 1, "deform_psroi_bwd_fp64acc: batch (%d) must be at least 1", batch);
  a.top_diff = top_diff; a.data_diff = data_diff; a.trans_diff = trans_diff;
  if (!fast_nhwc_ok(a) || ((uintptr_t)data_diff & 15) != 0 || ((uintptr_t)top_diff & 15) != 0) {
    sn::set_error("deformable psroi bwd fp64acc: shape / alignment does not qualify for the NHWC kernels");
    return -2;
  }
  const long data_elems = (long)batch * height * width * channels;
  const long trans_elems = no_trans ? 0 : (long)num_rois * 2 * a.part_size * a.part_size;
  SN_CHECK(acc != nullptr && acc_elems >= data_elems + trans_elems,
           "deformable psroi bwd fp64acc: acc needs %ld elements, %ld given", data_elems + trans_elems, acc_elems);
  SN_CHECK(((uintptr_t)acc & 7) == 0, "deform_psroi_bwd_fp64acc: acc must be 8-byte aligned");
  a.acc = acc; a.data_elems = data_elems;
  const long nbins = (long)num_rois * pooled_size * pooled_size;
  if (nbins == 0) return 0;
  const int g = fast_grid(nbins);
  if (channels == 128) deform_psroi_bwd_nhwc_kernel<1><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
  else if (channels == 256) deform_psroi_bwd_nhwc_kernel<2><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
  else deform_psroi_bwd_nhwc_kernel<4><<<g, 256, 0, (cudaStream_t)stream>>>(a, nbins);
  SN_LAUNCH_CHECK();
  long gg = (data_elems + 255) / 256;
  if (gg > (long)sn::kNumSMs * 16) gg = (long)sn::kNumSMs * 16;
  ps_add_f64_kernel<<<(int)gg, 256, 0, (cudaStream_t)stream>>>(data_diff, acc, data_elems);
  if (trans_elems)
    ps_add_f64_kernel<<<(int)((trans_elems + 255) / 256), 256, 0, (cudaStream_t)stream>>>(trans_diff, acc + data_elems,
                                                                                           trans_elems);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_psroi_fwd(const float* data, const float* rois, int num_rois, int channels, int height, int width,
                     float spatial_scale, int output_dim, int group_size, int pooled_size, int layout,
                     float* top_data, int32_t* bins, void* stream) {
  PsArgs a;
  if (fill_common(a, data, rois, nullptr, num_rois, channels, height, width, spatial_scale, output_dim, group_size,
                  pooled_size, pooled_size, 1, 0.0f, 1, 1, layout))
    return -1;
  SN_CHECK(data != nullptr && top_data != nullptr, "psroi_fwd: data / top_data must not be null");
  a.top_data = top_data; a.sample_idx = bins;
  const long count = (long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return 0;
  psroi_fwd_kernel<<<grid_for(count), 256, 0, (cudaStream_t)stream>>>(a, count);
  SN_LAUNCH_CHECK();
  return 0;
}

int sniper_psroi_bwd(const float* top_diff, const float* rois, int num_rois, int channels, int height, int width,
                     float spatial_scale, int output_dim, int group_size, int pooled_size, int layout,
                     float* data_diff, void* stream) {
  PsArgs a;
  if (fill_common(a, nullptr, rois, nullptr, num_rois, channels, height, width, spatial_scale, output_dim, group_size,
                  pooled_size, pooled_size, 1, 0.0f, 1, 1, layout))
    return -1;
  SN_CHECK(top_diff != nullptr && data_diff != nullptr, "psroi_bwd: top_diff / data_diff must not be null");
  a.top_diff = top_diff; a.data_diff = data_diff;
  const long count = (long)num_rois * output_dim * pooled_size * pooled_size;
  if (count == 0) return 0;
  psroi_bwd_kernel<<<grid_for(count), 256, 0, (cudaStream_t)stream>>>(a, count);
  SN_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
