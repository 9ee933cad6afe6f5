// wgmma tensor-core contraction kernel for sm_90a: GEMM / implicit-GEMM convolution (NHWC) /
// weight-gradient, operands staged global->shared by TMA (cp.async.bulk.tensor, 128B swizzle) into an
// mbarrier-synchronised ring, wgmma.mma_async from shared-memory descriptors, fp32 accumulators in registers.
//
// Replaces the reference's library calls on the hot path: cudnnConvolutionForward/BackwardData/
// BackwardFilter (SNIPER-mxnet/src/operator/nn/cudnn/cudnn_convolution-inl.h:144,211-266), cuBLAS
// via FullyConnected (nn/fully_connected-inl.h) and linalg_gemm in DeformableConvolution
// (contrib/deformable_convolution-inl.h:148-160).
//
// One CTA = one 128 x BLOCK_N output tile at a time (persistent over tiles).  384 threads: warpgroup 0 = TMA
// producer (one elected lane of warp 0 issues the copies), warpgroups 1 and 2 = consumers, each issuing the
// wgmma of 64 output rows x BLOCK_N columns and running the epilogue of those rows straight from its registers.
//
//   mode 0  GEMM    C[M,N]  = A[M,K] * B[N,K]^T             A,B K-major
//   mode 1  CONV    C[pix,N] = sum_taps A[n,h+dh,w+dw,c] * B[N,(tap,c)]   A 4-D NHWC, K-major; TMA zero
//                   fill implements padding, elementStrides implement stride
//   mode 2  WGRAD   C[Co,(tap,ci)] += sum_pix dY[pix,Co] * X[n,h+dh,w+dw,ci]   split-K.  bf16: both operands
//                   MN-major, wgmma reads the tiles directly (transpose bits).  tf32 (wgmma takes K-major tf32 only),
//                   stride-1 multi-tap layers over rows of Wo % 32 == 0 pixels: a copy kernel first writes dY^T and X^T
//                   channel-major into the stream's workspace and the TMA loads those K-major (see WgradFeed); other
//                   layers (wg_xpose): the consumers transpose each MN-major ring stage into a second, K-major ring
//                   while the wgmma of the previous stage run
//
// The tile width BN is a template parameter, so each compiled mainloop issues one wgmma shape (4 per k-block, one
// commit group).  The column pieces of a tail tile (PN columns) run a second, separately instantiated mainloop and
// epilogue of the same kernel, chosen once per work unit.
#include "common.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>

#include <algorithm>

namespace {

enum { MODE_GEMM = 0, MODE_CONV = 1, MODE_WGRAD = 2 };
enum { DT_TF32 = 0, DT_BF16 = 1 };
constexpr int kMaxTaps = 16;
constexpr int kStageABytes = 128 * 128;  // 128 rows x 128 B
constexpr int kStatsBytes = 8 * 2 * 256 * 4;   // per-warp column sums / sums of squares (fused BatchNorm statistics)
constexpr int kThreads = 384;            // producer warpgroup + 2 consumer warpgroups
constexpr int kMmasPerKb = 4;            // a k-block is 128 B of K per row: 4 x k8 (tf32) / k16 (bf16) wgmma
constexpr int kXStages = 2;              // tf32 WGRAD, wg_xpose: stages of the K-major ring the consumers transpose into

struct GemmParams {
  int mode, dtype;
  int M, N;               // logical output extent (rows, cols)
  int block_n;            // 64 / 128 / 256 (the kernel's BN)
  int num_kb;             // k-blocks per tile
  int stages;
  int tiles_m, tiles_n, splits;
  uint32_t stage_tx_bytes;  // bytes credited to the full barrier per ring stage
  // ---- producer geometry
  int elems_per_128B;     // 32 (tf32) / 64 (bf16)
  int cblocks;            // CONV: channel blocks per tap (Cin / elems_per_128B)
  int ntaps;
  int tap_dh[kMaxTaps], tap_dw[kMaxTaps];
  int conv_stride;        // input coordinate = out * conv_stride + tap offset
  int tile_w, tile_h;     // output pixels per tile = tile_w * tile_h (=128 CONV, = kp WGRAD)
  int tiles_w, tiles_per_img;
  int Ho, Wo;             // output spatial extent (CONV/WGRAD pixel space)
  int kp;                 // WGRAD: pixels per k-block
  int wg_cin_blocks;      // WGRAD: N tiles per tap = Cin / block_n
  // tf32 WGRAD from the channel-major copies (WgradFeed): X^T row block of each tap, input rows padded to wg_hp with
  // wg_padh of them before the first
  int wg_hp, wg_padh;
  int wg_tapblk[kMaxTaps];
  int wg_xpose;           // tf32 WGRAD without copies: MN-major boxes, transposed by the consumers
  // ---- descriptors (16-byte units)
  uint32_t a_lbo, a_sbo, b_lbo, b_sbo;
  uint32_t a_kadv, b_kadv;              // per wgmma k-step
  uint32_t a_half;                      // offset of the second consumer's 64 rows of A
  int a_boxes, b_boxes;                 // TMA boxes per stage
  uint32_t a_box_bytes, b_box_bytes;
  // ---- epilogue
  float* C;
  long ldc;
  const float* scale;     // per-column multiplier (optional)
  const float* bias;      // per-column addend (optional)
  const float* residual;  // same row mapping as C (optional)
  long ldr;
  int relu;
  int atomic;             // accumulate with red.global.add instead of store
  // row mapping for CONV: output pixel (n,oh,ow) -> row ((n*out_H + oh*out_s + out_oh)*out_W + ow*out_s + out_ow)
  int out_H, out_W, out_s, out_oh, out_ow;
  int out_bf16;           // store bf16 instead of fp32
  // ---- tail split: work units [0, tail_first) are whole tiles, every tile >= tail_first (the last, partial wave
  // over the persistent grid) is cut into column pieces (tail_p below)
  int tail_first;
  float4* tail_ws;
  int* tail_cnt;
  // ---- tail N-split (preferred when block_n = 256): every tile >= tail_first is cut into tail_p column pieces of
  // block_n / tail_p columns (own TMA box tma_bp, narrower wgmma), one piece per CTA.  Same K order as a whole tile
  // -> bit-identical results, no fix-up.  tail_p = 0: off.
  int tail_p;
  // ---- deterministic split-K (WGRAD, splits > 1): every split parks its partial tile in tail_ws (counted in tail_cnt);
  // the last split to arrive sums the partials in split order and adds the sum to C once (no order-dependent atomics)
  int split_park;
  double* stats;          // optional [2*N]: += per-column sum and sum of squares of the stored values
                          // (train-mode BatchNorm statistics of the consumer, fused into the producer)
};

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// one lane of a converged warp (the same one every time for a full mask)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// the 256 consumer threads (named barrier 1; barrier 0 is __syncthreads)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory matrix descriptor of wgmma: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base offset 0
// (stages are 1024-byte aligned), layout [62,64): 1 = SWIZZLE_128B
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo16, uint32_t sbo16) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);
  d |= (uint64_t)(lbo16 & 0x3fff) << 16;
  d |= (uint64_t)(sbo16 & 0x3fff) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// wgmma.mma_async m64nNk8 (tf32, K-major operands) / m64nNk16 (bf16; TR = 1: both operands MN-major), D += A * B.
// The accumulator array holds the instruction's N / 2 floats per thread.
template <int DT, int TR>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t da, uint64_t db) {
  if (DT == DT_TF32) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, 1, 1, 1;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                 : "l"(da), "l"(db));
  } else {
    asm volatile("wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, 1, 1, 1, %130, %131;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                 : "l"(da), "l"(db), "n"(TR), "n"(TR));
  }
}
template <int DT, int TR>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db) {
  if (DT == DT_TF32) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db));
  } else {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, %66, %67;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "n"(TR), "n"(TR));
  }
}
template <int DT, int TR>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db) {
  if (DT == DT_TF32) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db));
  } else {
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, %34, %35;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "n"(TR), "n"(TR));
  }
}

template <int DT, int TR, int W>
__device__ __forceinline__ void wgmma_tile(float (&d)[W / 2], uint64_t da, uint64_t db) {
  static_assert(W == 64 || W == 128 || W == 256, "wgmma width");
  if constexpr (W == 256) wgmma_n256<DT, TR>(d, da, db);
  else if constexpr (W == 128) wgmma_n128<DT, TR>(d, da, db);
  else wgmma_n64<DT, TR>(d, da, db);
}

struct TileCoord {
  int tile_m, tile_n, split;
  int kb0, nkb;       // k-block range of this work unit
  int slice, tail;    // split-K: split index and tile index (slice = -1: whole K range, no parking)
  int col0, ncols;    // output columns of this work unit (K-major modes)
  int piece;          // 1 if this unit is a column piece of a tail tile
};

__device__ __forceinline__ TileCoord tile_coord(const GemmParams& p, int u) {
  TileCoord c;
  c.kb0 = 0; c.nkb = p.num_kb; c.slice = -1; c.tail = 0;
  int pc = 0;
  c.piece = 0;
  c.ncols = p.block_n;
  if (p.tail_p > 0 && u >= p.tail_first) {
    const int v = u - p.tail_first;
    const int tt = v / p.tail_p;
    pc = v - tt * p.tail_p;
    c.piece = 1;
    c.ncols = p.block_n / p.tail_p;
    u = p.tail_first + tt;
  }
  c.tile_n = u % p.tiles_n;
  const int r = u / p.tiles_n;
  c.tile_m = r % p.tiles_m;
  c.split = r / p.tiles_m;
  c.col0 = c.tile_n * p.block_n + pc * c.ncols;
  if (p.split_park) {
    c.slice = c.split;
    c.tail = c.tile_m * p.tiles_n + c.tile_n;
  }
  return c;
}

// tf32 weight gradient: the TMA lands both operands MN-major (a 4 KB box = 32 pixel rows of 128 B = 32 channels, 128B
// swizzle; A = 4 boxes of dY channels, then B = BN / 32 boxes of X channels); wgmma takes tf32 K-major only, so the 8
// consumer warps (w = 0..7) rewrite the stage as (128 + BN) channel rows x 32 pixels (128 B, 128B swizzle) -- the layout
// of a K-major stage.  Work item = (box j, pixel quad q), lane = channel c of the box.  Banks:
//   loads: element (pix, c) is at byte pix * 128 + (((c >> 2) ^ (pix & 7)) << 4) + (c & 3) * 4 of its box, so for one
//          pix the 32 lanes hit banks ((c >> 2) ^ (pix & 7)) * 4 + (c & 3): all 32 distinct, one wavefront per load;
//   store: lane c writes pixels 4q..4q+3 as 16 B to row r = 32 j + c, 16-byte chunk q ^ (r & 7); the 8 lanes of each
//          quarter-warp phase have distinct r & 7, hence distinct chunks: the warp's 512 B take the minimum 4 wavefronts.
// Each warp loads kBatch items before it stores them, so that several loads are in flight.
template <int BN>
__device__ __forceinline__ void transpose_stage_tf32(const uint8_t* src, uint8_t* dst, int w, int lane) {
  constexpr int kItems = (128 + BN) / 32 * 8;
  constexpr int kBatch = 4;
  const int c = lane;
  for (int it0 = w; it0 < kItems; it0 += 8 * kBatch) {
    float v[kBatch][4];
#pragma unroll
    for (int b = 0; b < kBatch; ++b) {
      const int it = it0 + 8 * b;
      if (it < kItems) {
        const uint8_t* box = src + (it >> 3) * 4096;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int pix = 4 * (it & 7) + e;
          v[b][e] = *reinterpret_cast<const float*>(box + pix * 128 + (((c >> 2) ^ (pix & 7)) << 4) + (c & 3) * 4);
        }
      }
    }
#pragma unroll
    for (int b = 0; b < kBatch; ++b) {
      const int it = it0 + 8 * b;
      if (it < kItems) {
        const int r = 32 * (it >> 3) + c, q = it & 7;
        *reinterpret_cast<float4*>(dst + r * 128 + ((q ^ (r & 7)) << 4)) = make_float4(v[b][0], v[b][1], v[b][2], v[b][3]);
      }
    }
  }
}

// the shared-memory stages the consumers read (the TMA ring, or the K-major ring of a tf32 weight gradient)
struct Ring {
  uint8_t* base;
  uint32_t stride;
  int n;
  uint64_t* full;   // completes when a stage holds operands
  uint64_t* empty;  // one arrival per consumer warp when its wgmma have read the stage
};

// tf32 weight gradient: transpose the next TMA stage (raw ring position rs / rph) into the K-major ring at s / ph (the
// stage the consumers read next), then hand the TMA stage back
template <int BN>
__device__ __forceinline__ void xpose_next(const Ring& raw, int& rs, uint32_t& rph, const Ring& ring, int s, uint32_t ph) {
  const int lane = threadIdx.x & 31;
  mbar_wait(&raw.full[rs], rph);
  mbar_wait(&ring.empty[s], ph ^ 1u);   // both warpgroups' wgmma that read this K-major stage have completed
  transpose_stage_tf32<BN>(raw.base + (size_t)rs * raw.stride, ring.base + (size_t)s * ring.stride,
                           (threadIdx.x - 128) >> 5, lane);
  fence_proxy_async();   // generic-proxy stores -> visible to the wgmma (async proxy) that read them
  __syncwarp();
  if (lane == 0) {
    mbar_arrive(&raw.empty[rs]);
    mbar_arrive(&ring.full[s]);
  }
  if (++rs == raw.n) { rs = 0; rph ^= 1u; }
}

// One work unit of W output columns (W = BN for a whole tile, PN for a column piece): mainloop, split-K parking and
// epilogue.  s / ph: position in the ring, carried across units.  XP (tf32 weight gradient kernels) with p.wg_xpose:
// the consumers read the K-major ring and fill it themselves from the TMA ring (raw, position rs / rph): the transpose
// of stage i + 1 runs while the tensor cores work on the wgmma of stage i.
template <int DT, int TR, int W, bool XP>
__device__ __forceinline__ void consume_unit(const GemmParams& p, const TileCoord& tc, const Ring& ring, int& s,
                                             uint32_t& ph, const Ring& raw, int& rs, uint32_t& rph, float* st_buf,
                                             int* bcast) {
  const int ct = threadIdx.x - 128;          // 0..255
  const int g = ct >> 7;
  const int lane = threadIdx.x & 31;
  const int wl = (ct >> 5) & 3;
  const int cq = 2 * (lane & 3);             // first of the two columns this thread holds per 8-column block
  const bool f_stats = p.stats != nullptr;
  float acc[W / 2];
#pragma unroll
  for (int i = 0; i < W / 2; ++i) acc[i] = 0.f;
  const bool xp = XP && p.wg_xpose;
  if (xp && tc.nkb > 0) xpose_next<W>(raw, rs, rph, ring, s, ph);
  for (int i = 0; i < tc.nkb; ++i) {
    mbar_wait(&ring.full[s], ph);
    const uint32_t sa = smem_u32(ring.base + (size_t)s * ring.stride);
    const uint32_t sb = sa + kStageABytes;
    const uint64_t da = make_smem_desc(sa + (uint32_t)g * p.a_half, p.a_lbo, p.a_sbo);
    const uint64_t db = make_smem_desc(sb, p.b_lbo, p.b_sbo);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kMmasPerKb; ++k)
      wgmma_tile<DT, TR, W>(acc, da + (uint64_t)(k * p.a_kadv), db + (uint64_t)(k * p.b_kadv));
    wgmma_commit();
    // the previous k-block's wgmma have completed: hand its stage back
    wgmma_wait<1>();
    if (i > 0 && lane == 0) mbar_arrive(&ring.empty[s == 0 ? ring.n - 1 : s - 1]);
    if (++s == ring.n) { s = 0; ph ^= 1u; }
    if (xp && i + 1 < tc.nkb) xpose_next<W>(raw, rs, rph, ring, s, ph);
  }
  wgmma_wait<0>();
  if (tc.nkb > 0 && lane == 0) mbar_arrive(&ring.empty[s == 0 ? ring.n - 1 : s - 1]);

  // ---------------- split of a split-K tile: park the raw accumulators; the last split to arrive sums all of them
  // in split order
  if (tc.slice >= 0) {
    const int nsl = p.splits;
    float* ws = reinterpret_cast<float*>(p.tail_ws);
    const size_t slice_elems = (size_t)128 * 256;
    const size_t base = (size_t)tc.tail * nsl * slice_elems + ct;
    float* dst = ws + base + (size_t)tc.slice * slice_elems;
#pragma unroll
    for (int i = 0; i < W / 2; ++i) dst[(size_t)i * 256] = acc[i];
    __threadfence();
    consumer_sync();
    if (ct == 0) *bcast = atomicAdd(p.tail_cnt + tc.tail, 1);
    consumer_sync();
    const int old = *bcast;
    if (old != nsl - 1) return;          // another slice finishes this tile
    if (ct == 0) p.tail_cnt[tc.tail] = 0;       // self-cleaning for the next launch
    __threadfence();
    // slice by slice, each slice's W / 2 loads independent of one another: a loop over the slices inside the loop over
    // the elements waited out one L2 round trip per load (nsl * W / 2 of them in a row, ~0.15 ms at 16 splits).  Every
    // element is still summed in split order from slice 0, so the result is unchanged bit for bit.
    const float* src = ws + base;
#pragma unroll
    for (int i = 0; i < W / 2; ++i) acc[i] = __ldcg(src + (size_t)i * 256);
    for (int sl = 1; sl < nsl; ++sl) {
      const float* part = src + (size_t)sl * slice_elems;
#pragma unroll
      for (int i = 0; i < W / 2; ++i) acc[i] += __ldcg(part + (size_t)i * 256);
    }
  }

  // ---------------- epilogue: this thread holds rows r0 and r0 + 8, columns 8 j + cq, 8 j + cq + 1
  const int r0 = 64 * g + 16 * wl + (lane >> 2);
  long row[2];
  bool row_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m_local = r0 + 8 * h;
    if (p.mode == MODE_CONV) {
      const int n_img = tc.tile_m / p.tiles_per_img;
      const int r = tc.tile_m - n_img * p.tiles_per_img;
      const int th = r / p.tiles_w;
      const int oh = th * p.tile_h + m_local / p.tile_w;
      const int ow = (r - th * p.tiles_w) * p.tile_w + m_local % p.tile_w;
      row[h] = ((long)n_img * p.out_H + (long)oh * p.out_s + p.out_oh) * p.out_W + (long)ow * p.out_s + p.out_ow;
      row_ok[h] = oh < p.Ho && ow < p.Wo;
    } else {
      row[h] = (long)tc.tile_m * 128 + m_local;
      row_ok[h] = row[h] < p.M;
    }
  }
  int col_base = tc.col0;
  if (p.mode == MODE_WGRAD) {
    const int tap = tc.tile_n / p.wg_cin_blocks;
    col_base = tap * (p.wg_cin_blocks * p.block_n) + (tc.tile_n - tap * p.wg_cin_blocks) * p.block_n;
  }
  const __nv_bfloat16* res16 = reinterpret_cast<const __nv_bfloat16*>(p.residual);
  // The residual may be the output itself (an in-place sum), so the compiler may not move a residual load above an
  // earlier store: loaded one pair at a time, each load would wait out a full memory round trip.  The residual of
  // kResChunk column blocks is therefore loaded into registers before any of their stores (each thread reads only the
  // elements it writes itself), which keeps 4 * kResChunk loads in flight per thread.
  constexpr int kResChunk = 8;
  static_assert((W / 8) % kResChunk == 0, "residual chunks");
#pragma unroll
  for (int j0 = 0; j0 < W / 8; j0 += kResChunk) {
    float res[kResChunk][4];
    if (p.residual) {
#pragma unroll
      for (int jj = 0; jj < kResChunk; ++jj) {
        const int n = col_base + 8 * (j0 + jj) + cq;
        const bool two = n + 1 < p.N;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float r0 = 0.f, r1 = 0.f;
          if (n < p.N && row_ok[h]) {
            // bf16 output implies a bf16 residual (mixed-precision activations); fp32 otherwise
            const long ri = row[h] * p.ldr + n;
            if (p.out_bf16) {
              r0 = __bfloat162float(res16[ri]);
              if (two) r1 = __bfloat162float(res16[ri + 1]);
            } else {
              r0 = p.residual[ri];
              if (two) r1 = p.residual[ri + 1];
            }
          }
          res[jj][2 * h] = r0;
          res[jj][2 * h + 1] = r1;
        }
      }
    }
#pragma unroll
    for (int jj = 0; jj < kResChunk; ++jj) {
      const int j = j0 + jj;
      const int n = col_base + 8 * j + cq;
      float sm0 = 0.f, sm1 = 0.f, sq0 = 0.f, sq1 = 0.f;
      if (n < p.N) {
        const bool two = n + 1 < p.N;
        const float sc0 = p.scale ? __ldg(p.scale + n) : 1.f, sc1 = (p.scale && two) ? __ldg(p.scale + n + 1) : 1.f;
        const float bi0 = p.bias ? __ldg(p.bias + n) : 0.f, bi1 = (p.bias && two) ? __ldg(p.bias + n + 1) : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!row_ok[h]) continue;
          float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
          if (p.scale) { x0 *= sc0; x1 *= sc1; }
          if (p.bias) { x0 += bi0; x1 += bi1; }
          const long ro = row[h];
          if (p.residual) {
            x0 += res[jj][2 * h];
            if (two) x1 += res[jj][2 * h + 1];
          }
          if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          if (p.out_bf16) {
            __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.C) + ro * p.ldc + n;
            const __nv_bfloat162 h2 = __floats2bfloat162_rn(x0, x1);
            x0 = __low2float(h2);   // statistics of the values the consumer reads
            x1 = __high2float(h2);
            if (two && (reinterpret_cast<uintptr_t>(o) & 3) == 0) *reinterpret_cast<__nv_bfloat162*>(o) = h2;
            else { o[0] = __low2bfloat16(h2); if (two) o[1] = __high2bfloat16(h2); }
          } else {
            float* o = p.C + ro * p.ldc + n;
            if (p.atomic) {
              atomicAdd(o, x0);
              if (two) atomicAdd(o + 1, x1);
            } else if (two && (reinterpret_cast<uintptr_t>(o) & 7) == 0) {
              *reinterpret_cast<float2*>(o) = make_float2(x0, x1);
            } else {
              o[0] = x0;
              if (two) o[1] = x1;
            }
          }
          if (f_stats) {
            sm0 += x0; sq0 = fmaf(x0, x0, sq0);
            if (two) { sm1 += x1; sq1 = fmaf(x1, x1, sq1); }
          }
        }
      }
      if (f_stats) {
        // column sums over the warp's 16 rows (lanes with equal lane & 3 hold the same columns), then over the CTA
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          sm0 += __shfl_xor_sync(0xffffffffu, sm0, o);
          sm1 += __shfl_xor_sync(0xffffffffu, sm1, o);
          sq0 += __shfl_xor_sync(0xffffffffu, sq0, o);
          sq1 += __shfl_xor_sync(0xffffffffu, sq1, o);
        }
        if (lane < 4) {
          // this warp's partial sums; summed over the 8 warps in a fixed order below (deterministic forward pass)
          float* w = st_buf + (ct >> 5) * 512 + 8 * j + cq;
          w[0] = sm0; w[1] = sm1; w[256] = sq0; w[257] = sq1;
        }
      }
    }
  }
  if (f_stats) {
    consumer_sync();
    if (ct < W && col_base + ct < p.N) {
      float a = 0.f, b = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) { a += st_buf[w * 512 + ct]; b += st_buf[w * 512 + 256 + ct]; }
      if (a != 0.f || b != 0.f) {
        atomicAdd(p.stats + col_base + ct, (double)a);
        atomicAdd(p.stats + p.N + col_base + ct, (double)b);
      }
    }
    consumer_sync();   // the slots are rewritten by the next tile
  }
}

// Persistent: each CTA walks work units blockIdx.x, blockIdx.x + gridDim.x, ...; the shared-memory ring runs across
// tile boundaries, so the producer loads the next tile's operands while the consumers run this tile's epilogue.
// MN = 1: WGRAD operands (MN-major, or K-major copies in tf32, see WgradFeed).  BN: tile width; PN: width of a tail
// tile's column pieces (0: no pieces).
template <int DT, int MN, int BN, int PN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
               const __grid_constant__ CUtensorMap tma_bp, const __grid_constant__ GemmParams p) {
  constexpr bool kXposeOk = MN == 1 && DT == DT_TF32;
  const bool xpose = kXposeOk && p.wg_xpose;
  constexpr uint32_t kStageBytes = kStageABytes + BN * 128u;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages x (A 16KB | B BN*128B)] | [wg_xpose: kXStages K-major stages] | statistics 16 KB | barriers
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* xbuf = smem + (size_t)p.stages * kStageBytes;
  float* st_buf = reinterpret_cast<float*>(xbuf + (xpose ? kXStages * kStageBytes : 0u));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(st_buf) + kStatsBytes);
  uint64_t* empty_bar = full_bar + p.stages;
  uint64_t* xfull_bar = empty_bar + p.stages;     // K-major ring of wg_xpose
  uint64_t* xempty_bar = xfull_bar + kXStages;
  int* bcast = reinterpret_cast<int*>(xempty_bar + kXStages);

  const int warp = threadIdx.x >> 5;
  const int total_whole = p.tiles_m * p.tiles_n * p.splits;
  const int tail_mult = p.tail_p > 0 ? p.tail_p : 1;
  const int total_units = p.tail_first + (total_whole - p.tail_first) * tail_mult;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    if (PN > 0 && p.tail_p > 0) tma_prefetch_desc(&tma_bp);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrival per consumer warp
    }
    if (xpose) {
      for (int s = 0; s < kXStages; ++s) {
        mbar_init(&xfull_bar[s], 8);
        mbar_init(&xempty_bar[s], 8);
      }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // =============================== TMA producer.  Warp 0 walks the (warp-uniform) loops so that indices and
    // coordinates live in uniform registers; one elected lane issues the copies.
    setmaxnreg_dec<40>();
    if (warp == 0) {
      const bool leader = elect_one();
      const int E = p.elems_per_128B;
      int s = 0;          // ring slot / phase, carried across tiles
      uint32_t ph = 0;
      for (int t = blockIdx.x; t < total_units; t += gridDim.x) {
        const TileCoord tc = tile_coord(p, t);
        int n_img = 0, oh0 = 0, ow0 = 0;
        if (p.mode == MODE_CONV) {
          n_img = tc.tile_m / p.tiles_per_img;
          const int r = tc.tile_m - n_img * p.tiles_per_img;
          const int th = r / p.tiles_w;
          oh0 = th * p.tile_h;
          ow0 = (r - th * p.tiles_w) * p.tile_w;
        }
        int wg_tap = 0, wg_ci0 = 0;
        if (p.mode == MODE_WGRAD) {
          wg_tap = tc.tile_n / p.wg_cin_blocks;
          wg_ci0 = (tc.tile_n - wg_tap * p.wg_cin_blocks) * p.block_n;
        }
        for (int i = 0; i < tc.nkb; ++i) {
          mbar_wait(&empty_bar[s], ph ^ 1u);
          uint8_t* sa = smem + (size_t)s * kStageBytes;
          uint8_t* sb = sa + kStageABytes;
          const int kb = tc.split * p.num_kb + tc.kb0 + i;
          if (!leader) {
            // nothing to issue
          } else if (p.mode == MODE_GEMM) {
            mbar_expect_tx(&full_bar[s], tc.piece ? (uint32_t)(kStageABytes + tc.ncols * 128) : p.stage_tx_bytes);
            tma_load_4d(sa, &tma_a, &full_bar[s], kb * E, tc.tile_m * 128, 0, 0);
            tma_load_4d(sb, tc.piece ? &tma_bp : &tma_b, &full_bar[s], kb * E, tc.col0, 0, 0);
          } else if (p.mode == MODE_CONV) {
            mbar_expect_tx(&full_bar[s], tc.piece ? (uint32_t)(kStageABytes + tc.ncols * 128) : p.stage_tx_bytes);
            const int tap = kb / p.cblocks, cb = kb - tap * p.cblocks;
            tma_load_4d(sa, &tma_a, &full_bar[s], cb * E, ow0 * p.conv_stride + p.tap_dw[tap],
                        oh0 * p.conv_stride + p.tap_dh[tap], n_img);
            tma_load_4d(sb, tc.piece ? &tma_bp : &tma_b, &full_bar[s], kb * E, tc.col0, 0, 0);
          } else if (DT == DT_TF32 && !p.wg_xpose) {
            // WGRAD from the K-major copies: k-block = kp = 32 consecutive output pixels = one 128-byte row of dY^T
            // (A: 128 output channels) and of X^T (B: BN rows of one tap)
            mbar_expect_tx(&full_bar[s], p.stage_tx_bytes);
            const int pix0 = kb * p.kp;
            tma_load_4d(sa, &tma_a, &full_bar[s], pix0, tc.tile_m * 128, 0, 0);
            // the TMA takes 16-byte aligned starts along a map's first dimension: the pixel coordinate stays a multiple
            // of 32, the tap's column offset is its row block
            const int img = pix0 / (p.Ho * p.Wo);
            const int rem = pix0 - img * (p.Ho * p.Wo);
            const int oh = rem / p.Wo, ow = rem - oh * p.Wo;
            const int xpix = (img * p.wg_hp + oh + p.tap_dh[wg_tap] + p.wg_padh) * p.Wo + ow;
            tma_load_4d(sb, &tma_b, &full_bar[s], xpix, p.wg_tapblk[wg_tap] * p.wg_cin_blocks * p.block_n + wg_ci0, 0, 0);
          } else {
            // bf16 / wg_xpose WGRAD: k-block = kp consecutive output pixels of one image row block, MN-major boxes
            mbar_expect_tx(&full_bar[s], p.stage_tx_bytes);
            const int pix0 = kb * p.kp;
            const int img = pix0 / (p.Ho * p.Wo);
            const int rem = pix0 - img * (p.Ho * p.Wo);
            const int oh = rem / p.Wo, ow = rem - oh * p.Wo;
            for (int j = 0; j < p.a_boxes; ++j)
              tma_load_4d(sa + (size_t)j * p.a_box_bytes, &tma_a, &full_bar[s], tc.tile_m * 128 + j * E, pix0, 0, 0);
            for (int j = 0; j < p.b_boxes; ++j)
              tma_load_4d(sb + (size_t)j * p.b_box_bytes, &tma_b, &full_bar[s], wg_ci0 + j * E,
                          ow * p.conv_stride + p.tap_dw[wg_tap], oh * p.conv_stride + p.tap_dh[wg_tap], img);
          }
          if (++s == p.stages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // =============================== consumers: warpgroup g = 0 / 1 owns rows 64 g .. 64 g + 63 of the tile
  setmaxnreg_inc<232>();
  const Ring raw{smem, kStageBytes, p.stages, full_bar, empty_bar};
  const Ring ring = xpose ? Ring{xbuf, kStageBytes, kXStages, xfull_bar, xempty_bar} : raw;
  constexpr int kTR = DT == DT_TF32 ? 0 : MN;    // tf32 weight gradients are consumed K-major
  int s = 0, rs = 0;
  uint32_t ph = 0, rph = 0;
  for (int t = blockIdx.x; t < total_units; t += gridDim.x) {
    const TileCoord tc = tile_coord(p, t);
    if constexpr (PN > 0) {
      if (tc.piece) {
        consume_unit<DT, kTR, PN, false>(p, tc, ring, s, ph, raw, rs, rph, st_buf, bcast);
        continue;
      }
    }
    consume_unit<DT, kTR, BN, kXposeOk>(p, tc, ring, s, ph, raw, rs, rph, st_buf, bcast);
  }
}

// ---------------------------------------------------------------- tf32 weight gradient: channel-major operand copies
// dst[t * C + c, p] = src[n, oh + dh[t], ow + dw[t], c] for pixel p = (n, oh, ow) of an NB x Ho x Wo grid, zero outside
// the map: the fp32 bits unchanged.  dY^T is the identity gather (one tap, H = Ho, W = Wo).
struct XposeJob {
  const float* src;
  long ld;                // source pixel row stride (elements)
  float* dst;
  long pitch;             // destination row stride (elements, a multiple of 4)
  int C;                  // channels per tap (a multiple of 32)
  int rows;               // destination rows = taps * C (X^T: one tap per row block)
  int P;                  // destination pixels = NB * Ho * Wo
  int H, W, Ho, Wo;
  int dh[kMaxTaps], dw[kMaxTaps];
};
struct XposeParams {
  XposeJob job[2];        // dY^T, X^T
  int split;              // blockIdx.y < split: 32-row blocks of job 0
};

constexpr int kXpPix = 64;   // pixels per copy block; channel rows per block: 32

// 256 threads per 32 rows x 64 pixels: 16-byte loads along channels (8 lanes read one pixel's 128 B), 16-byte stores
// along pixels (16 lanes write one row's 256 B)
__global__ void __launch_bounds__(256) wgrad_xpose_kernel(const __grid_constant__ XposeParams xp) {
  __shared__ __align__(16) float tile[32][kXpPix + 4];
  int rb = blockIdx.y;
  const XposeJob& j = rb < xp.split ? xp.job[0] : xp.job[1];
  if (rb >= xp.split) rb -= xp.split;
  const int p0 = blockIdx.x * kXpPix;
  if (p0 >= j.P) return;
  const int row0 = rb * 32;
  const int t = row0 / j.C, c0 = row0 - t * j.C;
  const int hw = j.Ho * j.Wo;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = threadIdx.x + 256 * r;
    const int pl = i >> 3, q = i & 7;
    const int pix = p0 + pl;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pix < j.P) {
      const int n = pix / hw, rem = pix - n * hw;
      const int oh = rem / j.Wo, ow = rem - oh * j.Wo;
      const int ih = oh + j.dh[t], iw = ow + j.dw[t];
      if (ih >= 0 && ih < j.H && iw >= 0 && iw < j.W)
        v = __ldg(reinterpret_cast<const float4*>(j.src + (((long)n * j.H + ih) * j.W + iw) * j.ld + c0 + 4 * q));
    }
    tile[4 * q + 0][pl] = v.x;
    tile[4 * q + 1][pl] = v.y;
    tile[4 * q + 2][pl] = v.z;
    tile[4 * q + 3][pl] = v.w;
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = threadIdx.x + 256 * r;
    const int row = i >> 4, pq = 4 * (i & 15);
    // pixels P..pitch-1 of a row are padding (never read through the TMA maps): a ragged last quad may write them
    if (p0 + pq < j.P)
      *reinterpret_cast<float4*>(j.dst + (long)(row0 + row) * j.pitch + p0 + pq) =
          *reinterpret_cast<const float4*>(&tile[row][pq]);
  }
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}


// 4-D tiled map, 128B swizzle; dims/strides innermost first; strides in bytes for dims 1..3
int make_map(CUtensorMap* m, int dtype, const void* base, const uint64_t dims[4], const uint64_t strides_bytes[3],
             const uint32_t box[4], const uint32_t estr[4]) {
  EncodeTiledFn enc = get_encode();
  SN_CHECK(enc != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t gd[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gs[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t es[4] = {estr[0], estr[1], estr[2], estr[3]};
  CUresult r = enc(m, dtype == DT_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                   const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SN_CHECK(r == CUDA_SUCCESS,
           "cuTensorMapEncodeTiled failed (%d): dims=%llu,%llu,%llu,%llu strides=%llu,%llu,%llu box=%u,%u,%u,%u es=%u,%u,%u,%u",
           (int)r, (unsigned long long)gd[0], (unsigned long long)gd[1], (unsigned long long)gd[2],
           (unsigned long long)gd[3], (unsigned long long)gs[0], (unsigned long long)gs[1], (unsigned long long)gs[2],
           bx[0], bx[1], bx[2], bx[3], es[0], es[1], es[2], es[3]);
  return 0;
}

constexpr int kSmemMax = 227 * 1024;       // opt-in dynamic shared memory per block (H100)
constexpr int kSmemFixed = 1024 + kStatsBytes + 512;   // alignment slack, statistics, barriers

// one persistent CTA per SM: fill shared memory with the operand ring (wg_xpose weight gradients also keep kXStages
// K-major stages for the transposed operands; at block_n = 256 that leaves a 2-stage TMA ring)
int pick_stages(int block_n, int xpose = 0) {
  const int stage = kStageABytes + block_n * 128;
  const int s = (kSmemMax - kSmemFixed) / stage - (xpose ? kXStages : 0);
  return s > 8 ? 8 : s;
}

size_t smem_bytes(int stages, int block_n, int xpose) {
  return (size_t)(stages + (xpose ? kXStages : 0)) * (kStageABytes + block_n * 128) + kSmemFixed;
}

// Decide the tail split of a K-major launch (see GemmParams::tail_*).  SNIPER_GEMM_TAIL=0 disables it.  Only for
// widths that are a multiple of 32 columns (every layer of the training step; ragged widths keep whole tiles).
// (A K-slice split of the tail is not offered: its parked partials made graph-replayed steps differ run to run in
// the last bits, which the proposal stage amplifies across training steps.)
void plan_tail(GemmParams& p, long tiles, long grid_units) {
  p.tail_p = 0; p.tail_first = (int)tiles;
  if (p.split_park) return;   // the split-K workspace is already assigned
  p.tail_ws = nullptr; p.tail_cnt = nullptr;
  const char* e = getenv("SNIPER_GEMM_TAIL");   // 0 = off, otherwise (default) column pieces
  const int mode = e ? atoi(e) : 2;
  if (mode == 0) return;
  if (p.mode == MODE_WGRAD || p.N % 32 != 0 || p.splits != 1) return;
  const long tail = tiles % grid_units;
  if (tail == 0 || tail * 2 > grid_units) return;
  if (p.block_n == 256 && tiles > grid_units) {
    // column pieces: 4 x 64 columns if they fit one wave, else 2 x 128
    p.tail_p = tail * 4 <= grid_units ? 4 : 2;
    p.tail_first = (int)(tiles - tail);
  }
}

// K-major B operand [N rows, K] as launch() needs it to build the TMA map of a column piece
struct BOperand {
  const void* ptr;
  uint64_t K, N, ld_bytes;
};

int launch(const CUtensorMap& ma, const CUtensorMap& mb, GemmParams& p, dim3 tiles, cudaStream_t stream,
           const BOperand* bop = nullptr) {
  CUtensorMap mbp;
  memset(&mbp, 0, sizeof(mbp));
  p.tiles_m = (int)tiles.x; p.tiles_n = (int)tiles.y; p.splits = (int)tiles.z;
  long units = (long)tiles.x * tiles.y * tiles.z;
  const long max_units = sn::kNumSMs;
  plan_tail(p, units, max_units);
  if (p.tail_p > 0 && !bop) { p.tail_p = 0; p.tail_first = (int)units; }
  if (p.tail_p > 0) {
    const uint64_t d[4] = {bop->K, bop->N, 1, 1};
    const uint64_t st[3] = {bop->ld_bytes, bop->ld_bytes * bop->N, bop->ld_bytes * bop->N};
    const uint32_t b[4] = {(uint32_t)p.elems_per_128B, (uint32_t)(p.block_n / p.tail_p), 1, 1};
    const uint32_t ones[4] = {1, 1, 1, 1};
    if (make_map(&mbp, p.dtype, bop->ptr, d, st, b, ones)) return -1;
  }
  if (p.tail_p > 0) units = p.tail_first + (units - p.tail_first) * p.tail_p;
  const size_t smem = smem_bytes(p.stages, p.block_n, p.wg_xpose);
  typedef void (*KernelFn)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const GemmParams);
  // every instantiation: operand type, MN-major operands, tile width, column-piece width (tail splits of 256-wide
  // K-major tiles only)
  struct Instance { int dt, mn, bn, pn; KernelFn fn; };
  static const Instance kernels[] = {
      {DT_TF32, 0, 64, 0, gemm_tc_kernel<DT_TF32, 0, 64, 0>},     {DT_TF32, 0, 128, 0, gemm_tc_kernel<DT_TF32, 0, 128, 0>},
      {DT_TF32, 0, 256, 0, gemm_tc_kernel<DT_TF32, 0, 256, 0>},   {DT_TF32, 0, 256, 64, gemm_tc_kernel<DT_TF32, 0, 256, 64>},
      {DT_TF32, 0, 256, 128, gemm_tc_kernel<DT_TF32, 0, 256, 128>},
      {DT_TF32, 1, 64, 0, gemm_tc_kernel<DT_TF32, 1, 64, 0>},     {DT_TF32, 1, 128, 0, gemm_tc_kernel<DT_TF32, 1, 128, 0>},
      {DT_TF32, 1, 256, 0, gemm_tc_kernel<DT_TF32, 1, 256, 0>},
      {DT_BF16, 0, 64, 0, gemm_tc_kernel<DT_BF16, 0, 64, 0>},     {DT_BF16, 0, 128, 0, gemm_tc_kernel<DT_BF16, 0, 128, 0>},
      {DT_BF16, 0, 256, 0, gemm_tc_kernel<DT_BF16, 0, 256, 0>},   {DT_BF16, 0, 256, 64, gemm_tc_kernel<DT_BF16, 0, 256, 64>},
      {DT_BF16, 0, 256, 128, gemm_tc_kernel<DT_BF16, 0, 256, 128>},
      {DT_BF16, 1, 64, 0, gemm_tc_kernel<DT_BF16, 1, 64, 0>},     {DT_BF16, 1, 128, 0, gemm_tc_kernel<DT_BF16, 1, 128, 0>},
      {DT_BF16, 1, 256, 0, gemm_tc_kernel<DT_BF16, 1, 256, 0>}};
  constexpr int kNumKernels = (int)(sizeof(kernels) / sizeof(kernels[0]));
  // per-device one-time setup (a process may drive several GPUs)
  static bool attr_done[64] = {false};
  int dev = 0;
  SN_CUDA(cudaGetDevice(&dev));
  if (dev >= 0 && dev < 64 && !attr_done[dev]) {
    for (int i = 0; i < kNumKernels; ++i)
      SN_CUDA(cudaFuncSetAttribute(kernels[i].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
    attr_done[dev] = true;
  }
  const int mn = p.mode == MODE_WGRAD ? 1 : 0, pn = p.tail_p > 0 ? p.block_n / p.tail_p : 0;
  KernelFn fn = nullptr;
  for (int i = 0; i < kNumKernels; ++i)
    if (kernels[i].dt == p.dtype && kernels[i].mn == mn && kernels[i].bn == p.block_n && kernels[i].pn == pn)
      fn = kernels[i].fn;
  SN_CHECK(fn != nullptr, "gemm: no kernel for block_n %d with %d-column tail pieces", p.block_n, pn);
  const unsigned grid = (unsigned)(units < max_units ? units : max_units);
  fn<<<grid, kThreads, smem, stream>>>(ma, mb, mbp, p);
  SN_LAUNCH_CHECK();
  return 0;
}

// Tile width: wide tiles move fewer L2 -> shared-memory bytes per flop (a 128 x 128 tile moves 1.33x the bytes per
// flop of a 128 x 256 tile), so 256 columns wherever N allows it.
int pick_block_n(int N) {
  if (N <= 128) return N <= 64 ? 64 : 128;
  if (N % 256 == 0 || N > 1024) return 256;
  return 128;
}

// K-major operands, 128B swizzle: rows of 128 B, 8-row groups 1024 B apart (SBO); one wgmma consumes 32 B of K
void fill_kmajor(GemmParams& p, int dtype, int block_n) {
  p.dtype = dtype;
  p.block_n = block_n;
  p.elems_per_128B = dtype == DT_TF32 ? 32 : 64;
  p.a_lbo = 1; p.a_sbo = 64; p.b_lbo = 1; p.b_sbo = 64;
  p.a_kadv = 2; p.b_kadv = 2;
  p.a_half = 64 * 128;                                   // the second consumer's rows 64..127
  p.a_boxes = 1; p.b_boxes = 1;
  p.a_box_bytes = kStageABytes;
  p.b_box_bytes = (uint32_t)block_n * 128u;
  p.stage_tx_bytes = kStageABytes + p.b_box_bytes;
  p.stages = pick_stages(block_n);
}

// tf32 weight gradient operand feed.  wgmma reads tf32 K-major only and both operands are pixel-major.  For stride-1
// layers with several taps whose output rows are Wo % 32 == 0 pixels (the 3 x 3 layers of the ResNet-101 step), a copy
// kernel first writes them channel-major into the copy area of the stream's workspace:
//   dY^T [Cout, P], P = NB * Ho * Wo output pixels in k-block order;
//   X^T  [cols * Cin, NB * Hp * Wo]: one row block per distinct column offset dw of the taps, X^T[j * Cin + ci,
//        (n, hp, ow)] = X[n, hp - padh, ow + dw_j, ci] over the input rows zero-padded to Hp (padh before the first), so
//        that tap (dh, dw_j) of the k-block at (n, oh, ow) is the 32 pixels from (n, oh + dh + padh, ow) of row block j.
// Both are read through 2-D maps {pixels, rows} with boxes of 32 pixels x 128 / BN rows at pixel coordinates that are
// multiples of 32 (the TMA needs 16-byte aligned starts along the first dimension, which rules out shifting a box by
// dw).  Row pitches are rounded up to 16 bytes.  The k-block composition (32 consecutive output pixels, wgmma k-step j
// covering pixels 8 j .. 8 j + 7) is that of the transposing path, so both give the same bits.  Other layers keep the
// in-kernel transpose (wg_xpose): for 1 x 1 layers the copies' HBM traffic measured slower than the transpose, and a
// tap-gathered copy (taps x the input bytes) left the stride-2 layers of the ResNet-101 step no faster and slowed the
// MobileNetV2 step, whose RPN 3 x 3 runs on a 16-pixel-wide map.
struct WgradFeed {
  int padh, hp;               // zero rows before the first input row, padded height
  int blocks;                 // row blocks of Cin rows: distinct dw
  int blk_dw[kMaxTaps];       // column offset of each row block
  int tapblk[kMaxTaps];       // row block each tap reads
  long x_pixels;              // pixels per X^T row
  long p_pitch, x_pitch;      // elements per row of dY^T / X^T
  size_t xt_off, bytes;       // X^T offset in the copy area (256-byte aligned), total bytes
};

bool wgrad_copies(int dtype, int ntaps, int stride, int Wo) {
  return dtype == DT_TF32 && ntaps > 1 && stride == 1 && Wo % 32 == 0;
}

WgradFeed wgrad_feed(int NB, int H, int Cin, int Cout, int ntaps, const int* tap_dh, const int* tap_dw, int Ho,
                     int Wo) {
  WgradFeed f;
  memset(&f, 0, sizeof(f));
  const long P = (long)NB * Ho * Wo;
  int lo = 0, hi = 0;
  for (int t = 0; t < ntaps; ++t) {
    lo = std::max(lo, -tap_dh[t]);
    hi = std::max(hi, Ho - 1 + tap_dh[t] - (H - 1));
    int j = 0;
    while (j < f.blocks && f.blk_dw[j] != tap_dw[t]) ++j;
    if (j == f.blocks) f.blk_dw[f.blocks++] = tap_dw[t];
    f.tapblk[t] = j;
  }
  f.padh = lo;
  f.hp = H + lo + hi;
  f.x_pixels = (long)NB * f.hp * Wo;
  f.p_pitch = (P + 3) / 4 * 4;
  f.x_pitch = (f.x_pixels + 3) / 4 * 4;
  f.xt_off = ((size_t)Cout * f.p_pitch * 4 + 255) / 256 * 256;
  f.bytes = f.xt_off + (size_t)f.blocks * Cin * f.x_pitch * 4;
  return f;
}

struct Epilogue {
  const float* scale;
  const float* bias;
  const float* residual;
  long ldr;
  int relu;
  int atomic;
  int out_bf16;
};

}  // namespace

extern "C" {

// C[M,N] (ldc) = epilogue(A[M,K] (lda) * B[N,K]^T (ldb)).  dtype 0: fp32 storage / TF32 math, 1: bf16.
// K must be a multiple of 32 (tf32) / 64 (bf16) elements; lda/ldb in elements, 16-byte aligned rows.
int sniper_gemm_nt(const void* A, long lda, const void* B, long ldb, float* C, long ldc, int M, int N, int K,
                   int dtype, const float* scale, const float* bias, const float* residual, long ldr, int relu,
                   int accumulate, int out_bf16, double* stats, void* stream) {
  SN_CHECK(dtype == DT_TF32 || dtype == DT_BF16, "gemm: dtype must be 0 (tf32) or 1 (bf16)");
  const int esz = dtype == DT_TF32 ? 4 : 2;
  const int E = 128 / esz;
  SN_CHECK(K % E == 0 && K > 0, "gemm: K (%d) must be a positive multiple of %d", K, E);
  SN_CHECK(M > 0 && N > 0, "gemm: empty problem");
  SN_CHECK((lda * esz) % 16 == 0 && (ldb * esz) % 16 == 0, "gemm: row strides must be 16-byte multiples");
  SN_CHECK(!(accumulate && out_bf16), "gemm: accumulate needs an fp32 output (bf16 outputs are stored, not added to)");
  GemmParams p;
  memset(&p, 0, sizeof(p));
  const int bn = pick_block_n(N);
  fill_kmajor(p, dtype, bn);
  p.mode = MODE_GEMM; p.M = M; p.N = N; p.num_kb = K / E;
  p.C = C; p.ldc = ldc; p.scale = scale; p.bias = bias; p.residual = residual; p.ldr = ldr; p.relu = relu;
  p.atomic = accumulate; p.out_bf16 = out_bf16; p.stats = stats;
  CUtensorMap ma, mb;
  const uint32_t ones[4] = {1, 1, 1, 1};
  {
    const uint64_t d[4] = {(uint64_t)K, (uint64_t)M, 1, 1};
    const uint64_t s[3] = {(uint64_t)lda * esz, (uint64_t)lda * esz * M, (uint64_t)lda * esz * M};
    const uint32_t b[4] = {(uint32_t)E, 128, 1, 1};
    if (make_map(&ma, dtype, A, d, s, b, ones)) return -1;
  }
  {
    const uint64_t d[4] = {(uint64_t)K, (uint64_t)N, 1, 1};
    const uint64_t s[3] = {(uint64_t)ldb * esz, (uint64_t)ldb * esz * N, (uint64_t)ldb * esz * N};
    const uint32_t b[4] = {(uint32_t)E, (uint32_t)bn, 1, 1};
    if (make_map(&mb, dtype, B, d, s, b, ones)) return -1;
  }
  dim3 grid(sn::div_up(M, 128), sn::div_up(N, bn), 1);
  const BOperand bop = {B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * esz};
  return launch(ma, mb, p, grid, (cudaStream_t)stream, &bop);
}

// NHWC implicit-GEMM convolution forward (also used for stride-1 data gradients with flipped weights):
//   Y[n,oh,ow,co] = epi( sum_{t<ntaps, c<Cin} X[n, oh*stride + dh[t], ow*stride + dw[t], c] * Wt[co, t*Cin + c] )
// X: [NB,H,W,Cin] contiguous; Wt: [Cout, ntaps*Cin]; Y row (n,oh,ow) is written at
// ((n*out_H + oh*out_s + out_oh)*out_W + ow*out_s + out_ow) * ldc.  Out-of-range taps read zeros (TMA fill).
int sniper_conv2d_nhwc(const void* X, long x_ld, int NB, int H, int W, int Cin, const void* Wt, int Cout, int ntaps,
                       const int* tap_dh, const int* tap_dw, int stride, int Ho, int Wo, float* Y, long ldc,
                       int out_H, int out_W, int out_s, int out_oh, int out_ow, int dtype, const float* scale,
                       const float* bias, const float* residual, long ldr, int relu, int accumulate, int out_bf16,
                       double* stats, void* stream) {
  SN_CHECK(dtype == DT_TF32 || dtype == DT_BF16, "conv: dtype must be 0 (tf32) or 1 (bf16)");
  const int esz = dtype == DT_TF32 ? 4 : 2;
  const int E = 128 / esz;
  SN_CHECK(Cin % E == 0, "conv: Cin (%d) must be a multiple of %d", Cin, E);
  SN_CHECK(ntaps >= 1 && ntaps <= kMaxTaps, "conv: ntaps (%d) out of range", ntaps);
  SN_CHECK(stride == 1 || stride == 2, "conv: stride must be 1 or 2");
  SN_CHECK(!(accumulate && out_bf16), "conv: accumulate needs an fp32 output (bf16 outputs are stored, not added to)");
  // 128 output pixels per tile as tile_h rows x tile_w columns, tile_w = the largest power of two <= 128 dividing Wo
  // (training shapes: Wo = 32 ... 128 -> whole rows; inference canvases of any width that is a multiple of 8 pixels at
  // this layer's stride: narrower, taller tiles; rows past Ho are zero-filled by the TMA and not stored)
  int tile_w = 128;
  while (tile_w > 1 && Wo % tile_w != 0) tile_w >>= 1;
  SN_CHECK(tile_w >= 8, "conv: Wo (%d) must be a multiple of 8", Wo);
  int tile_h = 128 / tile_w;
  SN_CHECK(tile_w * stride <= 256, "conv: TMA box too wide");
  GemmParams p;
  memset(&p, 0, sizeof(p));
  const int bn = pick_block_n(Cout);
  fill_kmajor(p, dtype, bn);
  p.mode = MODE_CONV; p.N = Cout; p.cblocks = Cin / E; p.ntaps = ntaps; p.num_kb = ntaps * p.cblocks;
  for (int t = 0; t < ntaps; ++t) { p.tap_dh[t] = tap_dh[t]; p.tap_dw[t] = tap_dw[t]; }
  p.conv_stride = stride; p.tile_w = tile_w; p.tile_h = tile_h;
  p.tiles_w = Wo / tile_w; p.tiles_per_img = p.tiles_w * sn::div_up(Ho, tile_h);
  p.Ho = Ho; p.Wo = Wo; p.M = NB * Ho * Wo;
  p.C = Y; p.ldc = ldc; p.scale = scale; p.bias = bias; p.residual = residual; p.ldr = ldr; p.relu = relu;
  p.atomic = accumulate; p.out_bf16 = out_bf16; p.stats = stats;
  p.out_H = out_H; p.out_W = out_W; p.out_s = out_s; p.out_oh = out_oh; p.out_ow = out_ow;
  CUtensorMap ma, mb;
  {
    SN_CHECK(x_ld >= Cin && (x_ld * esz) % 16 == 0, "conv: bad x_ld");
    const uint64_t d[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
    const uint64_t s[3] = {(uint64_t)x_ld * esz, (uint64_t)x_ld * esz * W, (uint64_t)x_ld * esz * W * H};
    // with elementStrides the box extent is in un-strided elements
    const uint32_t b[4] = {(uint32_t)E, (uint32_t)(tile_w * stride), (uint32_t)(tile_h * stride), 1};
    const uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
    if (make_map(&ma, dtype, X, d, s, b, es)) return -1;
  }
  {
    const uint64_t K = (uint64_t)ntaps * Cin;
    const uint64_t d[4] = {K, (uint64_t)Cout, 1, 1};
    const uint64_t s[3] = {K * esz, K * esz * Cout, K * esz * Cout};
    const uint32_t b[4] = {(uint32_t)E, (uint32_t)bn, 1, 1};
    const uint32_t ones[4] = {1, 1, 1, 1};
    if (make_map(&mb, dtype, Wt, d, s, b, ones)) return -1;
  }
  dim3 grid(NB * p.tiles_per_img, sn::div_up(Cout, bn), 1);
  const BOperand bop = {Wt, (uint64_t)ntaps * Cin, (uint64_t)Cout, (uint64_t)ntaps * Cin * esz};
  return launch(ma, mb, p, grid, (cudaStream_t)stream, &bop);
}

// Weight gradient:  dW[co, t*Cin + ci] += sum_{n,oh,ow} dY[(n,oh,ow), co] * X[n, oh*stride+dh[t], ow*stride+dw[t], ci]
// dY: [NB*Ho*Wo, Cout] contiguous rows (ld = Cout); X: [NB,H,W,Cin]; the result is added to dW (zero it for a plain
// weight gradient).  Split-K partials are summed in split order, so the result does not depend on CTA timing.  ntaps = 1, dh=dw=0, H=Ho, W=Wo gives dY^T * X (FC layers).
int sniper_conv2d_wgrad_nhwc(const void* dY, long dy_ld, const void* X, long x_ld, int NB, int H, int W, int Cin,
                             int Cout, int ntaps,
                             const int* tap_dh, const int* tap_dw, int stride, int Ho, int Wo, float* dW, int dtype,
                             int splits, void* stream) {
  SN_CHECK(dtype == DT_TF32 || dtype == DT_BF16, "wgrad: dtype must be 0 (tf32) or 1 (bf16)");
  const int esz = dtype == DT_TF32 ? 4 : 2;
  const int E = 128 / esz;       // elements per 128-byte MN chunk
  const int kp = dtype == DT_TF32 ? 32 : 64;  // pixels per k-block
  SN_CHECK(Cin % 64 == 0, "wgrad: Cin (%d) must be a multiple of 64", Cin);
  SN_CHECK(Cout % E == 0, "wgrad: Cout (%d) must be a multiple of %d", Cout, E);
  SN_CHECK(ntaps >= 1 && ntaps <= kMaxTaps, "wgrad: ntaps out of range");
  const long pixels = (long)NB * Ho * Wo;
  // k-blocks are kp consecutive output pixels.  Either they tile rows exactly, or the problem is a single
  // row (NB == 1, Ho == 1: FC layers viewed as [1,1,N,C]) where the tail is zero-filled by TMA.
  const bool single_row = (NB == 1 && Ho == 1);
  SN_CHECK(single_row || ((Wo % kp == 0 || kp % Wo == 0) && pixels % kp == 0 && (Wo >= kp || (Ho * Wo) % kp == 0)),
           "wgrad: output %dx%d does not tile by %d pixels", Ho, Wo, kp);
  const int bw = Wo >= kp ? kp : Wo, bh = kp / bw;
  // wide N tiles halve the operand traffic per flop of the 128 x 128 tile and the number of split-K atomics
  const int bn = Cin % 256 == 0 ? 256 : (Cin % 128 == 0 ? 128 : 64);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.mode = MODE_WGRAD; p.dtype = dtype; p.block_n = bn; p.elems_per_128B = E;
  p.M = Cout; p.N = ntaps * Cin;
  const uint32_t chunk_bytes = (uint32_t)kp * 128u;
  const bool copies = wgrad_copies(dtype, ntaps, stride, Wo);
  p.wg_xpose = dtype == DT_TF32 && !copies;
  if (dtype == DT_TF32) {
    // K-major stages, A = 128 dY channel rows, B = BN X channel rows, 32 pixels (128 B) each: loaded so from the
    // channel-major copies (WgradFeed), or transposed by the consumers from MN-major boxes (see transpose_stage_tf32)
    p.a_lbo = 1; p.a_sbo = 64; p.b_lbo = 1; p.b_sbo = 64;
    p.a_kadv = 2; p.b_kadv = 2;
    p.a_half = 64 * 128;
  } else {
    // MN-major, 128B swizzle: LBO = stride between 64-element MN atoms (one TMA box of kp pixel rows), SBO = stride
    // between 8-pixel-row groups; one wgmma consumes 16 pixel rows (2 KB), kMmasPerKb of them the kp = 64 pixels of a
    // k-block; the second consumer's 64 output channels are the second box of A
    p.a_lbo = chunk_bytes >> 4; p.a_sbo = 64; p.b_lbo = chunk_bytes >> 4; p.b_sbo = 64;
    p.a_kadv = (16 * 128) >> 4; p.b_kadv = p.a_kadv;
    p.a_half = chunk_bytes;
  }
  if (copies) {
    p.a_boxes = 1; p.b_boxes = 1;
    p.a_box_bytes = kStageABytes; p.b_box_bytes = (uint32_t)bn * 128u;
  } else {
    p.a_boxes = 128 / E; p.b_boxes = bn / E;
    p.a_box_bytes = chunk_bytes; p.b_box_bytes = chunk_bytes;
  }
  p.stage_tx_bytes = (uint32_t)p.a_boxes * p.a_box_bytes + (uint32_t)p.b_boxes * p.b_box_bytes;
  p.stages = pick_stages(bn, p.wg_xpose);
  p.ntaps = ntaps;
  for (int t = 0; t < ntaps; ++t) { p.tap_dh[t] = tap_dh[t]; p.tap_dw[t] = tap_dw[t]; }
  p.conv_stride = stride; p.Ho = Ho; p.Wo = Wo; p.kp = kp; p.wg_cin_blocks = Cin / bn;
  const long total_kb = (pixels + kp - 1) / kp;
  if (splits < 1) {
    // auto: fill one wave of persistent CTAs (two if the tiles are tiny), at least 8 k-blocks per split
    const long base_tiles = (long)(Cout / 128 + (Cout % 128 ? 1 : 0)) * ntaps * p.wg_cin_blocks;
    long s = base_tiles >= sn::kNumSMs ? 1 : (sn::kNumSMs + base_tiles / 2) / base_tiles;
    if (s > total_kb / 8) s = total_kb / 8;
    splits = s < 1 ? 1 : (int)s;
  }
  // splits are summed deterministically through the stream's workspace (one 128 x 256 partial per split and tile, at
  // most kNumSMs of them)
  const long wg_tiles = (long)(Cout / 128 + (Cout % 128 ? 1 : 0)) * ntaps * p.wg_cin_blocks;
  while (splits > 1 && (total_kb % splits != 0 || wg_tiles * splits > sn::kNumSMs)) --splits;
  p.num_kb = (int)(total_kb / splits);
  p.C = dW; p.ldc = (long)ntaps * Cin; p.atomic = 1;
  SN_CHECK(dy_ld >= Cout && x_ld >= Cin && (dy_ld * esz) % 16 == 0 && (x_ld * esz) % 16 == 0, "wgrad: bad ld");
  sn::StreamWs ws = {};
  if ((splits > 1 || copies) && sn::stream_workspace(stream, &ws, "wgrad")) return -1;
  if (splits > 1) {
    p.split_park = 1;
    p.tail_ws = ws.partials;
    p.tail_cnt = ws.counters;
  }
  const uint32_t ones[4] = {1, 1, 1, 1};
  CUtensorMap ma, mb;
  dim3 grid(Cout / 128 + (Cout % 128 ? 1 : 0), ntaps * p.wg_cin_blocks, splits);
  if (!copies) {
    {
      const uint64_t d[4] = {(uint64_t)Cout, (uint64_t)pixels, 1, 1};
      const uint64_t s[3] = {(uint64_t)dy_ld * esz, (uint64_t)dy_ld * esz * pixels, (uint64_t)dy_ld * esz * pixels};
      const uint32_t b[4] = {(uint32_t)E, (uint32_t)kp, 1, 1};
      if (make_map(&ma, dtype, dY, d, s, b, ones)) return -1;
    }
    {
      const uint64_t d[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
      const uint64_t s[3] = {(uint64_t)x_ld * esz, (uint64_t)x_ld * esz * W, (uint64_t)x_ld * esz * W * H};
      const uint32_t b[4] = {(uint32_t)E, (uint32_t)(bw * stride), (uint32_t)(bh * stride), 1};
      const uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
      if (make_map(&mb, dtype, X, d, s, b, es)) return -1;
    }
    return launch(ma, mb, p, grid, (cudaStream_t)stream);
  }

  // channel-major copies of both operands into the copy area of the stream's workspace, then the K-major mainloop
  SN_CHECK((reinterpret_cast<uintptr_t>(dY) & 15) == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0,
           "wgrad: dY and X must be 16-byte aligned");
  const WgradFeed f = wgrad_feed(NB, H, Cin, Cout, ntaps, tap_dh, tap_dw, Ho, Wo);
  SN_CHECK(ws.copy_bytes >= f.bytes,
           "wgrad: the stream's workspace has a %zu-byte copy area, this call needs %zu (sniper_set_stream_workspace, "
           "sniper_conv2d_wgrad_scratch_bytes)", ws.copy_bytes, f.bytes);
  float* dyt = static_cast<float*>(ws.copies);
  float* xt = reinterpret_cast<float*>(static_cast<uint8_t*>(ws.copies) + f.xt_off);
  {
    const uint64_t pb = (uint64_t)f.p_pitch * 4;
    const uint64_t d[4] = {(uint64_t)pixels, (uint64_t)Cout, 1, 1};
    const uint64_t s[3] = {pb, pb * Cout, pb * Cout};
    const uint32_t b[4] = {(uint32_t)kp, 128, 1, 1};
    if (make_map(&ma, dtype, dyt, d, s, b, ones)) return -1;
  }
  const long x_rows = (long)f.blocks * Cin;
  {
    const uint64_t xb = (uint64_t)f.x_pitch * 4;
    const uint64_t d[4] = {(uint64_t)f.x_pixels, (uint64_t)x_rows, 1, 1};
    const uint64_t s[3] = {xb, xb * x_rows, xb * x_rows};
    const uint32_t b[4] = {(uint32_t)kp, (uint32_t)bn, 1, 1};
    if (make_map(&mb, dtype, xt, d, s, b, ones)) return -1;
  }
  p.wg_hp = f.hp; p.wg_padh = f.padh;
  for (int t = 0; t < ntaps; ++t) p.wg_tapblk[t] = f.tapblk[t];
  XposeParams xp;
  memset(&xp, 0, sizeof(xp));
  xp.job[0] = XposeJob{static_cast<const float*>(dY), dy_ld, dyt, f.p_pitch, Cout, Cout, (int)pixels, Ho, Wo, Ho, Wo};
  // X^T row block j: a gather over the Hp x Wo grid with offsets (-padh, dw_j)
  XposeJob& xj = xp.job[1];
  xj.src = static_cast<const float*>(X); xj.ld = x_ld; xj.dst = xt; xj.pitch = f.x_pitch;
  xj.C = Cin; xj.rows = (int)x_rows; xj.P = (int)f.x_pixels; xj.H = H; xj.W = W; xj.Ho = f.hp; xj.Wo = Wo;
  for (int j = 0; j < f.blocks; ++j) { xj.dh[j] = -f.padh; xj.dw[j] = f.blk_dw[j]; }
  xp.split = Cout / 32;
  const long xpix = pixels > xj.P ? pixels : xj.P;
  const dim3 xgrid((unsigned)sn::div_up(xpix, kXpPix), (unsigned)(xp.split + xj.rows / 32));
  wgrad_xpose_kernel<<<xgrid, 256, 0, (cudaStream_t)stream>>>(xp);
  SN_LAUNCH_CHECK();
  return launch(ma, mb, p, grid, (cudaStream_t)stream);
}

// Bytes of the tf32 operand copy area sniper_conv2d_wgrad_nhwc needs in the stream's workspace for a geometry (host
// only; 0 where the kernel reads the operands in place: bf16, and tf32 layers without copies, see WgradFeed).  Same
// arguments as that entry point.
size_t sniper_conv2d_wgrad_scratch_bytes(int NB, int H, int W, int Cin, int Cout, int ntaps, const int* tap_dh,
                                         const int* tap_dw, int stride, int Ho, int Wo, int dtype) {
  if (!wgrad_copies(dtype, ntaps, stride, Wo) || ntaps > kMaxTaps || !tap_dh || !tap_dw) return 0;
  return wgrad_feed(NB, H, Cin, Cout, ntaps, tap_dh, tap_dw, Ho, Wo).bytes;
}

// Host-only query of the launch plan sniper_gemm_nt would use for C[M,N] = A[M,K] * B[N,K]^T with 16-byte aligned,
// contiguous operands (no GPU needed; exercised by the CPU tests).  out[8] = {block_n, ring stages, 0 (reserved),
// tiles, persistent grid, tail mode (0 none, 2 column pieces), first tail tile, pieces per tail
// tile}.
int sniper_gemm_plan(int M, int N, int K, int dtype, int* out) {
  SN_CHECK(dtype == DT_TF32 || dtype == DT_BF16, "gemm_plan: dtype must be 0 (tf32) or 1 (bf16)");
  const int E = dtype == DT_TF32 ? 32 : 64;
  SN_CHECK(M > 0 && N > 0 && K > 0 && K % E == 0, "gemm_plan: K (%d) must be a positive multiple of %d", K, E);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  const int bn = pick_block_n(N);
  fill_kmajor(p, dtype, bn);
  p.mode = MODE_GEMM; p.M = M; p.N = N; p.num_kb = K / E;
  p.splits = 1;
  const long tiles = (long)sn::div_up(M, 128) * sn::div_up(N, bn);
  const long max_units = sn::kNumSMs;
  plan_tail(p, tiles, max_units);
  int mode = 0, factor = 1;
  if (p.tail_p > 0) { mode = 2; factor = p.tail_p; }
  const long units = p.tail_first + (tiles - p.tail_first) * factor;
  out[0] = bn;
  out[1] = p.stages;
  out[2] = 0;
  out[3] = (int)tiles;
  out[4] = (int)(units < max_units ? units : max_units);
  out[5] = mode;
  out[6] = p.tail_first;
  out[7] = factor;
  return 0;
}

}  // extern "C"
