// Shared helpers for the sniper_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace sn {

// thread-local last-error string, surfaced through sniper_last_error() (C-ABI mirror of
// MXGetLastError, SNIPER-mxnet/include/mxnet/c_api.h:196-204)
char* last_error_buf();
void set_error(const char* fmt, ...);

#define SN_CHECK(cond, ...)      \
  do {                           \
    if (!(cond)) {               \
      sn::set_error(__VA_ARGS__); \
      return -1;                 \
    }                            \
  } while (0)

#define SN_CUDA(call)                                                                  \
  do {                                                                                 \
    cudaError_t _e = (call);                                                           \
    if (_e != cudaSuccess) {                                                           \
      sn::set_error("%s:%d CUDA error: %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return -1;                                                                       \
    }                                                                                  \
  } while (0)

#define SN_LAUNCH_CHECK() SN_CUDA(cudaGetLastError())

static inline int div_up(long a, long b) { return (int)((a + b - 1) / b); }

// a host offset array off[0 .. n] (int or long long) that starts at 0 and never decreases
template <typename T>
bool offsets_ok(const T* off, long n) {
  if (off[0] != 0) return false;
  for (long i = 0; i < n; ++i)
    if (off[i + 1] < off[i]) return false;
  return true;
}

constexpr int kNumSMs = 132;   // H100 SXM

// Caller-owned device scratch, one buffer per (device, stream) registered with sniper_set_stream_workspace: launches on
// one stream run one after another and can share it; launches on different streams may overlap and must not.  Layout:
// a fixed part (the regions below, in this order, each 256-byte aligned), then the tf32 weight gradient's operand copy
// area up to the end of the buffer.
//   split-K parked partials of the wgmma weight gradient: at most kNumSMs (split, tile) pairs of 128 x 256 fp32;
constexpr size_t kTailWsBytes = (size_t)kNumSMs * 128 * 256 * 4;
//   split-K arrival counters, one per tile (zero when registered; every launch leaves them zero);
constexpr size_t kTailCntBytes = ((size_t)kNumSMs * 8 * sizeof(int) + 255) / 256 * 256;
//   the depthwise weight gradient's slab of block partials.  Its one-wave grid needs about kNumSMs * (blocks per SM) *
//   9 * 128 floats (a block covers at most 128 channels); at 126..158 registers per thread that is 1..2 blocks per SM,
//   so the cap (4 blocks per SM) binds only for grids the occupancy rule would not pick.
constexpr long kWgSlabFloats = (long)kNumSMs * 4 * 9 * 128;
constexpr size_t kStreamWsFixedBytes = kTailWsBytes + kTailCntBytes + ((size_t)kWgSlabFloats * 4 + 255) / 256 * 256;

struct StreamWs {
  float4* partials;
  int* counters;
  float* slab;
  void* copies;          // the tf32 operand copy area (256-byte aligned) and its size
  size_t copy_bytes;
};

// The workspace registered for (current device, stream); refuses (naming `who`) when there is none.
int stream_workspace(void* stream, StreamWs* ws, const char* who);

}  // namespace sn
