// Error reporting for the C-ABI (mirror of MXGetLastError, SNIPER-mxnet/include/mxnet/c_api.h:196-204) and the
// registry of the per-(device, stream) workspaces (common.cuh).
#include "common.cuh"
#include <stdarg.h>

namespace sn {
char* last_error_buf() {
  static thread_local char buf[1024] = {0};
  return buf;
}
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 1024, fmt, ap);
  va_end(ap);
}

namespace {
// Host-side table; the entry points are not re-entrant across host threads (one host thread drives a device's
// launches).  Entries are replaced, never removed.
constexpr int kStreamWsEntries = 256;
struct WsEntry {
  int device;
  cudaStream_t stream;
  uint8_t* base;
  size_t bytes;
};
WsEntry g_stream_ws[kStreamWsEntries];
int g_stream_ws_n = 0;
}  // namespace

int stream_workspace(void* stream, StreamWs* ws, const char* who) {
  const cudaStream_t st = (cudaStream_t)stream;
  // a stream nothing is registered for is refused before any CUDA call
  bool any = false;
  for (int i = 0; i < g_stream_ws_n; ++i) any |= g_stream_ws[i].stream == st;
  SN_CHECK(any, "%s: no workspace registered for this stream (sniper_set_stream_workspace)", who);
  int dev = -1;
  SN_CUDA(cudaGetDevice(&dev));
  const WsEntry* e = nullptr;
  for (int i = 0; i < g_stream_ws_n; ++i)
    if (g_stream_ws[i].device == dev && g_stream_ws[i].stream == st) e = &g_stream_ws[i];
  SN_CHECK(e != nullptr, "%s: no workspace registered for device %d and this stream (sniper_set_stream_workspace)", who,
           dev);
  ws->partials = reinterpret_cast<float4*>(e->base);
  ws->counters = reinterpret_cast<int*>(e->base + kTailWsBytes);
  ws->slab = reinterpret_cast<float*>(e->base + kTailWsBytes + kTailCntBytes);
  ws->copies = e->base + kStreamWsFixedBytes;
  ws->copy_bytes = e->bytes - kStreamWsFixedBytes;
  return 0;
}
}  // namespace sn

extern "C" {
const char* sniper_last_error(void) { return sn::last_error_buf(); }
int sniper_abi_version(void) { return 3; }

// Bytes of the fixed part of a stream workspace (split-K partials and counters, depthwise slab); the tf32 operand copy
// area a weight gradient needs (sniper_conv2d_wgrad_scratch_bytes) comes on top.
size_t sniper_stream_workspace_bytes(void) { return sn::kStreamWsFixedBytes; }

// Registers a caller-owned device buffer (256-byte aligned, at least sniper_stream_workspace_bytes() bytes) for the
// launches enqueued on `stream` of `device`; it must outlive them.  Its split-K counter region must be zero when it is
// registered; the kernels leave it zero.  Registering again for the same (device, stream) replaces the buffer.  The
// library itself never allocates.
int sniper_set_stream_workspace(void* ws, size_t bytes, int device, void* stream) {
  SN_CHECK(device >= 0, "set_stream_workspace: device (%d) must be >= 0", device);
  SN_CHECK(ws != nullptr, "set_stream_workspace: ws must not be null");
  SN_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "set_stream_workspace: ws must be 256-byte aligned");
  SN_CHECK(bytes >= sn::kStreamWsFixedBytes,
           "set_stream_workspace: bytes (%zu) is smaller than sniper_stream_workspace_bytes() (%zu)", bytes,
           sn::kStreamWsFixedBytes);
  const cudaStream_t st = (cudaStream_t)stream;
  uint8_t* base = static_cast<uint8_t*>(ws);
  for (int i = 0; i < sn::g_stream_ws_n; ++i)
    if (sn::g_stream_ws[i].device == device && sn::g_stream_ws[i].stream == st) {
      sn::g_stream_ws[i].base = base;
      sn::g_stream_ws[i].bytes = bytes;
      return 0;
    }
  SN_CHECK(sn::g_stream_ws_n < sn::kStreamWsEntries, "set_stream_workspace: more than %d (device, stream) pairs",
           sn::kStreamWsEntries);
  sn::g_stream_ws[sn::g_stream_ws_n++] = sn::WsEntry{device, st, base, bytes};
  return 0;
}
}
