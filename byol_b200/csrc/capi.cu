// byol_b200 — C-ABI plumbing shared by every entry point: thread-local error string, launch checks, version.
#include <stdarg.h>
#include <stdio.h>

#include "common.cuh"

namespace byol {

static thread_local char g_last_error[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

// Launch-configuration errors surface here; asynchronous faults surface at the caller's next sync.
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return -100;
  }
  return 0;
}

int device_slot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) dev = 0;
  return dev < kMaxDevices ? dev : kMaxDevices - 1;
}

int device_sm_count() {
  static int n[kMaxDevices] = {};
  const int slot = device_slot();
  if (n[slot] == 0) {
    int dev = 0, v = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[slot] = v;
  }
  return n[slot];
}

// Per-(device, stream) scratch for the fixed-point accumulators.  It only grows; a buffer that a captured CUDA graph
// may still reference is never freed.  Kernels on one stream run in order, so consecutive reductions on that stream
// reuse the same memory.  It is zeroed once when allocated; every consumer (fix_flush and the kernels that read the
// accumulators themselves) leaves what it read at zero, so no memset is needed per reduction.
namespace {
struct FixScratch {
  int dev;
  cudaStream_t stream;
  Fix128* p;
  int64_t n;
  bool leased;   // handed out and not yet marked complete by fix_done
};
static FixScratch g_fix[256];
static int g_fix_count = 0;
}  // namespace

Fix128* fix_scratch(cudaStream_t stream, int64_t n) {
  const int dev = device_slot();
  FixScratch* e = nullptr;
  for (int i = 0; i < g_fix_count; ++i)
    if (g_fix[i].dev == dev && g_fix[i].stream == stream) e = &g_fix[i];
  if (e == nullptr) {
    if (g_fix_count == 256) { set_last_error("fix_scratch: too many streams"); return nullptr; }
    e = &g_fix[g_fix_count++];
    e->dev = dev; e->stream = stream; e->p = nullptr; e->n = 0; e->leased = false;
  }
  if (e->n < n) {
    // cudaMalloc is not a stream operation: allowed even while the calling stream is being captured
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    Fix128* p = nullptr;
    const int64_t want = n + n / 2;
    cudaError_t err = cudaMalloc(&p, (size_t)want * sizeof(Fix128));
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (err != cudaSuccess) { set_last_error("fix_scratch: cudaMalloc failed: %s", cudaGetErrorString(err)); return nullptr; }
    if (cudaMemsetAsync(p, 0, (size_t)want * sizeof(Fix128), stream) != cudaSuccess) {
      set_last_error("fix_scratch: memset failed");
      return nullptr;
    }
    e->p = p;   // the previous buffer is kept alive (see above)
    e->n = want;
  } else if (e->leased) {
    // the previous reduction on this stream returned early (error path): its accumulators may be stale
    if (cudaMemsetAsync(e->p, 0, (size_t)e->n * sizeof(Fix128), stream) != cudaSuccess) {
      set_last_error("fix_scratch: memset failed");
      return nullptr;
    }
  }
  e->leased = true;
  return e->p;
}

int fix_done(cudaStream_t stream, int rc) {
  if (rc != 0) return rc;
  const int dev = device_slot();
  for (int i = 0; i < g_fix_count; ++i)
    if (g_fix[i].dev == dev && g_fix[i].stream == stream) g_fix[i].leased = false;
  return rc;
}

__global__ void fix_flush_kernel(Fix128* __restrict__ acc, float* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const Fix128 a = acc[i];
    acc[i] = Fix128{0ull, 0ll, 0.0};                                  // ready for the next reduction on this stream
    atomicAdd(dst + i, (float)fix_value(a));           // two streams may flush into one gradient
  }
}

int fix_flush(Fix128* acc, float* dst, int64_t n, cudaStream_t stream) {
  if (n <= 0) return 0;
  int64_t blocks = (n + 255) / 256;
  if (blocks > 4 * 1024) blocks = 4 * 1024;
  fix_flush_kernel<<<(int)blocks, 256, 0, stream>>>(acc, dst, n);
  return check_launch("fix_flush_kernel");
}

}  // namespace byol

extern "C" const char* byol_last_error(void) { return byol::g_last_error; }

extern "C" int byol_abi_version(void) { return 2; }

// number of SMs of the current device (used by the host side to size persistent grids); < 0 on error
extern "C" int byol_device_sm_count(void) {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  return n;
}
