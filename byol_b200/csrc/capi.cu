// byol_b200 — C-ABI plumbing shared by every entry point: thread-local error string, launch checks, version, and the
// host-side launch helpers (shared-memory opt-in, resident grids, tensor maps, fixed-point scratch).
#include <stdarg.h>
#include <stdio.h>

#include <atomic>
#include <map>
#include <mutex>
#include <utility>

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
  static std::atomic<int> n[kMaxDevices] = {};
  const int slot = device_slot();
  int v = n[slot].load(std::memory_order_relaxed);
  if (v == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[slot].store(v, std::memory_order_relaxed);
  }
  return v;
}

int smem_opt_in(const void* kernel, int bytes, const char* what) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> granted;   // (kernel, device slot) -> bytes
  const std::lock_guard<std::mutex> lock(mu);
  int& have = granted.emplace(std::make_pair(kernel, device_slot()), 48 * 1024).first->second;
  if (bytes <= have) return 0;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    set_last_error("%s: cudaFuncSetAttribute(%d bytes of shared memory) failed: %s", what, bytes,
                   cudaGetErrorString(e));
    return -2;
  }
  have = bytes;
  return 0;
}

int resident_blocks(const void* kernel, int threads, int smem_bytes, const char* what) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> known;   // (kernel, device slot) -> blocks on the device
  const std::lock_guard<std::mutex> lock(mu);
  int& n = known.emplace(std::make_pair(kernel, device_slot()), 0).first->second;
  if (n > 0) return n;
  int per_sm = 0;
  // not a stream operation: allowed while the calling stream is being captured (as in fix_scratch)
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  cudaThreadExchangeStreamCaptureMode(&mode);
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, (size_t)smem_bytes);
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (e != cudaSuccess || per_sm <= 0) {
    set_last_error("%s: no resident block of %d threads and %d bytes of shared memory (%s)", what, threads, smem_bytes,
                   cudaGetErrorString(e));
    return 0;
  }
  n = per_sm * device_sm_count();
  return n;
}

int tmap_bf16(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* byte_strides,
              const uint32_t* box, CUtensorMapSwizzle swizzle, const char* what) {
  // decltype only names the driver function's type: the library resolves it at run time and does not link libcuda
  static const auto encode = []() -> decltype(&cuTensorMapEncodeTiled) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<decltype(&cuTensorMapEncodeTiled)>(fn);
  }();
  if (encode == nullptr) {
    set_last_error("%s: cuTensorMapEncodeTiled entry point unavailable", what);
    return -3;
  }
  const cuuint32_t elem_strides[5] = {1u, 1u, 1u, 1u, 1u};
  const CUresult r = encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims,
                            byte_strides, box, elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char shape[384];   // at most 5 entries of < 72 characters
    int len = snprintf(shape, sizeof(shape), "%llu (box %u)", (unsigned long long)dims[0], box[0]);
    for (int i = 1; i < rank; ++i)
      len += snprintf(shape + len, sizeof(shape) - len, ", %llu (box %u, stride %llu B)", (unsigned long long)dims[i],
                      box[i], (unsigned long long)byte_strides[i - 1]);
    set_last_error("%s: cuTensorMapEncodeTiled failed (%d): dims %s, base %p", what, (int)r, shape, base);
    return -3;
  }
  return 0;
}

int tmap_2d(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
            uint32_t box_cols, const char* what) {
  const uint64_t dims[2] = {cols, rows};
  const uint64_t strides[1] = {ld * sizeof(bf16)};
  const uint32_t box[2] = {box_cols, box_rows};
  return tmap_bf16(tm, base, 2, dims, strides, box,
                   box_cols == 64u ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, what);
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

// Per-(device, stream) buffer of the wgrad partials.  Like fix_scratch it only grows and never frees a buffer a
// captured graph may still reference; it holds no state between reductions.
namespace {
struct PartScratch {
  int dev;
  cudaStream_t stream;
  float* p;
  int64_t n;
};
static PartScratch g_part[256];
static int g_part_count = 0;
}  // namespace

float* part_scratch(cudaStream_t stream, int64_t n) {
  const int dev = device_slot();
  PartScratch* e = nullptr;
  for (int i = 0; i < g_part_count; ++i)
    if (g_part[i].dev == dev && g_part[i].stream == stream) e = &g_part[i];
  if (e == nullptr) {
    if (g_part_count == 256) { set_last_error("part_scratch: too many streams"); return nullptr; }
    e = &g_part[g_part_count++];
    e->dev = dev; e->stream = stream; e->p = nullptr; e->n = 0;
  }
  if (e->n < n) {
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    float* p = nullptr;
    const int64_t want = n + n / 2;
    cudaError_t err = cudaMalloc(&p, (size_t)want * sizeof(float));
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (err != cudaSuccess) { set_last_error("part_scratch: cudaMalloc failed: %s", cudaGetErrorString(err)); return nullptr; }
    e->p = p;   // the previous buffer is kept alive (see above)
    e->n = want;
  }
  return e->p;
}

// Block pass: 256 / sl consecutive elements (coalesced loads), each summed by sl threads over every sl-th split; the
// sl partial accumulators of an element are then added up (integer words wrap; the side sums of multiples of 2^20 are
// exact), which gives the same words and side sum in any grouping.  sl > 1 keeps the SMs busy when there are few
// elements and many splits.
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int splits, float* __restrict__ dst, int64_t n,
                                    int sl) {
  __shared__ Fix128 acc[256];
  const int per = 256 / sl;
  const int e = threadIdx.x % per, j = threadIdx.x / per;
  for (int64_t base = blockIdx.x * (int64_t)per; base < n; base += (int64_t)gridDim.x * per) {
    const int64_t i = base + e;
    Fix128 a{0ull, 0ll, 0.0};
    if (i < n)
      for (int s = j; s < splits; s += sl) fix_add_reg(a, __ldg(part + s * n + i));
    acc[threadIdx.x] = a;
    __syncthreads();
    if (j == 0 && i < n) {
      for (int k = 1; k < sl; ++k) {
        const Fix128 b = acc[k * per + e];
        a.lo += b.lo;
        a.hi = (long long)((unsigned long long)a.hi + (unsigned long long)b.hi);
        a.spill += b.spill;
      }
      atomicAdd(dst + i, (float)fix_value(a));   // two streams may add into one gradient
    }
    __syncthreads();
  }
}

int wgrad_reduce(const float* part, int splits, float* dst, int64_t n, cudaStream_t stream) {
  if (n <= 0) return 0;
  int sl = 1;   // split lanes per element: about 2^18 threads in all, at most one per split
  while (sl < 32 && 2 * sl <= splits && n * sl < (1 << 18)) sl *= 2;
  const int per = 256 / sl;
  int64_t blocks = (n + per - 1) / per;
  if (blocks > 4 * 1024) blocks = 4 * 1024;
  wgrad_reduce_kernel<<<(int)blocks, 256, 0, stream>>>(part, splits, dst, n, sl);
  return check_launch("wgrad_reduce_kernel");
}

int fix_flush_stats(Fix128* acc, float* col_sum, float* col_sqsum, int64_t n, cudaStream_t stream) {
  const int rc = fix_flush(acc, col_sum, n, stream);
  if (rc != 0) return rc;
  return fix_done(stream, fix_flush(acc + n, col_sqsum, n, stream));
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
