// byol_b200 — sm_90a device helpers: mbarrier, TMA, wgmma, cp.async.
// Hand-written PTX wrappers; no CUTLASS/CuTe dependency.  Encodings follow the
// PTX ISA (wgmma shared-memory matrix descriptors).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace byol {

typedef __nv_bfloat16 bf16;

// ----------------------------------------------------------------------------
// error plumbing shared by all host wrappers (thread-local last error string)
// ----------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
int check_launch(const char* what);

// One process may drive several GPUs: per-kernel attributes (cudaFuncSetAttribute) and the SM count are per device,
// so the host wrappers cache them per device slot (capi.cu).
static constexpr int kMaxDevices = 64;
int device_slot();       // current CUDA device index, clamped to [0, kMaxDevices)
int device_sm_count();   // SM count of the current device (cached per device; 132 if the query fails)

// ----------------------------------------------------------------------------
// Deterministic reductions.  Partial sums from many blocks are accumulated in fixed point: an addend x = v * 2^50
// (rounded to an integer) is split into hi = floor(x / 2^32) and lo = x - hi * 2^32 in [0, 2^32], added to two
// independent 64-bit words (fire-and-forget reductions, no carry between them).  Integer addition is associative, so
// the totals do not depend on the order in which blocks arrive and every run gives the same bits; the value is
// hi * 2^-18 + lo * 2^-50 (resolution 8.9e-16).  Addends that are not finite or whose magnitude reaches kFixMax go to
// an fp64 side sum instead, so NaN / Inf propagate to the result and huge values keep their magnitude (that side sum
// is order-dependent in its last bits, which only happens on a diverging step).  With every fixed-point addend below
// 2^36 the integer part cannot overflow for fewer than 512 such addends per element.  The accumulators live in a
// per-stream scratch buffer (fix_scratch) and are added to their fp32 destination once by fix_flush.
// ----------------------------------------------------------------------------
struct Fix128 {
  unsigned long long lo;
  long long hi;
  double spill;   // non-finite / out-of-range addends
};
static constexpr double kFixMax = 68719476736.0;   // 2^36
// n zeroed accumulators on `stream` (stream-ordered), nullptr on error.  Whoever reads them leaves them at zero; a
// wrapper that got the scratch calls fix_done when its reduction is complete, otherwise the next fix_scratch on that
// stream zeroes the buffer again (an error path can not leave stale sums behind).
Fix128* fix_scratch(cudaStream_t stream, int64_t n);
int fix_done(cudaStream_t stream, int rc);   // marks the stream's scratch clean when rc == 0; returns rc
// dst[i] += value(acc[i]) for i < n (one fp32 addition per element); acc[i] is reset to zero
int fix_flush(Fix128* acc, float* dst, int64_t n, cudaStream_t stream);

__device__ __forceinline__ void fix_add_words(Fix128* acc, unsigned long long lo, long long hi) {
  atomicAdd(&acc->lo, lo);   // results unused: both compile to reductions
  atomicAdd(reinterpret_cast<unsigned long long*>(&acc->hi), (unsigned long long)hi);
}
__device__ __forceinline__ void fix_add(Fix128* acc, double v) {
  if (!(fabs(v) < kFixMax)) {   // NaN, Inf or too large for the fixed-point words
    atomicAdd(&acc->spill, v);
    return;
  }
  const double x = v * 0x1p50;                 // exact (power-of-two scaling)
  const double hi = floor(x * 0x1p-32);
  fix_add_words(acc, __double2ull_rn(x - hi * 0x1p32), (long long)hi);   // lo in [0, 2^32]
}
__device__ __forceinline__ void fix_add_raw(Fix128* acc, const Fix128& v) {
  fix_add_words(acc, v.lo, v.hi);
  if (v.spill != 0.0) atomicAdd(&acc->spill, v.spill);
}
__host__ __device__ __forceinline__ double fix_value(const Fix128& a) {
  return ((double)a.hi * 0x1p-18 + (double)a.lo * 0x1p-50) + a.spill;
}

#define BYOL_CHECK_ARG(cond, ...)                 \
  do {                                            \
    if (!(cond)) {                                \
      ::byol::set_last_error(__VA_ARGS__);        \
      return -1;                                  \
    }                                             \
  } while (0)

// ----------------------------------------------------------------------------
// small device utilities
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 %%rx;\n"
      ".reg .pred %%px;\n"
      "elect.sync %%rx|%%px, %1;\n"
      "@%%px mov.s32 %0, 1;\n"
      "}\n"
      : "+r"(pred)
      : "r"(0xffffffffu));
  return pred != 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a pipeline bug traps (reported as a launch failure) instead of
// hanging the GPU.  try_wait suspends in hardware, so the bound is generous.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // (2^28 polls: waits that span a grid barrier plus a cross-rank exchange — the MMA warp of mlp_fused_fwd_kernel under
  // SyncBatchNorm — can legitimately last as long as the rank skew, e.g. right after the CUDA-graph capture)
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 28)) __trap();
  }
}

// generic-proxy writes (st.shared / cp.async) -> visible to the async proxy (wgmma / TMA)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------
// cp.async (LDGSTS) 16-byte with zero-fill
// ----------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst_smem, const void* src, bool valid) {
  uint32_t sz = valid ? 16u : 0u;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), 2-D tiled, arrives on an mbarrier with complete_tx
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* tmap, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst_smem), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// TMA store smem -> global (bulk async group), 2-D tiled
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tmap, uint32_t src_smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tmap),
               "r"(src_smem), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until the bulk stores of this thread have finished READING their shared-memory source
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// same, but allow the most recent group to be still in flight (double-buffered staging)
__device__ __forceinline__ void tma_store_wait_read1() {
  asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------
// wgmma (sm_90a): one warpgroup (4 consecutive warps, the first a multiple of 4) computes a 64 x N tile with the
// fp32 accumulator in registers.  Fragment layout of a 64 x N fp32 accumulator: thread t of the warpgroup holds
// rows 16*(t/32) + (t%32)/4 and +8, columns 8j + 2*(t%4) and +1 for j < N/8, as d[4j .. 4j+3] =
// (row, c), (row, c+1), (row+8, c), (row+8, c+1).
// ----------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads across wg_wait
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 operands from shared-memory descriptors, fp32 accumulate.
// TA / TB = 1: the operand is MN-major (transposed) in shared memory.  accumulate = 0 overwrites D.
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(N == 32 || N == 64 || N == 128 || N == 192 || N == 256, "wgmma_bf16: unsupported N");
  if constexpr (N == 32) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
  if constexpr (N == 64) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
  if constexpr (N == 128) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
  if constexpr (N == 192) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %98, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, %99, %100;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
  if constexpr (N == 256) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
}

// Accumulator fragment of this warpgroup (rows row0 .. row0+63 of the tile) -> fp32 tile in shared memory
// ([rows][ld] floats, ld even), the hand-off to epilogue warps that own one tile row per lane.
template <int N>
__device__ __forceinline__ void acc_store_smem(float* buf, int ld, int row0, int col0, const float (&d)[N / 2]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + (t >> 5) * 16 + ((t & 31) >> 2);
  const int c = col0 + 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(buf + (int64_t)r * ld + c + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(buf + (int64_t)(r + 8) * ld + c + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// one tile row, 32 consecutive fp32 columns (16-byte aligned) -> registers
__device__ __forceinline__ void acc_load_row32(const float* src, uint32_t (&r)[32]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint4 q = *reinterpret_cast<const uint4*>(src + 4 * j);
    r[4 * j] = q.x; r[4 * j + 1] = q.y; r[4 * j + 2] = q.z; r[4 * j + 3] = q.w;
  }
}
// row stride (floats) of an accumulator tile with `cols` columns: 16-byte rows, row-per-lane loads conflict-free
__host__ __device__ constexpr int acc_ld(int cols) { return cols + 4; }

// ----------------------------------------------------------------------------
// descriptors
// ----------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, 128-byte swizzle.
//   start address  bits [0,14)   (>>4)
//   LBO            bits [16,30)  (>>4)
//   SBO            bits [32,46)  (>>4)
//   base offset    bits [49,52)  0: the swizzle pattern is a function of the absolute address bits
//   layout  = 1    bits [62,64)  (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// physical byte offset of (row, 16-byte chunk) inside a [rows][128 B] tile with
// the 128-byte swizzle (tile base must be 1024-byte aligned)
__device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return row * 128u + ((chunk ^ (row & 7u)) << 4);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ----------------------------------------------------------------------------
// 1-D bulk copy global -> shared (any multiple of 16 bytes), completes on an mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void bulk_load_1d(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tmap, uint32_t src_smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tmap),
               "r"(src_smem), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// Shared-memory matrix descriptor without swizzle: core matrix = 8 rows x 16 bytes, rows 16 bytes apart;
// K-major: LBO = byte step between the two 16-byte K chunks of one K = 16 MMA, SBO = step between 8-row groups.
// LBO / SBO may be smaller than the 128-byte core matrix, i.e. rows and chunks may overlap: the descriptor alone then
// forms the im2col of a 1-D window over 16-byte pixels.
__device__ __forceinline__ uint64_t make_smem_desc_none(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// ----------------------------------------------------------------------------
// epilogue statistics (shared by the igemm and stem kernels)
// ----------------------------------------------------------------------------
// packed fp32x2 helpers: the statistics loops carry two columns per 64-bit value
__device__ __forceinline__ uint64_t f2_pack(uint32_t lo, uint32_t hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(lo), "r"(hi));
  return r;
}
__device__ __forceinline__ float2 f2_unpack(uint64_t v) {
  uint32_t lo, hi;
  asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v));
  return make_float2(__uint_as_float(lo), __uint_as_float(hi));
}
__device__ __forceinline__ uint64_t f2_add(uint64_t a, uint64_t b) {
  const float2 x = f2_unpack(a), y = f2_unpack(b);
  return f2_pack(__float_as_uint(x.x + y.x), __float_as_uint(x.y + y.y));
}
__device__ __forceinline__ uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c) {
  const float2 x = f2_unpack(a), y = f2_unpack(b), z = f2_unpack(c);
  return f2_pack(__float_as_uint(fmaf(x.x, y.x, z.x)), __float_as_uint(fmaf(x.y, y.y, z.y)));
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t w;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(addr));
  return w;
}
// one staged word = two bf16 columns -> {sum, sum of squares} accumulators
__device__ __forceinline__ void stat_acc(uint32_t w, uint64_t& s1, uint64_t& s2) {
  const uint64_t x = f2_pack(w << 16, w & 0xffff0000u);
  s1 = f2_add(s1, x);
  s2 = f2_fma(x, x, s2);
}

// Column statistics of a staged narrow chunk ([32 rows][64 B], 16-byte chunk j of row r at j ^ ((r >> 1) & 3)).
// lane -> column pair cp = lane & 15 of rows with parity lane >> 4 (two adjacent rows per warp-wide load: all 32
// banks, no conflicts); the caller combines the two parities with one shuffle when it flushes.
__device__ __forceinline__ void stats_narrow(uint32_t stage_base, int lane, int rows_valid, uint64_t& s1,
                                             uint64_t& s2) {
  const uint32_t cp = (uint32_t)lane & 15u, rh = (uint32_t)lane >> 4;
  const uint32_t jc = cp >> 2, wq = cp & 3u;
  uint32_t offq[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) offq[q] = stage_base + rh * 64u + ((jc ^ (uint32_t)q) << 4) + wq * 4u;
  uint64_t a1 = 0ull, a2 = 0ull, b1 = 0ull, b2 = 0ull;
  if (rows_valid == 32) {
#pragma unroll
    for (int rr = 0; rr < 16; rr += 2) {   // row = 2*rr + rh, so (row >> 1) & 3 == rr & 3
      stat_acc(lds32(offq[rr & 3] + (uint32_t)rr * 128u), a1, a2);
      stat_acc(lds32(offq[(rr + 1) & 3] + (uint32_t)(rr + 1) * 128u), b1, b2);
    }
  } else {
    for (int rr = 0; rr < 16; ++rr)
      if (2 * rr + (int)rh < rows_valid) stat_acc(lds32(offq[rr & 3] + (uint32_t)rr * 128u), a1, a2);
  }
  s1 = f2_add(s1, f2_add(a1, b1));
  s2 = f2_add(s2, f2_add(a2, b2));
}


}  // namespace byol
