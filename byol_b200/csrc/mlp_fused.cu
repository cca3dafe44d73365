// byol_b200 — the projector / predictor MLP forward as ONE kernel:  Linear -> BatchNorm1d (batch statistics) -> ReLU -> Linear
//
// Replaces, per lane, the cuBLAS Linear + ATen batch_norm + ReLU + cuBLAS Linear chain the reference reaches through
// /root/reference/main.py:194-205 (head, predictor) and main.py:238-239 (4 launches + the BN statistics kernels each).
//
//   x [B, K1] bf16,  W1 [H, K1],  b1 [H],  gamma / beta [H],  W2 [O, H],  b2 [O]      (H % 128 == 0, O <= 256, B <= 128 * tiles_m)
//
// Cooperative grid of tiles_m x (H / 128) CTAs, one per SM (B = 512, H = 4096 -> 128 CTAs), 416 threads (warps 0-3
// epilogue, warps 4-11 two MMA warpgroups owning tile rows 0-63 / 64-127, warp 12 TMA producer):
//   phase 1  h-tile[128 x 128] = x-tile . W1-tile^T            wgmma, the fp32 accumulator is parked in shared memory
//   phase 2  per-column sum / sum of squares of h = acc + b1     smem -> registers, transpose-reduce, global atomics
//   ----- grid barrier (all M-tiles have contributed); under SyncBatchNorm CTA 0 then runs the peer-memory exchange of
//         csrc/xchg.cu on the statistics vector and a second grid barrier follows -----
//   phase 3  scale / shift per column (CTAs of M-tile 0 also update the running statistics and store the coefficients),
//            a = relu(h * scale + shift) from the SAME parked accumulator -> bf16 -> shared memory in the K-major 128-byte
//            swizzle, i.e. directly the A operand of the second GEMM (h and a are TMA-stored for the backward pass
//            only when the lane is differentiated)
//   phase 4  out-partial[128 x O] = a-tile[128 x 128] . W2[:, 128-column slice]^T   (K split over the H / 128 CTAs of a row
//            block), 64 output columns at a time, accumulated from the MMA registers in fixed point (+ b2 from the first
//            slice) and added to the fp32 output after the kernel
// Cross-CTA sums (statistics, output) are fixed point, so every run gives the same bits (common.cuh).
// The hidden activation never makes a round trip through HBM between the two GEMMs.
#include <cooperative_groups.h>
#include <string.h>

#include "common.cuh"

namespace byol {

static constexpr int MF_STAGE = 32768;                 // one ring stage: A [128 x 64] + B [128 x 64] bf16
static constexpr int MF_STAGES = 3;
static constexpr int MF_RING = MF_STAGES * MF_STAGE;   // 96 KB; after GEMM1: [a-tile 32 KB | W2 slice 64 KB]
static constexpr int MF_HSTAGE_OFF = MF_RING;          // 32 KB staging of h (bf16) for its TMA store
static constexpr int MF_COEF_OFF = MF_HSTAGE_OFF + 32768;   // scale[128], shift[128], bias1[128]
static constexpr int MF_ACC_LD = acc_ld(128);
static constexpr int MF_ACC_OFF = MF_COEF_OFF + 3 * 512;    // GEMM1 accumulator [128][MF_ACC_LD] fp32
static constexpr int MF_BAR_OFF = MF_ACC_OFF + 128 * MF_ACC_LD * 4;
static constexpr int MF_NEEDED = MF_BAR_OFF + 256;
static constexpr int MF_TOTAL = MF_NEEDED + 1024;
static constexpr int MF_THREADS = 13 * 32;
static_assert(MF_TOTAL <= 232448, "mlp_fused: shared memory");

struct MlpPeer {           // SyncBatchNorm exchange (csrc/xchg.cu layout); world <= 1: unused
  uint64_t p[8];
  int world, rank;
  int64_t cap_bytes;
  uint32_t* counter;
};

struct MlpParams {
  const float* b1;
  const float* gamma;
  const float* beta;
  const float* b2;
  float* stats;            // [2H] zeroed: sum | sum of squares of h (train) — after the kernel: the (global) sums
  float* running_mean;     // optional [H]
  float* running_var;
  float* coeffs;           // [4][H] scale, shift, mean, invstd (always written by the CTAs of M-tile 0)
  float* out;              // [B, O] fp32, zeroed by the caller
  uint32_t* grid_bar;      // [2] count, generation (zero-initialised once)
  Fix128* fx;           // fixed-point accumulators (fix_scratch): [2H] statistics, then [B, O] output
  int B, K1, H, O;
  int tiles_h;
  int train, save;
  float momentum, eps;
  double count;            // rows in the (global) batch
  MlpPeer peer;
};

__device__ __forceinline__ void grid_barrier(uint32_t* bar, int nblocks) {
  __syncthreads();
  if (threadIdx.x == 0) {
    volatile uint32_t* gen = bar + 1;
    const uint32_t g = *gen;
    __threadfence();
    if (atomicAdd(bar, 1u) == (uint32_t)nblocks - 1u) {
      bar[0] = 0u;
      __threadfence();
      atomicAdd(bar + 1, 1u);
    } else {
      unsigned long long spins = 0;
      while (*gen == g) {
        __nanosleep(32);
        if (++spins > (1ull << 26)) __trap();     // a missing CTA traps instead of hanging the GPU
      }
    }
    __threadfence();
  }
  __syncthreads();
}

// rank-ordered sum of `n` floats over the peers' symmetric buffers (same protocol as xchg_sum_kernel), one CTA
__device__ void peer_sum(float* vals, int n, const MlpPeer& pe) {
  constexpr int SLOTS = 4, MAXW = 8, FLAG_BYTES = 1024;
  const uint32_t seq = *pe.counter + 1u;
  const int slot = (int)(seq % SLOTS);
  uint8_t* mine = reinterpret_cast<uint8_t*>(pe.p[pe.rank]);
  float* my_data = reinterpret_cast<float*>(mine + FLAG_BYTES + (size_t)slot * pe.cap_bytes);
  for (int i = threadIdx.x; i < n; i += blockDim.x) my_data[i] = vals[i];
  __threadfence_system();
  __syncthreads();
  if ((int)threadIdx.x < pe.world) {
    const int r = (int)threadIdx.x;
    uint32_t* pf = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(pe.p[r])) + slot * MAXW + pe.rank;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(pf), "r"(seq) : "memory");
    const uint32_t* mf = reinterpret_cast<const uint32_t*>(mine) + slot * MAXW + r;
    unsigned long long spins = 0;
    for (;;) {
      uint32_t v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mf) : "memory");
      if (v == seq) break;
      __nanosleep(64);
      if (++spins > (1ull << 24)) __trap();
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float acc = 0.f;
    for (int r = 0; r < pe.world; ++r)
      acc += __ldcv(reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(pe.p[r]) + FLAG_BYTES +
                                                   (size_t)slot * pe.cap_bytes) + i);
    vals[i] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) *pe.counter = seq;
}

__global__ void __launch_bounds__(MF_THREADS, 1)
mlp_fused_fwd_kernel(const __grid_constant__ CUtensorMap tmapX, const __grid_constant__ CUtensorMap tmapW1,
                     const __grid_constant__ CUtensorMap tmapW2, const __grid_constant__ CUtensorMap tmapH,
                     const __grid_constant__ CUtensorMap tmapA, const MlpParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  if (smem + MF_NEEDED > smem_raw + MF_TOTAL) __trap();
  float* s_scale = reinterpret_cast<float*>(smem + MF_COEF_OFF);
  float* s_shift = s_scale + 128;
  float* s_b1 = s_shift + 128;
  uint64_t* full_bar = (uint64_t*)(smem + MF_BAR_OFF);
  uint64_t* empty_bar = full_bar + MF_STAGES;
  uint64_t* acc1_bar = empty_bar + MF_STAGES;    // GEMM1 accumulator parked in smem (also: the ring is free)
  uint64_t* w2_bar = acc1_bar + 1;               // W2 slice landed
  uint64_t* a_bar = w2_bar + 1;                  // a-tile written by the 128 epilogue threads
  float* accbuf = reinterpret_cast<float*>(smem + MF_ACC_OFF);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tile_h = blockIdx.x % p.tiles_h;
  const int tile_m = blockIdx.x / p.tiles_h;
  const int m0 = tile_m * 128, n0 = tile_h * 128;
  const int num_kb = p.K1 / 64;

  if (warp == 12 && lane == 0) {
    for (int s = 0; s < MF_STAGES; ++s) { mbar_init(&full_bar[s], 1u); mbar_init(&empty_bar[s], 2u); }
    mbar_init(acc1_bar, 256u);
    mbar_init(w2_bar, 1u);
    mbar_init(a_bar, 128u);
    fence_mbar_init();
    tma_prefetch_desc(&tmapX);
    tma_prefetch_desc(&tmapW1);
    tma_prefetch_desc(&tmapW2);
  }
  if (threadIdx.x < 128) s_b1[threadIdx.x] = p.b1 != nullptr ? p.b1[n0 + threadIdx.x] : 0.f;
  __syncthreads();
  const uint32_t ring = smem_u32(smem);
  const int wg = (warp - 4) >> 2;                       // MMA warpgroup (warps 4-11): tile rows 64*wg .. +63
  const bool wg_leader = (threadIdx.x & 127) == 0;

  if (warp == 12) {
    // ---------------- TMA producer ----------------
    if (lane == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % MF_STAGES;
        const uint32_t ph = (kb / MF_STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        mbar_arrive_expect_tx(&full_bar[s], (uint32_t)MF_STAGE);
        tma_load_2d(ring + s * MF_STAGE, &tmapX, &full_bar[s], kb * 64, m0);
        tma_load_2d(ring + s * MF_STAGE + 16384, &tmapW1, &full_bar[s], kb * 64, n0);
      }
      // the ring is free once every GEMM1 MMA has completed: W2[:, n0 .. n0 + 128) as two [O x 64] k-blocks
      mbar_wait(acc1_bar, 0);
      mbar_arrive_expect_tx(w2_bar, (uint32_t)(2 * p.O * 128));
      tma_load_2d(ring + 32768, &tmapW2, w2_bar, n0, 0);
      tma_load_2d(ring + 65536, &tmapW2, w2_bar, n0 + 64, 0);
    }
    __syncwarp();
  } else if (warp >= 4) {
    // ---------------- MMA warpgroups: GEMM1 ----------------
    float d[64];
    int prev_s = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      const int s = kb % MF_STAGES;
      const uint32_t ph = (kb / MF_STAGES) & 1;
      mbar_wait(&full_bar[s], ph);
      const uint64_t adesc = make_smem_desc_sw128(ring + s * MF_STAGE + wg * 8192, 16, 1024);
      const uint64_t bdesc = make_smem_desc_sw128(ring + s * MF_STAGE + 16384, 16, 1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_bf16<128, 0, 0>(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
      wg_commit();
      wg_wait<1>();
      if (wg_leader && prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
    }
    wg_wait<0>();
    wg_fence_acc(d);
    acc_store_smem<128>(accbuf, MF_ACC_LD, wg * 64, 0, d);
    mbar_arrive(acc1_bar);
  }
  // ---------------- phase 2: statistics of h (epilogue warps 0-3; lane = row) ----------------
  const int row = warp * 32 + lane;          // valid for warps 0-3
  const bool rvalid = warp < 4 && (m0 + row) < p.B;
  if (warp < 4) {
    mbar_wait(acc1_bar, 0);
    uint8_t* hst = smem + MF_HSTAGE_OFF;
#pragma unroll 1
    for (int c0 = 0; c0 < 128; c0 += 32) {
      uint32_t r[32];
      acc_load_row32(accbuf + row * MF_ACC_LD + c0, r);
      float v[32], q[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        v[j] = rvalid ? __uint_as_float(r[j]) + s_b1[c0 + j] : 0.f;
        q[j] = v[j] * v[j];
      }
      if (p.save) {
        // h (bf16) -> staging in the K-major 128-byte swizzle ([128 rows][64 cols] x 2), TMA-stored below
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          uint4 w;
          w.x = pack_bf16x2(v[j], v[j + 1]); w.y = pack_bf16x2(v[j + 2], v[j + 3]);
          w.z = pack_bf16x2(v[j + 4], v[j + 5]); w.w = pack_bf16x2(v[j + 6], v[j + 7]);
          const int c = c0 + j;
          *reinterpret_cast<uint4*>(hst + (c >> 6) * 16384 + sw128_offset((uint32_t)row, (uint32_t)((c & 63) >> 3))) = w;
        }
      }
      if (p.train) {
#pragma unroll
        for (int o = 16, n = 32; o >= 1; o >>= 1, n >>= 1) {
          const bool up = (lane & o) != 0;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            if (j < n / 2) {
              const float sv = up ? v[j] : v[j + n / 2], kv = up ? v[j + n / 2] : v[j];
              const float sq = up ? q[j] : q[j + n / 2], kq = up ? q[j + n / 2] : q[j];
              v[j] = kv + __shfl_xor_sync(0xffffffffu, sv, o);
              q[j] = kq + __shfl_xor_sync(0xffffffffu, sq, o);
            }
          }
        }
        fix_add(p.fx + n0 + c0 + lane, v[0]);
        fix_add(p.fx + p.H + n0 + c0 + lane, q[0]);
      }
    }
    if (p.save) {
      fence_proxy_async_smem();
    }
  }
  if (p.save) {
    __syncthreads();
    if (threadIdx.x == 0) {
      tma_store_2d(&tmapH, smem_u32(smem + MF_HSTAGE_OFF), n0, m0);
      tma_store_2d(&tmapH, smem_u32(smem + MF_HSTAGE_OFF + 16384), n0 + 64, m0);
      tma_store_commit();
    }
  }
  if (p.train) {
    grid_barrier(p.grid_bar, (int)gridDim.x);
    // the fixed-point sums (identical in every run, whatever the order of the CTAs) -> fp32 statistics
    if (tile_m == 0 && threadIdx.x < 128) {
      const int c = n0 + (int)threadIdx.x;
      const Fix128* f1 = p.fx + c;
      const Fix128* f2 = p.fx + p.H + c;
      p.stats[c] = (float)fix_value(Fix128{__ldcg(&f1->lo), __ldcg(&f1->hi), __ldcg(&f1->spill)});
      p.stats[p.H + c] = (float)fix_value(Fix128{__ldcg(&f2->lo), __ldcg(&f2->hi), __ldcg(&f2->spill)});
      p.fx[c] = Fix128{0ull, 0ll, 0.0};         // only these threads read them: leave the scratch zeroed (fix_scratch)
      p.fx[p.H + c] = Fix128{0ull, 0ll, 0.0};
    }
    grid_barrier(p.grid_bar, (int)gridDim.x);
    if (p.peer.world > 1) {
      if (blockIdx.x == 0) peer_sum(p.stats, 2 * p.H, p.peer);
      grid_barrier(p.grid_bar, (int)gridDim.x);
    }
  }
  // ---------------- phase 3: coefficients, a = relu(bn(h)) -> A operand of GEMM2 ----------------
  if (threadIdx.x < 128) {
    const int c = n0 + (int)threadIdx.x;
    float mean, invstd;
    if (p.train) {
      const double mu = (double)__ldcg(p.stats + c) / p.count;
      double var = (double)__ldcg(p.stats + p.H + c) / p.count - mu * mu;
      if (var < 0.0) var = 0.0;
      mean = (float)mu;
      invstd = (float)(1.0 / sqrt(var + (double)p.eps));
      if (tile_m == 0 && p.running_mean != nullptr) {
        const double unbiased = p.count > 1.0 ? var * p.count / (p.count - 1.0) : var;
        p.running_mean[c] = (1.f - p.momentum) * p.running_mean[c] + p.momentum * mean;
        p.running_var[c] = (1.f - p.momentum) * p.running_var[c] + p.momentum * (float)unbiased;
      }
    } else {
      mean = p.running_mean[c];
      invstd = 1.f / sqrtf(p.running_var[c] + p.eps);
    }
    const float sc = p.gamma[c] * invstd;
    const float sh = p.beta[c] - mean * sc;
    s_scale[threadIdx.x] = sc;
    s_shift[threadIdx.x] = sh;
    if (tile_m == 0) {
      p.coeffs[c] = sc;
      p.coeffs[p.H + c] = sh;
      p.coeffs[2 * p.H + c] = mean;
      p.coeffs[3 * p.H + c] = invstd;
    }
  }
  __syncthreads();
  if (warp < 4) {
#pragma unroll 1
    for (int c0 = 0; c0 < 128; c0 += 32) {
      uint32_t r[32];
      acc_load_row32(accbuf + row * MF_ACC_LD + c0, r);
#pragma unroll
      for (int j = 0; j < 32; j += 8) {
        float a[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float h = __uint_as_float(r[j + e]) + s_b1[c0 + j + e];
          a[e] = rvalid ? fmaxf(h * s_scale[c0 + j + e] + s_shift[c0 + j + e], 0.f) : 0.f;
        }
        uint4 w;
        w.x = pack_bf16x2(a[0], a[1]); w.y = pack_bf16x2(a[2], a[3]);
        w.z = pack_bf16x2(a[4], a[5]); w.w = pack_bf16x2(a[6], a[7]);
        const int c = c0 + j;
        *reinterpret_cast<uint4*>(smem + (c >> 6) * 16384 + sw128_offset((uint32_t)row, (uint32_t)((c & 63) >> 3))) = w;
      }
    }
    fence_proxy_async_smem();
    mbar_arrive(a_bar);
  }
  if (warp >= 4 && warp < 12) {
    // ---------------- phase 4: GEMM2 partial, K = this CTA's 128 hidden columns, 64 output columns at a time -----
    mbar_wait(a_bar, 0);
    mbar_wait(w2_bar, 0);
    const int t = threadIdx.x & 127;
    const int r0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);   // tile row of d[4j], d[4j+1]; +8 for d[4j+2 ..]
    float d2[32];
#pragma unroll 1
    for (int o0 = 0; o0 < p.O; o0 += 64) {
      wg_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb) {
        const uint64_t adesc = make_smem_desc_sw128(ring + kb * 16384 + wg * 8192, 16, 1024);
        const uint64_t bdesc = make_smem_desc_sw128(ring + 32768 + kb * 32768 + o0 * 128, 16, 1024);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_bf16<64, 0, 0>(d2, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(d2);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = o0 + 8 * j + 2 * (t & 3);
        if (c >= p.O) continue;   // O is a multiple of 16: c + 1 < O too
        float2 bb = make_float2(0.f, 0.f);
        if (tile_h == 0 && p.b2 != nullptr) bb = make_float2(p.b2[c], p.b2[c + 1]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rr = m0 + r0 + 8 * h;
          if (rr < p.B) {
            Fix128* acc = p.fx + 2 * p.H + (int64_t)rr * p.O + c;
            fix_add(acc, d2[4 * j + 2 * h] + bb.x);
            fix_add(acc + 1, d2[4 * j + 2 * h + 1] + bb.y);
          }
        }
      }
    }
  }
  if (warp < 4 && p.save) {
    if (threadIdx.x == 0) {
      // a (bf16) for the backward pass: the GEMM2 operand buffers are already in the TMA-storable layout
      mbar_wait(a_bar, 0);                 // all 128 rows written and fenced
      tma_store_2d(&tmapA, ring, n0, m0);
      tma_store_2d(&tmapA, ring + 16384, n0 + 64, m0);
      tma_store_commit();
      tma_store_wait_all();
    }
  }
}

typedef CUresult (*PFN_encodeTiledMF)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int mf_tmap(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  static PFN_encodeTiledMF fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess) {
      set_last_error("cuTensorMapEncodeTiled entry point unavailable");
      return -1;
    }
    fn = (PFN_encodeTiledMF)ptr;
  }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(bf16)};
  cuuint32_t box[2] = {64u, box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("mlp_fused: cuTensorMapEncodeTiled failed (%d): rows=%llu cols=%llu ld=%llu box_rows=%u", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows);
    return -1;
  }
  return 0;
}

}  // namespace byol

using namespace byol;

// 1 if byol_mlp_fused_fwd can run this shape on the current device (else use the unfused kernels)
extern "C" int byol_mlp_fused_supported(int B, int K1, int H, int O) {
  if (B <= 0 || K1 <= 0 || K1 % 64 != 0 || H <= 0 || H % 128 != 0 || O < 16 || O > 256 || O % 16 != 0) return 0;
  const int tiles = ((B + 127) / 128) * (H / 128);
  return tiles <= device_sm_count() ? 1 : 0;
}

// x [B, K1] bf16; w1 [H, ldw1 >= K1] bf16 (fprop layout); w2 [O, ldw2 >= H] bf16; b1 / gamma / beta [H], b2 [O] fp32.
// stats: [2H] fp32 ZEROED (train); out: [B, O] fp32 ZEROED; coeffs: [4, H]; h_save / a_save: optional bf16 [B, H].
// grid_bar: 2 zero-initialised uint32 (persistent).  count: rows of the global batch (B * world).
// peer_ptrs (host, [world]) / cap_bytes / counter: the SyncBatchNorm exchange of csrc/xchg.cu, or world <= 1.
extern "C" int byol_mlp_fused_fwd(const void* x, const void* w1, const float* b1, const float* gamma, const float* beta,
                                  const void* w2, const float* b2, float* stats, float* running_mean,
                                  float* running_var, float momentum, float eps, double count, float* coeffs,
                                  float* out, void* h_save, void* a_save, void* grid_bar, int B, int K1, int H, int O,
                                  int ldw1, int ldw2, int train, const uint64_t* peer_ptrs, int world, int rank,
                                  int64_t cap_bytes, void* counter, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && w1 && gamma && beta && w2 && coeffs && out && grid_bar, "byol_mlp_fused_fwd: null pointer");
  BYOL_CHECK_ARG(byol_mlp_fused_supported(B, K1, H, O), "byol_mlp_fused_fwd: unsupported shape B=%d K1=%d H=%d O=%d", B,
                 K1, H, O);
  BYOL_CHECK_ARG(!train || stats != nullptr, "byol_mlp_fused_fwd: train mode needs the statistics buffer");
  BYOL_CHECK_ARG(train || (running_mean && running_var), "byol_mlp_fused_fwd: eval mode needs the running statistics");
  BYOL_CHECK_ARG((h_save == nullptr) == (a_save == nullptr), "byol_mlp_fused_fwd: h_save and a_save go together");
  BYOL_CHECK_ARG(world <= 1 || (peer_ptrs && counter && world <= 8 && (int64_t)2 * H * 4 <= cap_bytes),
                 "byol_mlp_fused_fwd: bad peer exchange arguments");
  MlpParams p;
  memset(&p, 0, sizeof(p));
  p.b1 = b1; p.gamma = gamma; p.beta = beta; p.b2 = b2;
  p.stats = stats; p.running_mean = running_mean; p.running_var = running_var; p.coeffs = coeffs; p.out = out;
  p.grid_bar = (uint32_t*)grid_bar;
  p.B = B; p.K1 = K1; p.H = H; p.O = O;
  p.tiles_h = H / 128;
  p.train = train ? 1 : 0;
  p.save = h_save != nullptr ? 1 : 0;
  p.momentum = momentum; p.eps = eps; p.count = count;
  p.peer.world = world > 1 ? world : 1;
  p.peer.rank = rank;
  p.peer.cap_bytes = cap_bytes;
  p.peer.counter = (uint32_t*)counter;
  for (int r = 0; r < 8; ++r) p.peer.p[r] = (world > 1 && r < world) ? peer_ptrs[r] : 0ull;
  CUtensorMap tx, tw1, tw2, th, ta;
  if (mf_tmap(&tx, x, (uint64_t)B, (uint64_t)K1, (uint64_t)K1, 128u) != 0) return -3;
  if (mf_tmap(&tw1, w1, (uint64_t)H, (uint64_t)K1, (uint64_t)ldw1, 128u) != 0) return -3;
  if (mf_tmap(&tw2, w2, (uint64_t)O, (uint64_t)H, (uint64_t)ldw2, (uint32_t)O) != 0) return -3;
  if (p.save) {
    if (mf_tmap(&th, h_save, (uint64_t)B, (uint64_t)H, (uint64_t)H, 128u) != 0) return -3;
    if (mf_tmap(&ta, a_save, (uint64_t)B, (uint64_t)H, (uint64_t)H, 128u) != 0) return -3;
  } else {
    th = tx; ta = tx;
  }
  static bool attr_set[kMaxDevices] = {};
  const int dev_slot = device_slot();
  if (!attr_set[dev_slot]) {
    cudaError_t e = cudaFuncSetAttribute(mlp_fused_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MF_TOTAL);
    if (e != cudaSuccess) { set_last_error("cudaFuncSetAttribute(mlp_fused) failed: %s", cudaGetErrorString(e)); return -2; }
    attr_set[dev_slot] = true;
  }
  const int grid = ((B + 127) / 128) * p.tiles_h;
  // cooperative launch: every CTA must be resident for the grid barrier
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(MF_THREADS);
  cfg.dynamicSmemBytes = MF_TOTAL;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  p.fx = fix_scratch(stream, 2 * (int64_t)H + (int64_t)B * O);
  if (p.fx == nullptr) return -2;
  cudaError_t e = cudaLaunchKernelEx(&cfg, mlp_fused_fwd_kernel, tx, tw1, tw2, th, ta, p);
  if (e != cudaSuccess) {
    set_last_error("byol_mlp_fused_fwd: cooperative launch failed: %s", cudaGetErrorString(e));
    return -100;
  }
  if (check_launch("mlp_fused_fwd_kernel") != 0) return -100;
  return fix_done(stream, fix_flush(p.fx + 2 * (int64_t)H, out, (int64_t)B * O, stream));
}
