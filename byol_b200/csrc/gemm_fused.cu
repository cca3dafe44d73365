// byol_b200 — plain GEMM (1x1 / stride-1 convolution, both operands by TMA) with a residual epilogue, on wgmma.
//
//   out[M, N] = act( src[M, K] x wt[N, K]^T + bias[n] + (resid_mask ? resid : 0) ),
//   M = pixels, N = output channels (> 64), bf16 in / fp32 accumulate, bf16 out
//
// conv_igemm.cu routes here every 1x1 / stride-1 convolution with a bf16 residual, a bf16 output, no statistics and
// N > 64.  In training that is the conv1 dgrad of a torchvision Bottleneck block, which adds the (ReLU-masked)
// gradient of the residual branch.
//
// Why a separate kernel: in conv_igemm_kernel every epilogue lane fetched its residual row straight from global
// memory (32 rows x 16 B per warp-load, issued only after the accumulator arrived): 665 us instead of 187 us for the
// stage-1 conv1 dgrad of ResNet-50 (tools/time_dgrad_resid.py).  Here the residual tile comes by TMA into the warp's
// swizzled staging buffer — prefetched one chunk ahead, so its latency hides behind the MMA — and the same buffer is
// then reused to stage the output tile for the TMA store; the bias vector lives in shared memory.
//
// Warp roles (544 threads, 1 CTA / SM): warps 0-7 epilogue (tile row quarter w & 3, column half w >> 2), warps 8-15
// two MMA warpgroups (tile rows 0-63 / 64-127, accumulators in registers, handed to the epilogue through an fp32
// tile in shared memory), warp 16 TMA producer (2-stage operand ring, persistent tile loop).
#include <string.h>

#include "common.cuh"

namespace byol {

static constexpr int GF_BM = 128, GF_BN = 128, GF_BK = 64, GF_STAGES = 2;
static constexpr int GF_A_STAGE = GF_BM * 128, GF_B_STAGE = GF_BN * 128;
static constexpr int GF_EW = 8, GF_CPW = 2;
static constexpr int GF_A_OFF = 0;
static constexpr int GF_B_OFF = GF_STAGES * GF_A_STAGE;
static constexpr int GF_STAGE_OFF = GF_B_OFF + GF_STAGES * GF_B_STAGE;          // per warp 2 x 2048 B
static constexpr int GF_PARAM_OFF = GF_STAGE_OFF + GF_EW * 4096;                // per warp 64 bias floats
static constexpr int GF_ACC_LD = acc_ld(GF_BN);
static constexpr int GF_ACC_OFF = GF_PARAM_OFF + GF_EW * 256;                   // [GF_BM][GF_ACC_LD] fp32
static constexpr int GF_BAR_OFF = GF_ACC_OFF + GF_BM * GF_ACC_LD * 4;
static constexpr int GF_NEEDED = GF_BAR_OFF + 512;
static constexpr int GF_TOTAL = GF_NEEDED + 768;
static constexpr int GF_THREADS = 17 * 32;
static_assert(GF_TOTAL <= 232448, "one CTA per SM");

struct GemmFusedParams {
  const uint8_t* resid_mask;     // optional ReLU bits over the [M, ldc] index space of resid: add resid where set
  const float* bias;             // optional [N]
  int relu;
  int M, N, ldc, num_kb, tiles_n;
};

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

__global__ void __launch_bounds__(GF_THREADS, 1)
gemm_fused_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB,
                  const __grid_constant__ CUtensorMap tmapC, const __grid_constant__ CUtensorMap tmapR,
                  const GemmFusedParams p, const int num_tiles) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  if (smem + GF_NEEDED > smem_raw + GF_TOTAL) __trap();
  uint8_t* smemA = smem + GF_A_OFF;
  uint8_t* smemB = smem + GF_B_OFF;
  uint64_t* full_bar = (uint64_t*)(smem + GF_BAR_OFF);
  uint64_t* empty_bar = full_bar + GF_STAGES;
  uint64_t* tfull_bar = empty_bar + GF_STAGES;  // accumulator tile ready for the epilogue
  uint64_t* tempty_bar = tfull_bar + 1;         // accumulator tile drained
  uint64_t* rbar = tempty_bar + 1;              // [GF_EW][2] residual tile landed
  float* accbuf = reinterpret_cast<float*>(smem + GF_ACC_OFF);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int MMA_WARP = 8, TMA_WARP = 16;

  if (warp == TMA_WARP && lane == 0) {
    for (int s = 0; s < GF_STAGES; ++s) { mbar_init(&full_bar[s], 1u); mbar_init(&empty_bar[s], 2u); }
    mbar_init(tfull_bar, 256u);
    mbar_init(tempty_bar, (uint32_t)GF_EW);
    for (int i = 0; i < 2 * GF_EW; ++i) mbar_init(&rbar[i], 1u);
    fence_mbar_init();
    tma_prefetch_desc(&tmapA);
    tma_prefetch_desc(&tmapB);
    tma_prefetch_desc(&tmapC);
    tma_prefetch_desc(&tmapR);
  }
  __syncthreads();

  if (warp < GF_EW) {
    // ======================= epilogue =====================================================
    const int quarter = warp & 3;
    const int col_w0 = (warp >> 2) * (GF_CPW * 32);
    const uint32_t wstage = smem_u32(smem + GF_STAGE_OFF + warp * 4096);
    float* wbias = reinterpret_cast<float*>(smem + GF_PARAM_OFF + warp * 256);
    const uint32_t wbias_u32 = smem_u32(wbias);
    uint64_t* my_rbar = rbar + 2 * warp;
    // residual tiles are prefetched one chunk ahead: chunk sequence number q -> buffer q & 1
    auto chunk_valid = [&](int tile, int cl) -> bool {
      return tile < num_tiles && (tile % p.tiles_n) * GF_BN + col_w0 + cl * 32 < p.N;
    };
    auto issue_resid = [&](int tile, int cl, int buf) {
      if (lane == 0) {
        const int m0 = (tile / p.tiles_n) * GF_BM, n0 = (tile % p.tiles_n) * GF_BN;
        mbar_arrive_expect_tx(&my_rbar[buf], 2048u);
        tma_load_2d(wstage + (uint32_t)buf * 2048u, &tmapR, &my_rbar[buf], n0 + col_w0 + cl * 32, m0 + quarter * 32);
      }
    };
    auto next_chunk = [&](int& tile, int& cl) {     // the next VALID chunk after (tile, cl), or tile >= num_tiles
      for (;;) {
        if (++cl == GF_CPW) { cl = 0; tile += gridDim.x; }
        if (tile >= num_tiles || chunk_valid(tile, cl)) return;
      }
    };
    int q = 0;                       // valid chunks processed so far
    uint32_t rphase[2] = {0u, 0u};
    {
      int t0 = blockIdx.x, c0 = -1;
      next_chunk(t0, c0);            // first valid chunk of this warp (c0 = -1 -> starts at cl 0 of blockIdx.x)
      if (t0 < num_tiles) issue_resid(t0, c0, 0);
    }
    int bias_n0 = -1;
    int local = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++local) {
      const int m0 = (tile / p.tiles_n) * GF_BM;
      const int n0 = (tile % p.tiles_n) * GF_BN;
      if (bias_n0 != n0) {
        bias_n0 = n0;
        // this warp's 64 columns of the bias -> shared memory (read back as broadcast LDS.128)
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int c = n0 + col_w0 + lane + 32 * i;
          wbias[lane + 32 * i] = (c < p.N && p.bias != nullptr) ? __ldg(p.bias + c) : 0.f;
        }
        __syncwarp();
      }
      const int mrow0 = m0 + quarter * 32;
      const int m = mrow0 + lane;
      const bool mvalid = m < p.M;
      mbar_wait(tfull_bar, (uint32_t)(local & 1));
#pragma unroll
      for (int cl = 0; cl < GF_CPW; ++cl) {
        const int c0 = col_w0 + cl * 32;
        const int nbase = n0 + c0;
        const bool valid = nbase < p.N;          // warp-uniform
        const int buf = q & 1;
        const uint32_t sbuf = wstage + (uint32_t)buf * 2048u;
        uint32_t mbits = 0xffffffffu;
        if (valid) {
          // prefetch the NEXT valid chunk's residual tile into the other buffer (its last use, the output store of
          // chunk q - 1, must have finished reading shared memory)
          int nt = tile, nc = cl;
          next_chunk(nt, nc);
          if (nt < num_tiles) {
            if (lane == 0) tma_store_wait_read();
            issue_resid(nt, nc, buf ^ 1);
          }
          if (p.resid_mask != nullptr && mvalid) {
            const uint8_t* mp = p.resid_mask + (((int64_t)m * p.ldc + nbase) >> 3);
            if ((p.ldc & 31) == 0 && nbase + 32 <= p.N) {
              mbits = __ldg(reinterpret_cast<const uint32_t*>(mp));
            } else {
              mbits = 0u;
#pragma unroll
              for (int j = 0; j < 4; ++j)
                if (nbase + 8 * j < p.N) mbits |= (uint32_t)__ldg(mp + j) << (8 * j);
            }
          }
        }
        uint32_t r[32];
        acc_load_row32(accbuf + (quarter * 32 + lane) * GF_ACC_LD + c0, r);
        if (cl == GF_CPW - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(tempty_bar);
        }
        if (!valid) continue;
        // v = acc + bias (bias broadcast from this warp's shared-memory copy, 0 where absent)
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const uint4 bs = lds128(wbias_u32 + (uint32_t)(cl * 32 + j) * 4u);
          v[j] = __uint_as_float(r[j]) + __uint_as_float(bs.x);
          v[j + 1] = __uint_as_float(r[j + 1]) + __uint_as_float(bs.y);
          v[j + 2] = __uint_as_float(r[j + 2]) + __uint_as_float(bs.z);
          v[j + 3] = __uint_as_float(r[j + 3]) + __uint_as_float(bs.w);
        }
        // v += masked residual: this lane's row of the residual tile, 4 x 16 B at the 64-byte-swizzle positions (rows
        // >= M are TMA zeros).  A masked-off element adds +0.f instead of being skipped: a -0 sum becomes +0, as when
        // the masked residual is added as a tensor.
        mbar_wait(&my_rbar[buf], rphase[buf]);
        rphase[buf] ^= 1u;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 qv = lds128(sbuf + (uint32_t)lane * 64u + (uint32_t)((j ^ ((lane >> 1) & 3)) << 4));
          const uint32_t w4[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int c = 8 * j + 2 * e;
            const float lo = __uint_as_float(w4[e] << 16), hi = __uint_as_float(w4[e] & 0xffff0000u);
            v[c] += ((mbits >> c) & 1u) ? lo : 0.f;
            v[c + 1] += ((mbits >> (c + 1)) & 1u) ? hi : 0.f;
          }
        }
        if (p.relu) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        // stage the output tile in the SAME buffer (every lane has read its residual row), TMA store
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint4 qv;
          qv.x = pack_bf16x2(v[8 * j + 0], v[8 * j + 1]);
          qv.y = pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
          qv.z = pack_bf16x2(v[8 * j + 4], v[8 * j + 5]);
          qv.w = pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
          const uint32_t off = (uint32_t)lane * 64u + (uint32_t)((j ^ ((lane >> 1) & 3)) << 4);
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sbuf + off), "r"(qv.x), "r"(qv.y), "r"(qv.z),
                       "r"(qv.w)
                       : "memory");
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          tma_store_2d(&tmapC, sbuf, nbase, mrow0);
          tma_store_commit();
        }
        __syncwarp();
        ++q;
      }
    }
    if (lane == 0) tma_store_wait_all();
  } else if (warp >= MMA_WARP && warp < TMA_WARP) {
    // warpgroup wg: tile rows 64*wg .. +63 (A rows 8 KB further into the stage)
    const int wg = (warp - MMA_WARP) >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    float d[GF_BN / 2];
    int it = 0, local = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++local) {
      int prev_s = -1;
      for (int kb = 0; kb < p.num_kb; ++kb, ++it) {
        const int s = it % GF_STAGES;
        const uint32_t ph = (it / GF_STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint64_t adesc = make_smem_desc_sw128(smem_u32(smemA + s * GF_A_STAGE + wg * 8192), 16, 1024);
        const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smemB + s * GF_B_STAGE), 16, 1024);
        wg_fence();
#pragma unroll
        for (int k = 0; k < GF_BK / 16; ++k)
          wgmma_bf16<GF_BN, 0, 0>(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
        wg_commit();
        wg_wait<1>();
        if (leader && prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wg_wait<0>();
      wg_fence_acc(d);
      if (leader && prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
      mbar_wait(tempty_bar, (uint32_t)((local & 1) ^ 1));
      acc_store_smem<GF_BN>(accbuf, GF_ACC_LD, wg * 64, 0, d);
      mbar_arrive(tfull_bar);
    }
  } else if (warp == TMA_WARP) {
    if (lane == 0) {
      constexpr uint32_t tx = (uint32_t)(GF_A_STAGE + GF_B_STAGE);
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / p.tiles_n) * GF_BM, n0 = (tile % p.tiles_n) * GF_BN;
        for (int kb = 0; kb < p.num_kb; ++kb, ++it) {
          const int s = it % GF_STAGES;
          const uint32_t ph = (it / GF_STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], tx);
          tma_load_2d(smem_u32(smemB + s * GF_B_STAGE), &tmapB, &full_bar[s], kb * GF_BK, n0);
          tma_load_2d(smem_u32(smemA + s * GF_A_STAGE), &tmapA, &full_bar[s], kb * GF_BK, m0);
        }
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// true if the residual-epilogue kernel can run this GEMM (the caller falls back to conv_igemm_kernel otherwise)
bool gemm_fused_applicable(int M, int C, int Ndim, int ldw, int ldc) {
  return M > 0 && C % 8 == 0 && Ndim > 64 && Ndim % 8 == 0 && ldc % 8 == 0 && ldc >= Ndim && ldw % 8 == 0 && ldw >= C;
}

int gemm_fused_launch(const void* src, const void* wt, void* dst, const void* resid, const void* resid_mask,
                      const float* bias, int M, int C, int Ndim, int ldw, int ldc, int relu, cudaStream_t stream) {
  BYOL_CHECK_ARG(src && wt && dst && resid, "gemm_fused: null pointer (src, wt, dst and resid are required)");
  BYOL_CHECK_ARG(gemm_fused_applicable(M, C, Ndim, ldw, ldc), "gemm_fused: unsupported shape M=%d C=%d N=%d ldw=%d ldc=%d",
                 M, C, Ndim, ldw, ldc);
  GemmFusedParams p;
  memset(&p, 0, sizeof(p));
  p.resid_mask = (const uint8_t*)resid_mask;
  p.bias = bias;
  p.relu = relu;
  p.M = M; p.N = Ndim; p.ldc = ldc;
  p.num_kb = (C + GF_BK - 1) / GF_BK;
  p.tiles_n = (Ndim + GF_BN - 1) / GF_BN;
  const int tiles_m = (M + GF_BM - 1) / GF_BM;
  const int num_tiles = tiles_m * p.tiles_n;
  CUtensorMap ta, tb, tc, tr;
  if (tmap_2d(&ta, src, (uint64_t)M, (uint64_t)C, (uint64_t)C, GF_BM, 64u, "gemm_fused A") != 0) return -3;
  if (tmap_2d(&tb, wt, (uint64_t)Ndim, (uint64_t)C, (uint64_t)ldw, GF_BN, 64u, "gemm_fused B") != 0) return -3;
  if (tmap_2d(&tc, dst, (uint64_t)M, (uint64_t)Ndim, (uint64_t)ldc, 32u, 32u, "gemm_fused C") != 0) return -3;
  if (tmap_2d(&tr, resid, (uint64_t)M, (uint64_t)Ndim, (uint64_t)ldc, 32u, 32u, "gemm_fused R") != 0) return -3;
  if (smem_opt_in((const void*)gemm_fused_kernel, GF_TOTAL, "gemm_fused_kernel") != 0) return -2;
  int grid = device_sm_count();
  if (grid > num_tiles) grid = num_tiles;
  gemm_fused_kernel<<<grid, GF_THREADS, GF_TOTAL, stream>>>(ta, tb, tc, tr, p, num_tiles);
  return check_launch("gemm_fused_kernel");
}

}  // namespace byol
