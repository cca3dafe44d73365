// byol_b200 — plain GEMM (1x1 / stride-1 convolution, both operands by TMA) with a RICH epilogue, on wgmma.
//
//   out[M, N] = epilogue( src[M, K] x wt[N, K]^T ),   M = pixels, N = output channels (> 64), bf16 in / fp32 accumulate
//
// Used where the epilogue needs a second [M, N] tensor or per-column vectors (torchvision Bottleneck reached from
// /root/reference/main.py:237, and its backward under main.py:617):
//   * conv1 dgrad + the (ReLU-masked) gradient of the residual branch                 (resid, resid_mask)
//   * block-output BatchNorm fused into the expanding 1x1 convolution:
//       statistics-only pass (no_store), apply pass  out = relu(acc*scale + shift + resid), ReLU mask bits
//   * BatchNorm backward of that never-stored conv output, by recomputation:
//       reduce pass (bwd_reduce: sum dz, sum dz*xhat), apply pass  dy = A*dz + B*acc + Cc
//
// Why a separate kernel: in conv_igemm_kernel every epilogue lane fetched its residual row straight from global
// memory (32 rows x 16 B per warp-load, issued only after the accumulator arrived): 665 us instead of 187 us for the
// stage-1 conv1 dgrad of ResNet-50 (tools/time_dgrad_resid.py).  Here the residual tile comes by TMA into the warp's
// swizzled staging buffer — prefetched one chunk ahead, so its latency hides behind the MMA — and the same buffer is
// then reused to stage the output tile for the TMA store; per-column vectors live in shared memory.
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
static constexpr int GF_PARAM_OFF = GF_STAGE_OFF + GF_EW * 4096;                // per warp 3 x 64 floats
static constexpr int GF_ACC_LD = acc_ld(GF_BN);
static constexpr int GF_ACC_OFF = GF_PARAM_OFF + GF_EW * 768;                   // [GF_BM][GF_ACC_LD] fp32
static constexpr int GF_BAR_OFF = GF_ACC_OFF + GF_BM * GF_ACC_LD * 4;
static constexpr int GF_NEEDED = GF_BAR_OFF + 512;
static constexpr int GF_TOTAL = GF_NEEDED + 768;
static constexpr int GF_THREADS = 17 * 32;
static_assert(GF_TOTAL <= 232448, "one CTA per SM");

struct GemmFusedParams {
  const uint8_t* resid_mask;     // optional ReLU bits over the [M, ldc] index space of resid: add / use resid where set
  const float* colscale;         // optional [N]: t = acc * colscale + bias
  const float* bias;             // optional [N]
  const float* resid_colscale;   // optional [N]: residual term scaled per column
  uint8_t* mask_out;             // optional: bits (stored value > 0), [M * ldc / 8]
  float* col_sum;                // statistics / backward sums, [N]
  float* col_sqsum;
  Fix128* fx;                 // with col_sum: [2][N] fixed-point accumulators (fix_scratch)
  int has_resid, relu, no_store, bwd_reduce;
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
    if (!p.no_store && !p.bwd_reduce) tma_prefetch_desc(&tmapC);
    if (p.has_resid) tma_prefetch_desc(&tmapR);
  }
  __syncthreads();

  if (warp < GF_EW) {
    // ======================= epilogue =====================================================
    const int quarter = warp & 3;
    const int col_w0 = (warp >> 2) * (GF_CPW * 32);
    const uint32_t wstage = smem_u32(smem + GF_STAGE_OFF + warp * 4096);
    float* wparam = reinterpret_cast<float*>(smem + GF_PARAM_OFF + warp * 768);   // [colscale | bias | rscale][64]
    const uint32_t wparam_u32 = smem_u32(wparam);
    uint64_t* my_rbar = rbar + 2 * warp;
    const bool do_stats = p.col_sum != nullptr;
    const bool red_mode = p.bwd_reduce != 0;
    const bool storing = !p.no_store && !red_mode;
    uint64_t cs1[GF_CPW], cs2[GF_CPW];
    float racc1[GF_CPW], racc2[GF_CPW];
#pragma unroll
    for (int i = 0; i < GF_CPW; ++i) { cs1[i] = 0ull; cs2[i] = 0ull; racc1[i] = 0.f; racc2[i] = 0.f; }
    int stat_n0 = -1;
    auto flush_stats = [&]() {
#pragma unroll
      for (int i = 0; i < GF_CPW; ++i) {
        if (red_mode) {
          const int col = stat_n0 + col_w0 + i * 32 + lane;
          if (col < p.N) {
            fix_add(p.fx + col, racc1[i]);
            fix_add(p.fx + p.N + col, racc2[i]);
          }
          racc1[i] = 0.f; racc2[i] = 0.f;
        } else {
          float2 a = f2_unpack(cs1[i]), b = f2_unpack(cs2[i]);
          a.x += __shfl_xor_sync(0xffffffffu, a.x, 16);
          a.y += __shfl_xor_sync(0xffffffffu, a.y, 16);
          b.x += __shfl_xor_sync(0xffffffffu, b.x, 16);
          b.y += __shfl_xor_sync(0xffffffffu, b.y, 16);
          const int col = stat_n0 + col_w0 + i * 32 + 2 * (lane & 15);
          if (lane < 16 && col < p.N) {   // N is a multiple of 8: col + 1 is valid too
            fix_add(p.fx + col, a.x);
            fix_add(p.fx + col + 1, a.y);
            fix_add(p.fx + p.N + col, b.x);
            fix_add(p.fx + p.N + col + 1, b.y);
          }
          cs1[i] = 0ull; cs2[i] = 0ull;
        }
      }
    };
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
    if (p.has_resid) {
      int t0 = blockIdx.x, c0 = -1;
      next_chunk(t0, c0);            // first valid chunk of this warp (c0 = -1 -> starts at cl 0 of blockIdx.x)
      if (t0 < num_tiles) issue_resid(t0, c0, 0);
    }
    int local = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++local) {
      const int m0 = (tile / p.tiles_n) * GF_BM;
      const int n0 = (tile % p.tiles_n) * GF_BN;
      if (stat_n0 != n0) {
        if (do_stats && stat_n0 >= 0) flush_stats();
        stat_n0 = n0;
        // this warp's 64 columns of the per-column vectors -> shared memory (read back as broadcast LDS.128)
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int c = n0 + col_w0 + lane + 32 * i;
          const bool ok = c < p.N;
          wparam[lane + 32 * i] = (ok && p.colscale != nullptr) ? __ldg(p.colscale + c) : 1.f;
          wparam[64 + lane + 32 * i] = (ok && p.bias != nullptr) ? __ldg(p.bias + c) : 0.f;
          wparam[128 + lane + 32 * i] = (ok && p.resid_colscale != nullptr) ? __ldg(p.resid_colscale + c) : 1.f;
        }
        __syncwarp();
      }
      const int mrow0 = m0 + quarter * 32;
      const int m = mrow0 + lane;
      const bool mvalid = m < p.M;
      int rows_valid = p.M - mrow0;
      rows_valid = rows_valid < 0 ? 0 : (rows_valid > 32 ? 32 : rows_valid);
      mbar_wait(tfull_bar, (uint32_t)(local & 1));
#pragma unroll
      for (int cl = 0; cl < GF_CPW; ++cl) {
        const int c0 = col_w0 + cl * 32;
        const int nbase = n0 + c0;
        const bool valid = nbase < p.N;          // warp-uniform
        const int buf = q & 1;
        const uint32_t sbuf = wstage + (uint32_t)buf * 2048u;
        uint32_t mbits = 0xffffffffu;
        if (valid && p.has_resid) {
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
        float v[32];
        // t = acc * colscale + bias (vectors broadcast from this warp's shared-memory copy)
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const uint4 sc = lds128(wparam_u32 + (uint32_t)(cl * 32 + j) * 4u);
          const uint4 bs = lds128(wparam_u32 + 256u + (uint32_t)(cl * 32 + j) * 4u);
          v[j] = __uint_as_float(r[j]) * __uint_as_float(sc.x) + __uint_as_float(bs.x);
          v[j + 1] = __uint_as_float(r[j + 1]) * __uint_as_float(sc.y) + __uint_as_float(bs.y);
          v[j + 2] = __uint_as_float(r[j + 2]) * __uint_as_float(sc.z) + __uint_as_float(bs.z);
          v[j + 3] = __uint_as_float(r[j + 3]) * __uint_as_float(sc.w) + __uint_as_float(bs.w);
        }
        float dz[32];
        if (p.has_resid) {
          // this lane's row of the residual tile: 4 x 16 B at the 64-byte-swizzle positions (rows >= M are TMA zeros)
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
              dz[c] = ((mbits >> c) & 1u) ? lo : 0.f;
              dz[c + 1] = ((mbits >> (c + 1)) & 1u) ? hi : 0.f;
            }
          }
        }
        if (red_mode) {
          // BatchNorm-backward sums of the recomputed output: v = xhat, dz = masked gradient.  Column sums over the
          // warp's 32 rows by a transpose-reduce (after 5 exchange rounds lane l holds column l).
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] *= dz[j];
#pragma unroll
          for (int o = 16, n = 32; o >= 1; o >>= 1, n >>= 1) {
            const bool up = (lane & o) != 0;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              if (j < n / 2) {
                const float sd = up ? dz[j] : dz[j + n / 2], kd = up ? dz[j + n / 2] : dz[j];
                const float sv = up ? v[j] : v[j + n / 2], kv = up ? v[j + n / 2] : v[j];
                dz[j] = kd + __shfl_xor_sync(0xffffffffu, sd, o);
                v[j] = kv + __shfl_xor_sync(0xffffffffu, sv, o);
              }
            }
          }
          racc1[cl] += dz[0];
          racc2[cl] += v[0];
          ++q;
          continue;
        }
        if (p.has_resid) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const uint4 rs = lds128(wparam_u32 + 512u + (uint32_t)(cl * 32 + j) * 4u);
            v[j] += dz[j] * __uint_as_float(rs.x);
            v[j + 1] += dz[j + 1] * __uint_as_float(rs.y);
            v[j + 2] += dz[j + 2] * __uint_as_float(rs.z);
            v[j + 3] += dz[j + 3] * __uint_as_float(rs.w);
          }
        }
        if (p.relu) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        if (p.mask_out != nullptr && mvalid) {
          uint32_t bits = 0u;
#pragma unroll
          for (int j = 0; j < 32; ++j) bits |= (v[j] > 0.f ? 1u : 0u) << j;
          uint8_t* mo = p.mask_out + (((int64_t)m * p.ldc + nbase) >> 3);
          if ((p.ldc & 31) == 0 && nbase + 32 <= p.N) {
            *reinterpret_cast<uint32_t*>(mo) = bits;
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (nbase + 8 * j < p.N) mo[j] = (uint8_t)(bits >> (8 * j));
          }
        }
        // stage the output tile in the SAME buffer (every lane has read its residual row), TMA store, statistics
        __syncwarp();
        if (!p.has_resid && lane == 0) tma_store_wait_read1();   // without residual loads the two buffers alternate freely
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
        if (storing && lane == 0) {
          tma_store_2d(&tmapC, sbuf, nbase, mrow0);
          tma_store_commit();
        }
        if (do_stats) stats_narrow(sbuf, lane, rows_valid, cs1[cl], cs2[cl]);
        __syncwarp();
        ++q;
      }
    }
    if (do_stats && stat_n0 >= 0) flush_stats();
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
typedef CUresult (*PFN_encodeTiledGF)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiledGF gf_encode_fn() {
  static PFN_encodeTiledGF fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = (PFN_encodeTiledGF)ptr;
  }
  return fn;
}

static int gf_tmap(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                   uint32_t box_cols) {
  PFN_encodeTiledGF fn = gf_encode_fn();
  if (fn == nullptr) { set_last_error("cuTensorMapEncodeTiled entry point unavailable"); return -1; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(bf16)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, box_cols == 64u ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("gemm_fused: cuTensorMapEncodeTiled failed (%d): rows=%llu cols=%llu ld=%llu", (int)r,
                   (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld);
    return -1;
  }
  return 0;
}

// true if the rich-epilogue kernel can run this GEMM (the caller falls back to conv_igemm_kernel otherwise)
bool gemm_fused_applicable(int M, int C, int Ndim, int ldw, int ldc) {
  return M > 0 && C % 8 == 0 && Ndim > 64 && Ndim % 8 == 0 && ldc % 8 == 0 && ldc >= Ndim && ldw % 8 == 0 && ldw >= C;
}

int gemm_fused_launch(const void* src, const void* wt, void* dst, const void* resid, const void* resid_mask,
                      const float* colscale, const float* bias, const float* resid_colscale, void* mask_out,
                      float* col_sum, float* col_sqsum, int M, int C, int Ndim, int ldw, int ldc, int relu, int no_store,
                      int bwd_reduce, cudaStream_t stream) {
  const bool no_dst = no_store || bwd_reduce;
  BYOL_CHECK_ARG(src && wt && (dst || no_dst), "gemm_fused: null pointer");
  BYOL_CHECK_ARG(gemm_fused_applicable(M, C, Ndim, ldw, ldc), "gemm_fused: unsupported shape M=%d C=%d N=%d ldw=%d ldc=%d",
                 M, C, Ndim, ldw, ldc);
  BYOL_CHECK_ARG(resid_mask == nullptr || resid != nullptr, "gemm_fused: resid_mask without resid");
  BYOL_CHECK_ARG(!bwd_reduce || (resid != nullptr && col_sum != nullptr && col_sqsum != nullptr),
                 "gemm_fused: bwd_reduce needs the gradient tile (resid) and both sum buffers");
  BYOL_CHECK_ARG(!(no_store && resid != nullptr), "gemm_fused: the statistics-only pass takes no residual");
  BYOL_CHECK_ARG((col_sum == nullptr) == (col_sqsum == nullptr), "gemm_fused: col_sum and col_sqsum go together");
  GemmFusedParams p;
  memset(&p, 0, sizeof(p));
  p.resid_mask = (const uint8_t*)resid_mask;
  p.colscale = colscale;
  p.bias = bias;
  p.resid_colscale = resid_colscale;
  p.mask_out = (uint8_t*)mask_out;
  p.col_sum = col_sum;
  p.col_sqsum = col_sqsum;
  p.has_resid = resid != nullptr ? 1 : 0;
  p.relu = relu;
  p.no_store = no_store ? 1 : 0;
  p.bwd_reduce = bwd_reduce ? 1 : 0;
  p.M = M; p.N = Ndim; p.ldc = ldc;
  p.num_kb = (C + GF_BK - 1) / GF_BK;
  p.tiles_n = (Ndim + GF_BN - 1) / GF_BN;
  const int tiles_m = (M + GF_BM - 1) / GF_BM;
  const int num_tiles = tiles_m * p.tiles_n;
  CUtensorMap ta, tb, tc, tr;
  if (gf_tmap(&ta, src, (uint64_t)M, (uint64_t)C, (uint64_t)C, GF_BM, 64u) != 0) return -3;
  if (gf_tmap(&tb, wt, (uint64_t)Ndim, (uint64_t)C, (uint64_t)ldw, GF_BN, 64u) != 0) return -3;
  if (!no_dst) { if (gf_tmap(&tc, dst, (uint64_t)M, (uint64_t)Ndim, (uint64_t)ldc, 32u, 32u) != 0) return -3; }
  else tc = tb;
  if (resid != nullptr) { if (gf_tmap(&tr, resid, (uint64_t)M, (uint64_t)Ndim, (uint64_t)ldc, 32u, 32u) != 0) return -3; }
  else tr = tb;
  static bool attr_set[kMaxDevices] = {};
  const int dev_slot = device_slot();
  if (!attr_set[dev_slot]) {
    cudaError_t e = cudaFuncSetAttribute(gemm_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GF_TOTAL);
    if (e != cudaSuccess) { set_last_error("cudaFuncSetAttribute(gemm_fused) failed: %s", cudaGetErrorString(e)); return -2; }
    attr_set[dev_slot] = true;
  }
  int grid = device_sm_count();
  if (grid > num_tiles) grid = num_tiles;
  if (col_sum != nullptr) {
    p.fx = fix_scratch(stream, 2 * (int64_t)Ndim);
    if (p.fx == nullptr) return -2;
  }
  gemm_fused_kernel<<<grid, GF_THREADS, GF_TOTAL, stream>>>(ta, tb, tc, tr, p, num_tiles);
  int rc = check_launch("gemm_fused_kernel");
  if (rc != 0 || col_sum == nullptr) return rc;
  if ((rc = fix_flush(p.fx, col_sum, Ndim, stream)) != 0) return rc;
  return fix_done(stream, fix_flush(p.fx + Ndim, col_sqsum, Ndim, stream));
}

}  // namespace byol

using namespace byol;

// 1x1 / stride-1 convolution (plain GEMM: out[M, Ndim] = src[M, C] x wt[Ndim, C]^T, Ndim > 64) with a fused epilogue:
//     t   = acc * colscale[n] + bias[n]
//     out = act( t + resid_colscale[n] * (resid_mask ? resid : 0) )          -> dst (bf16), mask_out = bits (out > 0)
// no_store = 1  : nothing is written; only the column statistics (col_sum / col_sqsum of the bf16-rounded t) are
//                 produced — pass 1 of "statistics pass + recompute", which never materialises the raw conv output
// bwd_reduce = 1: nothing is written; with dz = (resid_mask ? resid : 0): col_sum += sum_m dz, col_sqsum += sum_m dz*t
//                 (t = xhat when colscale = invstd and bias = -mean*invstd): the BatchNorm-backward sums of a
//                 recomputed conv output
extern "C" int byol_conv_igemm_fused(const void* src, const void* wt, void* dst, const void* resid,
                                     const void* resid_mask, const float* colscale, const float* bias,
                                     const float* resid_colscale, void* mask_out, float* col_sum, float* col_sqsum,
                                     int M, int C, int Ndim, int ldw, int ldc, int relu, int no_store, int bwd_reduce,
                                     cudaStream_t stream) {
  return gemm_fused_launch(src, wt, dst, resid, resid_mask, colscale, bias, resid_colscale, mask_out, col_sum,
                           col_sqsum, M, C, Ndim, ldw, ldc, relu, no_store, bwd_reduce, stream);
}
