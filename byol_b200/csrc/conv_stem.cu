// byol_b200 — the ResNet stem: 7x7 / stride 2 / pad 3 convolution over <= 4-channel images (fprop + wgrad).
//
// The implicit-GEMM kernel re-gathers every input pixel ~12 times from L2 for this layer (7 kernel rows x ~1.75
// overlapping windows), which made the stem L2-bound at ~100 TFLOP/s.  Here the input is stored once as
// NHWC4 bf16 with the zero padding baked in ([N][H+6][264][4], 8 bytes per pixel).  Because the stride is 2 and a
// pixel is 8 bytes, the window of output pixel m along an input row starts 16 bytes after the window of pixel
// m - 1 — exactly the row pitch of a no-swizzle core matrix.  So with LBO = 16 and SBO = 128 the wgmma shared-memory
// matrix descriptor ALONE forms the im2col rows (rows and K chunks overlap in smem): an input row is bulk-copied
// into smem once and then read by the tensor core for all 128 output pixels x 8 window taps, and a row pair is
// loaded once per CTA for the 3-4 output rows that use it.  Per output row and warpgroup: 7 kernel rows x 2 MMAs
// (M = 64 pixels, N = 64 channels, K = 16 = 4 pixels x 4 ch).
//
//   warps 0-7  : epilogue (smem accumulator tile -> regs -> bf16 -> swizzled staging -> TMA store, fused BatchNorm
//                statistics)
//   warps 8-15 : two MMA warpgroups (output pixels 0-63 / 64-127 of the row)
//   warp 16    : producer (1-D bulk copies of input row pairs into an 8-slot ring; weights once)
// Replaces the cuDNN stem convolution reached from /root/reference/main.py:237 (torchvision resnet conv1) and its
// weight gradient under main.py:617.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace byol {

static constexpr int ST_WP = 264;                    // padded pixels per input row: 2*127 + 7 < 264
static constexpr int ST_ROW_BYTES = ST_WP * 8;       // 2112
static constexpr int ST_PAIR_BYTES = 2 * ST_ROW_BYTES;
static constexpr int ST_NP = 8;                      // row-pair ring slots
static constexpr int ST_W_BYTES = 7 * 4 * 64 * 16;   // [kh][k-chunk][cout][8] bf16 = 28672
static constexpr int ST_W_OFF = 0;
static constexpr int ST_RING_OFF = ST_W_BYTES;
static constexpr int ST_STAGE_OFF = ((ST_RING_OFF + ST_NP * ST_PAIR_BYTES + 1023) / 1024) * 1024;
static constexpr int ST_ACC_LD = acc_ld(64);
static constexpr int ST_ACC_OFF = ST_STAGE_OFF + 8 * 2 * 2048;    // [128][ST_ACC_LD] fp32 accumulator tile
static constexpr int ST_BAR_OFF = ST_ACC_OFF + 128 * ST_ACC_LD * 4;
static constexpr int ST_NEEDED = ST_BAR_OFF + 256;
static constexpr int ST_TOTAL = ST_NEEDED + 768;
static constexpr int ST_THREADS = 17 * 32;
static_assert(ST_TOTAL <= 232448, "one CTA per SM");

struct StemParams {
  const bf16* xs;   // [N][H+6][264][4]
  const bf16* w;    // [7][4][64][8]
  float* col_sum;   // optional [64]
  float* col_sqsum;
  Fix128* fx;    // with col_sum: [2][64] fixed-point accumulators (fix_scratch)
  int N, Ho, Wo;
  int pairs_per_img;   // (H + 6) / 2
  int num_tiles;       // N * Ho (one tile = one output row, Wo <= 128 pixels)
};

__global__ void __launch_bounds__(ST_THREADS, 1)
stem_fprop_kernel(const __grid_constant__ CUtensorMap tmapY, const StemParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  if (smem + ST_NEEDED > smem_raw + ST_TOTAL) __trap();
  uint8_t* sW = smem + ST_W_OFF;
  uint8_t* ring = smem + ST_RING_OFF;
  uint8_t* stage_out = smem + ST_STAGE_OFF;
  uint64_t* wfull = (uint64_t*)(smem + ST_BAR_OFF);
  uint64_t* full_bar = wfull + 1;
  uint64_t* empty_bar = full_bar + ST_NP;
  uint64_t* tfull_bar = empty_bar + ST_NP;   // accumulator tile ready for the epilogue
  uint64_t* tempty_bar = tfull_bar + 1;      // accumulator tile drained
  float* accbuf = reinterpret_cast<float*>(smem + ST_ACC_OFF);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // contiguous tile range per CTA: consecutive output rows share 5 of their 7 input rows
  const int t_begin = (int)((int64_t)blockIdx.x * p.num_tiles / gridDim.x);
  const int t_end = (int)((int64_t)(blockIdx.x + 1) * p.num_tiles / gridDim.x);

  if (warp == 16 && lane == 0) {
    mbar_init(wfull, 1u);
    for (int s = 0; s < ST_NP; ++s) { mbar_init(&full_bar[s], 1u); mbar_init(&empty_bar[s], 2u); }
    mbar_init(tfull_bar, 256u);
    mbar_init(tempty_bar, 8u);
    fence_mbar_init();
    tma_prefetch_desc(&tmapY);
  }
  __syncthreads();

  if (warp < 8) {
    // ======================= epilogue =====================================================
    const int quarter = warp & 3;          // tile rows (output pixels) 32*quarter ..
    const int c0 = (warp >> 2) * 32;       // output channels c0 .. c0+31
    const bool do_stats = p.col_sum != nullptr;
    const uint32_t stage_base0 = smem_u32(stage_out + warp * 4096);
    int rows_valid = p.Wo - quarter * 32;
    rows_valid = rows_valid < 0 ? 0 : (rows_valid > 32 ? 32 : rows_valid);
    uint64_t cs1 = 0ull, cs2 = 0ull;
    int sbuf = 0, local = 0;
    for (int t = t_begin; t < t_end; ++t, ++local) {
      mbar_wait(tfull_bar, (uint32_t)(local & 1));
      uint32_t r[32];
      acc_load_row32(accbuf + (quarter * 32 + lane) * ST_ACC_LD + c0, r);
      __syncwarp();
      if (lane == 0) mbar_arrive(tempty_bar);
      if (rows_valid == 0) continue;   // warp-uniform
      if (lane >= rows_valid) {
        // pixels beyond Wo see windows over the right padding: non-zero garbage that must not reach the statistics
#pragma unroll
        for (int j = 0; j < 32; ++j) r[j] = 0u;
      }
      const uint32_t stage_base = stage_base0 + (uint32_t)sbuf * 2048u;
      if (lane == 0) tma_store_wait_read1();
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 q;
        q.x = pack_bf16x2(__uint_as_float(r[8 * j + 0]), __uint_as_float(r[8 * j + 1]));
        q.y = pack_bf16x2(__uint_as_float(r[8 * j + 2]), __uint_as_float(r[8 * j + 3]));
        q.z = pack_bf16x2(__uint_as_float(r[8 * j + 4]), __uint_as_float(r[8 * j + 5]));
        q.w = pack_bf16x2(__uint_as_float(r[8 * j + 6]), __uint_as_float(r[8 * j + 7]));
        const uint32_t off = (uint32_t)lane * 64u + (uint32_t)((j ^ ((lane >> 1) & 3)) << 4);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(stage_base + off), "r"(q.x), "r"(q.y), "r"(q.z),
                     "r"(q.w)
                     : "memory");
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        tma_store_3d(&tmapY, stage_base, c0, quarter * 32, t);   // pixels >= Wo are clipped by TMA
        tma_store_commit();
      }
      if (do_stats) stats_narrow(stage_base, lane, rows_valid, cs1, cs2);
      sbuf ^= 1;
    }
    if (do_stats) {
      float2 a = f2_unpack(cs1), b = f2_unpack(cs2);
      a.x += __shfl_xor_sync(0xffffffffu, a.x, 16);
      a.y += __shfl_xor_sync(0xffffffffu, a.y, 16);
      b.x += __shfl_xor_sync(0xffffffffu, b.x, 16);
      b.y += __shfl_xor_sync(0xffffffffu, b.y, 16);
      if (lane < 16) {
        const int col = c0 + 2 * lane;
        fix_add(p.fx + col, a.x);
        fix_add(p.fx + col + 1, a.y);
        fix_add(p.fx + 64 + col, b.x);
        fix_add(p.fx + 64 + col + 1, b.y);
      }
    }
    if (lane == 0) tma_store_wait_all();
  } else if (warp < 16) {
    // ======================= MMA warpgroups ===============================================
    // warpgroup wg: output pixels 64*wg .. +63 of the row = A rows 64 * 16 B further into the row pair
    const int wg = (warp - 8) >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    mbar_wait(wfull, 0u);
    const uint32_t w_addr = smem_u32(sW);
    const uint32_t ring_addr = smem_u32(ring);
    // B: [k-chunk][cout][8]: chunk step 1024, 8-row group step 128; kh block 4096 B, K step (2 chunks) 2048 B
    const uint64_t bdesc0 = make_smem_desc_none(w_addr, 1024u, 128u);
    float d[32];
    int qb = 0, qn = 0, local = 0;
    for (int t = t_begin; t < t_end; ++t, ++local) {
      const int oh = t % p.Ho;
      const bool first = (t == t_begin) || (oh == 0);
      if (first) {
        qb = qn;
        qn += 4;
        for (int j = 0; j < 4; ++j) mbar_wait(&full_bar[(qb + j) % ST_NP], (uint32_t)(((qb + j) / ST_NP) & 1));
      } else {
        qb += 1;
        qn += 1;
        mbar_wait(&full_bar[(qb + 3) % ST_NP], (uint32_t)(((qb + 3) / ST_NP) & 1));
      }
      wg_fence();
#pragma unroll
      for (int kp = 0; kp < 4; ++kp) {   // row pair kp holds kernel rows 2*kp and 2*kp + 1
        // A: row m = output pixel m, 16-byte chunk c = input pixels 2m + 4s + 2c, +1 -> LBO 16, SBO 128 (overlapping)
        const uint64_t adesc0 = make_smem_desc_none(
            ring_addr + (uint32_t)(((qb + kp) % ST_NP) * ST_PAIR_BYTES) + (uint32_t)wg * 1024u, 16u, 128u);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int kh = 2 * kp + r;
          if (kh < 7) {
#pragma unroll
            for (int s = 0; s < 2; ++s)
              wgmma_bf16<64, 0, 0>(d, adesc0 + (uint64_t)((r * ST_ROW_BYTES + 32 * s) >> 4),
                                   bdesc0 + (uint64_t)((kh * 4096 + s * 2048) >> 4), (uint32_t)((kh | s) != 0));
          }
        }
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(d);
      const bool last = (t + 1 == t_end) || ((t + 1) % p.Ho == 0);
      if (leader) {
        if (last) {
          for (int j = 0; j < 4; ++j) mbar_arrive(&empty_bar[(qb + j) % ST_NP]);
        } else {
          mbar_arrive(&empty_bar[qb % ST_NP]);
        }
      }
      mbar_wait(tempty_bar, (uint32_t)((local & 1) ^ 1));
      acc_store_smem<64>(accbuf, ST_ACC_LD, wg * 64, 0, d);
      mbar_arrive(tfull_bar);
    }
  } else {
    // ======================= producer =====================================================
    if (lane == 0) {
      mbar_arrive_expect_tx(wfull, (uint32_t)ST_W_BYTES);
      bulk_load_1d(smem_u32(sW), p.w, (uint32_t)ST_W_BYTES, wfull);
      int q = 0;
      for (int t = t_begin; t < t_end; ++t) {
        const int n = t / p.Ho, oh = t % p.Ho;
        const bool first = (t == t_begin) || (oh == 0);
        const int p0 = first ? oh : oh + 3;
        const int cnt = first ? 4 : 1;
        for (int j = 0; j < cnt; ++j, ++q) {
          const int slot = q % ST_NP;
          mbar_wait(&empty_bar[slot], (uint32_t)(((q / ST_NP) & 1) ^ 1));
          mbar_arrive_expect_tx(&full_bar[slot], (uint32_t)ST_PAIR_BYTES);
          const bf16* src = p.xs + ((int64_t)n * p.pairs_per_img + p0 + j) * (ST_PAIR_BYTES / 2);
          bulk_load_1d(smem_u32(ring + slot * ST_PAIR_BYTES), src, (uint32_t)ST_PAIR_BYTES, &full_bar[slot]);
        }
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// Stem weight gradient: dW[co][c][kh][kw] += sum over pixels dY[n, oh, ow, co] * x[n, 2oh + kh - 3, 2ow + kw - 3, c].
// One work unit = one padded input row v of one image.  Row v meets the output rows oh = (v >> 1) - j with kernel row
// kh = (v & 1) + 2j (j = 0..3), so per unit two M = 128 MMA chains run over K = the pixels of the row:
//   A (M-major, 128-byte swizzle) = two ADJACENT dY row tiles [128 px][64 co] (LBO = tile size): rows (a-1, a) and
//     (a-3, a-2) with a = v >> 1; rows outside the image are TMA out-of-bounds zero tiles
//   B (N-major, no swizzle)       = the input row itself: N = 8 window pixels x 4 channels, pixel k's window starts
//     16 bytes after pixel k-1's (overlapping no-swizzle core matrices, as in the forward kernel)
//   D = four accumulators [128 = 2 kh x 64 co][32 = (kw, c)] (row parity x chain), kept in registers for the CTA's
//     whole contiguous range of units and added to the fp32 gradient with atomics at the end.
// The dY ring has 11 slots + a mirror of slot 0 behind slot 10, so that "row oh-1, row oh" are always adjacent in smem.
//   warps 0-7: two MMA warpgroups (warpgroup wg owns rows 64*wg .. +63 = the dY row tile wg of each pair), warp 8:
//   producer.
// ---------------------------------------------------------------------------------------------
static constexpr int SW_NS = 11;   // 4 rows in use + 7 rows of prefetch (dY streams from HBM: the ring depth hides its latency)
static constexpr int SW_TILE = 128 * 128;
static constexpr int SW_NX = 12;
static constexpr int SW_X_OFF = (SW_NS + 1) * SW_TILE;
static constexpr int SW_BAR_OFF = SW_X_OFF + SW_NX * ST_ROW_BYTES;
static constexpr int SW_NEEDED = SW_BAR_OFF + 256;
static constexpr int SW_TOTAL = SW_NEEDED + 1024;
static_assert(SW_BAR_OFF % 8 == 0 && SW_TOTAL <= 232448 - 1024, "stem wgrad smem");

struct StemWgradParams {
  const bf16* xs;   // [N][Hp][264][4]
  float* dw;        // [64][Cin][7][7] fp32, accumulated
  Fix128* fx;    // fixed-point accumulators over the whole dw (fix_scratch)
  int N, Ho, Wo, Hp, Cin;
  int num_units;    // N * Hp
  int ksteps;       // ceil(Wo / 16)
  uint32_t b_lbo, b_sbo;
};

__device__ __forceinline__ void tma_load_4d_stem(uint32_t dst_smem, const CUtensorMap* tmap, uint64_t* bar, int c0,
                                                 int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst_smem), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

static constexpr int SW_THREADS = 9 * 32;

__global__ void __launch_bounds__(SW_THREADS, 1)
stem_wgrad_kernel(const __grid_constant__ CUtensorMap tmapDY, const StemWgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  if (smem + SW_NEEDED > smem_raw + SW_TOTAL) __trap();
  uint8_t* sDY = smem;
  uint8_t* sX = smem + SW_X_OFF;
  uint64_t* dfull = (uint64_t*)(smem + SW_BAR_OFF);
  uint64_t* dempty = dfull + SW_NS;
  uint64_t* xfull = dempty + SW_NS;
  uint64_t* xempty = xfull + SW_NX;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int u_begin = (int)((int64_t)blockIdx.x * p.num_units / gridDim.x);
  const int u_end = (int)((int64_t)(blockIdx.x + 1) * p.num_units / gridDim.x);

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < SW_NS; ++s) { mbar_init(&dfull[s], 1u); mbar_init(&dempty[s], 2u); }   // 2 = both warpgroups
    for (int s = 0; s < SW_NX; ++s) { mbar_init(&xfull[s], 1u); mbar_init(&xempty[s], 2u); }
    fence_mbar_init();
    tma_prefetch_desc(&tmapDY);
  }
  __syncthreads();

  if (warp == 8) {
    // ======================= producer =====================================================
    if (lane == 0) {
      int q = 0, xq = 0;
      for (int u = u_begin; u < u_end; ++u) {
        const int n = u / p.Hp, v = u % p.Hp, a = v >> 1;
        const bool first = (u == u_begin) || (v == 0);
        const int r0 = first ? a - 3 : a;
        const int cnt = first ? 4 : ((v & 1) ? 0 : 1);
        for (int j = 0; j < cnt; ++j, ++q) {
          const int slot = q % SW_NS;
          mbar_wait(&dempty[slot], (uint32_t)(((q / SW_NS) & 1) ^ 1));
          mbar_arrive_expect_tx(&dfull[slot], (uint32_t)(slot == 0 ? 2 * SW_TILE : SW_TILE));
          tma_load_4d_stem(smem_u32(sDY + slot * SW_TILE), &tmapDY, &dfull[slot], 0, 0, r0 + j, n);
          if (slot == 0) tma_load_4d_stem(smem_u32(sDY + SW_NS * SW_TILE), &tmapDY, &dfull[slot], 0, 0, r0 + j, n);
        }
        const int xs = xq % SW_NX;
        mbar_wait(&xempty[xs], (uint32_t)(((xq / SW_NX) & 1) ^ 1));
        mbar_arrive_expect_tx(&xfull[xs], (uint32_t)ST_ROW_BYTES);
        bulk_load_1d(smem_u32(sX + xs * ST_ROW_BYTES), p.xs + (int64_t)u * (ST_ROW_BYTES / 2), (uint32_t)ST_ROW_BYTES,
                     &xfull[xs]);
        ++xq;
      }
    }
    __syncwarp();
  } else {
    // ======================= MMA warpgroups ===============================================
    const int wg = warp >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    const uint32_t dy_addr = smem_u32(sDY), x_addr = smem_u32(sX);
    float d[4][16];   // [par * 2 + chain]
    int qb = 0, qn = 0, xq = 0;
    uint32_t used = 0;
    for (int u = u_begin; u < u_end; ++u, ++xq) {
      const int v = u % p.Hp;
      const bool first = (u == u_begin) || (v == 0);
      if (first) {
        qb = qn;
        qn += 4;
        for (int j = 0; j < 4; ++j) mbar_wait(&dfull[(qb + j) % SW_NS], (uint32_t)(((qb + j) / SW_NS) & 1));
      } else if ((v & 1) == 0) {
        qb += 1;
        qn += 1;
        mbar_wait(&dfull[(qb + 3) % SW_NS], (uint32_t)(((qb + 3) / SW_NS) & 1));
      }
      const int xs = xq % SW_NX;
      mbar_wait(&xfull[xs], (uint32_t)((xq / SW_NX) & 1));
      // chain 0: dY rows (a-1, a) <-> kh = (par+2, par); chain 1: rows (a-3, a-2) <-> kh = (par+6, par+4)
      const int par = v & 1;
      const uint64_t bdesc = make_smem_desc_none(x_addr + (uint32_t)(xs * ST_ROW_BYTES), p.b_lbo, p.b_sbo);
      const uint32_t acc0 = (used >> par) & 1u;
      wg_fence();
#pragma unroll
      for (int chain = 0; chain < 2; ++chain) {
        const uint32_t tile0 = dy_addr + (uint32_t)(((qb + (chain == 0 ? 2 : 0)) % SW_NS) * SW_TILE);
        const uint64_t adesc = make_smem_desc_sw128(tile0 + (uint32_t)wg * SW_TILE, (uint32_t)SW_TILE, 1024u);
        // K step = 16 pixels: +2048 B in the dY tile, +256 B in the input row
        if (par == 0) {
          for (int ks = 0; ks < p.ksteps; ++ks)
            wgmma_bf16<32, 1, 1>(d[chain], adesc + (uint64_t)(128 * ks), bdesc + (uint64_t)(16 * ks), ks == 0 ? acc0 : 1u);
        } else {
          for (int ks = 0; ks < p.ksteps; ++ks)
            wgmma_bf16<32, 1, 1>(d[2 + chain], adesc + (uint64_t)(128 * ks), bdesc + (uint64_t)(16 * ks),
                                 ks == 0 ? acc0 : 1u);
        }
      }
      wg_commit();
      wg_wait<0>();
#pragma unroll
      for (int a = 0; a < 4; ++a) wg_fence_acc(d[a]);
      used |= 1u << par;
      if (leader) {
        mbar_arrive(&xempty[xs]);
        const bool last = (u + 1 == u_end) || (v == p.Hp - 1);
        if (last) {
          for (int j = 0; j < 4; ++j) mbar_arrive(&dempty[(qb + j) % SW_NS]);
        } else if (v & 1) {
          mbar_arrive(&dempty[qb % SW_NS]);
        }
      }
    }
    // ======================= epilogue (once): registers -> fp32 gradient ===================
    if (u_end > u_begin) {
      const int t = threadIdx.x & 127;
      const int co = (t >> 5) * 16 + ((t & 31) >> 2);   // + 8 for the second row of a fragment pair
      const bool both = (u_end - u_begin) >= 2;
      const int only_par = (u_begin % p.Hp) & 1;
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int par = a >> 1, chain = a & 1;
        if (!both && par != only_par) continue;   // this row parity never ran: the accumulator is uninitialised
        const int kh = par + (chain == 0 ? (wg == 0 ? 2 : 0) : (wg == 0 ? 6 : 4));
        if (kh > 6) continue;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int col = 8 * (i >> 2) + 2 * (t & 3) + (i & 1);
          const int row = co + ((i & 2) ? 8 : 0);
          const int kw = col >> 2, c = col & 3;
          if (kw < 7 && c < p.Cin) fix_add(p.fx + ((row * p.Cin + c) * 7 + kh) * 7 + kw, d[a][i]);
        }
      }
    }
  }
}

// fp32 NCHW image -> bf16 [N][H+6][264][4] with the conv padding (3 pixels / rows of zeros) and channel 3 = 0
__global__ void nchw_to_stem4_kernel(const float* __restrict__ x, bf16* __restrict__ y, int N, int Cin, int H, int W) {
  const int Hp = H + 6;
  const int64_t total = (int64_t)N * Hp * ST_WP;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int u = (int)(i % ST_WP);
    const int64_t t = i / ST_WP;
    const int v = (int)(t % Hp);
    const int n = (int)(t / Hp);
    const int ih = v - 3, iw = u - 3;
    float f[4] = {0.f, 0.f, 0.f, 0.f};
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < Cin) f[c] = __ldg(x + (((int64_t)n * Cin + c) * H + ih) * W + iw);
    }
    uint2 q;
    q.x = pack_bf16x2(f[0], f[1]);
    q.y = pack_bf16x2(f[2], f[3]);
    reinterpret_cast<uint2*>(y)[i] = q;
  }
}

// fp32 [64][Cin][7][7] -> bf16 [kh 7][k-chunk 4][cout 64][8]: element e of chunk kc = (kw = 2*kc + (e >> 2), c = e & 3)
__global__ void prep_weight_stem4_kernel(const float* __restrict__ w, bf16* __restrict__ ws, int Cin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 7 * 4 * 64 * 8) return;
  const int e = i & 7, n = (i >> 3) & 63, kc = (i >> 9) & 3, kh = i >> 11;
  const int kw = 2 * kc + (e >> 2), c = e & 3;
  float v = 0.f;
  if (c < Cin && kw < 7) v = w[((n * Cin + c) * 7 + kh) * 7 + kw];
  ws[i] = __float2bfloat16_rn(v);
}

}  // namespace byol

using namespace byol;

typedef CUresult (*PFN_encodeTiledStem)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiledStem stem_encode_fn() {
  static PFN_encodeTiledStem fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = (PFN_encodeTiledStem)ptr;
  }
  return fn;
}

static int stem_sm_count() { return device_sm_count(); }

// 1 if the stem kernels handle this geometry (otherwise use byol_conv_igemm / byol_conv_wgrad with the NHWC8 input)
extern "C" int byol_stem4_supported(int Cin, int Cout, int H, int W, int k, int stride, int pad) {
  return (Cin >= 1 && Cin <= 4 && Cout == 64 && k == 7 && stride == 2 && pad == 3 && H >= 2 && H % 2 == 0 &&
          W >= 2 && W % 2 == 0 && W <= 256) ? 1 : 0;
}

// padded pixels per row of the NHWC4 image tensor: its shape is [N][H + 6][byol_stem4_row_pixels()][4]
extern "C" int byol_stem4_row_pixels(void) { return ST_WP; }

extern "C" int byol_nchw_to_stem4(const float* x, void* xs, int N, int Cin, int H, int W, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && xs && N > 0 && byol_stem4_supported(Cin, 64, H, W, 7, 2, 3), "byol_nchw_to_stem4: bad args");
  const int64_t total = (int64_t)N * (H + 6) * ST_WP;
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  nchw_to_stem4_kernel<<<(int)blocks, 256, 0, stream>>>(x, (bf16*)xs, N, Cin, H, W);
  return check_launch("nchw_to_stem4_kernel");
}

extern "C" int byol_prep_weight_stem4(const float* w, void* ws, int Cin, cudaStream_t stream) {
  BYOL_CHECK_ARG(w && ws && Cin >= 1 && Cin <= 4, "byol_prep_weight_stem4: bad args");
  prep_weight_stem4_kernel<<<(7 * 4 * 64 * 8 + 255) / 256, 256, 0, stream>>>(w, (bf16*)ws, Cin);
  return check_launch("prep_weight_stem4_kernel");
}

// y[N, H/2, W/2, 64] (bf16) = conv7x7/s2/p3(xs, ws); optional fused per-channel sum / sum of squares of y
extern "C" int byol_stem_conv_fprop(const void* xs, const void* ws, void* y, float* col_sum, float* col_sqsum, int N,
                                    int H, int W, cudaStream_t stream) {
  BYOL_CHECK_ARG(xs && ws && y && N > 0 && byol_stem4_supported(3, 64, H, W, 7, 2, 3), "byol_stem_conv_fprop: bad args");
  BYOL_CHECK_ARG((col_sum == nullptr) == (col_sqsum == nullptr), "byol_stem_conv_fprop: need both statistics or none");
  const int Ho = H / 2, Wo = W / 2;
  BYOL_CHECK_ARG((int64_t)N * Ho < (1ll << 31), "byol_stem_conv_fprop: too many rows");
  StemParams p;
  memset(&p, 0, sizeof(p));
  p.xs = (const bf16*)xs;
  p.w = (const bf16*)ws;
  p.col_sum = col_sum;
  p.col_sqsum = col_sqsum;
  p.N = N; p.Ho = Ho; p.Wo = Wo;
  p.pairs_per_img = (H + 6) / 2;
  p.num_tiles = N * Ho;
  PFN_encodeTiledStem fn = stem_encode_fn();
  if (fn == nullptr) { set_last_error("byol_stem_conv_fprop: cuTensorMapEncodeTiled unavailable"); return -3; }
  CUtensorMap tmY;
  cuuint64_t dims[3] = {64, (cuuint64_t)Wo, (cuuint64_t)N * Ho};
  cuuint64_t strides[2] = {128, (cuuint64_t)Wo * 128};
  cuuint32_t box[3] = {32, 32, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(&tmY, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, y, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("byol_stem_conv_fprop: tensor map encode failed (%d)", (int)r); return -3; }
  static bool attr_set[kMaxDevices] = {};
  const int dev_slot = device_slot();
  if (!attr_set[dev_slot]) {
    cudaError_t e = cudaFuncSetAttribute(stem_fprop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ST_TOTAL);
    if (e != cudaSuccess) { set_last_error("cudaFuncSetAttribute(stem_fprop) failed: %s", cudaGetErrorString(e)); return -2; }
    attr_set[dev_slot] = true;
  }
  int grid = stem_sm_count();
  if (grid > p.num_tiles) grid = p.num_tiles;
  if (col_sum != nullptr) {
    p.fx = fix_scratch(stream, 128);
    if (p.fx == nullptr) return -2;
  }
  stem_fprop_kernel<<<grid, ST_THREADS, ST_TOTAL, stream>>>(tmY, p);
  int rc = check_launch("stem_fprop_kernel");
  if (rc != 0 || col_sum == nullptr) return rc;
  if ((rc = fix_flush(p.fx, col_sum, 64, stream)) != 0) return rc;
  return fix_done(stream, fix_flush(p.fx + 64, col_sqsum, 64, stream));
}

// dw[64][Cin][7][7] (fp32) += dY^T * im2col(xs); dy: [N, H/2, W/2, 64] bf16
extern "C" int byol_stem_conv_wgrad(const void* xs, const void* dy, float* dw, int N, int Cin, int H, int W,
                                    cudaStream_t stream) {
  BYOL_CHECK_ARG(xs && dy && dw && N > 0 && byol_stem4_supported(Cin, 64, H, W, 7, 2, 3), "byol_stem_conv_wgrad: bad args");
  const int Ho = H / 2, Wo = W / 2, Hp = H + 6;
  BYOL_CHECK_ARG((int64_t)N * Hp < (1ll << 31), "byol_stem_conv_wgrad: too many rows");
  StemWgradParams p;
  memset(&p, 0, sizeof(p));
  p.xs = (const bf16*)xs;
  p.dw = dw;
  p.N = N; p.Ho = Ho; p.Wo = Wo; p.Hp = Hp; p.Cin = Cin;
  p.num_units = N * Hp;
  p.ksteps = (Wo + 15) / 16;
  // no-swizzle MN-major B: LBO = step between 8-pixel (K) groups, SBO = step between 16-byte N chunks
  // (for no-swizzle MN-major operands the roles are swapped w.r.t. K-major)
  p.b_lbo = 128u;
  p.b_sbo = 16u;
  PFN_encodeTiledStem fn = stem_encode_fn();
  if (fn == nullptr) { set_last_error("byol_stem_conv_wgrad: cuTensorMapEncodeTiled unavailable"); return -3; }
  CUtensorMap tmDY;
  cuuint64_t dims[4] = {64, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)N};
  cuuint64_t strides[3] = {128, (cuuint64_t)Wo * 128, (cuuint64_t)Ho * Wo * 128};
  cuuint32_t box[4] = {64, 128, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(&tmDY, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(dy), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("byol_stem_conv_wgrad: tensor map encode failed (%d)", (int)r); return -3; }
  static bool attr_set[kMaxDevices] = {};
  const int dev_slot = device_slot();
  if (!attr_set[dev_slot]) {
    cudaError_t e = cudaFuncSetAttribute(stem_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SW_TOTAL);
    if (e != cudaSuccess) { set_last_error("cudaFuncSetAttribute(stem_wgrad) failed: %s", cudaGetErrorString(e)); return -2; }
    attr_set[dev_slot] = true;
  }
  int grid = stem_sm_count();
  if (grid > p.num_units) grid = p.num_units;
  const int64_t ndw = (int64_t)64 * Cin * 49;
  p.fx = fix_scratch(stream, ndw);
  if (p.fx == nullptr) return -2;
  stem_wgrad_kernel<<<grid, SW_THREADS, SW_TOTAL, stream>>>(tmDY, p);
  const int rc = check_launch("stem_wgrad_kernel");
  return fix_done(stream, rc != 0 ? rc : fix_flush(p.fx, dw, ndw, stream));
}
