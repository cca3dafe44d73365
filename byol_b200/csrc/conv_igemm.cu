// byol_b200 — implicit-GEMM convolution / linear layers on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces the cuDNN conv fwd/dgrad/wgrad and cuBLAS Linear calls reached from the reference at
// /root/reference/main.py:229-240 (BYOL.prediction: base_network -> head -> predictor).
//
// Data layout: activations NHWC bf16 (channels padded to a multiple of 8), weights bf16
// [Cout][KH*KW*Cin] K-major (prepared from the fp32 master by byol_prep_weight).
//
//   out[m, n] = sum_{tap, c} src[pix(m, tap), c] * Wt[n, tap*C + c]          (fprop and dgrad)
//   dW[n, tap, c] += sum_m dY[m, n] * src[pix(m, tap), c]                     (wgrad)
//
// One CTA computes a 128 x BN tile.  smem operand tiles use the 128-byte swizzle; two MMA warpgroups (wgmma) own
// 64 tile rows each and keep their accumulators in registers; a finished tile is handed to the epilogue warps
// (one tile row per lane) through an fp32 tile in shared memory, or, when the epilogue only stores bf16 values and
// their statistics, as bf16 store blocks (SmemLayout, H16).
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace byol {

static constexpr int BM = 128;           // output rows (pixels) per CTA
static constexpr int BK = 64;            // bf16 elements per k-block (= one 128-byte swizzle row)
static constexpr int A_STAGE_BYTES = BM * 128;
static constexpr int GATHER_LAG = 2;     // cp.async groups in flight per producer thread

struct ConvGemmParams {
  const bf16* src;     // gathered operand, NHWC [Nimg, Hs, Ws, C]
  void* dst;           // output [M, ldc] row-major (bf16 or fp32)
  const bf16* resid;   // optional, [M, ldc] bf16, added in the epilogue
  const uint8_t* resid_mask;   // optional ReLU mask bits over the same [M, ldc] index space: add resid only where set
  int resid_up;                // 1: resid is [Nimg, Ho/2, Wo/2, ldc] and belongs to the even (h, w) pixels only
  const float* resid_f32;      // optional fp32 residual over the same index space (fp32 outputs only)
  const float* bias;   // optional, [Ndim]
  float* col_sum;      // optional, [Ndim] fp32: += sum over rows of the stored value
  float* col_sqsum;    // optional, [Ndim] fp32: += sum over rows of value^2
  Fix128* fx;       // with col_sum: [2][Ndim] fixed-point accumulators of both sums (fix_scratch)
  int Nimg, Hs, Ws, C;
  int Ho, Wo;
  int KH, KW;
  int mul, base, dk, div;  // src coord = o*mul + base + k*dk ; valid iff >=0, %div==0, /div < Hs|Ws
  int M, Ndim, Kg;
  int ldc;
  int num_kb;
  int tiles_n;
  int out_fp32;
  int relu;
  int small_src;   // 1: the gathered tensor has < 2^31 elements (32-bit element offsets are safe)
  int local_stats; // H16 with statistics: the CTA sums its fixed-point words in shared memory (SmemLayout)
  // stride-2 dgrad by output parity ("parity mode"): the M dimension enumerates the pixels of dX class by class
  // (class = (ih & 1, iw & 1)); a tile belongs to ONE class, for which only the taps with the parity of
  // (coordinate + pad) contribute, so every role skips the other taps entirely.
  int fold;        // 1: stem layout: C == 8, one k-block per kh, K column = kw*8 + c (kw padded to 8)
  int parity;      // 1: enabled
  int Hh, Wh;      // dX spatial size / 2
  int Mc;          // pixels per class = Nimg*Hh*Wh (a multiple of BM)
  int ncls;        // number of classes with at least one tap
  int cls_list[4]; // their ids (ph*2 + pw)
};

// per-tile geometry shared by all warp roles
struct TileInfo {
  int m0, n0, nkb;
  int cls_idx, ph, pw, kh0, kw0, nkw;   // parity mode only
};

// GROUPED (grouped 3x3 convolutions with Cin == Cout == C and C / groups dividing 64): the weight of a 64-column
// output tile [n0, n0 + 64) is block-diagonal and needs only the input channels [n0, n0 + 64), so a tile's K loop is
// one 64-channel k-block per tap, starting at channel n0.  The weight layout is [C][taps * 64], column
// tap * 64 + (c - n0) (byol_prep_weights_grouped); BN is 64.
template <bool GROUPED = false>
__device__ __forceinline__ TileInfo tile_info(const ConvGemmParams& p, int tile, int BN_) {
  TileInfo t;
  t.m0 = (tile / p.tiles_n) * BM;
  t.n0 = (tile % p.tiles_n) * BN_;
  t.nkb = p.num_kb;
  t.cls_idx = 0; t.ph = 0; t.pw = 0; t.kh0 = 0; t.kw0 = 0; t.nkw = p.KW;
  if (p.parity) {
    t.cls_idx = t.m0 / p.Mc;
    const int cls = p.cls_list[t.cls_idx];
    t.ph = cls >> 1;
    t.pw = cls & 1;
    t.kh0 = (t.ph + p.base) & 1;            // p.base == pad in dgrad mode
    t.kw0 = (t.pw + p.base) & 1;
    const int nkh = (p.KH - t.kh0 + 1) >> 1;
    t.nkw = (p.KW - t.kw0 + 1) >> 1;
    t.nkb = nkh * t.nkw * (GROUPED ? 1 : p.C / BK);
  }
  return t;
}

// Epilogue geometry.  The TMA-operand variant (plain GEMM: 1x1 / stride 1 convolutions and the MLP layers) has no
// gather warps and is bound by its epilogue (few k-blocks per tile, outputs up to 4x the inputs), so it runs EIGHT
// epilogue warps: warps w and w + 4 share the row quarter w & 3 of the tile and split its columns.
// Output staging: [32 rows][32 cols] chunks with the 64-byte swizzle, NBUF staging buffers per warp.  (A variant with
// 128-byte staging rows and a 2-stage operand ring was measured slower for every K >= 128 and removed.)
// H16 (bf16 hand-off): when the epilogue only stores the bf16 value and sums its statistics (no bias, residual, ReLU
// or fp32 output), the MMA warpgroups round the accumulators to bf16 themselves and write them straight into the
// staging blocks, and the epilogue warps only issue the TMA stores and read the statistics.  Two such tiles
// ([quarter][chunk] blocks, 32 KB at BN = 128) replace the fp32 tile and the per-warp staging, so the MMA warpgroups
// can hand off tile i+1 while tile i is being stored.
// With statistics, a CTA whose tiles alternate between column tiles (Ndim of 1024 / 2048: 8 / 16 column tiles, 132
// CTAs) flushes its partial sums after every tile; with global fixed-point atomics those flushes cost more than the
// GEMM.  So the H16 kernel adds its flushes to fixed-point words of its own (local_stats: [2 * Ndim][lo, hi], 32 * Ndim
// bytes of dynamic shared memory from NEEDED on) and adds them to the global accumulators once, when it ends.
template <int BN, int STAGES, bool A_TMA, bool H16 = false>
struct SmemLayout {
  static constexpr int EW = A_TMA ? 8 : 4;                // epilogue warps
  static constexpr int CPW = (BN / 32) / (EW / 4);        // 32-column chunks per epilogue warp
  static constexpr int NBUF = (A_TMA && BN == 128) ? 1 : 2;
  static constexpr int STAGE_PER_WARP = NBUF * 2048;
  static constexpr int B_STAGE_BYTES = BN * 128;
  static constexpr int A_OFF = 0;
  static constexpr int B_OFF = STAGES * A_STAGE_BYTES;
  // output staging.  The TMA swizzle patterns repeat every 512 B (64-byte mode) / 1024 B (128-byte mode), so every
  // buffer starts on such a boundary (1024-aligned base + multiples of 2048 / 4096).
  static constexpr int STAGE_OUT_OFF = B_OFF + STAGES * B_STAGE_BYTES;
  // finished accumulator tile [BM][ACC_LD] fp32 (MMA warpgroups -> epilogue warps)
  static constexpr int ACC_LD = acc_ld(BN);
  static constexpr int ACC_OFF = STAGE_OUT_OFF + EW * STAGE_PER_WARP;
  // H16: two bf16 output tiles from STAGE_OUT_OFF instead of the staging buffers and the fp32 tile
  static constexpr int OUT_TILE_BYTES = BM * BN * 2;
  static constexpr int BAR_OFF = H16 ? STAGE_OUT_OFF + 2 * OUT_TILE_BYTES : ACC_OFF + BM * ACC_LD * 4;
  static constexpr int NEEDED = BAR_OFF + 256;
  static constexpr int TOTAL = NEEDED + 768;   // slack for the run-time 1024-byte alignment of the base
  static_assert(TOTAL <= 232448, "one CTA per SM: <= 227 KB of dynamic shared memory");
};

// ---------------------------------------------------------------------------------------------
// fprop / dgrad kernel — persistent: each CTA loops over output tiles (tile = blockIdx.x + i*gridDim.x,
// n-tile fastest so that concurrently running CTAs share the A tile through L2).  The smem operand ring runs across
// tile boundaries and the accumulators of tile i+1 build up in registers while the epilogue warps drain tile i from
// shared memory, so producers, tensor cores and epilogue overlap.
//   warps 0 .. EW-1     : epilogue (tile rows 32*(w & 3) .. +31, column group w >> 2)
//   warps 4-7 (!A_TMA)  : A-operand gather producers
//   warps 8-15          : two MMA warpgroups (tile rows 0-63 / 64-127)
//   warp 16             : barrier init + TMA producer
// ---------------------------------------------------------------------------------------------
static constexpr int IG_THREADS = 17 * 32;

// named barrier 1 over the epilogue warps (threads 0 .. n-1) only; barrier 0 is __syncthreads
__device__ __forceinline__ void epilogue_bar_sync(int n) { asm volatile("bar.sync 1, %0;" ::"r"(n) : "memory"); }

template <int BN, int STAGES, bool A_TMA, bool GROUPED = false, bool H16 = false>
__global__ void __launch_bounds__(IG_THREADS, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB,
                  const __grid_constant__ CUtensorMap tmapC, const ConvGemmParams p, const int num_tiles) {
  static_assert(!GROUPED || (BN == 64 && !A_TMA), "grouped mode: 64-column tiles, gathered A operand");
  static_assert(!H16 || A_TMA, "bf16 hand-off: plain GEMM only (no parity mode)");
  using L = SmemLayout<BN, STAGES, A_TMA, H16>;
  constexpr int EW = L::EW;
  constexpr int CPW = L::CPW;
  constexpr int MMA_WARP = 8;
  constexpr int TMA_WARP = MMA_WARP + 8;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  if (smem + L::NEEDED > smem_raw + L::TOTAL) __trap();   // the dynamic smem base was less aligned than assumed
  uint8_t* smemA = smem + L::A_OFF;
  uint8_t* smemB = smem + L::B_OFF;
  uint64_t* full_bar = (uint64_t*)(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* tfull_bar = empty_bar + STAGES;   // accumulator tile ready for the epilogue
  uint64_t* tempty_bar = tfull_bar + 1;       // accumulator tile drained
  uint64_t* ofull_bar = tempty_bar + 1;       // H16: bf16 tile b staged (b = 0, 1)
  uint64_t* oempty_bar = ofull_bar + 2;       // H16: bf16 tile b stored and read
  uint8_t* stage_out = smem + L::STAGE_OUT_OFF;   // 1024-byte aligned
  float* accbuf = reinterpret_cast<float*>(smem + L::ACC_OFF);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = p.num_kb;

  if (warp == TMA_WARP && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], A_TMA ? 1u : 129u);
      mbar_init(&empty_bar[s], 2u);   // one arrival per MMA warpgroup
    }
    mbar_init(tfull_bar, 256u);       // every MMA thread, after storing its fragment
    mbar_init(tempty_bar, (uint32_t)EW);   // one arrival per epilogue warp
    for (int b = 0; b < 2; ++b) {
      mbar_init(&ofull_bar[b], 256u);
      mbar_init(&oempty_bar[b], (uint32_t)EW);
    }
    fence_mbar_init();
    tma_prefetch_desc(&tmapB);
    if (A_TMA) tma_prefetch_desc(&tmapA);
    if (!p.out_fp32) tma_prefetch_desc(&tmapC);
  }
  __syncthreads();

  if (warp < EW) {
    // ======================= epilogue =====================================================
    // Per 32-column chunk: shared-memory accumulator tile -> registers -> (bias / residual / ReLU) -> bf16 -> this warp's swizzled smem
    // staging -> TMA store (no LSU global stores).  While the TMA engine reads the staging tile, the warp sums its
    // 32 rows per column from the same tile for the fused BatchNorm statistics (packed fp32x2 arithmetic on two
    // columns per lane); the sums stay in registers across all tiles of this CTA that share a column block.
    const bool do_stats = p.col_sum != nullptr;
    const int quarter = warp & 3;                 // tile rows 32*quarter ..
    const int col_w0 = (warp >> 2) * (CPW * 32);  // first tile column of this warp
    const uint32_t stage_base0 = smem_u32(stage_out + warp * L::STAGE_PER_WARP);
    int sbuf = 0;
    constexpr int NACC = CPW;
    uint64_t cs1[NACC], cs2[NACC];   // packed {even, odd} column sums / sums of squares
#pragma unroll
    for (int i = 0; i < NACC; ++i) { cs1[i] = 0ull; cs2[i] = 0ull; }
    int local = 0;
    int stat_n0 = -1;   // column offset the register accumulators currently belong to
    const bool local_stats = H16 && do_stats && p.local_stats;
    unsigned long long* lstats = reinterpret_cast<unsigned long long*>(smem + L::NEEDED);
    if (local_stats) {
      for (int i = threadIdx.x; i < 4 * p.Ndim; i += EW * 32) lstats[i] = 0ull;
      epilogue_bar_sync(EW * 32);
    }
    auto flush_stats = [&]() {
#pragma unroll
      for (int i = 0; i < NACC; ++i) {
        float2 a = f2_unpack(cs1[i]), b = f2_unpack(cs2[i]);
        // lanes l and l ^ 16 hold the two row parities of the same column pair
        a.x += __shfl_xor_sync(0xffffffffu, a.x, 16);
        a.y += __shfl_xor_sync(0xffffffffu, a.y, 16);
        b.x += __shfl_xor_sync(0xffffffffu, b.x, 16);
        b.y += __shfl_xor_sync(0xffffffffu, b.y, 16);
        const int col = stat_n0 + col_w0 + i * 32 + 2 * (lane & 15);
        const bool owner = lane < 16;
        if (owner && col < p.Ndim && local_stats) {   // Ndim is a multiple of 8: col + 1 is valid too
          fix_add_local(p.fx + col, lstats + 2 * col, a.x);
          fix_add_local(p.fx + col + 1, lstats + 2 * (col + 1), a.y);
          fix_add_local(p.fx + p.Ndim + col, lstats + 2 * (p.Ndim + col), b.x);
          fix_add_local(p.fx + p.Ndim + col + 1, lstats + 2 * (p.Ndim + col + 1), b.y);
        } else if (owner && col < p.Ndim) {
          fix_add(p.fx + col, a.x);
          fix_add(p.fx + col + 1, a.y);
          fix_add(p.fx + p.Ndim + col, b.x);
          fix_add(p.fx + p.Ndim + col + 1, b.y);
        }
        cs1[i] = 0ull; cs2[i] = 0ull;
      }
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++local) {
      const TileInfo ti = tile_info<GROUPED>(p, tile, BN);
      const int m0 = ti.m0;
      const int n0 = ti.n0;
      if (do_stats && stat_n0 != n0) {
        if (stat_n0 >= 0) flush_stats();
        stat_n0 = n0;
      }
      if constexpr (H16) {
        // the MMA warpgroups staged this warp's blocks (and fenced them for the TMA engine): store, then sum
        // the statistics from the same bytes while the TMA engine reads them
        const int buf = local & 1;
        mbar_wait(&ofull_bar[buf], (uint32_t)((local >> 1) & 1));
        const int mrow0 = m0 + quarter * 32;
        int rows_valid = p.M - mrow0;
        rows_valid = rows_valid < 0 ? 0 : (rows_valid > 32 ? 32 : rows_valid);
        const uint32_t qbase = smem_u32(stage_out + buf * L::OUT_TILE_BYTES) + (uint32_t)quarter * (BN / 32) * 2048u;
#pragma unroll
        for (int cl = 0; cl < CPW; ++cl) {
          const int c0 = col_w0 + cl * 32;
          const int nbase = n0 + c0;
          if (nbase >= p.Ndim) continue;  // warp-uniform
          const uint32_t blk = qbase + (uint32_t)(c0 / 32) * 2048u;
          if (lane == 0) {
            tma_store_2d(&tmapC, blk, nbase, mrow0);   // rows >= M and columns >= Ndim are clipped by TMA
            tma_store_commit();
          }
          if (do_stats) stats_narrow(blk, lane, rows_valid, cs1[cl], cs2[cl]);
        }
        // the TMA engine has read the blocks and every lane is past its statistics: hand the buffer back
        if (lane == 0) tma_store_wait_read();
        __syncwarp();
        if (lane == 0) mbar_arrive(&oempty_bar[buf]);
        continue;
      }
      mbar_wait(tfull_bar, (uint32_t)(local & 1));
      const int mrow0 = m0 + quarter * 32;
      int m = mrow0 + lane;
      const bool mvalid = m < p.M;
      if (p.parity) {
        // row of the class-major enumeration -> row of dX: pixel (n, 2a + ph, 2b + pw)
        const int mc = m - ti.cls_idx * p.Mc;
        const int b = mc % p.Wh;
        const int t2 = mc / p.Wh;
        const int a = t2 % p.Hh;
        const int n = t2 / p.Hh;
        m = (n * p.Ho + 2 * a + ti.ph) * p.Wo + 2 * b + ti.pw;
      }
      int rows_valid = p.M - mrow0;
      rows_valid = rows_valid < 0 ? 0 : (rows_valid > 32 ? 32 : rows_valid);
      // residual row of this thread's output row (resid_up: the compact gradient of a stride-2 branch is scattered
      // to the even pixels of the full-resolution map)
      bool rvalid = mvalid;
      int64_t rrow = m;
      if (p.resid_up) {
        const int w = m % p.Wo;
        const int t2 = m / p.Wo;
        const int h = t2 % p.Ho;
        const int n = t2 / p.Ho;
        rvalid = mvalid && ((h | w) & 1) == 0;
        rrow = ((int64_t)n * (p.Ho >> 1) + (h >> 1)) * (p.Wo >> 1) + (w >> 1);
      }
#pragma unroll
      for (int cl = 0; cl < CPW; ++cl) {
        const int c0 = col_w0 + cl * 32;
        uint32_t r[32];
        acc_load_row32(accbuf + (quarter * 32 + lane) * L::ACC_LD + c0, r);
        if (cl == CPW - 1) {
          // last read of this tile: hand the accumulator tile back to the MMA warpgroups
          __syncwarp();
          if (lane == 0) mbar_arrive(tempty_bar);
        }
        const int nbase = n0 + c0;
        if (nbase >= p.Ndim) continue;  // warp-uniform
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
        if (p.bias != nullptr) {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (nbase + j < p.Ndim) v[j] += __ldg(p.bias + nbase + j);
        }
        if (p.resid != nullptr && rvalid) {
          const bf16* rp = p.resid + rrow * p.ldc + nbase;
          const uint8_t* mp = p.resid_mask != nullptr ? p.resid_mask + ((rrow * p.ldc + nbase) >> 3) : nullptr;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            if (nbase + j < p.Ndim) {
              uint4 q = *reinterpret_cast<const uint4*>(rp + j);
              const uint32_t mb = mp != nullptr ? (uint32_t)__ldg(mp + (j >> 3)) : 0xffu;
              const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                float2 f = __bfloat1622float2(h[e]);
                v[j + 2 * e] += ((mb >> (2 * e)) & 1u) ? f.x : 0.f;
                v[j + 2 * e + 1] += ((mb >> (2 * e + 1)) & 1u) ? f.y : 0.f;
              }
            }
          }
        }
        if (p.resid_f32 != nullptr && rvalid) {
          const float* rp = p.resid_f32 + rrow * p.ldc + nbase;
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (nbase + j < p.Ndim) v[j] += rp[j];
        }
        if (p.relu) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        if (p.parity) {
          // rows of one tile are not contiguous in dX: plain 16-byte stores (six layers per backward pass only)
          if (mvalid) {
            bf16* op = reinterpret_cast<bf16*>(p.dst) + (int64_t)m * p.ldc + nbase;
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              if (nbase + j < p.Ndim) {
                uint4 q;
                q.x = pack_bf16x2(v[j], v[j + 1]);
                q.y = pack_bf16x2(v[j + 2], v[j + 3]);
                q.z = pack_bf16x2(v[j + 4], v[j + 5]);
                q.w = pack_bf16x2(v[j + 6], v[j + 7]);
                *reinterpret_cast<uint4*>(op + j) = q;
              }
            }
          }
        } else if (p.out_fp32) {
          if (mvalid) {
            float* op = reinterpret_cast<float*>(p.dst) + (int64_t)m * p.ldc + nbase;
            const bool vec = (p.ldc & 3) == 0;   // 16-byte aligned rows; otherwise (e.g. a 10-class classifier) scalar
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              if (vec && nbase + j + 3 < p.Ndim) {
                *reinterpret_cast<float4*>(op + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
              } else {
#pragma unroll
                for (int e = 0; e < 4; ++e)
                  if (nbase + j + e < p.Ndim) op[j + e] = v[j + e];
              }
            }
          }
        } else {
          // stage this warp's [32 rows][32 cols] bf16 block: row = lane, 16-byte chunk j at (j ^ ((row >> 1) & 3))
          // (= the TMA 64-byte swizzle), which also spreads the 32 row-writes over all banks
          const uint32_t stage_base = stage_base0 + (uint32_t)sbuf * 2048u;
          // the store that last used THIS buffer has read it (and every lane is past its statistics loop)
          if (lane == 0) { if (L::NBUF == 2) tma_store_wait_read1(); else tma_store_wait_read(); }
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint4 q;
            q.x = pack_bf16x2(v[8 * j + 0], v[8 * j + 1]);
            q.y = pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
            q.z = pack_bf16x2(v[8 * j + 4], v[8 * j + 5]);
            q.w = pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
            const uint32_t off = (uint32_t)lane * 64u + (uint32_t)((j ^ ((lane >> 1) & 3)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(stage_base + off), "r"(q.x), "r"(q.y),
                         "r"(q.z), "r"(q.w)
                         : "memory");
          }
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            tma_store_2d(&tmapC, stage_base, nbase, mrow0);   // rows >= M and columns >= Ndim are clipped by TMA
            tma_store_commit();
          }
          if (do_stats) stats_narrow(stage_base, lane, rows_valid, cs1[cl], cs2[cl]);
          if (L::NBUF == 2) sbuf ^= 1;
        }
      }
    }
    if (do_stats && stat_n0 >= 0) flush_stats();
    if (local_stats) {   // every epilogue warp has flushed: the CTA's words -> the global accumulators, once
      epilogue_bar_sync(EW * 32);
      for (int i = threadIdx.x; i < 2 * p.Ndim; i += EW * 32) {
        const unsigned long long lo = lstats[2 * i], hi = lstats[2 * i + 1];
        if ((lo | hi) != 0ull) fix_add_words(p.fx + i, lo, (long long)hi);
      }
    }
    if (lane == 0) tma_store_wait_all();   // global writes complete before the kernel exits
  } else if (!A_TMA && warp >= EW && warp < EW + 4) {
    // ======================= A gather producers ==========================================
    const int tid = threadIdx.x - 128;
    const int chunk = tid & 7;   // 16-byte chunk inside the 128-byte k-row
    const int row0 = tid >> 3;   // rows row0 + 16*i
    int it = 0;                  // k-block iteration counter across tiles
    // Fast path (stride-1 source mapping, C a multiple of 64, <= 32 taps, < 2^31 elements): one k-block is 64
    // channels of ONE tap, so the tap counters advance without divisions, every row needs just
    // "base offset + tap offset", and padding is a per-row bitmask over the taps computed once per tile.
    // The stride-2 dgrad mapping (div == 2) fits too: a tap is valid only if it has the parity of (o + pad), and
    // then src = ((o + pad) >> 1) - (k >> 1), i.e. again "row base + tap offset"; parity goes into the bitmask.
    // (grouped mode: the host guarantees the fast-path conditions)
    const bool fast = GROUPED || ((p.C % BK == 0) && (p.KH * p.KW <= 32) && p.small_src);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileInfo ti = tile_info<GROUPED>(p, tile, BN);
      const int m0 = ti.m0;
      if (!GROUPED && p.fold) {
        // stem: k-block = kh, this thread's 16-byte chunk = kw: the 8 chunks of a row are 128 contiguous bytes
        uint32_t mask[8];   // bit kh: (kh, this thread's kw) lies inside the image
        int roff[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int m = m0 + row0 + 16 * i;
          mask[i] = 0u;
          roff[i] = 0;
          if (m < p.M) {
            const int ow = m % p.Wo;
            const int t = m / p.Wo;
            const int oh = t % p.Ho;
            const int n = t / p.Ho;
            const int bh = oh * p.mul + p.base, bw = ow * p.mul + p.base;
            const int sw = bw + chunk;
            roff[i] = ((n * p.Hs + bh) * p.Ws + sw) * 8;
            if (chunk < p.KW && sw >= 0 && sw < p.Ws)
              for (int kh = 0; kh < p.KH; ++kh)
                if (bh + kh >= 0 && bh + kh < p.Hs) mask[i] |= 1u << kh;
          }
        }
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          if (it >= GATHER_LAG) {
            cp_async_wait<GATHER_LAG - 1>();
            fence_proxy_async_smem();
            mbar_arrive(&full_bar[(it - GATHER_LAG) % STAGES]);
          }
          mbar_wait(&empty_bar[s], ph ^ 1);
          const int tapoff = kb * p.Ws * 8;
          const uint32_t stage_base = smem_u32(smemA + s * A_STAGE_BYTES);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const bool v = (mask[i] >> kb) & 1u;
            const bf16* g = v ? p.src + (roff[i] + tapoff) : p.src;
            cp_async16_zfill(stage_base + sw128_offset(row0 + 16 * i, chunk), g, v);
          }
          cp_async_commit();
        }
      } else if (p.parity) {
        uint32_t mask[8];
        int roff[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int mc = m0 + row0 + 16 * i - ti.cls_idx * p.Mc;
          const int b = mc % p.Wh;
          const int t2 = mc / p.Wh;
          const int a = t2 % p.Hh;
          const int n = t2 / p.Hh;
          roff[i] = ((n * p.Hs + a) * p.Ws + b) * p.C;
          mask[i] = 0u;
          int tapi = 0;
          for (int kh = ti.kh0; kh < p.KH; kh += 2)
            for (int kw = ti.kw0; kw < p.KW; kw += 2, ++tapi) {
              const int sh = a + ((ti.ph + p.base - kh) >> 1), sw = b + ((ti.pw + p.base - kw) >> 1);
              if (sh >= 0 && sh < p.Hs && sw >= 0 && sw < p.Ws) mask[i] |= 1u << tapi;
            }
        }
        int kh = ti.kh0, kw = ti.kw0, cc = GROUPED ? ti.n0 : 0, tapi = 0;
        for (int kb = 0; kb < ti.nkb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          if (it >= GATHER_LAG) {
            cp_async_wait<GATHER_LAG - 1>();
            fence_proxy_async_smem();
            mbar_arrive(&full_bar[(it - GATHER_LAG) % STAGES]);
          }
          mbar_wait(&empty_bar[s], ph ^ 1);
          const int tapoff = (((ti.ph + p.base - kh) >> 1) * p.Ws + ((ti.pw + p.base - kw) >> 1)) * p.C + cc + chunk * 8;
          const uint32_t stage_base = smem_u32(smemA + s * A_STAGE_BYTES);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const bool v = (mask[i] >> tapi) & 1u;
            const bf16* g = v ? p.src + (roff[i] + tapoff) : p.src;
            cp_async16_zfill(stage_base + sw128_offset(row0 + 16 * i, chunk), g, v);
          }
          cp_async_commit();
          if (!GROUPED) cc += BK;
          if (GROUPED || cc >= p.C) {
            if (!GROUPED) cc = 0;
            ++tapi;
            kw += 2;
            if (kw >= p.KW) { kw = ti.kw0; kh += 2; }
          }
        }
      } else if (fast) {
        uint32_t mask[8];
        int roff[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int m = m0 + row0 + 16 * i;
          mask[i] = 0u;
          roff[i] = 0;
          if (m < p.M) {
            const int ow = m % p.Wo;
            const int t = m / p.Wo;
            const int oh = t % p.Ho;
            const int n = t / p.Ho;
            const int bh = oh * p.mul + p.base, bw = ow * p.mul + p.base;
            const int sft = p.div == 2 ? 1 : 0;
            roff[i] = ((n * p.Hs + (bh >> sft)) * p.Ws + (bw >> sft)) * p.C;
            int tapi = 0;
            for (int kh = 0; kh < p.KH; ++kh)
              for (int kw = 0; kw < p.KW; ++kw, ++tapi) {
                int sh = bh + kh * p.dk, sw = bw + kw * p.dk;
                bool ok = sh >= 0 && sw >= 0;
                if (p.div == 2) { ok = ok && ((sh | sw) & 1) == 0; sh >>= 1; sw >>= 1; }
                if (ok && sh < p.Hs && sw < p.Ws) mask[i] |= 1u << tapi;
              }
          }
        }
        int kh = 0, kw = 0, cc = GROUPED ? ti.n0 : 0, tapi = 0;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          if (it >= GATHER_LAG) {
            cp_async_wait<GATHER_LAG - 1>();
            fence_proxy_async_smem();
            mbar_arrive(&full_bar[(it - GATHER_LAG) % STAGES]);
          }
          mbar_wait(&empty_bar[s], ph ^ 1);
          const int tapoff = (p.div == 2 ? -((kh >> 1) * p.Ws + (kw >> 1)) : (kh * p.Ws + kw) * p.dk) * p.C + cc +
                             chunk * 8;
          const uint32_t stage_base = smem_u32(smemA + s * A_STAGE_BYTES);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const bool v = (mask[i] >> tapi) & 1u;
            const bf16* g = v ? p.src + (roff[i] + tapoff) : p.src;
            cp_async16_zfill(stage_base + sw128_offset(row0 + 16 * i, chunk), g, v);
          }
          cp_async_commit();
          if (!GROUPED) cc += BK;
          if (GROUPED || cc >= p.C) {
            if (!GROUPED) cc = 0;
            ++tapi;
            if (++kw == p.KW) { kw = 0; ++kh; }
          }
        }
      } else if (!GROUPED) {
        int bh[8], bw[8];
        int64_t ioff[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          int m = m0 + row0 + 16 * i;
          if (m < p.M) {
            int ow = m % p.Wo;
            int t = m / p.Wo;
            int oh = t % p.Ho;
            int n = t / p.Ho;
            bh[i] = oh * p.mul + p.base;
            bw[i] = ow * p.mul + p.base;
            ioff[i] = (int64_t)n * p.Hs * p.Ws * p.C;
          } else {
            bh[i] = -(1 << 28);  // never valid
            bw[i] = -(1 << 28);
            ioff[i] = 0;
          }
        }
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          // Publish the stage issued GATHER_LAG iterations ago BEFORE blocking on a free slot: otherwise the MMA
          // warp would wait for this thread to come round the loop although the data landed long ago.
          if (it >= GATHER_LAG) {
            cp_async_wait<GATHER_LAG - 1>();
            fence_proxy_async_smem();
            mbar_arrive(&full_bar[(it - GATHER_LAG) % STAGES]);
          }
          mbar_wait(&empty_bar[s], ph ^ 1);
          const int k0 = kb * BK + chunk * 8;
          const bool kvalid = k0 < p.Kg;
          const int tap = k0 / p.C;
          const int cc = k0 - tap * p.C;
          const int kh = tap / p.KW;
          const int kw = tap - kh * p.KW;
          const int dh = kh * p.dk, dw = kw * p.dk;
          const uint32_t stage_base = smem_u32(smemA + s * A_STAGE_BYTES);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            int sh = bh[i] + dh, sw = bw[i] + dw;
            bool v = kvalid && sh >= 0 && sw >= 0;
            if (p.div == 2) {
              v = v && ((sh | sw) & 1) == 0;
              sh >>= 1;
              sw >>= 1;
            }
            v = v && sh < p.Hs && sw < p.Ws;
            const bf16* g = v ? p.src + ioff[i] + ((int64_t)sh * p.Ws + sw) * p.C + cc : p.src;
            cp_async16_zfill(stage_base + sw128_offset(row0 + 16 * i, chunk), g, v);
          }
          cp_async_commit();
        }
      }
    }
    cp_async_wait<0>();
    fence_proxy_async_smem();
    for (int j = (it > GATHER_LAG ? it - GATHER_LAG : 0); j < it; ++j) mbar_arrive(&full_bar[j % STAGES]);
  } else if (warp >= MMA_WARP && warp < TMA_WARP) {
    // ======================= MMA warpgroups ===============================================
    // warpgroup wg multiplies tile rows 64*wg .. +63 (A rows 8 KB further into the stage) with the whole B tile
    const int wg = (warp - MMA_WARP) >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    float d[BN / 2];
    int it = 0, local = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++local) {
      const int nkb_tile = tile_info<GROUPED>(p, tile, BN).nkb;
      int prev_s = -1;
      for (int kb = 0; kb < nkb_tile; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint64_t adesc = make_smem_desc_sw128(smem_u32(smemA + s * A_STAGE_BYTES + wg * 8192), 16, 1024);
        const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smemB + s * L::B_STAGE_BYTES), 16, 1024);
        wg_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // advance 16 bf16 = 32 bytes along K inside the swizzle row: +2 in the (addr >> 4) field
          wgmma_bf16<BN, 0, 0>(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
        }
        wg_commit();
        wg_wait<1>();   // the previous k-block's MMAs are done: release its stage
        if (leader && prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wg_wait<0>();
      wg_fence_acc(d);
      if (leader && prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
      if constexpr (H16) {
        const int buf = local & 1;
        mbar_wait(&oempty_bar[buf], (uint32_t)(((local >> 1) & 1) ^ 1));
        // this warpgroup's two row quarters: blocks 2 * wg * (BN / 32) ..
        acc_store_bf16_sw64<BN>(smem_u32(stage_out + buf * L::OUT_TILE_BYTES) + (uint32_t)wg * 2 * (BN / 32) * 2048u, d);
        fence_proxy_async_smem();   // the epilogue's TMA stores (async proxy) read these writes
        mbar_arrive(&ofull_bar[buf]);
      } else {
        mbar_wait(tempty_bar, (uint32_t)((local & 1) ^ 1));
        acc_store_smem<BN>(accbuf, L::ACC_LD, wg * 64, 0, d);
        mbar_arrive(tfull_bar);
      }
    }
  } else if (warp == TMA_WARP) {
    // ======================= TMA producer =================================================
    if (lane == 0) {
      constexpr uint32_t tx = (uint32_t)L::B_STAGE_BYTES + (A_TMA ? (uint32_t)A_STAGE_BYTES : 0u);
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileInfo ti = tile_info<GROUPED>(p, tile, BN);
        const int n0 = ti.n0;
        const int m0 = ti.m0;
        int kh = ti.kh0, kw = ti.kw0, cc = 0;
        for (int kb = 0; kb < ti.nkb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], tx);
          int kcol = kb * BK;
          if (p.parity) {   // weight columns of the current class tap
            kcol = (kh * p.KW + kw) * (GROUPED ? BK : p.C) + cc;
            if (!GROUPED) cc += BK;
            if (GROUPED || cc >= p.C) { cc = 0; kw += 2; if (kw >= p.KW) { kw = ti.kw0; kh += 2; } }
          }
          tma_load_2d(smem_u32(smemB + s * L::B_STAGE_BYTES), &tmapB, &full_bar[s], kcol, n0);
          if (A_TMA) tma_load_2d(smem_u32(smemA + s * A_STAGE_BYTES), &tmapA, &full_bar[s], kb * BK, m0);
        }
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// wgrad kernel:  dW[co, tap, ci] += sum over pixels of dY[m, co] * src[pix(m, tap), ci]
//   A = dY  (MN-major: smem rows are pixels, 64-channel chunks along M)   via TMA
//   B = src (MN-major: smem rows are pixels, 64-channel chunks along N)   via TMA (plain GEMM) or gather
//   D[co 128][ci BN] accumulated in registers of two MMA warpgroups (co rows 0-63 / 64-127) over this CTA's pixel
//   range, then stored from the registers as this split's partial of the fp32 gradient, in the reference's
//   [Cout][Cin][KH][KW] parameter layout (wgrad_reduce), or with one split added to the gradient directly.
//   warps 0-3: B gather (when B is not loaded by TMA), warps 4-11: MMA warpgroups, warp 12: TMA producer.
// ---------------------------------------------------------------------------------------------
struct WgradParams {
  const bf16* src;   // NHWC [Nimg, Hs, Ws, C] forward input of the conv
  float* dw;         // fp32 gradient, [Cout][Cin_real][KH][KW]
  int Nimg, Hs, Ws, C;
  int Ho, Wo;
  int KH, KW;
  int stride, pad;
  int M;             // Nimg*Ho*Wo
  int Cout, Cin_real;
  int tiles_co, tiles_n;
  int splits, kb_per_split, num_kb_total;
  int Cg;            // channels per column group: C, or 64 in folded (stem) mode
  int groups;        // number of column groups: KH*KW taps, or KH in folded mode
  int fold_kw;       // 1: C == 8 and the KW taps are folded into the 64-wide column group: column = kw*8 + c
  int small_src;     // 1: 32-bit element offsets are safe
  float* part;       // splits > 1: [splits][Cout * Cin_real * KH * KW] fp32 partials (part_scratch), see wgrad_reduce
  int64_t ndw;
  // split-operand plane layouts (byol_conv_wgrad_planes): the product terms are an outer K loop.  K-block kb belongs
  // to term kb / kb_per_term, which reads dY columns from term * dy_term on and src channels from src_term[term] on.
  // Plain bf16 operands: terms = 1, ldsrc = C.
  int terms, kb_per_term;
  int ldsrc;         // src pixel pitch in elements
  int dy_term;
  int src_term[6];
};

static constexpr int WG_KROWS = 64;  // pixels per k-block
static constexpr int WG_A_STAGE = 2 * WG_KROWS * 128;  // two 64-channel chunks (co tile = 128)

// The GEMM N dimension is the concatenation of all taps: column = group*Cg + c (group = tap), tiled by BN, so a
// CTA whose BN spans several taps re-uses its dY tile (A operand) for all of them.
static constexpr int WG_THREADS = 13 * 32;

// GROUPED (grouped 3x3 convolutions, Cin == Cout == C, Cin_real = C / groups dividing 64): BN = 128, one tap per
// N-tile (Cg = 128), and the B chunk of warpgroup wg holds the input channels co0 + 64*wg .. +63, the only ones that
// share a group with its 64 output channels.  Each warpgroup runs a 64 x 64 MMA on its own chunk; only the in-group
// entries reach dW[Cout][Cin_real][KH][KW].
template <int BN, int STAGES, bool B_TMA, bool GROUPED = false>
__global__ void __launch_bounds__(WG_THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB,
                  const WgradParams p) {
  static_assert(!GROUPED || (BN == 128 && !B_TMA), "grouped mode: two 64-channel chunks, gathered B operand");
  constexpr int NCH = BN / 64;                       // 64-channel chunks along N
  constexpr int NMMA = GROUPED ? 64 : BN;            // MMA width per warpgroup
  constexpr int B_STAGE = NCH * WG_KROWS * 128;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + STAGES * WG_A_STAGE;
  uint64_t* full_bar = (uint64_t*)(smemB + STAGES * B_STAGE);
  uint64_t* empty_bar = full_bar + STAGES;

  // a warp index ptxas knows is warp-uniform: derived straight from threadIdx.x, the MMA branch counts as divergent
  // and ptxas serializes the wgmma of the TMA-operand variant (C7518)
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  int bid = blockIdx.x;
  const int tile_n = bid % p.tiles_n;    bid /= p.tiles_n;
  const int tile_co = bid % p.tiles_co;  bid /= p.tiles_co;
  const int split = bid;
  const int co0 = tile_co * 128;
  const int n0 = tile_n * BN;            // first column of this tile in the concatenated (group, channel) space
  const int kb_begin = split * p.kb_per_split;
  int kb_end = kb_begin + p.kb_per_split;
  if (kb_end > p.num_kb_total) kb_end = p.num_kb_total;
  const int nkb = kb_end - kb_begin;   // host guarantees nkb >= 1
  const int taps = p.KH * p.KW;

  if (warp == 12 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], B_TMA ? 1u : 129u);
      mbar_init(&empty_bar[s], 2u);   // one arrival per MMA warpgroup
    }
    fence_mbar_init();
    tma_prefetch_desc(&tmapA);
    if (B_TMA) tma_prefetch_desc(&tmapB);
  }
  __syncthreads();

  if (warp < 4) {
    if (!B_TMA) {
      // gather: 64 pixel rows x (NCH*8) 16-byte chunks per stage, 128 threads.  Thread t owns chunk column
      // (t % CHUNKS) -> a fixed (tap, channel) -> and PER_THREAD CONSECUTIVE pixels, so that coordinates and the
      // source offset advance by plain increments (one division pair per k-block, none per element).
      constexpr int CHUNKS = NCH * 8;
      constexpr int PER_THREAD = WG_KROWS * CHUNKS / 128;
      const int chunk = threadIdx.x % CHUNKS;
      const int rbase = (threadIdx.x / CHUNKS) * PER_THREAD;
      const int ch64 = chunk >> 3, c16 = chunk & 7;
      const int col = n0 + chunk * 8;
      const int group = col / p.Cg;
      const int cw = col - group * p.Cg;
      int kh, kw, ci;
      bool cvalid = group < p.groups;
      if (p.fold_kw) { kh = group; kw = cw >> 3; ci = 0; cvalid = cvalid && kw < p.KW; }
      else           { kh = group / p.KW; kw = group - kh * p.KW; ci = cw; }
      if (GROUPED) { ci += co0; cvalid = cvalid && ci < p.C; }
      const int dh = kh - p.pad, dw = kw - p.pad;
      const int64_t sC = (int64_t)p.stride * p.ldsrc;
      for (int it = 0; it < nkb; ++it) {
        const int kb = kb_begin + it;
        const int term = p.terms == 1 ? 0 : kb / p.kb_per_term;
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        if (it >= GATHER_LAG) {   // publish the older stage before blocking on a free slot (see conv_igemm_kernel)
          cp_async_wait<GATHER_LAG - 1>();
          fence_proxy_async_smem();
          mbar_arrive(&full_bar[(it - GATHER_LAG) % STAGES]);
        }
        mbar_wait(&empty_bar[s], ph ^ 1);
        const uint32_t stage_base = smem_u32(smemB + s * B_STAGE) + ch64 * (WG_KROWS * 128);
        const int cterm = ci + p.src_term[term];
        int m = (kb - term * p.kb_per_term) * WG_KROWS + rbase;
        int ow = m % p.Wo;
        int t = m / p.Wo;
        int oh = t % p.Ho;
        int n = t / p.Ho;
        int sw = ow * p.stride + dw;
        int sh = oh * p.stride + dh;
        bool hvalid = cvalid && sh >= 0 && sh < p.Hs;
        int64_t off = (((int64_t)n * p.Hs + sh) * p.Ws + sw) * p.ldsrc + cterm;
#pragma unroll
        for (int i = 0; i < PER_THREAD; ++i) {
          const bool v = hvalid && m < p.M && sw >= 0 && sw < p.Ws;
          cp_async16_zfill(stage_base + sw128_offset(rbase + i, c16), v ? p.src + off : p.src, v);
          ++m;
          sw += p.stride;
          off += sC;
          if (++ow == p.Wo) {
            ow = 0;
            if (++oh == p.Ho) { oh = 0; ++n; }
            sw = dw;
            sh = oh * p.stride + dh;
            hvalid = cvalid && sh >= 0 && sh < p.Hs;
            off = (((int64_t)n * p.Hs + sh) * p.Ws + sw) * p.ldsrc + cterm;
          }
        }
        cp_async_commit();
      }
      cp_async_wait<0>();
      fence_proxy_async_smem();
      for (int it = (nkb > GATHER_LAG ? nkb - GATHER_LAG : 0); it < nkb; ++it) mbar_arrive(&full_bar[it % STAGES]);
    }
  } else if (warp < 12) {
    // ======================= MMA warpgroups (co rows 64*wg .. +63) ========================
    const int wg = (warp - 4) >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    float d[NMMA / 2];
    int prev_s = -1;
    for (int it = 0; it < nkb; ++it) {
      const int s = it % STAGES;
      const uint32_t ph = (it / STAGES) & 1;
      mbar_wait(&full_bar[s], ph);
      // MN-major SW128: LBO = stride between 64-element MN chunks, SBO = stride between 8-row K groups; this
      // warpgroup's 64 co are the A chunk wg
      const uint64_t adesc =
          make_smem_desc_sw128(smem_u32(smemA + s * WG_A_STAGE + wg * WG_KROWS * 128), WG_KROWS * 128, 1024);
      const uint64_t bdesc = make_smem_desc_sw128(
          smem_u32(smemB + s * B_STAGE + (GROUPED ? wg * WG_KROWS * 128 : 0)), WG_KROWS * 128, 1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < WG_KROWS / 16; ++k) {
        // advance 16 pixel rows = 2048 bytes: +128 in the (addr >> 4) field
        wgmma_bf16<NMMA, 1, 1>(d, adesc + (uint64_t)(128 * k), bdesc + (uint64_t)(128 * k), (uint32_t)((it | k) != 0));
      }
      wg_commit();
      wg_wait<1>();
      if (leader && prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
    }
    wg_wait<0>();
    wg_fence_acc(d);
    // ---------------- epilogue: registers -> this split's partials (or, with one split, the gradient) ----------------
    const int t = threadIdx.x & 127;
    const int r0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
    float* const part = p.part != nullptr ? p.part + (int64_t)split * p.ndw : nullptr;
    auto add = [&](float* q, float v) {
      if (part != nullptr) part[q - p.dw] = v;
      else wgrad_add_single(q, v);
    };
    if (GROUPED) {
      // column c of warpgroup wg is input channel co0 + 64*wg + c
      const int gs = p.Cin_real;
      const int tap = n0 / BN;
#pragma unroll
      for (int j = 0; j < NMMA / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int co = co0 + r0 + 8 * h;
          if (co >= p.Cout) continue;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int ci = co0 + wg * 64 + 8 * j + 2 * (t & 3) + e;
            if (co / gs == ci / gs) add(p.dw + ((int64_t)co * gs + ci % gs) * taps + tap, d[4 * j + 2 * h + e]);
          }
        }
      }
      return;
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int co = co0 + r0 + 8 * h;
        const int colb = n0 + 8 * j + 2 * (t & 3);   // columns colb, colb + 1 lie in one group (Cg % 8 == 0)
        const int group = colb / p.Cg;
        const int cw = colb - group * p.Cg;
        const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
        if (co >= p.Cout || group >= p.groups) continue;
        if (p.fold_kw) {
          // column = kw*8 + ci ; the group index is kh
          float* gp = p.dw + ((int64_t)co * p.Cin_real) * taps + group * p.KW;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int kwj = (cw + e) >> 3, cj = (cw + e) & 7;
            if (kwj < p.KW && cj < p.Cin_real) add(gp + (int64_t)cj * taps + kwj, e ? v1 : v0);
          }
        } else {
          float* gp = p.dw + ((int64_t)co * p.Cin_real) * taps + group;
          if (cw < p.Cin_real) add(gp + (int64_t)cw * taps, v0);
          if (cw + 1 < p.Cin_real) add(gp + (int64_t)(cw + 1) * taps, v1);
        }
      }
    }
  } else {
    if (lane == 0) {
      constexpr uint32_t tx = (uint32_t)WG_A_STAGE + (B_TMA ? (uint32_t)B_STAGE : 0u);
      for (int it = 0; it < nkb; ++it) {
        const int kb = kb_begin + it;
        const int term = p.terms == 1 ? 0 : kb / p.kb_per_term;
        const int row = (kb - term * p.kb_per_term) * WG_KROWS;
        const int col_a = co0 + term * p.dy_term;
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        mbar_arrive_expect_tx(&full_bar[s], tx);
        const uint32_t a_base = smem_u32(smemA + s * WG_A_STAGE);
        // with several terms, co rows past Cout read the next term's columns: those accumulator rows are discarded
        tma_load_2d(a_base, &tmapA, &full_bar[s], col_a, row);
        tma_load_2d(a_base + WG_KROWS * 128, &tmapA, &full_bar[s], col_a + 64, row);
        if (B_TMA) {
          const uint32_t b_base = smem_u32(smemB + s * B_STAGE);
#pragma unroll
          for (int c = 0; c < NCH; ++c)
            tma_load_2d(b_base + c * (WG_KROWS * 128), &tmapB, &full_bar[s], n0 + 64 * c + p.src_term[term], row);
        }
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// gemm_fused.cu: plain GEMM with a TMA-staged (masked) residual tile added in the epilogue
bool gemm_fused_applicable(int M, int C, int Ndim, int ldw, int ldc);
int gemm_fused_launch(const void* src, const void* wt, void* dst, const void* resid, const void* resid_mask,
                      const float* bias, int M, int C, int Ndim, int ldw, int ldc, int relu, cudaStream_t stream);

// conv_patch.cu
bool patch_conv_applicable(int H, int W, int C, int Ndim, int KH, int KW, int stride, int pad, int out_fp32,
                           const float* bias, int64_t src_elems);
int patch_conv_launch(const void* src, const void* wt, void* dst, const void* resid, float* col_sum, float* col_sqsum,
                      int Nimg, int H, int W, int C, int Ndim, int ldw, int ldc, int flip, int relu, int sms,
                      cudaStream_t stream, int grouped = 0);

bool patch_wgrad_applicable(int H, int W, int C, int Cin_real, int Cout, int KH, int KW, int stride, int pad);
int patch_wgrad_launch(const void* x, const void* dy, float* dw, int Nimg, int H, int W, int C, int Cout, int sms,
                       cudaStream_t stream, int gs = 0);

template <int BN, int STAGES, bool A_TMA, bool GROUPED = false, bool H16 = false>
static int launch_igemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
                        const ConvGemmParams& p, int tiles_m, cudaStream_t stream) {
  using L = SmemLayout<BN, STAGES, A_TMA, H16>;
  auto kern = conv_igemm_kernel<BN, STAGES, A_TMA, GROUPED, H16>;
  // block-local statistic words when they fit next to the tiles (Ndim <= 2112 at BN = 128); else global atomics
  ConvGemmParams q = p;
  const int64_t local_bytes = 32 * (int64_t)p.Ndim;
  q.local_stats = (H16 && p.col_sum != nullptr && L::TOTAL + local_bytes <= 232448) ? 1 : 0;
  const int smem = L::TOTAL + (q.local_stats ? (int)local_bytes : 0);
  if (smem_opt_in((const void*)kern, smem, "conv_igemm_kernel") != 0) return -2;
  const int num_tiles = tiles_m * p.tiles_n;
  int grid = device_sm_count();        // persistent: one CTA per SM (shared memory sized for it)
  if (grid > num_tiles) grid = num_tiles;
  kern<<<grid, IG_THREADS, smem, stream>>>(ta, tb, tc, q, num_tiles);
  return check_launch("conv_igemm_kernel");
}

}  // namespace byol

using namespace byol;

// out[M=Nimg*Ho*Wo, Ndim] = gather(src) x Wt^T  (+bias, +resid, relu, fused column statistics)
// mode 0 (fprop):  src coord = o*stride - pad + k
// mode 1 (dgrad):  src coord = (o + pad - k) / stride  (valid only when divisible); here `src` is dY,
//                  (Hs, Ws) its spatial size and (Ho, Wo) the spatial size of dX.
// resid_f32 (fp32 outputs only): an fp32 residual added in the epilogue (the fp32 backward's residual-branch gradient)
static int conv_igemm_impl(const void* src, const void* wt, void* dst, const void* resid, const float* resid_f32,
                           const void* resid_mask, int resid_up, const float* bias, float* col_sum, float* col_sqsum,
                           int Nimg, int Hs, int Ws, int C, int Ho, int Wo, int Ndim, int KH, int KW, int stride,
                           int pad, int mode, int ldw, int ldc, int out_fp32, int relu, int force_gather,
                           cudaStream_t stream, int grouped = 0) {
  BYOL_CHECK_ARG(src && wt && dst, "byol_conv_igemm: null pointer");
  BYOL_CHECK_ARG(resid_f32 == nullptr || (out_fp32 && resid == nullptr && !resid_up),
                 "byol_conv_igemm: an fp32 residual needs an fp32 output and no other residual");
  BYOL_CHECK_ARG(C % 8 == 0 && C >= 8, "byol_conv_igemm: C=%d must be a multiple of 8", C);
  // bf16 outputs are TMA-stored (16-byte row pitch); fp32 outputs (logits, MLP outputs) may have any width
  BYOL_CHECK_ARG(Ndim > 0 && (Ndim % 8 == 0 || (out_fp32 && resid == nullptr && col_sum == nullptr)),
                 "byol_conv_igemm: Ndim=%d must be a multiple of 8 (any width only for plain fp32 outputs)", Ndim);
  BYOL_CHECK_ARG(ldc >= Ndim && (ldc % 8 == 0 || out_fp32), "byol_conv_igemm: bad ldc=%d", ldc);
  BYOL_CHECK_ARG(!(out_fp32 && col_sum != nullptr), "byol_conv_igemm: fused statistics need a bf16 output");
  BYOL_CHECK_ARG((col_sum == nullptr) == (col_sqsum == nullptr), "byol_conv_igemm: need both statistics or none");
  BYOL_CHECK_ARG(stride == 1 || stride == 2, "byol_conv_igemm: stride %d unsupported", stride);
  BYOL_CHECK_ARG(mode == 0 || mode == 1, "byol_conv_igemm: bad mode %d", mode);
  const int64_t M64 = (int64_t)Nimg * Ho * Wo;
  BYOL_CHECK_ARG(M64 > 0 && M64 < (1ll << 31), "byol_conv_igemm: M out of range");
  BYOL_CHECK_ARG((int64_t)Nimg * Hs * Ws * C < (1ll << 40), "byol_conv_igemm: src too large");
  // 3x3 / stride 1 / pad 1 (fprop and its dgrad): shared-memory patch reuse instead of a 9x re-gather
  BYOL_CHECK_ARG(resid_mask == nullptr || (resid != nullptr && ldc % 8 == 0), "byol_conv_igemm: resid_mask without resid");
  BYOL_CHECK_ARG(!resid_up || (resid != nullptr && resid_mask == nullptr && Ho % 2 == 0 && Wo % 2 == 0 &&
                               !(mode == 1 && stride == 2)),
                 "byol_conv_igemm: resid_up needs resid, even output dims and a non-parity mode");
  // 1x1 / stride 1 with a residual tile in the epilogue (conv1 dgrad + the residual-branch gradient): the kernel that
  // stages the residual by TMA instead of per-lane global loads (3.5x faster at 56x56, tools/time_dgrad_resid.py)
  // (these two kernels take no fp32 residual: an fp32 residual always goes to conv_igemm_kernel)
  if (!force_gather && resid_f32 == nullptr && resid != nullptr && !resid_up && KH == 1 && KW == 1 && stride == 1 &&
      pad == 0 && !out_fp32 &&
      col_sum == nullptr && gemm_fused_applicable((int)M64, C, Ndim, ldw, ldc))
    return gemm_fused_launch(src, wt, dst, resid, resid_mask, bias, (int)M64, C, Ndim, ldw, ldc, relu, stream);
  if (!force_gather && resid_f32 == nullptr && resid_mask == nullptr && !resid_up && Hs == Ho && Ws == Wo &&
      ldw >= 9 * (grouped ? BK : C) &&
      patch_conv_applicable(Hs, Ws, C, Ndim, KH, KW, stride, pad, out_fp32, bias, (int64_t)Nimg * Hs * Ws * C))
    return patch_conv_launch(src, wt, dst, resid, col_sum, col_sqsum, Nimg, Hs, Ws, C, Ndim, ldw, ldc, mode, relu,
                             device_sm_count(), stream, grouped);
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.src = (const bf16*)src;
  p.dst = dst;
  p.resid = (const bf16*)resid;
  p.resid_mask = (const uint8_t*)resid_mask;
  p.resid_up = resid_up ? 1 : 0;
  p.resid_f32 = resid_f32;
  p.bias = bias;
  p.col_sum = col_sum;
  p.col_sqsum = col_sqsum;
  p.Nimg = Nimg; p.Hs = Hs; p.Ws = Ws; p.C = C; p.Ho = Ho; p.Wo = Wo; p.KH = KH; p.KW = KW;
  if (mode == 0) { p.mul = stride; p.base = -pad; p.dk = 1; p.div = 1; }
  else           { p.mul = 1; p.base = pad; p.dk = -1; p.div = stride; }
  p.M = (int)M64;
  p.Ndim = Ndim;
  p.Kg = KH * KW * (grouped ? BK : C);   // grouped: one 64-channel k-block per tap
  // stem layout (weights made by byol_prep_weight with fold = 1): K = KH * 64, column = kh*64 + kw*8 + c
  p.fold = (mode == 0 && C == 8 && KW > 1 && KW <= 8 && KH <= 32 && ldw == KH * 64 &&
            (int64_t)Nimg * Hs * Ws * C < (1ll << 31) - (1ll << 24)) ? 1 : 0;
  if (p.fold) p.Kg = KH * 64;
  BYOL_CHECK_ARG(ldw >= p.Kg && ldw % 8 == 0, "byol_conv_igemm: bad ldw=%d (Kg=%d)", ldw, p.Kg);
  p.ldc = ldc;
  p.num_kb = (p.Kg + BK - 1) / BK;
  p.out_fp32 = out_fp32;
  p.relu = relu;
  p.small_src = ((int64_t)Nimg * Hs * Ws * C < (1ll << 31) - (1ll << 24)) ? 1 : 0;
  const int BN = (Ndim > 64 && !grouped) ? 128 : 64;
  p.tiles_n = (Ndim + BN - 1) / BN;
  int tiles_m = (p.M + BM - 1) / BM;
  // the dX parity classes with at least one tap (a 1x1 / stride-2 / pad-0 dgrad has only class (0, 0))
  int ncls = 0, cls_list[4];
  for (int cls = 0; cls < 4; ++cls) {
    const int ph = cls >> 1, pw = cls & 1;
    const int nkh = (KH - ((ph + pad) & 1) + 1) >> 1, nkw = (KW - ((pw + pad) & 1) + 1) >> 1;
    if (nkh > 0 && nkw > 0) cls_list[ncls++] = cls;
  }
  // Parity mode launches tiles for the classes with taps only, so the residual of a pixel without taps would never
  // be added: with a residual, a layer with tap-less classes takes the gathered path, which visits every dX pixel.
  if (mode == 1 && stride == 2 && Ho % 2 == 0 && Wo % 2 == 0 && C % BK == 0 && p.small_src && KH <= 3 && KW <= 3 &&
      ((int64_t)Nimg * (Ho / 2) * (Wo / 2)) % BM == 0 && !out_fp32 && (resid == nullptr || ncls == 4)) {
    p.parity = 1;
    p.Hh = Ho / 2;
    p.Wh = Wo / 2;
    p.Mc = Nimg * p.Hh * p.Wh;
    p.ncls = ncls;
    for (int i = 0; i < ncls; ++i) p.cls_list[i] = cls_list[i];
    if (p.ncls < 4) {   // pixels of classes without any tap receive zero gradient (no residual here)
      cudaError_t e = cudaMemsetAsync(dst, 0, (size_t)p.M * ldc * sizeof(bf16), stream);
      if (e != cudaSuccess) { set_last_error("byol_conv_igemm: memset failed: %s", cudaGetErrorString(e)); return -2; }
    }
    tiles_m = p.ncls * (p.Mc / BM);
  }
  const bool a_tma = !force_gather && KH == 1 && KW == 1 && stride == 1 && pad == 0;   // never true in parity mode
  // bf16 hand-off (SmemLayout): the epilogue only stores the rounded accumulator and sums its statistics
  const bool h16 = a_tma && !out_fp32 && bias == nullptr && resid == nullptr && resid_mask == nullptr &&
                   resid_f32 == nullptr && !relu;

  CUtensorMap ta, tb, tc;
  memset(&ta, 0, sizeof(ta));
  if (tmap_2d(&tb, wt, (uint64_t)Ndim, (uint64_t)p.Kg, (uint64_t)ldw, (uint32_t)BN, 64u, "conv_igemm B") != 0) return -3;
  if (!out_fp32) {
    if (tmap_2d(&tc, dst, (uint64_t)p.M, (uint64_t)Ndim, (uint64_t)ldc, 32u, 32u, "conv_igemm C") != 0) return -3;
  } else {
    tc = tb;
  }
  if (a_tma) {
    if (tmap_2d(&ta, src, (uint64_t)p.M, (uint64_t)C, (uint64_t)C, (uint32_t)BM, 64u, "conv_igemm A") != 0) return -3;
  } else {
    ta = tb;
  }
  if (col_sum != nullptr) {
    p.fx = fix_scratch(stream, 2 * (int64_t)Ndim);
    if (p.fx == nullptr) return -2;
  }
  int rc;
  if (grouped) {
    rc = launch_igemm<64, 4, false, true>(ta, tb, tc, p, tiles_m, stream);
  } else if (BN == 128) {
    rc = h16     ? launch_igemm<128, 3, true, false, true>(ta, tb, tc, p, tiles_m, stream)
         : a_tma ? launch_igemm<128, 3, true>(ta, tb, tc, p, tiles_m, stream)
                 : launch_igemm<128, 3, false>(ta, tb, tc, p, tiles_m, stream);
  } else {
    rc = h16     ? launch_igemm<64, 3, true, false, true>(ta, tb, tc, p, tiles_m, stream)
         : a_tma ? launch_igemm<64, 3, true>(ta, tb, tc, p, tiles_m, stream)
                 : launch_igemm<64, 4, false>(ta, tb, tc, p, tiles_m, stream);
  }
  if (rc != 0 || col_sum == nullptr) return rc;
  return fix_flush_stats(p.fx, col_sum, col_sqsum, Ndim, stream);
}

extern "C" int byol_conv_igemm(const void* src, const void* wt, void* dst, const void* resid,
                               const void* resid_mask, int resid_up, const float* bias, float* col_sum, float* col_sqsum, int Nimg, int Hs, int Ws, int C, int Ho, int Wo,
                               int Ndim, int KH, int KW, int stride, int pad, int mode, int ldw, int ldc,
                               int out_fp32, int relu, int force_gather, cudaStream_t stream) {
  return conv_igemm_impl(src, wt, dst, resid, nullptr, resid_mask, resid_up, bias, col_sum, col_sqsum, Nimg, Hs, Ws, C,
                         Ho, Wo, Ndim, KH, KW, stride, pad, mode, ldw, ldc, out_fp32, relu, force_gather, stream);
}

// Grouped 3x3 convolutions (ResNeXt conv2): Cin == Cout == C, a multiple of 64; C / groups divides 64; pad 1;
// stride 1 or 2.  (H, W) is the input size, (Ho, Wo) the output size.  Every check runs before any launch.
static bool grouped_geometry_ok(const char* what, int Nimg, int H, int W, int C, int Ho, int Wo, int KH, int KW,
                                int stride, int pad) {
  if (Nimg <= 0 || H <= 0 || W <= 0 || C < 64 || C % 64 != 0 || KH != 3 || KW != 3 || pad != 1 ||
      (stride != 1 && stride != 2) || Ho != (H - 1) / stride + 1 || Wo != (W - 1) / stride + 1) {
    set_last_error("%s: unsupported geometry (N=%d H=%d W=%d C=%d Ho=%d Wo=%d KH=%d KW=%d stride=%d pad=%d): needs "
                   "C %% 64 == 0, 3x3, pad 1, stride 1 or 2", what, Nimg, H, W, C, Ho, Wo, KH, KW, stride, pad);
    return false;
  }
  const int64_t big = (int64_t)Nimg * (H > Ho ? H : Ho) * (W > Wo ? W : Wo) * C;
  if (big >= (1ll << 31) - (1ll << 24)) {
    set_last_error("%s: tensor of %lld elements too large for 32-bit offsets", what, (long long)big);
    return false;
  }
  return true;
}

// y[Nimg, Ho, Wo, C] = grouped conv(x[Nimg, H, W, C], wt); wt: bf16 [C / 64][64][9 * 64] (byol_prep_weights_grouped);
// col_sum / col_sqsum (both or none): += per-channel sum / sum of squares of the stored bf16 y
extern "C" int byol_conv_fprop_grouped(const void* x, const void* wt, void* y, float* col_sum, float* col_sqsum,
                                       int Nimg, int H, int W, int C, int Ho, int Wo, int KH, int KW, int stride,
                                       int pad, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && wt && y, "byol_conv_fprop_grouped: null pointer");
  if (!grouped_geometry_ok("byol_conv_fprop_grouped", Nimg, H, W, C, Ho, Wo, KH, KW, stride, pad)) return -1;
  return conv_igemm_impl(x, wt, y, nullptr, nullptr, nullptr, 0, nullptr, col_sum, col_sqsum, Nimg, H, W, C, Ho, Wo,
                         C, KH, KW, stride, pad, 0, KH * KW * BK, C, 0, 0, 0, stream, 1);
}

// dx[Nimg, H, W, C] = transpose of the grouped conv applied to dy[Nimg, Ho, Wo, C]; wd: bf16 [C / 64][64][9 * 64]
// (the dgrad layout of byol_prep_weights_grouped)
extern "C" int byol_conv_dgrad_grouped(const void* dy, const void* wd, void* dx, int Nimg, int Ho, int Wo, int C,
                                       int H, int W, int KH, int KW, int stride, int pad, cudaStream_t stream) {
  BYOL_CHECK_ARG(dy && wd && dx, "byol_conv_dgrad_grouped: null pointer");
  if (!grouped_geometry_ok("byol_conv_dgrad_grouped", Nimg, H, W, C, Ho, Wo, KH, KW, stride, pad)) return -1;
  return conv_igemm_impl(dy, wd, dx, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, Nimg, Ho, Wo, C, H, W,
                         C, KH, KW, stride, pad, 1, KH * KW * BK, C, 0, 0, 0, stream, 1);
}

// fp32-accurate dgrad: dx[Nimg, H, W, Cin] (fp32) = conv_transpose(dY, W) (+ resid_f32, fp32 [Nimg, H, W, Cin]).
// dy: bf16 planes [Nimg, Hs, Ws, T*Cout] (activation pattern), wd: bf16 [Cin, taps*T*Cout] (byol_prep_weight_dgrad_planes).
// One implicit GEMM over T*Cout channels.  Stride-2 layers take the gather path (the parity mode stores bf16 only).
extern "C" int byol_conv_dgrad_planes(const void* dy, const void* wd, float* dx, const float* resid_f32, int Nimg,
                                      int Hs, int Ws, int Cout, int H, int W, int Cin, int KH, int KW, int stride,
                                      int pad, int T, cudaStream_t stream) {
  BYOL_CHECK_ARG((T == 3 || T == 6) && Cout % 8 == 0 && Cin % 8 == 0, "byol_conv_dgrad_planes: bad args (T=%d Cout=%d Cin=%d)",
                 T, Cout, Cin);
  return conv_igemm_impl(dy, wd, dx, nullptr, resid_f32, nullptr, 0, nullptr, nullptr, nullptr, Nimg, Hs, Ws, T * Cout,
                         H, W, Cin, KH, KW, stride, pad, 1, KH * KW * T * Cout, Cin, 1, 0, 0, stream);
}

template <int BN, bool B_TMA, bool GROUPED = false>
static int launch_wgrad(const CUtensorMap& ta, const CUtensorMap& tb, const WgradParams& p, int grid,
                        cudaStream_t stream) {
  constexpr int STAGES = 4;
  constexpr int SMEM = STAGES * (WG_A_STAGE + (BN / 64) * WG_KROWS * 128) + 256 + 1024;
  auto kern = conv_wgrad_kernel<BN, STAGES, B_TMA, GROUPED>;
  if (smem_opt_in((const void*)kern, SMEM, "conv_wgrad_kernel") != 0) return -2;
  kern<<<grid, WG_THREADS, SMEM, stream>>>(ta, tb, p);
  return check_launch("conv_wgrad_kernel");
}

// dW[Cout][Cin_real][KH][KW] (fp32) += dY^T x gather(src);  dy: [M, Cout] bf16, src: NHWC [Nimg,Hs,Ws,C]
// ldy: row pitch of dy in elements (0 = Cout); a pitch > Cout lets Cout be any width (TMA zero-fills the columns
// beyond Cout), e.g. the gradient of a 10-class classifier stored with a pitch of 16.
// T: 0 = plain bf16 operands; 3 / 6 = split-operand planes (byol_conv_wgrad_planes)
static int conv_wgrad_impl(const void* src, const void* dy, float* dw, int Nimg, int Hs, int Ws, int C, int Cin_real,
                           int Ho, int Wo, int Cout, int ldy, int KH, int KW, int stride, int pad, int force_gather,
                           int T, cudaStream_t stream, int gs = 0) {
  BYOL_CHECK_ARG(src && dy && dw, "byol_conv_wgrad: null pointer");
  if (ldy == 0) ldy = Cout;
  // gs > 0: grouped 3x3 convolution with gs = Cin_real input channels per group (byol_conv_wgrad_grouped)
  if (gs > 0) {
    if (!force_gather && Hs == Ho && Ws == Wo && patch_wgrad_applicable(Hs, Ws, C, C, Cout, KH, KW, stride, pad))
      return patch_wgrad_launch(src, dy, dw, Nimg, Hs, Ws, C, Cout, device_sm_count(), stream, gs);
  }
  BYOL_CHECK_ARG(C % 8 == 0 && ldy % 8 == 0 && ldy >= Cout && Cout > 0,
                 "byol_conv_wgrad: C=%d and the dy pitch %d must be multiples of 8 (Cout=%d)", C, ldy, Cout);
  BYOL_CHECK_ARG(Cin_real <= C, "byol_conv_wgrad: Cin_real > C");
  BYOL_CHECK_ARG(T == 0 || T == 3 || T == 6, "byol_conv_wgrad: bad T=%d", T);
  const int64_t M64 = (int64_t)Nimg * Ho * Wo;
  BYOL_CHECK_ARG(M64 > 0 && M64 < (1ll << 31), "byol_conv_wgrad: M out of range");
  // 3x3 / stride 1 / pad 1: shifted-window kernel over TMA patches (no gather)
  if (T == 0 && !force_gather && ldy == Cout && Hs == Ho && Ws == Wo && patch_wgrad_applicable(Hs, Ws, C, Cin_real, Cout, KH, KW, stride, pad))
    return patch_wgrad_launch(src, dy, dw, Nimg, Hs, Ws, C, Cout, device_sm_count(), stream);
  const int terms = T == 0 ? 1 : T;
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.terms = terms;
  p.ldsrc = C * terms;
  p.dy_term = ldy;
  // Term j pairs plane A_PAT[j] of dY (column j of its activation-pattern planes) with plane B_PAT[j] of src, which
  // its activation-pattern planes hold at column perm[j] (A_PAT[perm[j]] == B_PAT[j], csrc/split.cu).
  const int perm3[3] = {0, 2, 1}, perm6[6] = {0, 2, 1, 3, 5, 4};
  for (int j = 0; j < terms; ++j) p.src_term[j] = (T == 3 ? perm3[j] : T == 6 ? perm6[j] : 0) * C;
  p.src = (const bf16*)src;
  p.dw = dw;
  p.Nimg = Nimg; p.Hs = Hs; p.Ws = Ws; p.C = C; p.Ho = Ho; p.Wo = Wo; p.KH = KH; p.KW = KW;
  p.stride = stride; p.pad = pad;
  p.M = (int)M64;
  p.Cout = Cout;
  p.Cin_real = Cin_real;
  p.fold_kw = (C == 8 && KW <= 8 && KW > 1) ? 1 : 0;
  BYOL_CHECK_ARG(p.fold_kw || C % 64 == 0 || KH * KW == 1, "byol_conv_wgrad: C=%d must be 8 (stem) or a multiple of 64", C);
  p.Cg = p.fold_kw ? 64 : gs > 0 ? 128 : C;               // grouped: one 128-wide column group (two chunks) per tap
  p.groups = p.fold_kw ? KH : KH * KW;
  const int ncols = p.groups * p.Cg;                       // concatenated (tap, channel) columns
  // (a 128 x 256 tile would need 128 accumulator registers per MMA thread: more than the register file leaves)
  const int BN = ncols > 64 ? 128 : 64;
  p.tiles_co = (Cout + 127) / 128;
  p.tiles_n = (ncols + BN - 1) / BN;
  p.kb_per_term = (p.M + WG_KROWS - 1) / WG_KROWS;
  p.num_kb_total = terms * p.kb_per_term;
  p.small_src = ((int64_t)Nimg * Hs * Ws * p.ldsrc < (1ll << 31) - (1ll << 24)) ? 1 : 0;
  const int taps = KH * KW;
  const int base_ctas = p.tiles_co * p.tiles_n;
  // Every split stores 128 x BN partials per CTA that wgrad_reduce reads back, so the split count trades
  // parallelism against reduction traffic: exactly one resident wave (one CTA per SM), rounded DOWN so that no
  // second, nearly empty wave appears.  The split count fixes the bits of dW (each split is one fp32 partial).
  const int target_ctas = device_sm_count();
  int splits = target_ctas / base_ctas;
  int max_splits = (p.num_kb_total + 7) / 8;                // at least 8 k-blocks (512 pixels) per CTA
  if (max_splits < 1) max_splits = 1;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  p.kb_per_split = (p.num_kb_total + splits - 1) / splits;
  p.splits = (p.num_kb_total + p.kb_per_split - 1) / p.kb_per_split;  // no empty split
  const int grid = base_ctas * p.splits;
  const bool b_tma = !force_gather && KH == 1 && KW == 1 && stride == 1 && pad == 0;

  BYOL_CHECK_ARG(!b_tma || C % 8 == 0, "byol_conv_wgrad: bad C");
  CUtensorMap ta, tb;
  // plain operands: the map ends at column Cout (TMA zero-fills a co tile past it); planes: all terms side by side
  const uint64_t dy_cols = T == 0 ? (uint64_t)Cout : (uint64_t)terms * ldy;
  if (tmap_2d(&ta, dy, (uint64_t)p.M, dy_cols, (uint64_t)terms * ldy, (uint32_t)WG_KROWS, 64u, "conv_wgrad dY") != 0)
    return -3;
  if (b_tma) {
    if (tmap_2d(&tb, src, (uint64_t)p.M, (uint64_t)p.ldsrc, (uint64_t)p.ldsrc, (uint32_t)WG_KROWS, 64u, "conv_wgrad X") != 0)
      return -3;
  } else {
    tb = ta;
  }
  p.ndw = (int64_t)Cout * Cin_real * taps;
  if (p.splits > 1) {
    p.part = part_scratch(stream, p.splits * p.ndw);
    if (p.part == nullptr) return -2;
  }
  const int rc = gs > 0 ? launch_wgrad<128, false, true>(ta, tb, p, grid, stream)
               : BN == 128 ? (b_tma ? launch_wgrad<128, true>(ta, tb, p, grid, stream) : launch_wgrad<128, false>(ta, tb, p, grid, stream))
                           : (b_tma ? launch_wgrad<64, true>(ta, tb, p, grid, stream) : launch_wgrad<64, false>(ta, tb, p, grid, stream));
  if (rc != 0 || p.splits == 1) return rc;
  return wgrad_reduce(p.part, p.splits, dw, p.ndw, stream);
}

// Grouped 3x3 wgrad: dw[C][Cg][KH][KW] (fp32, the real parameter, accumulated) += the in-group entries of
// dY^T x im2col(x); x [Nimg, H, W, C], dy [Nimg, Ho, Wo, C].  Nothing outside the C * Cg * 9 entries is written.
extern "C" int byol_conv_wgrad_grouped(const void* x, const void* dy, float* dw, int Nimg, int H, int W, int C, int Cg,
                                       int Ho, int Wo, int KH, int KW, int stride, int pad, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && dy && dw, "byol_conv_wgrad_grouped: null pointer");
  BYOL_CHECK_ARG(Cg >= 1 && Cg <= 64 && 64 % Cg == 0, "byol_conv_wgrad_grouped: Cg=%d must divide 64", Cg);
  if (!grouped_geometry_ok("byol_conv_wgrad_grouped", Nimg, H, W, C, Ho, Wo, KH, KW, stride, pad)) return -1;
  return conv_wgrad_impl(x, dy, dw, Nimg, H, W, C, Cg, Ho, Wo, C, C, KH, KW, stride, pad, 0, 0, stream, Cg);
}

extern "C" int byol_conv_wgrad(const void* src, const void* dy, float* dw, int Nimg, int Hs, int Ws, int C,
                               int Cin_real, int Ho, int Wo, int Cout, int ldy, int KH, int KW, int stride, int pad,
                               int force_gather, cudaStream_t stream) {
  return conv_wgrad_impl(src, dy, dw, Nimg, Hs, Ws, C, Cin_real, Ho, Wo, Cout, ldy, KH, KW, stride, pad, force_gather,
                         0, stream);
}

// fp32-accurate wgrad: dW (fp32) += sum over the T product terms of dY-plane^T x im2col(src-plane).
// src: bf16 planes [Nimg, Hs, Ws, T*C], dy: bf16 planes [Nimg, Ho, Wo, T*ldy] (both in the activation pattern of
// byol_split_planes; ldy >= Cout, a multiple of 8).  All terms accumulate into one fixed-point sum per element and
// reach dw with ONE fp32 addition per element.  Always the gather / TMA kernel (no 3x3 patch kernel); a 7x7 stem over 8 padded
// channels keeps its folded (kw, c) columns.
extern "C" int byol_conv_wgrad_planes(const void* src, const void* dy, float* dw, int Nimg, int Hs, int Ws, int C,
                                      int Cin_real, int Ho, int Wo, int Cout, int ldy, int KH, int KW, int stride,
                                      int pad, int T, cudaStream_t stream) {
  BYOL_CHECK_ARG(T == 3 || T == 6, "byol_conv_wgrad_planes: T=%d must be 3 or 6", T);
  return conv_wgrad_impl(src, dy, dw, Nimg, Hs, Ws, C, Cin_real, Ho, Wo, Cout, ldy, KH, KW, stride, pad, 0, T, stream);
}
