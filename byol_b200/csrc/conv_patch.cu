// byol_b200 — 3x3 / stride-1 / pad-1 convolution (fprop and its dgrad) with shared-memory PATCH REUSE.
//
// The implicit-GEMM kernel in conv_igemm.cu gathers a fresh A tile per filter tap, i.e. it re-reads every input
// pixel 9 times from L2 — which is what bounds the 3x3 layers.  Here each CTA TMA-loads, per 64-channel chunk, ONE
// halo patch [(TH+2) rows][W+2 cols][64 ch] of the input (4-D tensor map; the zero padding is TMA out-of-bounds
// fill) into a 128B-swizzled smem image with one 128-byte row per pixel.  With the GEMM rows enumerated as
// m = orow*(W+2) + ocol (two "garbage" columns per image row, discarded in the epilogue), the A operand of tap
// (kh, kw) is the SAME smem image shifted by (kh*(W+2) + kw) rows: the wgmma shared-memory descriptor simply starts
// (kh*(W+2)+kw)*128 bytes later.  The 128-byte swizzle is a function of the smem address bits only, so a start
// address that is 128-byte (not 1024-byte) aligned works with base_offset = 0.  Operand traffic from L2 drops from
// 9x to (TH+2)/TH x the input.
//
//   warps 0-3  : epilogue (smem accumulator tile -> regs -> bf16 -> global; fused BN column statistics through a
//                smem staging tile)
//   warps 4-11 : two MMA warpgroups (tile rows 0-63 / 64-127, accumulators of both M-tiles of a pair in registers)
//   warp 12    : TMA producer (patch ring + weight-tile ring)
// Replaces the cuDNN 3x3 conv fwd / dgrad calls reached from /root/reference/main.py:237 and main.py:617.
#include <string.h>

#include "common.cuh"

namespace byol {

struct PatchParams {
  void* dst;            // [Nimg, H, W, Ndim] bf16
  const bf16* resid;    // optional, same shape as dst
  float* col_sum;       // optional [Ndim]
  float* col_sqsum;
  Fix128* fx;        // with col_sum: [2][Ndim] fixed-point accumulators (fix_scratch)
  int Nimg, H, W, C;    // input == output spatial size (stride 1, pad 1)
  int Ndim, ldc;
  int Wp, TH, HB;       // W + 2, output rows per tile, tiles per image = ceil(H / TH)
  int tiles_n, num_tiles;   // num_tiles counts PAIR tiles: two consecutive M-tiles x one N-tile
  int num_mt;               // number of M-tiles = Nimg * HB
  int nchunks;          // C / 64
  int flip;             // 0: fprop tap shift kh*Wp + kw ; 1: dgrad (2-kh)*Wp + (2-kw)
  int relu;
  uint32_t patch_bytes; // 128 * Wp * (TH + 2)
};

static constexpr int P_PATCH_SLOT = 32768;   // bytes per patch slot (>= 128 * (128 + 2*Wp + 2))
static constexpr int P_PSTAGES = 2;          // patch GROUP stages; a group = the patches of the (up to) 2 M-tiles of a pair
static constexpr int P_BSTAGES = 2;
static constexpr int P_THREADS = 13 * 32;
static constexpr int P_ACC_LD = acc_ld(128);   // accumulator tile: [128 rows][2 M-tiles x 64 columns] fp32

__device__ __forceinline__ void tma_load_4d(uint32_t dst_smem, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst_smem), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

template <int BN>
__global__ void __launch_bounds__(P_THREADS, 1)
conv3x3_patch_kernel(const __grid_constant__ CUtensorMap tmapX, const __grid_constant__ CUtensorMap tmapB,
                     const PatchParams p) {
  constexpr int B_STAGE = BN * 128;
  constexpr int PATCH_OFF = 0;
  constexpr int B_OFF = P_PSTAGES * 2 * P_PATCH_SLOT;
  constexpr int STAGE_OUT_OFF = B_OFF + P_BSTAGES * B_STAGE;   // 4 warps x [32 rows][64 B]
  constexpr int ACC_OFF = STAGE_OUT_OFF + 4 * 2048;
  constexpr int BAR_OFF = ACC_OFF + 128 * P_ACC_LD * 4;
  static_assert(2 * BN <= 128, "the accumulator tile holds two 64-column M-tiles");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* smemP = smem + PATCH_OFF;
  uint8_t* smemB = smem + B_OFF;
  uint8_t* stage_out = smem + STAGE_OUT_OFF;
  uint64_t* pfull = (uint64_t*)(smem + BAR_OFF);
  uint64_t* pempty = pfull + P_PSTAGES;
  uint64_t* bfull = pempty + P_PSTAGES;
  uint64_t* bempty = bfull + P_BSTAGES;
  uint64_t* tfull = bempty + P_BSTAGES;   // accumulator tile ready for the epilogue
  uint64_t* tempty = tfull + 1;           // accumulator tile drained
  float* accbuf = reinterpret_cast<float*>(smem + ACC_OFF);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 12 && lane == 0) {
    for (int s = 0; s < P_PSTAGES; ++s) { mbar_init(&pfull[s], 1u); mbar_init(&pempty[s], 2u); }
    for (int s = 0; s < P_BSTAGES; ++s) { mbar_init(&bfull[s], 1u); mbar_init(&bempty[s], 2u); }
    mbar_init(tfull, 256u);
    mbar_init(tempty, 4u);
    fence_mbar_init();
    tma_prefetch_desc(&tmapX);
    tma_prefetch_desc(&tmapB);
  }
  __syncthreads();

  if (warp < 4) {
    // ======================= epilogue =====================================================
    const bool do_stats = p.col_sum != nullptr;
    const uint32_t stage_base = smem_u32(stage_out + warp * 2048);
    float csum[BN / 32], csq[BN / 32];
#pragma unroll
    for (int i = 0; i < BN / 32; ++i) { csum[i] = 0.f; csq[i] = 0.f; }
    int local = 0;
    int stat_n0 = -1;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++local) {
      const int tile_n = tile % p.tiles_n;
      const int mt0 = (tile / p.tiles_n) * 2;
      const int npair = (mt0 + 1 < p.num_mt) ? 2 : 1;
      const int n0 = tile_n * BN;
      if (do_stats && stat_n0 != n0) {
        if (stat_n0 >= 0) {
#pragma unroll
          for (int i = 0; i < BN / 32; ++i) {
            if (stat_n0 + i * 32 + lane < p.Ndim) {
              fix_add(p.fx + stat_n0 + i * 32 + lane, csum[i]);
              fix_add(p.fx + p.Ndim + stat_n0 + i * 32 + lane, csq[i]);
            }
            csum[i] = 0.f; csq[i] = 0.f;
          }
        }
        stat_n0 = n0;
      }
      mbar_wait(tfull, (uint32_t)(local & 1));
      for (int jp = 0; jp < npair; ++jp) {
      const int mt = mt0 + jp;
      const int n = mt / p.HB;
      const int h0 = (mt - n * p.HB) * p.TH;
      // GEMM row -> output pixel (rows with ocol >= W, orow >= TH or beyond the image are garbage)
      const int ml = warp * 32 + lane;
      const int orow = ml / p.Wp;
      const int ocol = ml - orow * p.Wp;
      const bool rvalid = orow < p.TH && ocol < p.W && (h0 + orow) < p.H;
      const int64_t opix = ((int64_t)n * p.H + h0 + orow) * p.W + ocol;
      const uint32_t vmask = __ballot_sync(0xffffffffu, rvalid);
#pragma unroll
      for (int ci = 0; ci < BN / 32; ++ci) {
        const int c0 = ci * 32;
        uint32_t r[32];
        acc_load_row32(accbuf + (warp * 32 + lane) * P_ACC_LD + jp * BN + c0, r);
        if (ci == BN / 32 - 1 && jp == npair - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(tempty);
        }
        const int nbase = n0 + c0;
        if (nbase >= p.Ndim) continue;  // warp-uniform
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
        if (p.resid != nullptr && rvalid) {
          const bf16* rp = p.resid + opix * p.ldc + nbase;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            if (nbase + j < p.Ndim) {
              uint4 q = *reinterpret_cast<const uint4*>(rp + j);
              const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                float2 f = __bfloat1622float2(h[e]);
                v[j + 2 * e] += f.x;
                v[j + 2 * e + 1] += f.y;
              }
            }
          }
        }
        if (p.relu) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        uint4 q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          q[j].x = pack_bf16x2(v[8 * j + 0], v[8 * j + 1]);
          q[j].y = pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
          q[j].z = pack_bf16x2(v[8 * j + 4], v[8 * j + 5]);
          q[j].w = pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
        }
        if (rvalid) {
          bf16* op = reinterpret_cast<bf16*>(p.dst) + opix * p.ldc + nbase;
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (nbase + 8 * j < p.Ndim) *reinterpret_cast<uint4*>(op + 8 * j) = q[j];
        }
        if (do_stats) {
          // stage the bf16 block (row = lane, 16-byte chunk j at j ^ ((row >> 1) & 3)) and sum valid rows per column
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint32_t off = (uint32_t)lane * 64u + (uint32_t)((j ^ ((lane >> 1) & 3)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(stage_base + off), "r"(q[j].x), "r"(q[j].y),
                         "r"(q[j].z), "r"(q[j].w)
                         : "memory");
          }
          __syncwarp();
          const uint32_t jc = (uint32_t)lane >> 3, e2 = ((uint32_t)lane & 7u) * 2u;
          uint32_t offq[4];
#pragma unroll
          for (int qq = 0; qq < 4; ++qq) offq[qq] = stage_base + ((jc ^ (uint32_t)qq) << 4) + e2;
          float s1 = 0.f, s2 = 0.f;
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            uint16_t hv;
            asm volatile("ld.shared.u16 %0, [%1];" : "=h"(hv) : "r"(offq[(rr >> 1) & 3] + (uint32_t)rr * 64u));
            float x = __uint_as_float((uint32_t)hv << 16);
            x = ((vmask >> rr) & 1u) ? x : 0.f;
            s1 += x;
            s2 = fmaf(x, x, s2);
          }
          csum[ci] += s1;
          csq[ci] += s2;
        }
      }
      }   // jp
    }
    if (do_stats && stat_n0 >= 0) {
#pragma unroll
      for (int i = 0; i < BN / 32; ++i) {
        if (stat_n0 + i * 32 + lane < p.Ndim) {
          fix_add(p.fx + stat_n0 + i * 32 + lane, csum[i]);
          fix_add(p.fx + p.Ndim + stat_n0 + i * 32 + lane, csq[i]);
        }
      }
    }
  } else if (warp < 12) {
    // ======================= MMA warpgroups ===============================================
    // warpgroup wg: tile rows 64*wg .. +63 = the patch image 64 rows (8 KB) further on
    const int wg = (warp - 4) >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    float d[2][BN / 2];
    int pit = 0, bit = 0, local = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++local) {
      const int mt0 = (tile / p.tiles_n) * 2;
      const int npair = (mt0 + 1 < p.num_mt) ? 2 : 1;
      for (int cc = 0; cc < p.nchunks; ++cc, ++pit) {
        const int ps = pit % P_PSTAGES;
        mbar_wait(&pfull[ps], (uint32_t)((pit / P_PSTAGES) & 1));
        const uint32_t patch = smem_u32(smemP + ps * 2 * P_PATCH_SLOT) + (uint32_t)wg * 8192u;
        int prev_bs = -1;
        for (int tap = 0; tap < 9; ++tap, ++bit) {
          const int bs = bit % P_BSTAGES;
          mbar_wait(&bfull[bs], (uint32_t)((bit / P_BSTAGES) & 1));
          const int kh = tap / 3, kw = tap - kh * 3;
          const int shift = p.flip ? ((2 - kh) * p.Wp + (2 - kw)) : (kh * p.Wp + kw);
          const uint64_t bdesc = make_smem_desc_sw128(smem_u32(smemB + bs * B_STAGE), 16, 1024);
          wg_fence();
          // the same weight tile multiplies the patches of both M-tiles of the pair.  Both are always issued (a branch
          // around wgmma makes ptxas serialise every MMA); for a single-tile pair the second result is discarded.
#pragma unroll
          for (int jp = 0; jp < 2; ++jp) {
            // shifted window over the swizzled patch image: start address only 128-byte aligned, base_offset 0
            const uint64_t adesc =
                make_smem_desc_sw128(patch + (uint32_t)jp * P_PATCH_SLOT + (uint32_t)shift * 128u, 16, 1024);
#pragma unroll
            for (int k = 0; k < 4; ++k)
              wgmma_bf16<BN, 0, 0>(d[jp], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k),
                                   (uint32_t)((cc | tap | k) != 0));
          }
          wg_commit();
          wg_wait<1>();   // the previous tap's MMAs are done with their weight stage
          if (leader && prev_bs >= 0) mbar_arrive(&bempty[prev_bs]);
          prev_bs = bs;
        }
        wg_wait<0>();
        if (leader) {
          mbar_arrive(&bempty[prev_bs]);
          mbar_arrive(&pempty[ps]);
        }
      }
      wg_fence_acc(d[0]);
      wg_fence_acc(d[1]);
      mbar_wait(tempty, (uint32_t)((local & 1) ^ 1));
      acc_store_smem<BN>(accbuf, P_ACC_LD, wg * 64, 0, d[0]);
      if (npair == 2) acc_store_smem<BN>(accbuf, P_ACC_LD, wg * 64, BN, d[1]);
      mbar_arrive(tfull);
    }
  } else {
    // ======================= TMA producer =================================================
    // Flat loop over this CTA's (tile, channel-chunk) pairs.  The patch of the NEXT pair is requested while the
    // weight tiles of the current pair are still streaming (at tap 4: by then the MMA warp has certainly left the
    // pair that previously occupied that patch slot, so the wait on pempty cannot stall the weight stream).
    if (lane == 0) {
      const int my_tiles = (p.num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
      const int total = my_tiles * p.nchunks;
      auto issue_patch = [&](int g) {
        const int tile = blockIdx.x + (g / p.nchunks) * gridDim.x;
        const int cc = g % p.nchunks;
        const int mt0 = (tile / p.tiles_n) * 2;
        const int npair = (mt0 + 1 < p.num_mt) ? 2 : 1;
        const int ps = g % P_PSTAGES;
        mbar_wait(&pempty[ps], (uint32_t)(((g / P_PSTAGES) & 1) ^ 1));
        mbar_arrive_expect_tx(&pfull[ps], p.patch_bytes * (uint32_t)npair);
        for (int jp = 0; jp < npair; ++jp) {
          const int mt = mt0 + jp;
          const int n = mt / p.HB;
          const int h0 = (mt - n * p.HB) * p.TH;
          tma_load_4d(smem_u32(smemP + (ps * 2 + jp) * P_PATCH_SLOT), &tmapX, &pfull[ps], cc * 64, -1, h0 - 1, n);
        }
      };
      int bit = 0;
      if (total > 0) issue_patch(0);
      for (int g = 0; g < total; ++g) {
        const int tile = blockIdx.x + (g / p.nchunks) * gridDim.x;
        const int cc = g % p.nchunks;
        const int n0 = (tile % p.tiles_n) * BN;
        for (int tap = 0; tap < 9; ++tap, ++bit) {
          if (tap == 4 && g + 1 < total) issue_patch(g + 1);
          const int bs = bit % P_BSTAGES;
          mbar_wait(&bempty[bs], (uint32_t)(((bit / P_BSTAGES) & 1) ^ 1));
          mbar_arrive_expect_tx(&bfull[bs], (uint32_t)B_STAGE);
          tma_load_2d(smem_u32(smemB + bs * B_STAGE), &tmapB, &bfull[bs], (tap * p.nchunks + cc) * 64, n0);
        }
      }
    }
    __syncwarp();
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled patch_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = (PFN_encodeTiled)ptr;
  }
  return fn;
}

template <int BN>
static int launch_patch(const CUtensorMap& tx, const CUtensorMap& tb, const PatchParams& p, int sms,
                        cudaStream_t stream) {
  constexpr int SMEM = P_PSTAGES * 2 * P_PATCH_SLOT + P_BSTAGES * BN * 128 + 4 * 2048 + 128 * P_ACC_LD * 4 + 256 + 1024;
  static_assert(SMEM <= 232448, "conv3x3_patch_kernel: shared memory");
  auto kern = conv3x3_patch_kernel<BN>;
  static bool attr_set[kMaxDevices] = {};
  const int dev_slot = device_slot();
  if (!attr_set[dev_slot]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(conv3x3_patch) failed: %s", cudaGetErrorString(e));
      return -2;
    }
    attr_set[dev_slot] = true;
  }
  int grid = sms < p.num_tiles ? sms : p.num_tiles;
  kern<<<grid, P_THREADS, SMEM, stream>>>(tx, tb, p);
  return check_launch("conv3x3_patch_kernel");
}

// Is the patch formulation applicable / worthwhile for this geometry?
bool patch_conv_applicable(int H, int W, int C, int Ndim, int KH, int KW, int stride, int pad, int out_fp32,
                           const float* bias, int64_t src_elems) {
  if (KH != 3 || KW != 3 || stride != 1 || pad != 1 || out_fp32 || bias != nullptr) return false;
  if (C % 64 != 0 || Ndim % 8 != 0) return false;
  const int Wp = W + 2;
  // at 14x14 and below few of the 128 tile rows are valid: the gather kernel is used there
  if (Wp > 128 || W < 12) return false;
  const int TH = 128 / Wp;
  if (128 * (128 + 2 * Wp + 2) > P_PATCH_SLOT) return false;
  if (128 * Wp * (TH + 2) > P_PATCH_SLOT) return false;
  (void)H; (void)src_elems;
  return true;
}

// src: NHWC [Nimg,H,W,C]; wt: [Ndim][9*C] K-major (k = tap*C + c); dst: [Nimg,H,W,Ndim] bf16
int patch_conv_launch(const void* src, const void* wt, void* dst, const void* resid, float* col_sum, float* col_sqsum,
                      int Nimg, int H, int W, int C, int Ndim, int ldw, int ldc, int flip, int relu, int sms,
                      cudaStream_t stream) {
  PFN_encodeTiled fn = patch_encode_fn();
  if (fn == nullptr) { set_last_error("cuTensorMapEncodeTiled entry point unavailable"); return -3; }
  PatchParams p;
  memset(&p, 0, sizeof(p));
  p.dst = dst; p.resid = (const bf16*)resid; p.col_sum = col_sum; p.col_sqsum = col_sqsum;
  p.Nimg = Nimg; p.H = H; p.W = W; p.C = C; p.Ndim = Ndim; p.ldc = ldc;
  p.Wp = W + 2;
  p.TH = 128 / p.Wp;
  if (p.TH > H) p.TH = H;
  p.HB = (H + p.TH - 1) / p.TH;
  // 64 columns: the accumulators of both M-tiles of a pair (2 x 64 x BN per warpgroup) must fit in registers
  const int BN = 64;
  p.tiles_n = (Ndim + BN - 1) / BN;
  p.num_mt = Nimg * p.HB;
  p.num_tiles = ((p.num_mt + 1) / 2) * p.tiles_n;
  p.nchunks = C / 64;
  p.flip = flip;
  p.relu = relu;
  p.patch_bytes = 128u * (uint32_t)p.Wp * (uint32_t)(p.TH + 2);

  CUtensorMap tx, tb;
  {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)Nimg};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {64u, (cuuint32_t)p.Wp, (cuuint32_t)(p.TH + 2), 1u};
    cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult r = fn(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(src), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("patch conv: 4-D tensor map encode failed (%d)", (int)r); return -3; }
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)(9 * C), (cuuint64_t)Ndim};
    cuuint64_t strides[1] = {(cuuint64_t)ldw * 2};
    cuuint32_t box[2] = {64u, (cuuint32_t)BN};
    cuuint32_t estr[2] = {1u, 1u};
    CUresult r = fn(&tb, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(wt), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("patch conv: weight tensor map encode failed (%d)", (int)r); return -3; }
  }
  if (col_sum != nullptr) {
    p.fx = fix_scratch(stream, 2 * (int64_t)Ndim);
    if (p.fx == nullptr) return -2;
  }
  int rc = launch_patch<64>(tx, tb, p, sms, stream);
  if (rc != 0 || col_sum == nullptr) return rc;
  if ((rc = fix_flush(p.fx, col_sum, Ndim, stream)) != 0) return rc;
  return fix_done(stream, fix_flush(p.fx + Ndim, col_sqsum, Ndim, stream));
}

}  // namespace byol

// =================================================================================================
// 3x3 / stride-1 / pad-1 WGRAD with the same shifted-window trick.
//   dW[co, ci, kh, kw] += sum_pixels dY[pix, co] * X[pix + (kh-1, kw-1), ci]
// Per M-tile (TH image rows, GEMM K rows = orow*(W+2)+ocol, 128 of them):
//   A = dY tile  [128 pixel rows][128 co]  MN-major, TMA box {64 co, W+2, TH, 1}: the two garbage columns and rows
//       beyond the image are out-of-bounds -> ZERO, so garbage rows contribute nothing
//   B = X patch  [(TH+2)*(W+2) pixel rows][64*NB ci] MN-major; tap (kh,kw) = the same image shifted by kh*(W+2)+kw rows
//   D[128 co][kw*64*NB + ci] for the three taps of ONE kh row per CTA, accumulated in the registers of two MMA
//   warpgroups (co rows 0-63 / 64-127; warps 0-7) over the CTA's range of M-tiles, then added to the fp32 gradient
//   with L2 reductions.  Warp 8 is the TMA producer.
// Rows of the smem slots that TMA never writes (beyond the boxes) are zeroed once, so stale shared memory can not
// inject Inf/NaN through the zero rows of A.
// =================================================================================================
namespace byol {

struct WPatchParams {
  float* dw;            // [Cout][Cin][3][3] fp32
  Fix128* fx;        // fixed-point accumulators over the whole dw (fix_scratch)
  int Nimg, H, W, C, Cout;
  int Wp, TH, HB, num_mt;
  int co_tiles, ci_groups;
  int splits, mt_per_split;
  uint32_t patch_bytes; // 128 * Wp * (TH + 2)
  uint32_t dy_bytes;    // 128 * Wp * TH
};

static constexpr int WP_STAGES = 2;

static constexpr int WP_THREADS = 9 * 32;

template <int NB>
__global__ void __launch_bounds__(WP_THREADS, 1)
conv3x3_wgrad_patch_kernel(const __grid_constant__ CUtensorMap tmapX, const __grid_constant__ CUtensorMap tmapDY,
                           const WPatchParams p) {
  constexpr int X_STAGE = NB * P_PATCH_SLOT;
  constexpr int DY_STAGE = 2 * 16384;
  constexpr int DY_OFF = WP_STAGES * X_STAGE;
  constexpr int BAR_OFF = DY_OFF + WP_STAGES * DY_STAGE;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* smemX = smem;
  uint8_t* smemDY = smem + DY_OFF;
  uint64_t* full_bar = (uint64_t*)(smem + BAR_OFF);
  uint64_t* empty_bar = full_bar + WP_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int bid = blockIdx.x;
  const int kh = bid % 3;               bid /= 3;
  const int cig = bid % p.ci_groups;    bid /= p.ci_groups;
  const int tile_co = bid % p.co_tiles; bid /= p.co_tiles;
  const int split = bid;
  const int co0 = tile_co * 128;
  const int ci0 = cig * 64 * NB;
  const int mt_begin = split * p.mt_per_split;
  int mt_end = mt_begin + p.mt_per_split;
  if (mt_end > p.num_mt) mt_end = p.num_mt;
  const int ntiles = mt_end - mt_begin;   // host guarantees >= 1

  // zero every operand slot once (see header comment)
  for (int i = threadIdx.x; i < BAR_OFF / 16; i += blockDim.x) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_smem();
  if (warp == 8 && lane == 0) {
    for (int s = 0; s < WP_STAGES; ++s) { mbar_init(&full_bar[s], 1u); mbar_init(&empty_bar[s], 2u); }
    fence_mbar_init();
    tma_prefetch_desc(&tmapX);
    tma_prefetch_desc(&tmapDY);
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      for (int it = 0; it < ntiles; ++it) {
        const int mt = mt_begin + it;
        const int n = mt / p.HB;
        const int h0 = (mt - n * p.HB) * p.TH;
        const int s = it % WP_STAGES;
        mbar_wait(&empty_bar[s], (uint32_t)(((it / WP_STAGES) & 1) ^ 1));
        mbar_arrive_expect_tx(&full_bar[s], (uint32_t)NB * p.patch_bytes + 2u * p.dy_bytes);
#pragma unroll
        for (int c = 0; c < NB; ++c)
          tma_load_4d(smem_u32(smemX + s * X_STAGE + c * P_PATCH_SLOT), &tmapX, &full_bar[s], ci0 + 64 * c, -1, h0 - 1, n);
#pragma unroll
        for (int j = 0; j < 2; ++j)
          tma_load_4d(smem_u32(smemDY + s * DY_STAGE + j * 16384), &tmapDY, &full_bar[s], co0 + 64 * j, 0, h0, n);
      }
    }
    __syncwarp();
  } else {
    const int wg = warp >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    float d[3][32 * NB];
    int prev_s = -1;
    for (int it = 0; it < ntiles; ++it) {
      const int s = it % WP_STAGES;
      mbar_wait(&full_bar[s], (uint32_t)((it / WP_STAGES) & 1));
      const uint32_t a_base = smem_u32(smemDY + s * DY_STAGE) + (uint32_t)wg * 16384u;   // this warpgroup's 64 co
      const uint32_t x_base = smem_u32(smemX + s * X_STAGE);
      wg_fence();
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const uint32_t shift = (uint32_t)(kh * p.Wp + kw) * 128u;
        // A: co chunks 16384 B apart; B: NB ci chunks P_PATCH_SLOT apart; 8-row groups 1024 B apart
        const uint64_t adesc = make_smem_desc_sw128(a_base, 16384, 1024);
        const uint64_t bdesc = make_smem_desc_sw128(x_base + shift, P_PATCH_SLOT, 1024);
#pragma unroll
        for (int k = 0; k < 8; ++k)   // 16 pixel rows = 2048 bytes per step
          wgmma_bf16<64 * NB, 1, 1>(d[kw], adesc + (uint64_t)(128 * k), bdesc + (uint64_t)(128 * k),
                                    (uint32_t)((it | k) != 0));
      }
      wg_commit();
      wg_wait<1>();
      if (leader && prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
    }
    wg_wait<0>();
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) wg_fence_acc(d[kw]);
    // ---------------- epilogue: registers -> L2 reductions into dW[co][ci][kh][kw] ----------------
    const int t = threadIdx.x & 127;
    const int r0 = co0 + wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
#pragma unroll
      for (int i = 0; i < 32 * NB; ++i) {
        const int co = r0 + ((i & 2) ? 8 : 0);
        const int ci = ci0 + 8 * (i >> 2) + 2 * (t & 3) + (i & 1);
        if (co < p.Cout && ci < p.C) fix_add(p.fx + ((int64_t)co * p.C + ci) * 9 + kh * 3 + kw, d[kw][i]);
      }
    }
  }
}

template <int NB>
static int launch_wpatch(const CUtensorMap& tx, const CUtensorMap& ty, const WPatchParams& p, int grid,
                         cudaStream_t stream) {
  constexpr int SMEM = WP_STAGES * (NB * P_PATCH_SLOT + 2 * 16384) + 256 + 1024;
  auto kern = conv3x3_wgrad_patch_kernel<NB>;
  static bool attr_set[kMaxDevices] = {};
  const int dev_slot = device_slot();
  if (!attr_set[dev_slot]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(conv3x3_wgrad_patch) failed: %s", cudaGetErrorString(e));
      return -2;
    }
    attr_set[dev_slot] = true;
  }
  kern<<<grid, WP_THREADS, SMEM, stream>>>(tx, ty, p);
  return check_launch("conv3x3_wgrad_patch_kernel");
}

bool patch_wgrad_applicable(int H, int W, int C, int Cin_real, int Cout, int KH, int KW, int stride, int pad) {
  if (KH != 3 || KW != 3 || stride != 1 || pad != 1) return false;
  if (C % 64 != 0 || C != Cin_real || Cout % 8 != 0) return false;
  const int Wp = W + 2;
  if (Wp > 128 || W < 12) return false;
  if (128 * (128 + 2 * Wp + 2) > P_PATCH_SLOT) return false;
  (void)H;
  return true;
}

// x: NHWC [Nimg,H,W,C]; dy: [Nimg,H,W,Cout]; dw: fp32 [Cout][C][3][3] (accumulated)
int patch_wgrad_launch(const void* x, const void* dy, float* dw, int Nimg, int H, int W, int C, int Cout, int sms,
                       cudaStream_t stream) {
  PFN_encodeTiled fn = patch_encode_fn();
  if (fn == nullptr) { set_last_error("cuTensorMapEncodeTiled entry point unavailable"); return -3; }
  WPatchParams p;
  memset(&p, 0, sizeof(p));
  p.dw = dw; p.Nimg = Nimg; p.H = H; p.W = W; p.C = C; p.Cout = Cout;
  p.Wp = W + 2;
  p.TH = 128 / p.Wp;
  if (p.TH > H) p.TH = H;
  p.HB = (H + p.TH - 1) / p.TH;
  p.num_mt = Nimg * p.HB;
  // one 64-channel chunk per CTA: 3 taps x 64 x 64 accumulators per warpgroup already take 96 registers per thread
  constexpr int NB = 1;
  p.co_tiles = (Cout + 127) / 128;
  p.ci_groups = C / (64 * NB);
  const int base = p.co_tiles * p.ci_groups * 3;
  int splits = sms / base;
  if (splits < 1) splits = 1;
  if (splits > p.num_mt) splits = p.num_mt;
  p.mt_per_split = (p.num_mt + splits - 1) / splits;
  p.splits = (p.num_mt + p.mt_per_split - 1) / p.mt_per_split;
  p.patch_bytes = 128u * (uint32_t)p.Wp * (uint32_t)(p.TH + 2);
  p.dy_bytes = 128u * (uint32_t)p.Wp * (uint32_t)p.TH;
  CUtensorMap tx, ty;
  for (int which = 0; which < 2; ++which) {
    const int ch = which == 0 ? C : Cout;
    cuuint64_t dims[4] = {(cuuint64_t)ch, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)Nimg};
    cuuint64_t strides[3] = {(cuuint64_t)ch * 2, (cuuint64_t)W * ch * 2, (cuuint64_t)H * W * ch * 2};
    cuuint32_t box[4] = {64u, (cuuint32_t)p.Wp, (cuuint32_t)(which == 0 ? p.TH + 2 : p.TH), 1u};
    cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult r = fn(which == 0 ? &tx : &ty, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                    const_cast<void*>(which == 0 ? x : dy), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("patch wgrad: tensor map encode failed (%d)", (int)r); return -3; }
  }
  const int grid = base * p.splits;
  const int64_t ndw = (int64_t)Cout * C * 9;
  p.fx = fix_scratch(stream, ndw);
  if (p.fx == nullptr) return -2;
  const int rc = launch_wpatch<NB>(tx, ty, p, grid, stream);
  return fix_done(stream, rc != 0 ? rc : fix_flush(p.fx, dw, ndw, stream));
}

}  // namespace byol
