// byol_b200 — BatchNorm (train-mode, optionally cross-rank) kernels over NHWC bf16 activations.
//
// Replaces the ATen/cuDNN batch_norm and SyncBatchNorm kernels reached from
// /root/reference/main.py:237-239 (BatchNorm2d x53 in the encoder, BatchNorm1d(4096) in head / predictor,
// main.py:196,202) and main.py:433 (SyncBatchNorm; math in torch/nn/modules/_functions.py:10-205).
//
// Forward is split so that a cross-rank reduction of the raw sums can sit between the two halves:
//   bn_stats     : per-channel sum / sum of squares over the rows of x            (HBM-bound, 2 B/elem)
//   [all-reduce of the 2C sums across ranks when SyncBN is on]
//   bn_finalize  : mean / invstd / (scale, shift), running-stat update            (tiny)
//   bn_apply     : y = relu(x*scale + shift (+ resid | resid*rscale + rshift))    (HBM-bound)
// Backward likewise:
//   bn_bwd_reduce: s1 = sum dz, s2 = sum dz * xhat  (dz = g masked by ReLU)       (HBM-bound)
//   [all-reduce of s1, s2 across ranks when SyncBN is on]
//   bn_bwd_apply : dy = gamma*invstd*(dz - s1/n - xhat*s2/n)  (optionally also writes dz)
#include "common.cuh"

namespace byol {

// ---------------------------------------------------------------------------------------------
// column statistics: x [M, C] bf16 (C % 8 == 0).  Each thread owns one 8-channel group and strides
// over rows; a block covers ROWS_PER_BLOCK rows.  Partial sums are combined with fp32 atomics.
// ---------------------------------------------------------------------------------------------
__global__ void bn_stats_kernel(const bf16* __restrict__ x, Fix128* __restrict__ sum, Fix128* __restrict__ sqsum,
                                int M, int C, int rows_per_block) {
  extern __shared__ Fix128 red[];               // [2][C] block-level partial sums (fixed point)
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) red[c] = Fix128{0ull, 0ll, 0.0};
  __syncthreads();
  const int groups = C >> 3;                       // 8-channel groups per row
  const int tpr = groups < (int)blockDim.x ? groups : (int)blockDim.x;  // threads used per row pass
  const int row_lanes = blockDim.x / tpr;          // rows processed concurrently by the block
  const int g_in = threadIdx.x % tpr;
  const int rlane = threadIdx.x / tpr;
  const int row_begin = blockIdx.x * rows_per_block;
  int row_end = row_begin + rows_per_block;
  if (row_end > M) row_end = M;
  if (rlane < row_lanes) {
    for (int g = g_in; g < groups; g += tpr) {
      float s[8], q[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) { s[e] = 0.f; q[e] = 0.f; }
      for (int r = row_begin + rlane; r < row_end; r += row_lanes) {
        uint4 v = __ldg(reinterpret_cast<const uint4*>(x + (int64_t)r * C + g * 8));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __bfloat1622float2(h[e]);
          s[2 * e] += f.x; q[2 * e] += f.x * f.x;
          s[2 * e + 1] += f.y; q[2 * e + 1] += f.y * f.y;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        fix_add(red + g * 8 + e, s[e]);
        fix_add(red + C + g * 8 + e, q[e]);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    fix_add_raw(sum + c, red[c]);
    fix_add_raw(sqsum + c, red[C + c]);
  }
}

// Statistics -> coefficients for up to 4 "lanes" (forward passes that ran this layer in lock-step, each with its own gamma/beta set and
// its own batch statistics) in ONE launch; the running statistics are updated lane after lane, i.e. in the order
// the reference's four sequential forward passes would update them (main.py:244-247).
struct LanePtrs { const float* p[4]; };
__global__ void bn_finalize_lanes_kernel(const float* __restrict__ stats, double count, LanePtrs gamma, LanePtrs beta,
                                         float* __restrict__ running_mean, float* __restrict__ running_var,
                                         float momentum, float eps, float* __restrict__ coeffs, int C, int L) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float rm = running_mean != nullptr ? running_mean[c] : 0.f;
  float rv = running_var != nullptr ? running_var[c] : 0.f;
  for (int l = 0; l < L; ++l) {
    const float* st = stats + (int64_t)l * 2 * C;
    double mean = (double)st[c] / count;
    double var = (double)st[C + c] / count - mean * mean;   // biased
    if (var < 0.0) var = 0.0;
    float invstd = (float)(1.0 / sqrt(var + (double)eps));
    float sc = gamma.p[l][c] * invstd;
    float* co = coeffs + (int64_t)l * 4 * C;
    co[c] = sc;
    co[C + c] = beta.p[l][c] - (float)mean * sc;
    co[2 * C + c] = (float)mean;
    co[3 * C + c] = invstd;
    double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    rm = (1.f - momentum) * rm + momentum * (float)mean;
    rv = (1.f - momentum) * rv + momentum * (float)unbiased;
  }
  if (running_mean != nullptr) {
    running_mean[c] = rm;
    running_var[c] = rv;
  }
}

// eval mode: scale/shift from running statistics
__global__ void bn_eval_coeffs_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                                      const float* __restrict__ running_mean, const float* __restrict__ running_var,
                                      float eps, float* __restrict__ scale, float* __restrict__ shift, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float invstd = 1.f / sqrtf(running_var[c] + eps);
  float sc = gamma[c] * invstd;
  scale[c] = sc;
  shift[c] = beta[c] - running_mean[c] * sc;
}

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float2 t = __bfloat1622float2(h[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 q;
  q.x = pack_bf16x2(f[0], f[1]);
  q.y = pack_bf16x2(f[2], f[3]);
  q.z = pack_bf16x2(f[4], f[5]);
  q.w = pack_bf16x2(f[6], f[7]);
  return q;
}

// bit e = (o[e] > 0): the ReLU mask of one 8-channel vector (one byte per vector, same linear order as the data)
__device__ __forceinline__ uint8_t positive_bits(const float* o) {
  uint32_t b = 0;
#pragma unroll
  for (int e = 0; e < 8; ++e) b |= (o[e] > 0.f ? 1u : 0u) << e;
  return (uint8_t)b;
}

// y = act(x*scale + shift + residual);  residual = resid (rscale == null) or resid*rscale + rshift
// Each thread handles one 8-channel vector; grid-stride over M*C/8 vectors.
__global__ void bn_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ scale,
                                const float* __restrict__ shift, const bf16* __restrict__ resid,
                                const float* __restrict__ rscale, const float* __restrict__ rshift,
                                bf16* __restrict__ y, float* __restrict__ y_f32, uint8_t* __restrict__ mask_out,
                                int64_t nvec, int C, int relu) {
  const int groups = C >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    float xv[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x) + i), xv);
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + g * 8));
    const float4 s1 = __ldg(reinterpret_cast<const float4*>(scale + g * 8 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(shift + g * 8));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(shift + g * 8 + 4));
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float sh[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = xv[e] * sc[e] + sh[e];
    if (resid != nullptr) {
      float rv[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(resid) + i), rv);
      if (rscale != nullptr) {
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] += rv[e] * __ldg(rscale + g * 8 + e) + __ldg(rshift + g * 8 + e);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] += rv[e];
      }
    }
    if (relu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = fmaxf(o[e], 0.f);
    }
    if (y != nullptr) reinterpret_cast<uint4*>(y)[i] = pack8(o);
    if (mask_out != nullptr) mask_out[i] = positive_bits(o);
    if (y_f32 != nullptr) {
      reinterpret_cast<float4*>(y_f32)[2 * i] = make_float4(o[0], o[1], o[2], o[3]);
      reinterpret_cast<float4*>(y_f32)[2 * i + 1] = make_float4(o[4], o[5], o[6], o[7]);
    }
  }
}

// Vectors in flight per thread of bn_apply_fixed_kernel<*, false>: each thread loads the 16-byte vectors i, i + T,
// ..., i + (kFixedVecs - 1) T of the grid's T threads (every operand) before any arithmetic, so each warp still reads
// and writes 512 contiguous bytes per vector and each thread stays on one channel group.  Its grid is at most one wave
// of resident blocks (fixed_wave_grid).
static constexpr int kFixedVecs = 4;

// Same as bn_apply_kernel, for launches where (gridDim.x * blockDim.x) % (C/8) == 0: every thread then stays on
// ONE 8-channel group for its whole grid-stride loop and keeps the per-channel coefficients in registers
// (the generic kernel re-loads them per vector, which makes it LSU-bound rather than HBM-bound).
// <true, true> (block outputs with a downsample-BN residual) already ran at 85 % of the HBM bound with one vector per
// thread and the fixed_grid launch, and kFixedVecs vectors on one wave did not make it faster: it keeps that schedule.
template <bool RESID, bool RAFFINE>
__global__ void __launch_bounds__(256)
bn_apply_fixed_kernel(const bf16* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ shift,
                      const bf16* __restrict__ resid, const float* __restrict__ rscale,
                      const float* __restrict__ rshift, bf16* __restrict__ y, uint8_t* __restrict__ mask_out,
                      int64_t nvec, int C, int relu) {
  const int groups = C >> 3;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int g = (int)(tid % groups);
  float sc[8], sh[8], rs[8], rb[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    sc[e] = scale[g * 8 + e];
    sh[e] = shift[g * 8 + e];
    rs[e] = RAFFINE ? rscale[g * 8 + e] : 1.f;
    rb[e] = RAFFINE ? rshift[g * 8 + e] : 0.f;
  }
  constexpr int V = RAFFINE ? 1 : kFixedVecs;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < nvec; i += V * stride) {
    uint4 xq[V], rq[V];
#pragma unroll
    for (int u = 0; u < V; ++u) {
      const int64_t j = i + u * stride;
      const bool ok = j < nvec;
      xq[u] = ok ? __ldg(reinterpret_cast<const uint4*>(x) + j) : make_uint4(0u, 0u, 0u, 0u);
      if (RESID) rq[u] = ok ? __ldg(reinterpret_cast<const uint4*>(resid) + j) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < V; ++u) {
      const int64_t j = i + u * stride;
      if (j < nvec) {
        float xv[8], o[8];
        unpack8(xq[u], xv);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = xv[e] * sc[e] + sh[e];
        if (RESID) {
          float rv[8];
          unpack8(rq[u], rv);
#pragma unroll
          for (int e = 0; e < 8; ++e) o[e] += RAFFINE ? (rv[e] * rs[e] + rb[e]) : rv[e];
        }
        if (relu) {
#pragma unroll
          for (int e = 0; e < 8; ++e) o[e] = fmaxf(o[e], 0.f);
        }
        reinterpret_cast<uint4*>(y)[j] = pack8(o);
        if (mask_out != nullptr) mask_out[j] = positive_bits(o);
      }
    }
  }
}

// dy = A*dz + B*x + Cc with per-channel A = gamma*invstd, B = -gamma*invstd^2*s2/n,
// Cc = gamma*invstd*(mean*invstd*s2/n - s1/n); same thread <-> channel-group pinning as bn_apply_fixed_kernel.
template <int MASK>
__global__ void __launch_bounds__(256)
bn_bwd_apply_fixed_kernel(const bf16* __restrict__ g, const bf16* __restrict__ x, const bf16* __restrict__ act,
                          const float* __restrict__ scale, const float* __restrict__ shift,
                          const float* __restrict__ mean, const float* __restrict__ invstd,
                          const float* __restrict__ gamma, const float* __restrict__ s1,
                          const float* __restrict__ s2, float inv_count, bf16* __restrict__ dy,
                          bf16* __restrict__ dz_out, int64_t nvec, int C, const float* __restrict__ s1_local,
                          const float* __restrict__ s2_local, float* __restrict__ dgamma,
                          float* __restrict__ dbeta) {
  const int groups = C >> 3;
  if (blockIdx.x == 0 && dgamma != nullptr) {
    // atomics: the two online views may run concurrently; each adds once per element to the zeroed gradient, and two
    // additions onto zero give the same bits in either order
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      atomicAdd(dgamma + c, s2_local[c]);
      atomicAdd(dbeta + c, s1_local[c]);
    }
  }
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int gi = (int)(tid % groups);
  float A[8], B[8], Cc[8], sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = gi * 8 + e;
    const float is = invstd[c], mu = mean[c], ga = gamma[c];
    const float m1 = s1[c] * inv_count, m2 = s2[c] * inv_count;
    A[e] = ga * is;
    B[e] = -ga * is * is * m2;
    Cc[e] = ga * is * (mu * is * m2 - m1);
    sc[e] = MASK == 1 ? scale[c] : 0.f;
    sh[e] = MASK == 1 ? shift[c] : 0.f;
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < nvec; i += stride) {
    float gv[8], xv[8], o[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(g) + i), gv);
    unpack8(__ldg(reinterpret_cast<const uint4*>(x) + i), xv);
    if (MASK == 3) {
      const uint32_t mb = __ldg(reinterpret_cast<const uint8_t*>(act) + i);
#pragma unroll
      for (int e = 0; e < 8; ++e) gv[e] = ((mb >> e) & 1u) ? gv[e] : 0.f;
    } else if (MASK == 2) {
      float av[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(act) + i), av);
#pragma unroll
      for (int e = 0; e < 8; ++e) gv[e] = av[e] > 0.f ? gv[e] : 0.f;
    } else if (MASK == 1) {
#pragma unroll
      for (int e = 0; e < 8; ++e) gv[e] = (xv[e] * sc[e] + sh[e]) > 0.f ? gv[e] : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = A[e] * gv[e] + (B[e] * xv[e] + Cc[e]);
    reinterpret_cast<uint4*>(dy)[i] = pack8(o);
    if (dz_out != nullptr) reinterpret_cast<uint4*>(dz_out)[i] = pack8(gv);
  }
}

// mask_mode: 0 = none (dz = g), 1 = ReLU mask recomputed from x (x*scale+shift > 0), 2 = mask from act > 0,
// 3 = mask bits written by bn_apply (`act` = uint8 [M*C/8], bit e of byte i = element 8*i + e)
template <int MASK>
__global__ void bn_bwd_reduce_kernel(const bf16* __restrict__ g, const bf16* __restrict__ x,
                                     const bf16* __restrict__ act, const float* __restrict__ scale,
                                     const float* __restrict__ shift, const float* __restrict__ mean,
                                     const float* __restrict__ invstd, Fix128* __restrict__ s1,
                                     Fix128* __restrict__ s2, int M, int C, int rows_per_block) {
  extern __shared__ Fix128 red[];                   // [2][C]
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) red[c] = Fix128{0ull, 0ll, 0.0};
  __syncthreads();
  const int groups = C >> 3;
  const int tpr = groups < (int)blockDim.x ? groups : (int)blockDim.x;
  const int row_lanes = blockDim.x / tpr;
  const int g_in = threadIdx.x % tpr;
  const int rlane = threadIdx.x / tpr;
  const int row_begin = blockIdx.x * rows_per_block;
  int row_end = row_begin + rows_per_block;
  if (row_end > M) row_end = M;
  for (int gi = g_in; gi < groups && rlane < row_lanes; gi += tpr) {
    float a1[8], a2[8], mu[8], is[8], sc[8], sh[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      a1[e] = 0.f; a2[e] = 0.f;
      mu[e] = mean[gi * 8 + e];
      is[e] = invstd[gi * 8 + e];
      sc[e] = MASK == 1 ? scale[gi * 8 + e] : 0.f;
      sh[e] = MASK == 1 ? shift[gi * 8 + e] : 0.f;
    }
    // four rows per iteration, all loads issued before the arithmetic (memory-level parallelism: the loop carries
    // only the accumulators); rows past the end contribute zeros
    for (int r = row_begin + rlane; r < row_end; r += 4 * row_lanes) {
      uint4 gq[4], xq[4], aq[4];
      uint32_t mb[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int rr = r + u * row_lanes;
        const bool ok = rr < row_end;
        const int64_t off = ((int64_t)(ok ? rr : r) * C + gi * 8) >> 3;
        gq[u] = ok ? __ldg(reinterpret_cast<const uint4*>(g) + off) : make_uint4(0u, 0u, 0u, 0u);
        xq[u] = __ldg(reinterpret_cast<const uint4*>(x) + off);
        if (MASK == 3) mb[u] = __ldg(reinterpret_cast<const uint8_t*>(act) + off);
        if (MASK == 2) aq[u] = __ldg(reinterpret_cast<const uint4*>(act) + off);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float gv[8], xv[8];
        unpack8(gq[u], gv);
        unpack8(xq[u], xv);
        if (MASK == 3) {
#pragma unroll
          for (int e = 0; e < 8; ++e) gv[e] = ((mb[u] >> e) & 1u) ? gv[e] : 0.f;
        } else if (MASK == 2) {
          float av[8];
          unpack8(aq[u], av);
#pragma unroll
          for (int e = 0; e < 8; ++e) gv[e] = av[e] > 0.f ? gv[e] : 0.f;
        } else if (MASK == 1) {
#pragma unroll
          for (int e = 0; e < 8; ++e) gv[e] = (xv[e] * sc[e] + sh[e]) > 0.f ? gv[e] : 0.f;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          a1[e] += gv[e];
          a2[e] += gv[e] * (xv[e] - mu[e]) * is[e];
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      fix_add(red + gi * 8 + e, a1[e]);
      fix_add(red + C + gi * 8 + e, a2[e]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    fix_add_raw(s1 + c, red[c]);
    fix_add_raw(s2 + c, red[C + c]);
  }
}

// Same reduction with the access pattern of the "fixed" elementwise kernels: the grid sweeps the tensor front to back
// instead of giving each block a private row range (1184 private sequential streams per operand cost DRAM row
// locality).  Its result is defined by S = `chains` = fixed_grid(nvec, C/8) * 256 fp32 partial sums: chain t < S sums
// the 8-channel vectors t, t+S, t+2S, ... in that order, four vectors per iteration (past the end an iteration adds
// zero gradients), and every chain's a1[e] / a2[e] goes into fixed point.  Fixed-point addition is exact and
// order-free, so how chains map onto threads and blocks does not change a bit:
//  - a warp runs 32 consecutive chains (512 contiguous bytes per vector and operand); chain t is on channel group
//    t % (C/8), so warps whose first chain is equal modulo C/8 ("class": one of max(C/256, 1)) have the same channels
//    in every lane and the 8 warps of a block are always of one class;
//  - a warp runs `rounds` such chain sets one after another, and the grid is at most one wave of resident blocks;
//  - each thread turns a finished chain into fixed-point words in registers and adds them, as plain 64-bit integers,
//    to its own slots of a shared-memory slab (the part of an addend beyond the words goes straight to the fp64 side
//    sum in global memory, fix_take_spill); at the end the block adds the slots of each channel, over its warps and
//    the lanes that share the channel, and issues one fix_add_words per channel and sum.
// The integer sums wrap mod 2^64 in any grouping, so s1 / s2 end with the same words and side sums as when every
// chain went to them on its own.
static constexpr int kReduceWarps = 8;
static constexpr int kReduceSlab = 2 * kReduceWarps * 16 * 32;   // lo and hi words: [2][warp][16 sums][32 lanes]
template <int MASK>
__global__ void __launch_bounds__(256)
bn_bwd_reduce_fixed_kernel(const bf16* __restrict__ g, const bf16* __restrict__ x, const bf16* __restrict__ act,
                           const float* __restrict__ scale, const float* __restrict__ shift,
                           const float* __restrict__ mean, const float* __restrict__ invstd, Fix128* __restrict__ s1,
                           Fix128* __restrict__ s2, int64_t nvec, int C, int64_t chains, int rounds) {
  extern __shared__ unsigned long long slab[];
  const int groups = C >> 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int classes = groups > 32 ? groups / 32 : 1;
  const int cls = (int)(blockIdx.x % classes);
  const int64_t per_class = chains / 32 / classes;                       // warps of chains in each class
  const int64_t first = (int64_t)(blockIdx.x / classes) * rounds * kReduceWarps;
  unsigned long long* lo_w = slab + warp * 16 * 32 + lane;               // this thread's 16 slots, 32 words apart
  unsigned long long* hi_w = lo_w + kReduceSlab / 2;
#pragma unroll
  for (int v = 0; v < 16; ++v) { lo_w[32 * v] = 0ull; hi_w[32 * v] = 0ull; }
  const int gi = (cls * 32 + lane) % groups;
  float mu[8], is[8], sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    mu[e] = mean[gi * 8 + e];
    is[e] = invstd[gi * 8 + e];
    sc[e] = MASK == 1 ? scale[gi * 8 + e] : 0.f;
    sh[e] = MASK == 1 ? shift[gi * 8 + e] : 0.f;
  }
  for (int k = 0; k < rounds; ++k) {
    const int64_t wj = first + (int64_t)k * kReduceWarps + warp;
    if (wj >= per_class) break;
    const int64_t t = (wj * classes + cls) * 32 + lane;                  // this thread's chain
    float a1[8], a2[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { a1[e] = 0.f; a2[e] = 0.f; }
    // Two of the chain's four-vector iterations per pass, all 8 loads issued first (short chains wait on memory
    // half as often).  The second iteration is added only when the chain has it; within an iteration a vector past
    // the end loads a zero gradient and the x of the iteration's first vector, exactly as one iteration at a time.
    for (int64_t i0 = t; i0 < nvec; i0 += 8 * chains) {
      uint4 gq[8], xq[8], aq[8];
      uint32_t mb[8];
      const bool second = i0 + 4 * chains < nvec;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int64_t i = u < 4 ? i0 : i0 + 4 * chains;
        const int64_t j = i + (u & 3) * chains;
        const bool ok = j < nvec;
        const bool in_chain = u < 4 || second;
        const int64_t off = ok ? j : (in_chain ? i : i0);
        gq[u] = ok ? __ldg(reinterpret_cast<const uint4*>(g) + off) : make_uint4(0u, 0u, 0u, 0u);
        xq[u] = __ldg(reinterpret_cast<const uint4*>(x) + off);
        if (MASK == 3) mb[u] = __ldg(reinterpret_cast<const uint8_t*>(act) + off);
        if (MASK == 2) aq[u] = __ldg(reinterpret_cast<const uint4*>(act) + off);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (u >= 4 && !second) break;
        float gv[8], xv[8];
        unpack8(gq[u], gv);
        unpack8(xq[u], xv);
        if (MASK == 3) {
#pragma unroll
          for (int e = 0; e < 8; ++e) gv[e] = ((mb[u] >> e) & 1u) ? gv[e] : 0.f;
        } else if (MASK == 2) {
          float av[8];
          unpack8(aq[u], av);
#pragma unroll
          for (int e = 0; e < 8; ++e) gv[e] = av[e] > 0.f ? gv[e] : 0.f;
        } else if (MASK == 1) {
#pragma unroll
          for (int e = 0; e < 8; ++e) gv[e] = (xv[e] * sc[e] + sh[e]) > 0.f ? gv[e] : 0.f;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          a1[e] += gv[e];
          a2[e] += gv[e] * (xv[e] - mu[e]) * is[e];
        }
      }
    }
#pragma unroll
    for (int v = 0; v < 16; ++v) {
      double a = v < 8 ? (double)a1[v] : (double)a2[v - 8];
      if (!fix_take_spill((v < 8 ? s1 : s2) + gi * 8 + (v & 7), a)) continue;
      unsigned long long lo;
      long long hi;
      fix_words(a, lo, hi);
      lo_w[32 * v] += lo;
      hi_w[32 * v] += (unsigned long long)hi;
    }
  }
  __syncthreads();
  const int win = groups < 32 ? groups : 32;                             // channel groups of the block
  for (int idx = threadIdx.x; idx < 16 * win; idx += blockDim.x) {
    const int v = idx / win, p = idx - v * win;
    unsigned long long lo = 0ull, hi = 0ull;
    for (int w = 0; w < kReduceWarps; ++w)
      for (int l = p; l < 32; l += win) {
        lo += slab[(w * 16 + v) * 32 + l];
        hi += slab[kReduceSlab / 2 + (w * 16 + v) * 32 + l];
      }
    fix_add_words((v < 8 ? s1 : s2) + (cls * 32 + p) * 8 + (v & 7), lo, (long long)hi);
  }
}

// dy = gamma*invstd*(dz - s1/n - xhat*s2/n);  optional dz output (bf16) for the residual path
template <int MASK>
__global__ void bn_bwd_apply_kernel(const bf16* __restrict__ g, const bf16* __restrict__ x,
                                    const bf16* __restrict__ act, const float* __restrict__ scale,
                                    const float* __restrict__ shift, const float* __restrict__ mean,
                                    const float* __restrict__ invstd, const float* __restrict__ gamma,
                                    const float* __restrict__ s1, const float* __restrict__ s2, float inv_count,
                                    bf16* __restrict__ dy, bf16* __restrict__ dz_out, int64_t nvec, int C,
                                    const float* __restrict__ s1_local, const float* __restrict__ s2_local,
                                    float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int groups = C >> 3;
  if (blockIdx.x == 0 && dgamma != nullptr) {
    // parameter gradients come from the rank-LOCAL sums (SyncBatchNorm.backward, _functions.py:122-170)
    // atomics: the two online views may run concurrently; each adds once per element to the zeroed gradient, and two
    // additions onto zero give the same bits in either order
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      atomicAdd(dgamma + c, s2_local[c]);
      atomicAdd(dbeta + c, s1_local[c]);
    }
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int gi = (int)(i % groups);
    float gv[8], xv[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(g) + i), gv);
    unpack8(__ldg(reinterpret_cast<const uint4*>(x) + i), xv);
    if (MASK == 3) {
      const uint32_t mb = __ldg(reinterpret_cast<const uint8_t*>(act) + i);
#pragma unroll
      for (int e = 0; e < 8; ++e) gv[e] = ((mb >> e) & 1u) ? gv[e] : 0.f;
    } else if (MASK == 2) {
      float av[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(act) + i), av);
#pragma unroll
      for (int e = 0; e < 8; ++e) gv[e] = av[e] > 0.f ? gv[e] : 0.f;
    } else if (MASK == 1) {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        gv[e] = (xv[e] * __ldg(scale + gi * 8 + e) + __ldg(shift + gi * 8 + e)) > 0.f ? gv[e] : 0.f;
    }
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = gi * 8 + e;
      const float is = __ldg(invstd + c);
      const float xhat = (xv[e] - __ldg(mean + c)) * is;
      o[e] = __ldg(gamma + c) * is * (gv[e] - __ldg(s1 + c) * inv_count - xhat * __ldg(s2 + c) * inv_count);
    }
    reinterpret_cast<uint4*>(dy)[i] = pack8(o);
    if (dz_out != nullptr) reinterpret_cast<uint4*>(dz_out)[i] = pack8(gv);
  }
}

// column sum of a bf16 or fp32 [M, C] matrix (bias gradients): out[c] += sum_r x[r, c]
template <typename T>
__global__ void col_sum_kernel(const T* __restrict__ x, Fix128* __restrict__ out, int M, int C, int ld,
                               int rows_per_block) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int row_begin = blockIdx.x * rows_per_block;
  int row_end = row_begin + rows_per_block;
  if (row_end > M) row_end = M;
  float s = 0.f;
  for (int r = row_begin; r < row_end; ++r) s += (float)x[(int64_t)r * ld + c];
  fix_add(out + c, s);
}

// grid for the "fixed channel group" elementwise kernels: (grid*256) % groups == 0, or 0 if impossible
static inline int fixed_grid(int64_t nvec, int groups) {
  int unit = groups > 256 ? groups / 256 : 1;          // blocks per channel period
  if (groups > 256 ? (groups % 256 != 0) : (256 % groups != 0)) return 0;
  int64_t b = (nvec + 255) / 256;
  int64_t cap = 132 * 8;
  if (b > cap) b = cap;
  b = (b + unit - 1) / unit * unit;
  if (b < unit) b = unit;
  return (int)b;
}

// launch grid of bn_apply_fixed_kernel<*, false>: enough blocks for kFixedVecs vectors per thread, at most
// `resident` (one wave), a multiple of the blocks per channel period so that (grid*256) % groups == 0
static inline int fixed_wave_grid(int64_t nvec, int groups, int resident) {
  const int unit = groups > 256 ? groups / 256 : 1;
  int64_t b = (nvec + 256 * kFixedVecs - 1) / (256 * kFixedVecs);
  if (b > resident) b = resident;
  b = b / unit * unit;
  return (int)(b < unit ? unit : b);
}

static inline int grid_for(int64_t n, int block, int max_blocks = 132 * 16) {
  int64_t b = (n + block - 1) / block;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace byol

using namespace byol;

// stats must be zeroed by the caller; accumulates sum into stats[0:C], sqsum into stats[C:2C]
extern "C" int byol_bn_stats(const void* x, float* stats, int M, int C, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && stats && M > 0 && C % 8 == 0 && C <= 4800, "byol_bn_stats: bad args (M=%d C=%d)", M, C);
  int rows_per_block = (M + 132 * 8 - 1) / (132 * 8);
  if (rows_per_block < 32) rows_per_block = 32;
  const int blocks = (M + rows_per_block - 1) / rows_per_block;
  const size_t red_bytes = 2 * (size_t)C * sizeof(Fix128);
  if (smem_opt_in((const void*)bn_stats_kernel, (int)red_bytes, "bn_stats_kernel") != 0) return -2;
  Fix128* fx = fix_scratch(stream, 2 * (int64_t)C);
  if (fx == nullptr) return -2;
  bn_stats_kernel<<<blocks, 256, red_bytes, stream>>>((const bf16*)x, fx, fx + C, M, C, rows_per_block);
  if (check_launch("bn_stats_kernel") != 0) return -100;
  return fix_done(stream, fix_flush(fx, stats, 2 * (int64_t)C, stream));
}

// stats: [L][2C]; coeffs: [L][4][C]; gamma_l / beta_l for l < L (L <= 4)
extern "C" int byol_bn_finalize_lanes(const float* stats, double count, int L, const float* gamma0, const float* beta0,
                                      const float* gamma1, const float* beta1, const float* gamma2,
                                      const float* beta2, const float* gamma3, const float* beta3,
                                      float* running_mean, float* running_var, float momentum, float eps,
                                      float* coeffs, int C, cudaStream_t stream) {
  BYOL_CHECK_ARG(stats && coeffs && L >= 1 && L <= 4 && C > 0 && count > 0, "byol_bn_finalize_lanes: bad args");
  LanePtrs g, b;
  g.p[0] = gamma0; g.p[1] = gamma1; g.p[2] = gamma2; g.p[3] = gamma3;
  b.p[0] = beta0; b.p[1] = beta1; b.p[2] = beta2; b.p[3] = beta3;
  for (int l = 0; l < L; ++l) BYOL_CHECK_ARG(g.p[l] && b.p[l], "byol_bn_finalize_lanes: null gamma/beta for lane %d", l);
  bn_finalize_lanes_kernel<<<(C + 127) / 128, 128, 0, stream>>>(stats, count, g, b, running_mean, running_var, momentum,
                                                               eps, coeffs, C, L);
  return check_launch("bn_finalize_lanes_kernel");
}

extern "C" int byol_bn_eval_coeffs(const float* gamma, const float* beta, const float* running_mean,
                                   const float* running_var, float eps, float* scale, float* shift, int C,
                                   cudaStream_t stream) {
  BYOL_CHECK_ARG(gamma && beta && running_mean && running_var && scale && shift && C > 0,
                 "byol_bn_eval_coeffs: bad args");
  bn_eval_coeffs_kernel<<<(C + 127) / 128, 128, 0, stream>>>(gamma, beta, running_mean, running_var, eps, scale,
                                                            shift, C);
  return check_launch("bn_eval_coeffs_kernel");
}

extern "C" int byol_bn_apply(const void* x, const float* scale, const float* shift, const void* resid,
                             const float* rscale, const float* rshift, void* y, float* y_f32, void* mask_out,
                             int M, int C, int relu, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && scale && shift && (y || y_f32) && M > 0 && C % 8 == 0, "byol_bn_apply: bad args");
  uint8_t* mo = (uint8_t*)mask_out;
  const int64_t nvec = (int64_t)M * C / 8;
  const int fg = (y != nullptr && y_f32 == nullptr) ? fixed_grid(nvec, C / 8) : 0;
  if (fg > 0) {
    const bf16 *xp = (const bf16*)x, *rp = (const bf16*)resid;
    if (rscale != nullptr) {
      bn_apply_fixed_kernel<true, true><<<fg, 256, 0, stream>>>(xp, scale, shift, rp, rscale, rshift, (bf16*)y, mo, nvec, C, relu);
      return check_launch("bn_apply_fixed_kernel");
    }
    const auto kern = resid == nullptr ? bn_apply_fixed_kernel<false, false> : bn_apply_fixed_kernel<true, false>;
    const int resident = resident_blocks((const void*)kern, 256, 0, "bn_apply_fixed_kernel");
    if (resident <= 0) return -2;
    kern<<<fixed_wave_grid(nvec, C / 8, resident), 256, 0, stream>>>(xp, scale, shift, rp, rscale, rshift, (bf16*)y,
                                                                     mo, nvec, C, relu);
    return check_launch("bn_apply_fixed_kernel");
  }
  bn_apply_kernel<<<grid_for(nvec, 256), 256, 0, stream>>>((const bf16*)x, scale, shift, (const bf16*)resid, rscale,
                                                           rshift, (bf16*)y, y_f32, mo, nvec, C, relu);
  return check_launch("bn_apply_kernel");
}

// sums must be zeroed by the caller: s12[0:C] = sum dz, s12[C:2C] = sum dz*xhat
extern "C" int byol_bn_bwd_reduce(const void* g, const void* x, const void* act, const float* scale,
                                  const float* shift, const float* mean, const float* invstd, float* s12, int M,
                                  int C, int mask_mode, cudaStream_t stream) {
  BYOL_CHECK_ARG(g && x && mean && invstd && s12 && M > 0 && C % 8 == 0, "byol_bn_bwd_reduce: bad args");
  BYOL_CHECK_ARG(mask_mode >= 0 && mask_mode <= 3, "byol_bn_bwd_reduce: bad mask_mode %d", mask_mode);
  BYOL_CHECK_ARG(mask_mode < 2 || act, "byol_bn_bwd_reduce: mask_mode 2/3 needs act");
  BYOL_CHECK_ARG(mask_mode != 1 || (scale && shift), "byol_bn_bwd_reduce: mask_mode 1 needs scale/shift");
  int rows_per_block = (M + 132 * 8 - 1) / (132 * 8);
  if (rows_per_block < 32) rows_per_block = 32;
  const int blocks = (M + rows_per_block - 1) / rows_per_block;
  const bf16 *gp = (const bf16*)g, *xp = (const bf16*)x, *ap = (const bf16*)act;
  const size_t red_bytes = 2 * (size_t)C * sizeof(Fix128);
  const int64_t nvec = (int64_t)M * C / 8;
  Fix128* fx = fix_scratch(stream, 2 * (int64_t)C);
  if (fx == nullptr) return -2;
  BYOL_CHECK_ARG(red_bytes <= 226 * 1024, "byol_bn_bwd_reduce: C=%d too wide (at most 4800 channels)", C);
  const int fg = fixed_grid(nvec, C / 8);
  if (fg > 0) {
    static const decltype(&bn_bwd_reduce_fixed_kernel<0>) fixed_kernels[4] = {
        bn_bwd_reduce_fixed_kernel<0>, bn_bwd_reduce_fixed_kernel<1>, bn_bwd_reduce_fixed_kernel<2>,
        bn_bwd_reduce_fixed_kernel<3>};
    const auto kern = fixed_kernels[mask_mode];
    const int slab = kReduceSlab * (int)sizeof(unsigned long long);
    if (smem_opt_in((const void*)kern, slab, "bn_bwd_reduce_fixed_kernel") != 0) return -2;
    const int resident = resident_blocks((const void*)kern, 256, slab, "bn_bwd_reduce_fixed_kernel");
    if (resident <= 0) return -2;
    // fixed_grid defines the chains (and so the bits); the launch is the fewest rounds that fit in one wave: at most
    // resident / classes blocks per class, and at least one (a device holding fewer blocks than there are classes
    // runs one block per class, in more than one wave)
    const int64_t chains = (int64_t)fg * 256;
    const int64_t classes = C / 8 > 32 ? C / 8 / 32 : 1, per_class = chains / 32 / classes;
    const int64_t class_blocks = resident / classes > 0 ? resident / classes : 1;
    const int64_t rounds = (per_class + kReduceWarps * class_blocks - 1) / (kReduceWarps * class_blocks);
    const int blocks = (int)(classes * ((per_class + kReduceWarps * rounds - 1) / (kReduceWarps * rounds)));
    kern<<<blocks, 256, slab, stream>>>(gp, xp, ap, scale, shift, mean, invstd, fx, fx + C, nvec, C, chains,
                                        (int)rounds);
    if (check_launch("bn_bwd_reduce_fixed_kernel") != 0) return -100;
    return fix_done(stream, fix_flush(fx, s12, 2 * (int64_t)C, stream));
  }
  static const decltype(&bn_bwd_reduce_kernel<0>) kernels[4] = {bn_bwd_reduce_kernel<0>, bn_bwd_reduce_kernel<1>,
                                                                 bn_bwd_reduce_kernel<2>, bn_bwd_reduce_kernel<3>};
  const auto kern = kernels[mask_mode];
  if (smem_opt_in((const void*)kern, (int)red_bytes, "bn_bwd_reduce_kernel") != 0) return -2;
  kern<<<blocks, 256, red_bytes, stream>>>(gp, xp, ap, scale, shift, mean, invstd, fx, fx + C, M, C, rows_per_block);
  if (check_launch("bn_bwd_reduce_kernel") != 0) return -100;
  return fix_done(stream, fix_flush(fx, s12, 2 * (int64_t)C, stream));
}

// s12: global (cross-rank) sums used for dy; s12_local: this rank's sums accumulated into dgamma/dbeta
// (both optional; s12_local == nullptr means "same as s12").
extern "C" int byol_bn_bwd_apply(const void* g, const void* x, const void* act, const float* scale,
                                 const float* shift, const float* mean, const float* invstd, const float* gamma,
                                 const float* s12, double count, void* dy, void* dz_out, int M, int C, int mask_mode,
                                 const float* s12_local, float* dgamma, float* dbeta, cudaStream_t stream) {
  if (s12_local == nullptr) s12_local = s12;
  BYOL_CHECK_ARG(g && x && mean && invstd && gamma && s12 && dy && M > 0 && C % 8 == 0, "byol_bn_bwd_apply: bad args");
  BYOL_CHECK_ARG(mask_mode >= 0 && mask_mode <= 3 && (mask_mode < 2 || act), "byol_bn_bwd_apply: bad mask_mode %d", mask_mode);
  const int64_t nvec = (int64_t)M * C / 8;
  const float inv_count = (float)(1.0 / count);
  const bf16 *gp = (const bf16*)g, *xp = (const bf16*)x, *ap = (const bf16*)act;
  const int fg = fixed_grid(nvec, C / 8);
  if (fg > 0) {
    if (mask_mode == 0)
      bn_bwd_apply_fixed_kernel<0><<<fg, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
    else if (mask_mode == 1)
      bn_bwd_apply_fixed_kernel<1><<<fg, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
    else if (mask_mode == 2)
      bn_bwd_apply_fixed_kernel<2><<<fg, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
    else
      bn_bwd_apply_fixed_kernel<3><<<fg, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
    return check_launch("bn_bwd_apply_fixed_kernel");
  }
  const int grid = grid_for(nvec, 256);
  if (mask_mode == 0)
    bn_bwd_apply_kernel<0><<<grid, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
  else if (mask_mode == 1)
    bn_bwd_apply_kernel<1><<<grid, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
  else if (mask_mode == 2)
    bn_bwd_apply_kernel<2><<<grid, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
  else
    bn_bwd_apply_kernel<3><<<grid, 256, 0, stream>>>(gp, xp, ap, scale, shift, mean, invstd, gamma, s12, s12 + C, inv_count, (bf16*)dy, (bf16*)dz_out, nvec, C, s12_local, s12_local + C, dgamma, dbeta);
  return check_launch("bn_bwd_apply_kernel");
}

// out[c] += sum_r x[r, c]   (x bf16 when is_f32 == 0)
extern "C" int byol_col_sum(const void* x, float* out, int M, int C, int ld, int is_f32, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && out && M > 0 && C > 0 && ld >= C, "byol_col_sum: bad args");
  int rows_per_block = (M + 63) / 64;
  if (rows_per_block < 16) rows_per_block = 16;
  dim3 grid((M + rows_per_block - 1) / rows_per_block, (C + 127) / 128);
  Fix128* fx = fix_scratch(stream, C);
  if (fx == nullptr) return -2;
  if (is_f32)
    col_sum_kernel<float><<<grid, 128, 0, stream>>>((const float*)x, fx, M, C, ld, rows_per_block);
  else
    col_sum_kernel<bf16><<<grid, 128, 0, stream>>>((const bf16*)x, fx, M, C, ld, rows_per_block);
  if (check_launch("col_sum_kernel") != 0) return -100;
  return fix_done(stream, fix_flush(fx, out, C, stream));
}
