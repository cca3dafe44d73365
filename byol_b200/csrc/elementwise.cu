// byol_b200 — layout conversion, weight preparation and pooling kernels (NHWC bf16 activations).
//
// These replace the ATen elementwise / pooling kernels under torchvision's ResNet stem and tail reached from
// /root/reference/main.py:237 (`self.base_network(augmentation)`): MaxPool2d(3, 2, 1), AdaptiveAvgPool2d(1),
// plus the NCHW fp32 -> NHWC bf16 input conversion and the fp32 master -> bf16 K-major weight layouts the
// tensor-core (wgmma) kernels consume.  All are HBM-bound streaming kernels: 16-byte vector accesses, grid-stride loops.
#include <stdlib.h>
#include "common.cuh"

namespace byol {

static inline int grid_for(int64_t n, int block, int max_blocks = 132 * 16) {
  int64_t b = (n + block - 1) / block;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return (int)b;
}

// x: [N, Cin, H, W] fp32 (Cin <= 8)  ->  y: [N, H, W, 8] bf16, channels >= Cin zero
__global__ void nchw_to_nhwc8_kernel(const float* __restrict__ x, bf16* __restrict__ y, int64_t npix, int Cin,
                                     int HW) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npix; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / HW;
    const int hw = (int)(i - n * HW);
    float v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = c < Cin ? __ldg(x + (n * Cin + c) * HW + hw) : 0.f;
    uint4 q;
    q.x = pack_bf16x2(v[0], v[1]);
    q.y = pack_bf16x2(v[2], v[3]);
    q.z = pack_bf16x2(v[4], v[5]);
    q.w = pack_bf16x2(v[6], v[7]);
    reinterpret_cast<uint4*>(y)[i] = q;
  }
}

// w: fp32 [Cout][Cin][KH][KW]  ->  wf: bf16 [Cout][KH*KW*Cpad] (fprop, K-major)
//                                  wd: bf16 [Cin][KH*KW*Cout]  (dgrad, K-major; optional)
__global__ void prep_weight_kernel(const float* __restrict__ w, bf16* __restrict__ wf, bf16* __restrict__ wd,
                                   int Cout, int Cin, int Cpad, int taps) {
  if (taps <= 9 && Cpad == Cin) {
    // Tiled through shared memory: a 32 (cout) x 32 (cin) tile for all taps.  Reads follow the master's
    // [cout][cin][tap] order (contiguous), the fprop layout is written along cin and the dgrad layout along cout
    // (64 contiguous bytes each); the element-per-thread loop below scattered 2-byte writes with a stride of Cout.
    __shared__ float tile[9][32][33];
    const int tiles_c = (Cin + 31) / 32, tiles_o = (Cout + 31) / 32;
    for (int tix = blockIdx.x; tix < tiles_c * tiles_o; tix += gridDim.x) {
      const int o0 = (tix / tiles_c) * 32, c0 = (tix % tiles_c) * 32;
      __syncthreads();
      for (int i = threadIdx.x; i < 32 * 32 * taps; i += blockDim.x) {
        const int r = i / (32 * taps), rem = i % (32 * taps);        // r: cout row; rem = c * taps + tap (contiguous)
        const int c = rem / taps, tap = rem % taps;
        float v = 0.f;
        if (o0 + r < Cout && c0 + c < Cin) v = __ldg(w + ((int64_t)(o0 + r) * Cin + c0 + c) * taps + tap);
        tile[tap][r][c] = v;
      }
      __syncthreads();
      for (int i = threadIdx.x; i < 32 * 32 * taps; i += blockDim.x) {
        const int c = i & 31, r = (i >> 5) & 31, tap = i >> 10;
        if (o0 + r < Cout && c0 + c < Cin)
          wf[((int64_t)(o0 + r) * taps + tap) * Cpad + c0 + c] = __float2bfloat16_rn(tile[tap][r][c]);
      }
      if (wd != nullptr) {
        for (int i = threadIdx.x; i < 32 * 32 * taps; i += blockDim.x) {
          const int r = i & 31, c = (i >> 5) & 31, tap = i >> 10;
          if (o0 + r < Cout && c0 + c < Cin)
            wd[((int64_t)(c0 + c) * taps + tap) * Cout + o0 + r] = __float2bfloat16_rn(tile[tap][r][c]);
        }
      }
    }
    return;
  }
  const int64_t total = (int64_t)Cout * taps * Cpad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t t = i / Cpad;
    const int tap = (int)(t % taps);
    const int co = (int)(t / taps);
    float v = 0.f;
    if (c < Cin) v = __ldg(w + ((int64_t)co * Cin + c) * taps + tap);
    const bf16 b = __float2bfloat16_rn(v);
    wf[i] = b;
    if (wd != nullptr && c < Cin) wd[((int64_t)c * taps + tap) * Cout + co] = b;
  }
}

// stem (folded) fprop layout: w fp32 [Cout][Cin<=8][KH][KW<=8] -> wf bf16 [Cout][KH][8 kw slots][8 channels]
__global__ void prep_weight_fold_kernel(const float* __restrict__ w, bf16* __restrict__ wf, int Cout, int Cin, int KH,
                                        int KW) {
  const int64_t total = (int64_t)Cout * KH * 64;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i & 7);
    const int kw = (int)((i >> 3) & 7);
    const int64_t t = i >> 6;
    const int kh = (int)(t % KH);
    const int co = (int)(t / KH);
    float v = 0.f;
    if (c < Cin && kw < KW) v = __ldg(w + (((int64_t)co * Cin + c) * KH + kh) * KW + kw);
    wf[i] = __float2bfloat16_rn(v);
  }
}

// All conv / linear weights of one parameter set in ONE launch.  desc[u] = {src_off, dstf_off, dstd_off (-1: none),
// Cout, Cin, Cpad, taps, fold(KH,KW packed as KH*16+KW or 0)} (int64 each); blockIdx.y = unit, grid-stride in x.
__host__ __device__ inline int prep_unit_blocks(int Cout, int Cin, int Cpad, int taps, int fold) {
  if (!fold && taps <= 9 && Cpad == Cin) return ((Cin + 31) / 32) * ((Cout + 31) / 32);      // 32 x 32 tiles
  const int64_t total = fold ? (int64_t)Cout * (fold >> 4) * 64 : (int64_t)Cout * taps * Cpad;
  return (int)((total + 8191) / 8192);
}

__global__ void prep_weights_multi_kernel(const float* __restrict__ flat, bf16* __restrict__ pool_f,
                                          bf16* __restrict__ pool_d, const int64_t* __restrict__ desc, int num_units) {
  // Work is balanced over the units: every unit owns prep_unit_blocks() consecutive blocks of the 1-D grid (a
  // [2048 x 4096] Linear needs 8192 tiles, a BatchNorm-sized conv a handful), found by a scan over the <= ~60 units.
  __shared__ int s_unit, s_local, s_nb;
  if (threadIdx.x == 0) {
    int rem = (int)blockIdx.x, u = 0, nb = 0;
    for (; u < num_units; ++u) {
      const int64_t* du = desc + (int64_t)u * 8;
      nb = prep_unit_blocks((int)du[3], (int)du[4], (int)du[5], (int)du[6], (int)du[7]);
      if (rem < nb) break;
      rem -= nb;
    }
    s_unit = u; s_local = rem; s_nb = nb;
  }
  __syncthreads();
  if (s_unit >= num_units) return;
  const int bx = s_local, nbx = s_nb;          // this block's index / block count inside its unit
  const int64_t* d = desc + (int64_t)s_unit * 8;
  const float* w = flat + d[0];
  bf16* wf = pool_f + d[1];
  bf16* wd = d[2] >= 0 ? pool_d + d[2] : nullptr;
  const int Cout = (int)d[3], Cin = (int)d[4], Cpad = (int)d[5], taps = (int)d[6], fold = (int)d[7];
  if (fold) {
    const int KH = fold >> 4, KW = fold & 15;
    const int64_t total = (int64_t)Cout * KH * 64;
    for (int64_t i = bx * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)nbx * blockDim.x) {
      const int c = (int)(i & 7);
      const int kw = (int)((i >> 3) & 7);
      const int64_t t = i >> 6;
      const int kh = (int)(t % KH);
      const int co = (int)(t / KH);
      float v = 0.f;
      if (c < Cin && kw < KW) v = __ldg(w + (((int64_t)co * Cin + c) * KH + kh) * KW + kw);
      wf[i] = __float2bfloat16_rn(v);
    }
    return;
  }
  const int64_t total = (int64_t)Cout * taps * Cpad;
  for (int64_t i = bx * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)nbx * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t t = i / Cpad;
    const int tap = (int)(t % taps);
    const int co = (int)(t / taps);
    float v = 0.f;
    if (c < Cin) v = __ldg(w + ((int64_t)co * Cin + c) * taps + tap);
    const bf16 b = __float2bfloat16_rn(v);
    wf[i] = b;
    if (wd != nullptr && c < Cin) wd[((int64_t)c * taps + tap) * Cout + co] = b;
  }
}

// Grouped 3x3 convolutions (Cin == Cout == C, Cg = C / groups dividing 64), all units of one parameter set in ONE
// launch; blockIdx.y = unit.  desc[u] = {src_off, dstf_off, dstd_off (-1: none), C, Cg} (int64 each).  The weight of
// a 64-channel tile [n0, n0 + 64) is block-diagonal, so both layouts keep only that tile's 64 partner channels:
//   fprop wf[co][tap * 64 + (ci - n0)], n0 = co & ~63   = w[co][ci % Cg][tap] if co, ci share a group, else 0
//   dgrad wd[ci][tap * 64 + (co - n0)], n0 = ci & ~63   = w[co][ci % Cg][tap] if co, ci share a group, else 0
__global__ void prep_weights_grouped_kernel(const float* __restrict__ flat, bf16* __restrict__ pool_f,
                                            bf16* __restrict__ pool_d, const int64_t* __restrict__ desc) {
  const int64_t* d = desc + (int64_t)blockIdx.y * 5;
  const float* w = flat + d[0];
  bf16* wf = pool_f + d[1];
  bf16* wd = d[2] >= 0 ? pool_d + d[2] : nullptr;
  const int C = (int)d[3], Cg = (int)d[4];
  if (C <= 0 || C % 64 != 0 || Cg <= 0 || Cg > 64 || 64 % Cg != 0) return;   // rejected on the host
  const int64_t total = (int64_t)C * 9 * 64;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i & 63);
    const int tap = (int)((i >> 6) % 9);
    const int r = (int)(i / (9 * 64));
    const int c = (r & ~63) + j;   // the partner channel: ci of row co (fprop), co of row ci (dgrad)
    const bool same = r / Cg == c / Cg;
    wf[i] = __float2bfloat16_rn(same ? __ldg(w + ((int64_t)r * Cg + c % Cg) * 9 + tap) : 0.f);
    if (wd != nullptr) wd[i] = __float2bfloat16_rn(same ? __ldg(w + ((int64_t)c * Cg + r % Cg) * 9 + tap) : 0.f);
  }
}

// y[n, i, j, :] = x[n, 2i, 2j, :]: the pixels a 1x1 / stride-2 convolution reads, compacted so that the downsample
// branch runs as a plain (TMA-fed) GEMM.  One thread per 16-byte vector.
__global__ void subsample2_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int H, int W, int C) {
  const int groups = C >> 3, Ho = H >> 1, Wo = W >> 1;
  const int64_t total = (int64_t)N * Ho * Wo * groups;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    int64_t t = i / groups;
    const int j = (int)(t % Wo); t /= Wo;
    const int r = (int)(t % Ho);
    const int n = (int)(t / Ho);
    reinterpret_cast<uint4*>(y)[i] =
        __ldg(reinterpret_cast<const uint4*>(x + (((int64_t)n * H + 2 * r) * W + 2 * j) * C) + g);
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16_rn(x[i]);
}

// MaxPool (k x k, stride s, pad p) over NHWC bf16; one thread per (output pixel, 8-channel group).
// idx (uint8, window position kh*k+kw of the first maximum in scan order) is saved for the backward pass,
// matching ATen's max_pool2d_with_indices tie-breaking (first occurrence wins).
__global__ void maxpool_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, uint8_t* __restrict__ idx,
                                   int N, int H, int W, int C, int Ho, int Wo, int k, int s, int p) {
  const int groups = C >> 3;
  const int64_t total = (int64_t)N * Ho * Wo * groups;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    int64_t t = i / groups;
    const int ow = (int)(t % Wo); t /= Wo;
    const int oh = (int)(t % Ho);
    const int n = (int)(t / Ho);
    // a window whose in-image values are all -inf reports its first in-image position (ATen), never a padding one
    const int first = (p - oh * s > 0 ? p - oh * s : 0) * k + (p - ow * s > 0 ? p - ow * s : 0);
    float best[8];
    int bi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; bi[e] = first; }
    for (int kh = 0; kh < k; ++kh) {
      const int ih = oh * s - p + kh;
      if (ih < 0 || ih >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int iw = ow * s - p + kw;
        if (iw < 0 || iw >= W) continue;
        uint4 v = __ldg(reinterpret_cast<const uint4*>(x + (((int64_t)n * H + ih) * W + iw) * C + g * 8));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __bfloat1622float2(h[e]);
          if (f.x > best[2 * e] || f.x != f.x) { best[2 * e] = f.x; bi[2 * e] = kh * k + kw; }
          if (f.y > best[2 * e + 1] || f.y != f.y) { best[2 * e + 1] = f.y; bi[2 * e + 1] = kh * k + kw; }
        }
      }
    }
    uint4 q;
    q.x = pack_bf16x2(best[0], best[1]);
    q.y = pack_bf16x2(best[2], best[3]);
    q.z = pack_bf16x2(best[4], best[5]);
    q.w = pack_bf16x2(best[6], best[7]);
    reinterpret_cast<uint4*>(y)[i] = q;
    if (idx != nullptr) {
      uint2 pk;
      pk.x = (uint32_t)bi[0] | ((uint32_t)bi[1] << 8) | ((uint32_t)bi[2] << 16) | ((uint32_t)bi[3] << 24);
      pk.y = (uint32_t)bi[4] | ((uint32_t)bi[5] << 8) | ((uint32_t)bi[6] << 16) | ((uint32_t)bi[7] << 24);
      reinterpret_cast<uint2*>(idx)[i] = pk;
    }
  }
}

// Stem fusion: y = maxpool(relu(x*scale + shift)) without materialising the normalised map.  Candidates are rounded
// to bf16 before the comparison, so values AND argmax indices equal bn_apply followed by maxpool_fwd bit for bit.
__global__ void bn_relu_maxpool_fwd_kernel(const bf16* __restrict__ x, const float* __restrict__ scale,
                                           const float* __restrict__ shift, bf16* __restrict__ y,
                                           uint8_t* __restrict__ idx, int N, int H, int W, int C, int Ho, int Wo,
                                           int k, int s, int p) {
  const int groups = C >> 3;
  const int64_t total = (int64_t)N * Ho * Wo * groups;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    int64_t t = i / groups;
    const int ow = (int)(t % Wo); t /= Wo;
    const int oh = (int)(t % Ho);
    const int n = (int)(t / Ho);
    float sc[8], sh[8], best[8];
    int bi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      sc[e] = __ldg(scale + g * 8 + e);
      sh[e] = __ldg(shift + g * 8 + e);
      best[e] = -INFINITY;
      bi[e] = 0;
    }
    for (int kh = 0; kh < k; ++kh) {
      const int ih = oh * s - p + kh;
      if (ih < 0 || ih >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int iw = ow * s - p + kw;
        if (iw < 0 || iw >= W) continue;
        uint4 v = __ldg(reinterpret_cast<const uint4*>(x + (((int64_t)n * H + ih) * W + iw) * C + g * 8));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __bfloat1622float2(h[e]);
          const float a0 = __bfloat162float(__float2bfloat16_rn(fmaxf(f.x * sc[2 * e] + sh[2 * e], 0.f)));
          const float a1 = __bfloat162float(__float2bfloat16_rn(fmaxf(f.y * sc[2 * e + 1] + sh[2 * e + 1], 0.f)));
          if (a0 > best[2 * e] || a0 != a0) { best[2 * e] = a0; bi[2 * e] = kh * k + kw; }
          if (a1 > best[2 * e + 1] || a1 != a1) { best[2 * e + 1] = a1; bi[2 * e + 1] = kh * k + kw; }
        }
      }
    }
    uint4 q;
    q.x = pack_bf16x2(best[0], best[1]);
    q.y = pack_bf16x2(best[2], best[3]);
    q.z = pack_bf16x2(best[4], best[5]);
    q.w = pack_bf16x2(best[6], best[7]);
    reinterpret_cast<uint4*>(y)[i] = q;
    if (idx != nullptr) {
      uint2 pk;
      pk.x = (uint32_t)bi[0] | ((uint32_t)bi[1] << 8) | ((uint32_t)bi[2] << 16) | ((uint32_t)bi[3] << 24);
      pk.y = (uint32_t)bi[4] | ((uint32_t)bi[5] << 8) | ((uint32_t)bi[6] << 16) | ((uint32_t)bi[7] << 24);
      reinterpret_cast<uint2*>(idx)[i] = pk;
    }
  }
}

// Same without the argmax (target lanes keep nothing for a backward pass): candidates are packed to bf16x2 right
// after the normalisation and reduced with packed max — half the instructions of the index-tracking kernel.
__global__ void __launch_bounds__(256)
bn_relu_maxpool_fwd_noidx_kernel(const bf16* __restrict__ x, const float* __restrict__ scale,
                                 const float* __restrict__ shift, bf16* __restrict__ y, int N, int H, int W, int C,
                                 int Ho, int Wo, int k, int s, int p) {
  const int groups = C >> 3;
  const int64_t total = (int64_t)N * Ho * Wo * groups;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    int64_t t = i / groups;
    const int ow = (int)(t % Wo); t /= Wo;
    const int oh = (int)(t % Ho);
    const int n = (int)(t / Ho);
    float sc[8], sh[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { sc[e] = __ldg(scale + g * 8 + e); sh[e] = __ldg(shift + g * 8 + e); }
    __nv_bfloat162 best[4];
    bool any = false;
    for (int kh = 0; kh < k; ++kh) {
      const int ih = oh * s - p + kh;
      if (ih < 0 || ih >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int iw = ow * s - p + kw;
        if (iw < 0 || iw >= W) continue;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + (((int64_t)n * H + ih) * W + iw) * C + g * 8));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(h[e]);
          const __nv_bfloat162 c2 = __floats2bfloat162_rn(fmaxf(f.x * sc[2 * e] + sh[2 * e], 0.f),
                                                          fmaxf(f.y * sc[2 * e + 1] + sh[2 * e + 1], 0.f));
          best[e] = any ? __hmax2_nan(best[e], c2) : c2;
        }
        any = true;
      }
    }
    uint4 q;
    q.x = *reinterpret_cast<uint32_t*>(&best[0]);
    q.y = *reinterpret_cast<uint32_t*>(&best[1]);
    q.z = *reinterpret_cast<uint32_t*>(&best[2]);
    q.w = *reinterpret_cast<uint32_t*>(&best[3]);
    reinterpret_cast<uint4*>(y)[i] = q;
  }
}

// dx[n, ih, iw, c] = sum over output windows (oh, ow) containing (ih, iw) whose saved argmax is this position
__global__ void maxpool_bwd_kernel(const bf16* __restrict__ dy, const uint8_t* __restrict__ idx,
                                   bf16* __restrict__ dx, int N, int H, int W, int C, int Ho, int Wo, int k, int s,
                                   int p) {
  const int groups = C >> 3;
  const int64_t total = (int64_t)N * H * W * groups;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    int64_t t = i / groups;
    const int iw = (int)(t % W); t /= W;
    const int ih = (int)(t % H);
    const int n = (int)(t / H);
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    // only window offsets kh == (ih + p) mod s (step s) can have produced this pixel: <= ceil(k/s)^2 candidates,
    // no division in the loops
    for (int kh = (ih + p) % s; kh < k; kh += s) {
      const int oh = (ih + p - kh) / s;
      if (oh < 0 || oh >= Ho) continue;
      for (int kw = (iw + p) % s; kw < k; kw += s) {
        const int ow = (iw + p - kw) / s;
        if (ow < 0 || ow >= Wo) continue;
        const int64_t o = (((int64_t)n * Ho + oh) * Wo + ow) * groups + g;
        const uint2 pk = __ldg(reinterpret_cast<const uint2*>(idx) + o);
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(dy) + o);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
        const int pos = kh * k + kw;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __bfloat1622float2(h[e]);
          const uint32_t word = e < 2 ? pk.x : pk.y;
          const int i0 = (word >> (16 * (e & 1))) & 0xff;
          const int i1 = (word >> (16 * (e & 1) + 8)) & 0xff;
          if (i0 == pos) acc[2 * e] += f.x;
          if (i1 == pos) acc[2 * e + 1] += f.y;
        }
      }
    }
    uint4 q;
    q.x = pack_bf16x2(acc[0], acc[1]);
    q.y = pack_bf16x2(acc[2], acc[3]);
    q.z = pack_bf16x2(acc[4], acc[5]);
    q.w = pack_bf16x2(acc[6], acc[7]);
    reinterpret_cast<uint4*>(dx)[i] = q;
  }
}

// Fast path for the ResNet stem pool (k = 3, s = 2, p = 1, H = 2 Ho, W = 2 Wo): one thread owns the 2 x 2 input block
// (2a .. 2a+1, 2b .. 2b+1) of one 8-channel group.  Exactly the four windows (a, b), (a, b+1), (a+1, b), (a+1, b+1) touch
// it, each at fixed window positions, so the thread reads 4 (argmax, dy) pairs and writes 4 gradient vectors — no loops,
// no divisions per tap, one (idx, dy) read per written pixel instead of 2.25 (the generic kernel ran at 1.2 TB/s).
__global__ void __launch_bounds__(256)
maxpool_bwd_k3s2_kernel(const bf16* __restrict__ dy, const uint8_t* __restrict__ idx, bf16* __restrict__ dx, int N,
                        int Ho, int Wo, int C) {
  const int groups = C >> 3;
  const int W = 2 * Wo;
  const int64_t total = (int64_t)N * Ho * Wo * groups;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    int64_t t = i / groups;
    const int b = (int)(t % Wo); t /= Wo;
    const int a = (int)(t % Ho);
    const int n = (int)(t / Ho);
    // windows: 0 = (a, b), 1 = (a, b+1), 2 = (a+1, b), 3 = (a+1, b+1)
    uint2 pk[4];
    uint4 gv[4];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int oh = a + (w >> 1), ow = b + (w & 1);
      const bool ok = oh < Ho && ow < Wo;
      const int64_t o = (((int64_t)n * Ho + (ok ? oh : a)) * Wo + (ok ? ow : b)) * groups + g;
      pk[w] = ok ? __ldg(reinterpret_cast<const uint2*>(idx) + o) : make_uint2(0xffffffffu, 0xffffffffu);
      gv[w] = __ldg(reinterpret_cast<const uint4*>(dy) + o);
    }
    // window position (kh*3 + kw) of each window that maps onto the block's pixels:
    //   pixel (2a, 2b)     <- w0 @ 4
    //   pixel (2a, 2b+1)   <- w0 @ 5, w1 @ 3
    //   pixel (2a+1, 2b)   <- w0 @ 7, w2 @ 1
    //   pixel (2a+1, 2b+1) <- w0 @ 8, w1 @ 6, w2 @ 2, w3 @ 0
    float acc[4][8];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[q][e] = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&gv[w]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t word = e < 4 ? pk[w].x : pk[w].y;
        const int id = (int)((word >> (8 * (e & 3))) & 0xffu);
        const float2 f2 = __bfloat1622float2(h[e >> 1]);
        const float f = (e & 1) ? f2.y : f2.x;
        if (w == 0) {
          if (id == 4) acc[0][e] += f;
          if (id == 5) acc[1][e] += f;
          if (id == 7) acc[2][e] += f;
          if (id == 8) acc[3][e] += f;
        } else if (w == 1) {
          if (id == 3) acc[1][e] += f;
          if (id == 6) acc[3][e] += f;
        } else if (w == 2) {
          if (id == 1) acc[2][e] += f;
          if (id == 2) acc[3][e] += f;
        } else {
          if (id == 0) acc[3][e] += f;
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint4 o4;
      o4.x = pack_bf16x2(acc[q][0], acc[q][1]);
      o4.y = pack_bf16x2(acc[q][2], acc[q][3]);
      o4.z = pack_bf16x2(acc[q][4], acc[q][5]);
      o4.w = pack_bf16x2(acc[q][6], acc[q][7]);
      const int ih = 2 * a + (q >> 1), iw = 2 * b + (q & 1);
      reinterpret_cast<uint4*>(dx)[(((int64_t)n * (2 * Ho) + ih) * W + iw) * groups + g] = o4;
    }
  }
}

// global average pool: x [N, HW, C] bf16 -> y_f32 [N, C] fp32 and y_bf16 [N, C] (both optional)
__global__ void avgpool_fwd_kernel(const bf16* __restrict__ x, float* __restrict__ y_f32, bf16* __restrict__ y_bf16,
                                   int N, int HW, int C) {
  const int groups = C >> 3;
  const int64_t total = (int64_t)N * groups;
  const float inv = 1.f / (float)HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const int64_t n = i / groups;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int r = 0; r < HW; ++r) {
      uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((int64_t)n * HW + r) * C + g * 8));
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __bfloat1622float2(h[e]);
        acc[2 * e] += f.x;
        acc[2 * e + 1] += f.y;
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] *= inv;
    if (y_f32 != nullptr) {
      float4* o = reinterpret_cast<float4*>(y_f32 + n * C + g * 8);
      o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    if (y_bf16 != nullptr) {
      uint4 q;
      q.x = pack_bf16x2(acc[0], acc[1]);
      q.y = pack_bf16x2(acc[2], acc[3]);
      q.z = pack_bf16x2(acc[4], acc[5]);
      q.w = pack_bf16x2(acc[6], acc[7]);
      *reinterpret_cast<uint4*>(y_bf16 + n * C + g * 8) = q;
    }
  }
}

// dx[n, r, c] = (g_a[n, c] (+ g_b[n, c])) / HW     (g_a bf16 from dgrad, g_b fp32 from autograd; either may be null)
__global__ void avgpool_bwd_kernel(const bf16* __restrict__ g_a, const float* __restrict__ g_b,
                                   bf16* __restrict__ dx, int N, int HW, int C) {
  const int groups = C >> 3;
  const int64_t total = (int64_t)N * HW * groups;
  const float inv = 1.f / (float)HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const int64_t n = i / ((int64_t)HW * groups);
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (g_a != nullptr) {
      uint4 q = __ldg(reinterpret_cast<const uint4*>(g_a + n * C + g * 8));
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __bfloat1622float2(h[e]);
        v[2 * e] += f.x;
        v[2 * e + 1] += f.y;
      }
    }
    if (g_b != nullptr) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] += __ldg(g_b + n * C + g * 8 + e);
    }
    uint4 q;
    q.x = pack_bf16x2(v[0] * inv, v[1] * inv);
    q.y = pack_bf16x2(v[2] * inv, v[3] * inv);
    q.z = pack_bf16x2(v[4] * inv, v[5] * inv);
    q.w = pack_bf16x2(v[6] * inv, v[7] * inv);
    reinterpret_cast<uint4*>(dx)[i] = q;
  }
}

}  // namespace byol

using namespace byol;

extern "C" int byol_nchw_to_nhwc8(const float* x, void* y, int N, int Cin, int H, int W, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y && N > 0 && Cin > 0 && Cin <= 8 && H > 0 && W > 0, "byol_nchw_to_nhwc8: bad args");
  const int64_t npix = (int64_t)N * H * W;
  nchw_to_nhwc8_kernel<<<grid_for(npix, 256), 256, 0, stream>>>(x, (bf16*)y, npix, Cin, H * W);
  return check_launch("nchw_to_nhwc8_kernel");
}

extern "C" int byol_prep_weight(const float* w, void* w_fprop, void* w_dgrad, int Cout, int Cin, int Cpad, int KH,
                                int KW, cudaStream_t stream) {
  BYOL_CHECK_ARG(w && w_fprop && Cout > 0 && Cin > 0 && Cpad >= Cin && Cpad % 8 == 0, "byol_prep_weight: bad args");
  BYOL_CHECK_ARG(w_dgrad == nullptr || Cout % 8 == 0, "byol_prep_weight: dgrad layout needs Cout %% 8 == 0");
  const int64_t total = (int64_t)Cout * KH * KW * Cpad;
  prep_weight_kernel<<<grid_for(total, 256), 256, 0, stream>>>(w, (bf16*)w_fprop, (bf16*)w_dgrad, Cout, Cin, Cpad,
                                                              KH * KW);
  return check_launch("prep_weight_kernel");
}

// stem layout for byol_conv_igemm's folded mode (C = 8 input channels, KW <= 8): w_fprop is [Cout][KH*64]
extern "C" int byol_prep_weight_fold(const float* w, void* w_fprop, int Cout, int Cin, int KH, int KW,
                                     cudaStream_t stream) {
  BYOL_CHECK_ARG(w && w_fprop && Cout > 0 && Cin > 0 && Cin <= 8 && KW <= 8 && KH > 0, "byol_prep_weight_fold: bad args");
  const int64_t total = (int64_t)Cout * KH * 64;
  prep_weight_fold_kernel<<<grid_for(total, 256), 256, 0, stream>>>(w, (bf16*)w_fprop, Cout, Cin, KH, KW);
  return check_launch("prep_weight_fold_kernel");
}

// desc: device array [num_units][8] int64 (see prep_weights_multi_kernel); pool_d may be null if no entry needs it
extern "C" int byol_prep_unit_blocks(int Cout, int Cin, int Cpad, int taps, int fold) {
  return prep_unit_blocks(Cout, Cin, Cpad, taps, fold);
}

extern "C" int byol_prep_weights_multi(const float* flat, void* pool_f, void* pool_d, const int64_t* desc,
                                       int num_units, int num_blocks, cudaStream_t stream) {
  BYOL_CHECK_ARG(flat && pool_f && desc && num_units > 0 && num_blocks > 0, "byol_prep_weights_multi: bad args");
  // num_blocks = sum over units of byol_prep_unit_blocks(...) (the host knows the shapes; desc lives on the device)
  prep_weights_multi_kernel<<<num_blocks, 256, 0, stream>>>(flat, (bf16*)pool_f, (bf16*)pool_d, desc, num_units);
  return check_launch("prep_weights_multi_kernel");
}

// desc: device int64 [num_units][5] (see prep_weights_grouped_kernel); max_c: the largest C among the units
extern "C" int byol_prep_weights_grouped(const float* flat, void* pool_f, void* pool_d, const int64_t* desc,
                                         int num_units, int max_c, cudaStream_t stream) {
  BYOL_CHECK_ARG(flat && pool_f && desc && num_units > 0 && num_units <= 65535 && max_c >= 64 && max_c % 64 == 0,
                 "byol_prep_weights_grouped: bad args (num_units=%d max_c=%d)", num_units, max_c);
  const dim3 grid((unsigned)grid_for((int64_t)max_c * 9 * 64, 256, 256), (unsigned)num_units);
  prep_weights_grouped_kernel<<<grid, 256, 0, stream>>>(flat, (bf16*)pool_f, (bf16*)pool_d, desc);
  return check_launch("prep_weights_grouped_kernel");
}

extern "C" int byol_subsample2(const void* x, void* y, int N, int H, int W, int C, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y && N > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "byol_subsample2: bad args");
  const int64_t total = (int64_t)N * (H / 2) * (W / 2) * (C / 8);
  subsample2_kernel<<<grid_for(total, 256), 256, 0, stream>>>((const bf16*)x, (bf16*)y, N, H, W, C);
  return check_launch("subsample2_kernel");
}

// y[r, c] = bf16(x[r, c]) for c < cols, 0 for cols <= c < ldy (row pitches ldx / ldy in elements)
__global__ void cast_f32_bf16_2d_kernel(const float* __restrict__ x, bf16* __restrict__ y, int rows, int cols, int ldx,
                                        int ldy) {
  const int64_t total = (int64_t)rows * ldy;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % ldy);
    const int64_t r = i / ldy;
    y[i] = c < cols ? __float2bfloat16_rn(x[r * ldx + c]) : __float2bfloat16_rn(0.f);
  }
}

extern "C" int byol_cast_f32_bf16_2d(const float* x, void* y, int rows, int cols, int ldx, int ldy,
                                     cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y && rows > 0 && cols > 0 && ldx >= cols && ldy >= cols, "byol_cast_f32_bf16_2d: bad args");
  cast_f32_bf16_2d_kernel<<<grid_for((int64_t)rows * ldy, 256), 256, 0, stream>>>(x, (bf16*)y, rows, cols, ldx, ldy);
  return check_launch("cast_f32_bf16_2d_kernel");
}

extern "C" int byol_cast_f32_bf16(const float* x, void* y, int64_t n, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y && n > 0, "byol_cast_f32_bf16: bad args");
  cast_f32_bf16_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, (bf16*)y, n);
  return check_launch("cast_f32_bf16_kernel");
}

extern "C" int byol_maxpool_fwd(const void* x, void* y, void* idx, int N, int H, int W, int C, int k, int s, int p,
                                cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y && C % 8 == 0 && k * k <= 255, "byol_maxpool_fwd: bad args");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
  const int64_t total = (int64_t)N * Ho * Wo * (C / 8);
  maxpool_fwd_kernel<<<grid_for(total, 256), 256, 0, stream>>>((const bf16*)x, (bf16*)y, (uint8_t*)idx, N, H, W, C,
                                                              Ho, Wo, k, s, p);
  return check_launch("maxpool_fwd_kernel");
}

// y = maxpool_kxk/s/p(relu(x*scale + shift)), idx as byol_maxpool_fwd (stem: BN-apply + ReLU + pool in one pass)
extern "C" int byol_bn_relu_maxpool_fwd(const void* x, const float* scale, const float* shift, void* y, void* idx,
                                        int N, int H, int W, int C, int k, int s, int p, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && scale && shift && y && C % 8 == 0 && k * k <= 255, "byol_bn_relu_maxpool_fwd: bad args");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
  const int64_t total = (int64_t)N * Ho * Wo * (C / 8);
  if (idx == nullptr) {
    bn_relu_maxpool_fwd_noidx_kernel<<<grid_for((int64_t)N * Ho * Wo * (C / 8), 256), 256, 0, stream>>>(
        (const bf16*)x, scale, shift, (bf16*)y, N, H, W, C, Ho, Wo, k, s, p);
    return check_launch("bn_relu_maxpool_fwd_noidx_kernel");
  }
  bn_relu_maxpool_fwd_kernel<<<grid_for(total, 256), 256, 0, stream>>>((const bf16*)x, scale, shift, (bf16*)y,
                                                                      (uint8_t*)idx, N, H, W, C, Ho, Wo, k, s, p);
  return check_launch("bn_relu_maxpool_fwd_kernel");
}

extern "C" int byol_maxpool_bwd(const void* dy, const void* idx, void* dx, int N, int H, int W, int C, int k, int s,
                                int p, cudaStream_t stream) {
  BYOL_CHECK_ARG(dy && idx && dx && C % 8 == 0, "byol_maxpool_bwd: bad args");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
  const int64_t total = (int64_t)N * H * W * (C / 8);
  if (k == 3 && s == 2 && p == 1 && H == 2 * Ho && W == 2 * Wo) {
    maxpool_bwd_k3s2_kernel<<<grid_for((int64_t)N * Ho * Wo * (C / 8), 256), 256, 0, stream>>>(
        (const bf16*)dy, (const uint8_t*)idx, (bf16*)dx, N, Ho, Wo, C);
    return check_launch("maxpool_bwd_k3s2_kernel");
  }
  maxpool_bwd_kernel<<<grid_for(total, 256), 256, 0, stream>>>((const bf16*)dy, (const uint8_t*)idx, (bf16*)dx, N, H,
                                                              W, C, Ho, Wo, k, s, p);
  return check_launch("maxpool_bwd_kernel");
}

extern "C" int byol_avgpool_fwd(const void* x, float* y_f32, void* y_bf16, int N, int HW, int C,
                                cudaStream_t stream) {
  BYOL_CHECK_ARG(x && (y_f32 || y_bf16) && C % 8 == 0 && HW > 0, "byol_avgpool_fwd: bad args");
  avgpool_fwd_kernel<<<grid_for((int64_t)N * (C / 8), 128), 128, 0, stream>>>((const bf16*)x, y_f32, (bf16*)y_bf16,
                                                                              N, HW, C);
  return check_launch("avgpool_fwd_kernel");
}

extern "C" int byol_avgpool_bwd(const void* g_bf16, const float* g_f32, void* dx, int N, int HW, int C,
                                cudaStream_t stream) {
  BYOL_CHECK_ARG((g_bf16 || g_f32) && dx && C % 8 == 0 && HW > 0, "byol_avgpool_bwd: bad args");
  avgpool_bwd_kernel<<<grid_for((int64_t)N * HW * (C / 8), 256), 256, 0, stream>>>((const bf16*)g_bf16, g_f32,
                                                                                    (bf16*)dx, N, HW, C);
  return check_launch("avgpool_bwd_kernel");
}
