// byol_b200 — GroupNorm (32 groups) and weight standardisation kernels for BYOL(norm="group_ws").
//
// GroupNorm normalises each image on its own (Wu & He 2018): the statistics of a conv output y [N, H, W, C] are per
// (image, group) over H * W * C/32 values, so an image's representation does not depend on the rest of its batch.
// Weight standardisation (Qiao et al. 2019) replaces every encoder conv weight row w_o (one output channel, fan-in
// Cin/groups * KH * KW values) by (w_o - mean(w_o)) / sqrt(var(w_o) + 1e-5), biased variance.
//
//   ws_fwd        : fp32 master rows -> standardised fp32 rows + (mean, rstd) per row           (one launch per set)
//   ws_bwd        : grad[w_o] += rstd * (dw^ - mean(dw^) - w^ * mean(dw^ * w^)) per row            (one launch)
//   gn_stats      : per (image, group) sum / sum of squares (fixed point) -> fp32 (mean, rstd)    (two launches)
//   gn_apply      : act(y * scale[n,c] + shift[n,c] (+ resid | + resid * rscale[n,c] + rshift[n,c])) + mask bits
//   gn_relu_maxpool_fwd : stem: maxpool(relu(gn(y))) without writing the normalised map
//   gn_bwd_reduce : per (image, group) s1 = sum gamma*dz, s2 = sum gamma*dz*xhat; per channel dbeta += sum dz,
//                   dgamma += sum dz*xhat
//   gn_bwd_apply  : dy = rstd * (gamma*dz - s1/m - xhat * s2/m)
//
// (the gradient of xhat is gamma_c * dz and differs between the channels of a group, so the group sums carry gamma)
//
// with scale = gamma_c * rstd[n, g] and shift = beta_c - mean[n, g] * scale.  Every fp32 operation is written with an
// explicit rounding intrinsic, so the tests restate the arithmetic exactly.  Sums that cross blocks go through the
// fixed-point scratch (fix_scratch / fix_flush): every run gives the same bits.
#include "common.cuh"

namespace byol {

static constexpr int kGroups = 32;
static constexpr int kThreads = 256;

__device__ __forceinline__ void gn_unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t = __bfloat1622float2(h[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 gn_pack8(const float (&f)[8]) {
  uint4 q;
  q.x = pack_bf16x2(f[0], f[1]);
  q.y = pack_bf16x2(f[2], f[3]);
  q.z = pack_bf16x2(f[4], f[5]);
  q.w = pack_bf16x2(f[6], f[7]);
  return q;
}

// fixed-order block sum of one double per thread (kThreads threads): warp butterflies, then warp 0 adds the eight
// warp partials in warp order.  Every thread gets the total.
__device__ __forceinline__ double block_sum_f64(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                       // sh may still be read by a previous call
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) t += sh[w];
  return t;
}

// the unit of row `row`: desc rows are {src offset in flat, offset in the scratch, Cout, fan-in, first row}
__device__ __forceinline__ int ws_unit(const int64_t* desc, int units, int64_t row) {
  int lo = 0, hi = units - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (desc[mid * 5 + 4] <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// One block per weight row.  Two passes in fp64 (mean, then the sum of squared deviations), each summed in a fixed
// order; w^ = (w - mean) * rstd in fp64, rounded once.  stats[row] = (fp32 mean, fp32 rstd), each rounded once.
__global__ void __launch_bounds__(kThreads)
ws_fwd_kernel(const float* __restrict__ flat, const int64_t* __restrict__ desc, int units, float* __restrict__ w_out,
              float* __restrict__ stats) {
  __shared__ double sh[kThreads / 32];
  const int64_t row = blockIdx.x;
  const int u = ws_unit(desc, units, row);
  const int64_t n = desc[u * 5 + 3];
  const int64_t r = row - desc[u * 5 + 4];
  const float* w = flat + desc[u * 5 + 0] + r * n;
  float* o = w_out + desc[u * 5 + 1] + r * n;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kThreads) s += (double)w[i];
  const double mean = block_sum_f64(s, sh) / (double)n;
  double q = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kThreads) {
    const double d = (double)w[i] - mean;
    q += d * d;
  }
  const double var = block_sum_f64(q, sh) / (double)n;
  const double rstd = 1.0 / sqrt(var + 1e-5);
  for (int64_t i = threadIdx.x; i < n; i += kThreads) o[i] = (float)(((double)w[i] - mean) * rstd);
  if (threadIdx.x == 0) {
    stats[2 * row] = (float)mean;
    stats[2 * row + 1] = (float)rstd;
  }
}

// One block per weight row: s1 = sum dw^, s2 = sum dw^ * w^ in fp64 (fixed order); grad += fp32 of
// rstd * (dw^ - s1/n - w^ * s2/n) evaluated in fp64.
__global__ void __launch_bounds__(kThreads)
ws_bwd_kernel(const float* __restrict__ dwhat, const float* __restrict__ what, const float* __restrict__ stats,
              const int64_t* __restrict__ desc, int units, float* __restrict__ grad) {
  __shared__ double sh[kThreads / 32];
  const int64_t row = blockIdx.x;
  const int u = ws_unit(desc, units, row);
  const int64_t n = desc[u * 5 + 3];
  const int64_t r = row - desc[u * 5 + 4];
  const int64_t so = desc[u * 5 + 1] + r * n;
  const float* g = dwhat + so;
  const float* wh = what + so;
  float* dst = grad + desc[u * 5 + 0] + r * n;
  double a = 0.0, b = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kThreads) {
    a += (double)g[i];
    b += (double)g[i] * (double)wh[i];
  }
  const double m1 = block_sum_f64(a, sh) / (double)n;
  const double m2 = block_sum_f64(b, sh) / (double)n;
  const double rstd = (double)stats[2 * row + 1];
  for (int64_t i = threadIdx.x; i < n; i += kThreads)
    dst[i] = __fadd_rn(dst[i], (float)(rstd * ((double)g[i] - m1 - (double)wh[i] * m2)));
}

// ---------------------------------------------------------------------------------------------
// GroupNorm.  Grid (blocks per image, N); block b of an image covers its 8-channel vectors [b * chunk, (b+1) * chunk)
// with chunk a multiple of kThreads, thread t the vectors t, t + 256, ...  When C/8 divides 256 (every C of the
// torchvision ResNets and ResNeXts: 64 ... 2048) a thread stays on one channel vector (and one or more whole groups)
// for its whole loop.  Other widths (C = 96, 4096, ...) are handled but change a thread's channel vector on every
// iteration: the coefficients are then reloaded and the backward reduction flushes its partials per vector, a slower
// route than the pinned one.
// ---------------------------------------------------------------------------------------------
struct GnGeom {
  int64_t vecs;     // 8-channel vectors per image = HW * C / 8
  int64_t chunk;    // vectors per block
  int cvecs;        // C / 8
  int cpg;          // channels per group = C / 32
};

// red: [32][2] Fix128 (sum, sum of squares) of this block's image
__device__ __forceinline__ void gn_stats_flush(Fix128* red, int cv, int cpg, const double (&s)[8],
                                               const double (&q)[8]) {
  double a = 0.0, b = 0.0;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int g = (cv * 8 + e) / cpg;
    a += s[e];
    b += q[e];
    if (e == 7 || (cv * 8 + e + 1) / cpg != g) {    // last channel of a group within this vector
      fix_add(red + 2 * g, a);
      fix_add(red + 2 * g + 1, b);
      a = 0.0;
      b = 0.0;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
gn_stats_kernel(const bf16* __restrict__ y, Fix128* __restrict__ acc, GnGeom gm) {
  __shared__ Fix128 red[2 * kGroups];
  if (threadIdx.x < 2 * kGroups) red[threadIdx.x] = Fix128{0ull, 0ll, 0.0};
  __syncthreads();
  const int n = blockIdx.y;
  const uint4* src = reinterpret_cast<const uint4*>(y) + (int64_t)n * gm.vecs;
  const int64_t beg = blockIdx.x * gm.chunk;
  const int64_t end = beg + gm.chunk < gm.vecs ? beg + gm.chunk : gm.vecs;
  int cur = -1;
  double s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { s[e] = 0.0; q[e] = 0.0; }
  for (int64_t i = beg + threadIdx.x; i < end; i += kThreads) {
    const int cv = (int)(i % gm.cvecs);
    if (cv != cur) {
      if (cur >= 0) gn_stats_flush(red, cur, gm.cpg, s, q);
#pragma unroll
      for (int e = 0; e < 8; ++e) { s[e] = 0.0; q[e] = 0.0; }
      cur = cv;
    }
    float v[8];
    gn_unpack8(__ldg(src + i), v);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const double d = (double)v[e];
      s[e] += d;
      q[e] = fma(d, d, q[e]);
    }
  }
  if (cur >= 0) gn_stats_flush(red, cur, gm.cpg, s, q);
  __syncthreads();
  if (threadIdx.x < 2 * kGroups) fix_add_raw(acc + (int64_t)n * 2 * kGroups + threadIdx.x, red[threadIdx.x]);
}

// (sum, sum of squares) of every (image, group) -> fp32 (mean, rstd), computed in fp64 and rounded once; the
// accumulators are left at zero.  sums64 (optional): the fp64 values of the sums.
__global__ void gn_finalize_kernel(Fix128* __restrict__ acc, float* __restrict__ out, double* __restrict__ sums64,
                                   int NG, double count, double eps) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= NG) return;
  const double s = fix_value(acc[2 * k]), q = fix_value(acc[2 * k + 1]);
  acc[2 * k] = Fix128{0ull, 0ll, 0.0};
  acc[2 * k + 1] = Fix128{0ull, 0ll, 0.0};
  const double mean = s / count;
  double var = q / count - mean * mean;
  if (var < 0.0) var = 0.0;
  out[2 * k] = (float)mean;
  out[2 * k + 1] = (float)(1.0 / sqrt(var + eps));
  if (sums64 != nullptr) {
    sums64[2 * k] = s;
    sums64[2 * k + 1] = q;
  }
}

// per-channel scale / shift of image n for the channels of vector cv
__device__ __forceinline__ void gn_coeffs(const float* __restrict__ gamma, const float* __restrict__ beta,
                                          const float* __restrict__ st, int cv, int cpg, float (&sc)[8],
                                          float (&sh)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = cv * 8 + e;
    const int g = c / cpg;
    sc[e] = __fmul_rn(__ldg(gamma + c), __ldg(st + 2 * g + 1));
    sh[e] = __fmaf_rn(-__ldg(st + 2 * g), sc[e], __ldg(beta + c));
  }
}

// RESID: 0 none, 1 plain bf16 residual, 2 GroupNorm-applied residual (rgamma, rbeta, rstats: the downsample branch)
template <int RESID>
__global__ void __launch_bounds__(kThreads)
gn_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                const float* __restrict__ stats, const bf16* __restrict__ resid, const float* __restrict__ rgamma,
                const float* __restrict__ rbeta, const float* __restrict__ rstats, bf16* __restrict__ y,
                uint8_t* __restrict__ mask_out, GnGeom gm, int relu) {
  const int n = blockIdx.y;
  const int64_t base = (int64_t)n * gm.vecs;
  const float* st = stats + n * 2 * kGroups;
  const float* rst = RESID == 2 ? rstats + n * 2 * kGroups : nullptr;
  const int64_t beg = blockIdx.x * gm.chunk;
  const int64_t end = beg + gm.chunk < gm.vecs ? beg + gm.chunk : gm.vecs;
  int cur = -1;
  float sc[8], sh[8], rs[8], rb[8];
  for (int64_t i = beg + threadIdx.x; i < end; i += kThreads) {
    const int cv = (int)(i % gm.cvecs);
    if (cv != cur) {
      gn_coeffs(gamma, beta, st, cv, gm.cpg, sc, sh);
      if (RESID == 2) gn_coeffs(rgamma, rbeta, rst, cv, gm.cpg, rs, rb);
      cur = cv;
    }
    float xv[8], o[8];
    gn_unpack8(__ldg(reinterpret_cast<const uint4*>(x) + base + i), xv);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = __fmaf_rn(xv[e], sc[e], sh[e]);
    if (RESID != 0) {
      float rv[8];
      gn_unpack8(__ldg(reinterpret_cast<const uint4*>(resid) + base + i), rv);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = __fadd_rn(o[e], RESID == 2 ? __fmaf_rn(rv[e], rs[e], rb[e]) : rv[e]);
    }
    if (relu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = fmaxf(o[e], 0.f);
    }
    reinterpret_cast<uint4*>(y)[base + i] = gn_pack8(o);
    if (mask_out != nullptr) {
      uint32_t b = 0;
#pragma unroll
      for (int e = 0; e < 8; ++e) b |= (o[e] > 0.f ? 1u : 0u) << e;
      mask_out[base + i] = (uint8_t)b;
    }
  }
}

// Stem: y = maxpool(relu(gn(x))), one thread per (output pixel, 8-channel vector).  Candidates are rounded to bf16
// before the comparison, so values and argmax indices equal gn_apply followed by maxpool_fwd bit for bit.
__global__ void __launch_bounds__(kThreads)
gn_relu_maxpool_fwd_kernel(const bf16* __restrict__ x, const float* __restrict__ gamma,
                           const float* __restrict__ beta, const float* __restrict__ stats, bf16* __restrict__ y,
                           uint8_t* __restrict__ idx, int N, int H, int W, int C, int Ho, int Wo, int k, int s, int p) {
  const int cvecs = C >> 3, cpg = C / kGroups;
  const int64_t total = (int64_t)N * Ho * Wo * cvecs;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % cvecs);
    int64_t t = i / cvecs;
    const int ow = (int)(t % Wo); t /= Wo;
    const int oh = (int)(t % Ho);
    const int n = (int)(t / Ho);
    float sc[8], sh[8], best[8];
    int bi[8];
    gn_coeffs(gamma, beta, stats + n * 2 * kGroups, cv, cpg, sc, sh);
    // a window whose in-image values are all -inf reports its first in-image position (maxpool_fwd)
    const int first = (p - oh * s > 0 ? p - oh * s : 0) * k + (p - ow * s > 0 ? p - ow * s : 0);
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; bi[e] = first; }
    for (int kh = 0; kh < k; ++kh) {
      const int ih = oh * s - p + kh;
      if (ih < 0 || ih >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int iw = ow * s - p + kw;
        if (iw < 0 || iw >= W) continue;
        float v[8];
        gn_unpack8(__ldg(reinterpret_cast<const uint4*>(x + (((int64_t)n * H + ih) * W + iw) * C + cv * 8)), v);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float a = __bfloat162float(__float2bfloat16_rn(fmaxf(__fmaf_rn(v[e], sc[e], sh[e]), 0.f)));
          if (a > best[e] || a != a) { best[e] = a; bi[e] = kh * k + kw; }
        }
      }
    }
    reinterpret_cast<uint4*>(y)[i] = gn_pack8(best);
    if (idx != nullptr) {
      uint2 pk;
      pk.x = (uint32_t)bi[0] | ((uint32_t)bi[1] << 8) | ((uint32_t)bi[2] << 16) | ((uint32_t)bi[3] << 24);
      pk.y = (uint32_t)bi[4] | ((uint32_t)bi[5] << 8) | ((uint32_t)bi[6] << 16) | ((uint32_t)bi[7] << 24);
      reinterpret_cast<uint2*>(idx)[i] = pk;
    }
  }
}

// dz = g masked: MASK 0 none, 1 ReLU recomputed (x * scale + shift > 0), 2 act > 0 (bf16), 3 mask bits (uint8)
template <int MASK>
__device__ __forceinline__ void gn_mask(float (&gv)[8], const float (&xv)[8], const bf16* __restrict__ act, int64_t i,
                                        const float (&sc)[8], const float (&sh)[8]) {
  if (MASK == 3) {
    const uint32_t mb = __ldg(reinterpret_cast<const uint8_t*>(act) + i);
#pragma unroll
    for (int e = 0; e < 8; ++e) gv[e] = ((mb >> e) & 1u) ? gv[e] : 0.f;
  } else if (MASK == 2) {
    float av[8];
    gn_unpack8(__ldg(reinterpret_cast<const uint4*>(act) + i), av);
#pragma unroll
    for (int e = 0; e < 8; ++e) gv[e] = av[e] > 0.f ? gv[e] : 0.f;
  } else if (MASK == 1) {
#pragma unroll
    for (int e = 0; e < 8; ++e) gv[e] = __fmaf_rn(xv[e], sc[e], sh[e]) > 0.f ? gv[e] : 0.f;
  }
}

__device__ __forceinline__ void gn_norm_params(const float* __restrict__ st, int cv, int cpg, float (&mu)[8],
                                               float (&rs)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int g = (cv * 8 + e) / cpg;
    mu[e] = __ldg(st + 2 * g);
    rs[e] = __ldg(st + 2 * g + 1);
  }
}

// red layout: [32][2] (s1, s2) of this block's image, then [C] sum dz, then [C] sum dz * xhat
__device__ __forceinline__ void gn_bwd_flush(Fix128* red, const float* __restrict__ gamma, int C, int cv, int cpg,
                                             const double (&a)[8], const double (&b)[8]) {
  double ga[8], gb[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    fix_add(red + 2 * kGroups + cv * 8 + e, a[e]);
    fix_add(red + 2 * kGroups + C + cv * 8 + e, b[e]);
    const double gm = (double)__ldg(gamma + cv * 8 + e);
    ga[e] = gm * a[e];
    gb[e] = gm * b[e];
  }
  gn_stats_flush(red, cv, cpg, ga, gb);
}

template <int MASK>
__global__ void __launch_bounds__(kThreads)
gn_bwd_reduce_kernel(const bf16* __restrict__ g, const bf16* __restrict__ x, const bf16* __restrict__ act,
                     const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ stats,
                     Fix128* __restrict__ acc_g, Fix128* __restrict__ acc_c, GnGeom gm) {
  extern __shared__ Fix128 red[];
  const int C = gm.cvecs * 8;
  for (int j = threadIdx.x; j < 2 * kGroups + 2 * C; j += kThreads) red[j] = Fix128{0ull, 0ll, 0.0};
  __syncthreads();
  const int n = blockIdx.y;
  const int64_t base = (int64_t)n * gm.vecs;
  const float* st = stats + n * 2 * kGroups;
  const int64_t beg = blockIdx.x * gm.chunk;
  const int64_t end = beg + gm.chunk < gm.vecs ? beg + gm.chunk : gm.vecs;
  int cur = -1;
  float sc[8], sh[8], mu[8], rs[8];
  double a[8], b[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { a[e] = 0.0; b[e] = 0.0; sc[e] = 0.f; sh[e] = 0.f; }
  for (int64_t i = beg + threadIdx.x; i < end; i += kThreads) {
    const int cv = (int)(i % gm.cvecs);
    if (cv != cur) {
      if (cur >= 0) gn_bwd_flush(red, gamma, C, cur, gm.cpg, a, b);
#pragma unroll
      for (int e = 0; e < 8; ++e) { a[e] = 0.0; b[e] = 0.0; }
      gn_norm_params(st, cv, gm.cpg, mu, rs);
      if (MASK == 1) gn_coeffs(gamma, beta, st, cv, gm.cpg, sc, sh);
      cur = cv;
    }
    float gv[8], xv[8];
    gn_unpack8(__ldg(reinterpret_cast<const uint4*>(g) + base + i), gv);
    gn_unpack8(__ldg(reinterpret_cast<const uint4*>(x) + base + i), xv);
    gn_mask<MASK>(gv, xv, act, base + i, sc, sh);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float xh = __fmul_rn(__fsub_rn(xv[e], mu[e]), rs[e]);
      a[e] += (double)gv[e];
      b[e] = fma((double)gv[e], (double)xh, b[e]);
    }
  }
  if (cur >= 0) gn_bwd_flush(red, gamma, C, cur, gm.cpg, a, b);
  __syncthreads();
  if (threadIdx.x < 2 * kGroups) fix_add_raw(acc_g + (int64_t)n * 2 * kGroups + threadIdx.x, red[threadIdx.x]);
  for (int j = threadIdx.x; j < 2 * C; j += kThreads) fix_add_raw(acc_c + j, red[2 * kGroups + j]);
}

// dy = rstd * (gamma*dz - s1/m - xhat * s2/m), with s12 [N][32][2] the image's (s1, s2)
template <int MASK>
__global__ void __launch_bounds__(kThreads)
gn_bwd_apply_kernel(const bf16* __restrict__ g, const bf16* __restrict__ x, const bf16* __restrict__ act,
                    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ stats,
                    const float* __restrict__ s12, float inv_m, bf16* __restrict__ dy, bf16* __restrict__ dz_out,
                    GnGeom gm) {
  const int n = blockIdx.y;
  const int64_t base = (int64_t)n * gm.vecs;
  const float* st = stats + n * 2 * kGroups;
  const float* ss = s12 + n * 2 * kGroups;
  const int64_t beg = blockIdx.x * gm.chunk;
  const int64_t end = beg + gm.chunk < gm.vecs ? beg + gm.chunk : gm.vecs;
  int cur = -1;
  float sc[8], sh[8], mu[8], rs[8], ga[8], m1[8], m2[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { sc[e] = 0.f; sh[e] = 0.f; }
  for (int64_t i = beg + threadIdx.x; i < end; i += kThreads) {
    const int cv = (int)(i % gm.cvecs);
    if (cv != cur) {
      gn_norm_params(st, cv, gm.cpg, mu, rs);
      if (MASK == 1) gn_coeffs(gamma, beta, st, cv, gm.cpg, sc, sh);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int c = cv * 8 + e, gi = c / gm.cpg;
        ga[e] = __ldg(gamma + c);
        m1[e] = __fmul_rn(__ldg(ss + 2 * gi), inv_m);
        m2[e] = __fmul_rn(__ldg(ss + 2 * gi + 1), inv_m);
      }
      cur = cv;
    }
    float gv[8], xv[8], o[8];
    gn_unpack8(__ldg(reinterpret_cast<const uint4*>(g) + base + i), gv);
    gn_unpack8(__ldg(reinterpret_cast<const uint4*>(x) + base + i), xv);
    gn_mask<MASK>(gv, xv, act, base + i, sc, sh);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float xh = __fmul_rn(__fsub_rn(xv[e], mu[e]), rs[e]);
      o[e] = __fmul_rn(rs[e], __fsub_rn(__fsub_rn(__fmul_rn(ga[e], gv[e]), m1[e]), __fmul_rn(xh, m2[e])));
    }
    reinterpret_cast<uint4*>(dy)[base + i] = gn_pack8(o);
    if (dz_out != nullptr) reinterpret_cast<uint4*>(dz_out)[base + i] = gn_pack8(gv);
  }
}

// About 32 vectors per thread.  The partition of an image over blocks and threads depends on its own shape (HW, C)
// only, never on the batch size N: the per-thread fp64 partials and their fixed-point rounding, and so the statistics'
// bits, are the same for an image computed alone and inside any batch.
static GnGeom gn_geom(int HW, int C) {
  GnGeom gm;
  gm.cvecs = C / 8;
  gm.cpg = C / kGroups;
  gm.vecs = (int64_t)HW * gm.cvecs;
  const int64_t per = (int64_t)kThreads * 32;
  const int64_t blocks = (gm.vecs + per - 1) / per;
  gm.chunk = (gm.vecs + blocks - 1) / blocks;
  gm.chunk = (gm.chunk + kThreads - 1) / kThreads * kThreads;
  return gm;
}
static dim3 gn_grid(const GnGeom& gm, int N) { return dim3((unsigned)((gm.vecs + gm.chunk - 1) / gm.chunk), (unsigned)N); }

static bool gn_shape_ok(int N, int HW, int C) {
  return N > 0 && N <= 65535 && HW > 0 && C > 0 && C % 8 == 0 && C % kGroups == 0;
}

}  // namespace byol

using namespace byol;

extern "C" int byol_ws_fwd(const float* flat, const int64_t* desc, int num_units, int64_t num_rows, float* w_out,
                           float* stats, cudaStream_t stream) {
  BYOL_CHECK_ARG(flat && desc && w_out && stats && num_units > 0 && num_rows > 0 && num_rows < (1ll << 31),
                 "byol_ws_fwd: bad args");
  ws_fwd_kernel<<<(unsigned)num_rows, kThreads, 0, stream>>>(flat, desc, num_units, w_out, stats);
  return check_launch("ws_fwd_kernel");
}

extern "C" int byol_ws_bwd(const float* dwhat, const float* what, const float* stats, const int64_t* desc,
                           int num_units, int64_t num_rows, float* grad, cudaStream_t stream) {
  BYOL_CHECK_ARG(dwhat && what && stats && desc && grad && num_units > 0 && num_rows > 0 && num_rows < (1ll << 31),
                 "byol_ws_bwd: bad args");
  ws_bwd_kernel<<<(unsigned)num_rows, kThreads, 0, stream>>>(dwhat, what, stats, desc, num_units, grad);
  return check_launch("ws_bwd_kernel");
}

extern "C" int byol_gn_stats(const void* y, float* stats, double* sums64, int N, int HW, int C, float eps,
                             cudaStream_t stream) {
  BYOL_CHECK_ARG(y && stats && gn_shape_ok(N, HW, C), "byol_gn_stats: bad args (N=%d HW=%d C=%d)", N, HW, C);
  const GnGeom gm = gn_geom(HW, C);
  const int NG = N * kGroups;
  Fix128* fx = fix_scratch(stream, 2 * (int64_t)NG);
  if (fx == nullptr) return -2;
  gn_stats_kernel<<<gn_grid(gm, N), kThreads, 0, stream>>>((const bf16*)y, fx, gm);
  if (check_launch("gn_stats_kernel") != 0) return -100;
  gn_finalize_kernel<<<(NG + 127) / 128, 128, 0, stream>>>(fx, stats, sums64, NG, (double)HW * (C / kGroups),
                                                          (double)eps);
  return fix_done(stream, check_launch("gn_finalize_kernel"));
}

extern "C" int byol_gn_apply(const void* x, const float* gamma, const float* beta, const float* stats,
                             const void* resid, const float* rgamma, const float* rbeta, const float* rstats, void* y,
                             void* mask_out, int N, int HW, int C, int relu, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && gamma && beta && stats && y && gn_shape_ok(N, HW, C), "byol_gn_apply: bad args");
  BYOL_CHECK_ARG(rgamma == nullptr || (resid && rbeta && rstats), "byol_gn_apply: rgamma needs resid, rbeta, rstats");
  const GnGeom gm = gn_geom(HW, C);
  const dim3 grid = gn_grid(gm, N);
  const bf16 *xp = (const bf16*)x, *rp = (const bf16*)resid;
  uint8_t* mo = (uint8_t*)mask_out;
  if (resid == nullptr)
    gn_apply_kernel<0><<<grid, kThreads, 0, stream>>>(xp, gamma, beta, stats, rp, rgamma, rbeta, rstats, (bf16*)y, mo, gm, relu);
  else if (rgamma == nullptr)
    gn_apply_kernel<1><<<grid, kThreads, 0, stream>>>(xp, gamma, beta, stats, rp, rgamma, rbeta, rstats, (bf16*)y, mo, gm, relu);
  else
    gn_apply_kernel<2><<<grid, kThreads, 0, stream>>>(xp, gamma, beta, stats, rp, rgamma, rbeta, rstats, (bf16*)y, mo, gm, relu);
  return check_launch("gn_apply_kernel");
}

extern "C" int byol_gn_relu_maxpool_fwd(const void* x, const float* gamma, const float* beta, const float* stats,
                                        void* y, void* idx, int N, int H, int W, int C, int k, int s, int p,
                                        cudaStream_t stream) {
  BYOL_CHECK_ARG(x && gamma && beta && stats && y && gn_shape_ok(N, H * W, C) && k * k <= 255,
                 "byol_gn_relu_maxpool_fwd: bad args");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
  const int64_t total = (int64_t)N * Ho * Wo * (C / 8);
  int64_t blocks = (total + kThreads - 1) / kThreads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  gn_relu_maxpool_fwd_kernel<<<(unsigned)blocks, kThreads, 0, stream>>>((const bf16*)x, gamma, beta, stats, (bf16*)y,
                                                                        (uint8_t*)idx, N, H, W, C, Ho, Wo, k, s, p);
  return check_launch("gn_relu_maxpool_fwd_kernel");
}

extern "C" int byol_gn_bwd_reduce(const void* g, const void* x, const void* act, const float* gamma, const float* beta,
                                  const float* stats, float* s12, float* dgamma, float* dbeta, int N, int HW, int C,
                                  int mask_mode, cudaStream_t stream) {
  BYOL_CHECK_ARG(g && x && gamma && beta && stats && s12 && gn_shape_ok(N, HW, C), "byol_gn_bwd_reduce: bad args");
  BYOL_CHECK_ARG(mask_mode >= 0 && mask_mode <= 3 && (mask_mode < 2 || act), "byol_gn_bwd_reduce: bad mask_mode %d",
                 mask_mode);
  // dgamma / dbeta are required: the kernel always accumulates the per-channel sums, and only their flush leaves the
  // stream's scratch zeroed for a CUDA graph captured earlier on this stream (its replay does not clear the scratch)
  BYOL_CHECK_ARG(dgamma && dbeta, "byol_gn_bwd_reduce: dgamma and dbeta are required");
  const GnGeom gm = gn_geom(HW, C);
  const int64_t ng2 = (int64_t)N * 2 * kGroups;
  const size_t red_bytes = (2 * kGroups + 2 * (size_t)C) * sizeof(Fix128);
  BYOL_CHECK_ARG(red_bytes <= 226 * 1024, "byol_gn_bwd_reduce: C=%d too wide", C);
  Fix128* fx = fix_scratch(stream, ng2 + 2 * (int64_t)C);
  if (fx == nullptr) return -2;
  static const decltype(&gn_bwd_reduce_kernel<0>) kernels[4] = {gn_bwd_reduce_kernel<0>, gn_bwd_reduce_kernel<1>,
                                                                 gn_bwd_reduce_kernel<2>, gn_bwd_reduce_kernel<3>};
  const auto kern = kernels[mask_mode];
  if (smem_opt_in((const void*)kern, (int)red_bytes, "gn_bwd_reduce_kernel") != 0) return -2;
  kern<<<gn_grid(gm, N), kThreads, red_bytes, stream>>>((const bf16*)g, (const bf16*)x, (const bf16*)act, gamma, beta,
                                                        stats, fx, fx + ng2, gm);
  if (check_launch("gn_bwd_reduce_kernel") != 0) return -100;
  if (fix_flush(fx, s12, ng2, stream) != 0) return -100;
  if (fix_flush(fx + ng2, dbeta, C, stream) != 0) return -100;
  if (fix_flush(fx + ng2 + C, dgamma, C, stream) != 0) return -100;
  return fix_done(stream, 0);
}

extern "C" int byol_gn_bwd_apply(const void* g, const void* x, const void* act, const float* gamma, const float* beta,
                                 const float* stats, const float* s12, void* dy, void* dz_out, int N, int HW, int C,
                                 int mask_mode, cudaStream_t stream) {
  BYOL_CHECK_ARG(g && x && gamma && beta && stats && s12 && dy && gn_shape_ok(N, HW, C), "byol_gn_bwd_apply: bad args");
  BYOL_CHECK_ARG(mask_mode >= 0 && mask_mode <= 3 && (mask_mode < 2 || act), "byol_gn_bwd_apply: bad mask_mode %d",
                 mask_mode);
  const GnGeom gm = gn_geom(HW, C);
  const dim3 grid = gn_grid(gm, N);
  const float inv_m = (float)(1.0 / ((double)HW * (C / kGroups)));
  const bf16 *gp = (const bf16*)g, *xp = (const bf16*)x, *ap = (const bf16*)act;
  static const decltype(&gn_bwd_apply_kernel<0>) kernels[4] = {gn_bwd_apply_kernel<0>, gn_bwd_apply_kernel<1>,
                                                                gn_bwd_apply_kernel<2>, gn_bwd_apply_kernel<3>};
  kernels[mask_mode]<<<grid, kThreads, 0, stream>>>(gp, xp, ap, gamma, beta, stats, s12, inv_m, (bf16*)dy,
                                                    (bf16*)dz_out, gm);
  return check_launch("gn_bwd_apply_kernel");
}
