// byol_b200 — the fp32-accurate forward path ("split-bf16"): elementwise kernels.
//
// BASELINE.json configs[1] asks for the reference's fp32 results (/root/reference/main.py:229-276 runs every conv /
// linear / BatchNorm in fp32) within 1e-3.  The tensor cores have no fp32 MMA, and single-pass TF32 misses that bar by two orders
// of magnitude on a randomly initialised ResNet-50 (DESIGN.md §4: 5-19 % relative error, bf16 30-80 %), so the
// accurate path keeps the bf16 tensor-core kernels and feeds them EXACT SPLITS of the fp32 operands instead:
//
//     x = x0 + x1 + x2 (+ 2^-24 |x|),   x0 = bf16(x), x1 = bf16(x - x0), x2 = bf16(x - x0 - x1)
//     x * w  ~=  x0 w0 + x0 w1 + x1 w0 + x1 w1 + x0 w2 + x2 w0        (T = 6 terms; dropped terms <= 2^-24 |x w|)
//
// Every product of two bf16 values is exact in the fp32 accumulator, so a convolution over K input channels becomes
// ONE ordinary implicit GEMM over T*K channels: the activation tensor stores T "planes" per channel
// (channel index j*C + c holds plane A_PAT[j] of channel c) and the weight matrix the matching planes B_PAT[j].
// T = 3 (A = 0,0,1 / B = 0,1,0) gives ~2^-16 operands ("bf16x2"), T = 6 the full 24 bits.  The existing
// conv_igemm_kernel runs unchanged (C := T*C, fp32 epilogue); this file holds the producers of the plane layout and
// fp32 versions of the BatchNorm / pooling passes (statistics accumulated in fp64).
#include "common.cuh"

namespace byol {

struct SplitPattern {
  int T;
  int a[6];   // plane index of term j on the activation side
  int b[6];   // plane index of term j on the weight side
};

static inline SplitPattern make_pattern(int T) {
  SplitPattern p;
  p.T = T;
  const int a3[6] = {0, 0, 1, 0, 0, 0}, b3[6] = {0, 1, 0, 0, 0, 0};
  const int a6[6] = {0, 0, 1, 1, 0, 2}, b6[6] = {0, 1, 0, 1, 2, 0};
  for (int j = 0; j < 6; ++j) {
    p.a[j] = T == 3 ? a3[j] : a6[j];
    p.b[j] = T == 3 ? b3[j] : b6[j];
  }
  return p;
}

// A finite |x| >= 0x7F7F8000 (~3.3962e38) rounds to +-inf in bf16: x0 is then the largest finite bf16 of x's sign
// instead, so that x - x0 stays exact (Sterbenz) and the planes still sum to x.  Non-finite x keeps its planes
// (+-inf, NaN, NaN) / (NaN, NaN, NaN): every output such an element reaches is NaN.
__device__ __forceinline__ void split3(float x, bf16 (&pl)[3]) {
  const uint32_t u = __float_as_uint(x);
  // |x| in [0x7F7F8000, 0x7F7FFFFF]: truncating to the top 16 bits gives +-0x7F7F
  pl[0] = (u & 0x7FFFFFFFu) - 0x7F7F8000u < 0x8000u ? __ushort_as_bfloat16((unsigned short)(u >> 16))
                                                    : __float2bfloat16_rn(x);
  const float r1 = x - __bfloat162float(pl[0]);          // exact (Sterbenz-like: |r1| <= 2^-9 |x|)
  pl[1] = __float2bfloat16_rn(r1);
  const float r2 = r1 - __bfloat162float(pl[1]);         // exact
  pl[2] = __float2bfloat16_rn(r2);
}

static inline int grid_for(int64_t n, int block, int max_blocks = 132 * 16) {
  int64_t b = (n + block - 1) / block;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return (int)b;
}

// ---------------------------------------------------------------------------------------------
// fp32 [M, C] (row pitch ldx) -> planes bf16 [M, T*Cpad]  (+ optional plain bf16 copy [M, C] for the backward pass)
// one thread per (row, channel)
// ---------------------------------------------------------------------------------------------
__global__ void split_planes_kernel(const float* __restrict__ x, bf16* __restrict__ planes, bf16* __restrict__ copy,
                                    int64_t M, int C, int Cpad, int ldx, SplitPattern pat) {
  const int64_t total = M * Cpad;
  const int64_t row_elems = (int64_t)pat.T * Cpad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t m = i / Cpad;
    bf16 pl[3];
    split3(c < C ? x[m * ldx + c] : 0.f, pl);
    bf16* o = planes + m * row_elems + c;
#pragma unroll
    for (int j = 0; j < 6; ++j)
      if (j < pat.T) o[(int64_t)j * Cpad] = pl[pat.a[j]];
    if (copy != nullptr && c < C) copy[m * C + c] = pl[0];
  }
}

// fp32 NCHW image [N, Cin, H, W] -> planes NHWC bf16 [N, H, W, T*Cpad] (Cpad = 8: zero channels beyond Cin)
__global__ void nchw_to_planes_kernel(const float* __restrict__ x, bf16* __restrict__ planes, int N, int Cin, int H,
                                      int W, int Cpad, SplitPattern pat) {
  const int64_t npix = (int64_t)N * H * W;
  const int64_t total = npix * Cpad;
  const int64_t row_elems = (int64_t)pat.T * Cpad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t pix = i / Cpad;
    const int64_t hw = pix % ((int64_t)H * W);
    const int64_t n = pix / ((int64_t)H * W);
    bf16 pl[3];
    split3(c < Cin ? x[(n * Cin + c) * (int64_t)H * W + hw] : 0.f, pl);
    bf16* o = planes + pix * row_elems + c;
#pragma unroll
    for (int j = 0; j < 6; ++j)
      if (j < pat.T) o[(int64_t)j * Cpad] = pl[pat.a[j]];
  }
}

// fp32 weight [Cout, Cin, taps] (the reference's [Cout, Cin, KH, KW]) -> bf16 [Cout, taps * T * Cpad],
// column (tap*T + j)*Cpad + c = plane B_PAT[j] of w[n, c, tap]
__global__ void prep_weight_planes_kernel(const float* __restrict__ w, bf16* __restrict__ out, int Cout, int Cin,
                                          int Cpad, int taps, SplitPattern pat) {
  const int64_t total = (int64_t)Cout * taps * Cpad;
  const int64_t row_elems = (int64_t)taps * pat.T * Cpad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    int64_t t = i / Cpad;
    const int tap = (int)(t % taps);
    const int64_t n = t / taps;
    bf16 pl[3];
    split3(c < Cin ? w[(n * Cin + c) * taps + tap] : 0.f, pl);
    bf16* o = out + n * row_elems + (int64_t)tap * pat.T * Cpad + c;
#pragma unroll
    for (int j = 0; j < 6; ++j)
      if (j < pat.T) o[(int64_t)j * Cpad] = pl[pat.b[j]];
  }
}

// ---------------------------------------------------------------------------------------------
// BatchNorm statistics of an fp32 [M, C] matrix, accumulated in fp64: stats[0:C] += sum, stats[C:2C] += sum of squares
// block = 256 threads = (256 / CT) row lanes x CT columns (CT = min(C, 256)); grid.x strides rows, grid.y tiles columns
// ---------------------------------------------------------------------------------------------
// part: [gridDim.x][2][C] fp64 partial sums, one slot per row block (summed in block order by stats_f32_sum_kernel, so
// the statistics are the same bits in every run at full fp64 precision)
__global__ void stats_f32_kernel(const float* __restrict__ y, double* __restrict__ part, int64_t M, int C, int CT,
                                 int64_t rows_per_block) {
  const int col = blockIdx.y * CT + (int)(threadIdx.x % CT);
  const int rlane = (int)(threadIdx.x / CT);
  const int lanes = (int)(blockDim.x / CT);
  const int64_t r0 = blockIdx.x * rows_per_block;
  int64_t r1 = r0 + rows_per_block;
  if (r1 > M) r1 = M;
  double s = 0.0, q = 0.0;
  if (col < C) {
    for (int64_t r = r0 + rlane; r < r1; r += lanes) {
      const double v = (double)y[r * C + col];
      s += v;
      q += v * v;
    }
  }
  __shared__ double sh[2][256];
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = q;
  __syncthreads();
  if (rlane == 0 && col < C) {
    for (int l = 1; l < lanes; ++l) {
      s += sh[0][l * CT + (threadIdx.x % CT)];
      q += sh[1][l * CT + (threadIdx.x % CT)];
    }
    part[(int64_t)blockIdx.x * 2 * C + col] = s;
    part[(int64_t)blockIdx.x * 2 * C + C + col] = q;
  }
}

// fp64 statistics -> [scale, shift, mean, invstd] per lane, running statistics updated lane after lane
// (same contract as bn_finalize_lanes_kernel in bn.cu, which takes the fp32 sums of the bf16 path)
struct LanePtrs64 { const float* p[4]; };
__global__ void bn_finalize_lanes_f64_kernel(const double* __restrict__ stats, double count, LanePtrs64 gamma,
                                             LanePtrs64 beta, float* __restrict__ running_mean,
                                             float* __restrict__ running_var, float momentum, float eps,
                                             float* __restrict__ coeffs, int C, int L) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float rm = running_mean != nullptr ? running_mean[c] : 0.f;
  float rv = running_var != nullptr ? running_var[c] : 0.f;
  for (int l = 0; l < L; ++l) {
    const double* st = stats + (int64_t)l * 2 * C;
    const double mean = st[c] / count;
    double var = st[C + c] / count - mean * mean;   // biased
    if (var < 0.0) var = 0.0;
    // the reference (ATen batch_norm, fp32) computes invstd = 1/sqrt(var + eps) in fp32 from fp32 mean / var
    const float invstd = (float)(1.0 / sqrt(var + (double)eps));
    const float sc = gamma.p[l][c] * invstd;
    float* co = coeffs + (int64_t)l * 4 * C;
    co[c] = sc;
    co[C + c] = (float)((double)beta.p[l][c] - mean * (double)sc);
    co[2 * C + c] = (float)mean;
    co[3 * C + c] = invstd;
    const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    rm = (1.f - momentum) * rm + momentum * (float)mean;
    rv = (1.f - momentum) * rv + momentum * (float)unbiased;
  }
  if (running_mean != nullptr) {
    running_mean[c] = rm;
    running_var[c] = rv;
  }
}

// ---------------------------------------------------------------------------------------------
// o = act(y*scale + shift (+ resid | resid*rscale + rshift)) on fp32 [M, C]; any subset of the outputs:
//   out32 (fp32 [M, C]), planes (bf16 [M, T*C]), copy (bf16 [M, C]), mask (bit e of byte i = element 8i+e > 0)
// one thread per 8 consecutive channels
// ---------------------------------------------------------------------------------------------
__global__ void bn_apply_f32_kernel(const float* __restrict__ y, const float* __restrict__ scale,
                                    const float* __restrict__ shift, const float* __restrict__ resid,
                                    const float* __restrict__ rscale, const float* __restrict__ rshift,
                                    float* __restrict__ out32, bf16* __restrict__ planes, bf16* __restrict__ copy,
                                    uint8_t* __restrict__ mask, int64_t nvec, int C, int relu, SplitPattern pat) {
  const int groups = C >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const int64_t m = i / groups;
    float o[8];
    const float4 y0 = __ldg(reinterpret_cast<const float4*>(y) + 2 * i);
    const float4 y1 = __ldg(reinterpret_cast<const float4*>(y) + 2 * i + 1);
    const float yv[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = yv[e] * __ldg(scale + g * 8 + e) + __ldg(shift + g * 8 + e);
    if (resid != nullptr) {
      const float4 r0 = __ldg(reinterpret_cast<const float4*>(resid) + 2 * i);
      const float4 r1 = __ldg(reinterpret_cast<const float4*>(resid) + 2 * i + 1);
      const float rv[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e)
        o[e] += rscale != nullptr ? (rv[e] * __ldg(rscale + g * 8 + e) + __ldg(rshift + g * 8 + e)) : rv[e];
    }
    if (relu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = fmaxf(o[e], 0.f);
    }
    if (out32 != nullptr) {
      reinterpret_cast<float4*>(out32)[2 * i] = make_float4(o[0], o[1], o[2], o[3]);
      reinterpret_cast<float4*>(out32)[2 * i + 1] = make_float4(o[4], o[5], o[6], o[7]);
    }
    if (planes != nullptr || copy != nullptr) {
      bf16 pl[8][3];
#pragma unroll
      for (int e = 0; e < 8; ++e) split3(o[e], pl[e]);
      if (planes != nullptr) {
        bf16* base = planes + m * (int64_t)pat.T * C + g * 8;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          if (j < pat.T) {
            const int a = pat.a[j];
            uint4 q;
            __nv_bfloat162 h0 = __halves2bfloat162(pl[0][a], pl[1][a]), h1 = __halves2bfloat162(pl[2][a], pl[3][a]);
            __nv_bfloat162 h2 = __halves2bfloat162(pl[4][a], pl[5][a]), h3 = __halves2bfloat162(pl[6][a], pl[7][a]);
            q.x = *reinterpret_cast<uint32_t*>(&h0);
            q.y = *reinterpret_cast<uint32_t*>(&h1);
            q.z = *reinterpret_cast<uint32_t*>(&h2);
            q.w = *reinterpret_cast<uint32_t*>(&h3);
            *reinterpret_cast<uint4*>(base + (int64_t)j * C) = q;
          }
        }
      }
      if (copy != nullptr) {
        uint4 q;
        __nv_bfloat162 h0 = __halves2bfloat162(pl[0][0], pl[1][0]), h1 = __halves2bfloat162(pl[2][0], pl[3][0]);
        __nv_bfloat162 h2 = __halves2bfloat162(pl[4][0], pl[5][0]), h3 = __halves2bfloat162(pl[6][0], pl[7][0]);
        q.x = *reinterpret_cast<uint32_t*>(&h0);
        q.y = *reinterpret_cast<uint32_t*>(&h1);
        q.z = *reinterpret_cast<uint32_t*>(&h2);
        q.w = *reinterpret_cast<uint32_t*>(&h3);
        reinterpret_cast<uint4*>(copy)[i] = q;
      }
    }
    if (mask != nullptr) {
      uint32_t b = 0;
#pragma unroll
      for (int e = 0; e < 8; ++e) b |= (o[e] > 0.f ? 1u : 0u) << e;
      mask[i] = (uint8_t)b;
    }
  }
}

// max-pool (k x k, stride s, pad p) over fp32 NHWC; idx = window position of the first maximum (uint8, like the bf16 path)
__global__ void maxpool_f32_kernel(const float* __restrict__ x, float* __restrict__ y, uint8_t* __restrict__ idx, int N,
                                   int H, int W, int C, int Ho, int Wo, int k, int s, int p) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t t = i / C;
    const int ow = (int)(t % Wo); t /= Wo;
    const int oh = (int)(t % Ho);
    const int n = (int)(t / Ho);
    float best = -INFINITY;
    int bi = (p - oh * s > 0 ? p - oh * s : 0) * k + (p - ow * s > 0 ? p - ow * s : 0);   // all -inf: first in-image
    for (int kh = 0; kh < k; ++kh) {
      const int ih = oh * s - p + kh;
      if (ih < 0 || ih >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int iw = ow * s - p + kw;
        if (iw < 0 || iw >= W) continue;
        const float v = x[(((int64_t)n * H + ih) * W + iw) * C + c];
        if (v > best || v != v) { best = v; bi = kh * k + kw; }
      }
    }
    y[i] = best;
    if (idx != nullptr) idx[i] = (uint8_t)bi;
  }
}

// global average pool of fp32 [N, HW, C] -> fp32 [N, C]
__global__ void avgpool_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int HW, int C) {
  const int64_t total = (int64_t)N * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t n = i / C;
    float acc = 0.f;
    for (int r = 0; r < HW; ++r) acc += x[(n * HW + r) * C + c];
    y[i] = acc / (float)HW;
  }
}

}  // namespace byol

using namespace byol;

#define BYOL_CHECK_T(T) BYOL_CHECK_ARG((T) == 3 || (T) == 6, "split path: T=%d must be 3 or 6", (T))

extern "C" int byol_split_planes(const float* x, void* planes, void* copy_bf16, int64_t M, int C, int Cpad, int ldx,
                                 int T, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && planes && M > 0 && C > 0 && Cpad >= C && ldx >= C, "byol_split_planes: bad args");
  BYOL_CHECK_T(T);
  split_planes_kernel<<<grid_for(M * Cpad, 256), 256, 0, stream>>>(x, (bf16*)planes, (bf16*)copy_bf16, M, C, Cpad, ldx,
                                                                   make_pattern(T));
  return check_launch("split_planes_kernel");
}

extern "C" int byol_nchw_to_planes(const float* x, void* planes, int N, int Cin, int H, int W, int Cpad, int T,
                                   cudaStream_t stream) {
  BYOL_CHECK_ARG(x && planes && N > 0 && Cin > 0 && Cpad >= Cin && (T * Cpad) % 8 == 0, "byol_nchw_to_planes: bad args");
  BYOL_CHECK_T(T);
  nchw_to_planes_kernel<<<grid_for((int64_t)N * H * W * Cpad, 256), 256, 0, stream>>>(x, (bf16*)planes, N, Cin, H, W,
                                                                                     Cpad, make_pattern(T));
  return check_launch("nchw_to_planes_kernel");
}

extern "C" int byol_prep_weight_planes(const float* w, void* out, int Cout, int Cin, int Cpad, int taps, int T,
                                       cudaStream_t stream) {
  BYOL_CHECK_ARG(w && out && Cout > 0 && Cin > 0 && Cpad >= Cin && taps > 0, "byol_prep_weight_planes: bad args");
  BYOL_CHECK_T(T);
  prep_weight_planes_kernel<<<grid_for((int64_t)Cout * taps * Cpad, 256), 256, 0, stream>>>(w, (bf16*)out, Cout, Cin,
                                                                                           Cpad, taps, make_pattern(T));
  return check_launch("prep_weight_planes_kernel");
}

__global__ void stats_f32_sum_kernel(double* __restrict__ part, double* __restrict__ stats, int nblocks, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int k = 0; k < nblocks; ++k) {
    s += part[(int64_t)k * n + i];
    part[(int64_t)k * n + i] = 0.0;   // the scratch is left zeroed (fix_scratch)
  }
  stats[i] += s;
}

// stats: 2C doubles, zeroed by the caller
extern "C" int byol_stats_f32(const float* y, double* stats, int64_t M, int C, cudaStream_t stream) {
  BYOL_CHECK_ARG(y && stats && M > 0 && C > 0, "byol_stats_f32: bad args");
  int CT = 1;
  while (CT < C && CT < 256) CT <<= 1;           // power of two <= 256 covering min(C, 256) columns per block
  const int lanes = 256 / CT;
  int64_t rows_per_block = (M + 132 * 4 - 1) / (132 * 4);
  if (rows_per_block < 4 * lanes) rows_per_block = 4 * lanes;
  dim3 grid((unsigned)((M + rows_per_block - 1) / rows_per_block), (unsigned)((C + CT - 1) / CT));
  // the scratch of the fixed-point reductions holds the 2 * grid.x * C fp64 partials (three doubles per entry)
  Fix128* scratch = fix_scratch(stream, ((int64_t)grid.x * C * 2 + 2) / 3);
  if (scratch == nullptr) return -2;
  double* part = reinterpret_cast<double*>(scratch);
  stats_f32_kernel<<<grid, 256, 0, stream>>>(y, part, M, C, CT, rows_per_block);
  stats_f32_sum_kernel<<<(2 * C + 255) / 256, 256, 0, stream>>>(part, stats, (int)grid.x, 2 * C);
  return fix_done(stream, check_launch("stats_f32_kernel"));
}

extern "C" int byol_bn_finalize_lanes_f64(const double* stats, double count, int L, const float* gamma0,
                                          const float* beta0, const float* gamma1, const float* beta1,
                                          const float* gamma2, const float* beta2, const float* gamma3,
                                          const float* beta3, float* running_mean, float* running_var, float momentum,
                                          float eps, float* coeffs, int C, cudaStream_t stream) {
  BYOL_CHECK_ARG(stats && coeffs && L >= 1 && L <= 4 && C > 0 && count > 0, "byol_bn_finalize_lanes_f64: bad args");
  LanePtrs64 g, b;
  g.p[0] = gamma0; g.p[1] = gamma1; g.p[2] = gamma2; g.p[3] = gamma3;
  b.p[0] = beta0; b.p[1] = beta1; b.p[2] = beta2; b.p[3] = beta3;
  for (int l = 0; l < L; ++l) BYOL_CHECK_ARG(g.p[l] && b.p[l], "byol_bn_finalize_lanes_f64: null gamma/beta, lane %d", l);
  bn_finalize_lanes_f64_kernel<<<(C + 127) / 128, 128, 0, stream>>>(stats, count, g, b, running_mean, running_var,
                                                                   momentum, eps, coeffs, C, L);
  return check_launch("bn_finalize_lanes_f64_kernel");
}

extern "C" int byol_bn_apply_f32(const float* y, const float* scale, const float* shift, const float* resid,
                                 const float* rscale, const float* rshift, float* out32, void* planes, void* copy_bf16,
                                 void* mask, int64_t M, int C, int relu, int T, cudaStream_t stream) {
  BYOL_CHECK_ARG(y && scale && shift && M > 0 && C % 8 == 0 && (out32 || planes || copy_bf16),
                 "byol_bn_apply_f32: bad args");
  BYOL_CHECK_T(T);
  const int64_t nvec = M * C / 8;
  bn_apply_f32_kernel<<<grid_for(nvec, 256), 256, 0, stream>>>(y, scale, shift, resid, rscale, rshift, out32,
                                                               (bf16*)planes, (bf16*)copy_bf16, (uint8_t*)mask, nvec, C,
                                                               relu, make_pattern(T));
  return check_launch("bn_apply_f32_kernel");
}

extern "C" int byol_maxpool_f32(const float* x, float* y, void* idx, int N, int H, int W, int C, int k, int s, int p,
                                cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y && k * k <= 255, "byol_maxpool_f32: bad args");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
  maxpool_f32_kernel<<<grid_for((int64_t)N * Ho * Wo * C, 256), 256, 0, stream>>>(x, y, (uint8_t*)idx, N, H, W, C, Ho,
                                                                                 Wo, k, s, p);
  return check_launch("maxpool_f32_kernel");
}

extern "C" int byol_avgpool_f32(const float* x, float* y, int N, int HW, int C, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y && N > 0 && HW > 0 && C > 0, "byol_avgpool_f32: bad args");
  avgpool_f32_kernel<<<grid_for((int64_t)N * C, 256), 256, 0, stream>>>(x, y, N, HW, C);
  return check_launch("avgpool_f32_kernel");
}

// =============================================================================================
// fp32-accurate backward path (BYOL(backward_precision="fp32")): the same split scheme on the backward GEMMs.
//   dgrad  dX = dY * W^T : dY in activation-pattern planes, W in the dgrad plane layout below (weight pattern)
//   wgrad  dW = dY^T * X : the planes of dY and X as they are (byol_conv_wgrad_planes pairs the columns)
// BatchNorm backward reads the fp32 conv output and the fp32 incoming gradient; its per-channel sums are per-block
// fp64 partials added in block order (same bits in every run, no float atomics).
// =============================================================================================
namespace byol {

// fp32 weight [Cout, Cin, taps] -> bf16 [Cin, taps * T * Cout]: column (tap*T + j)*Cout + co = plane B_PAT[j] of
// w[co, ci, tap] (the dgrad layout of byol_prep_weight with T planes per output channel)
__global__ void prep_weight_dgrad_planes_kernel(const float* __restrict__ w, bf16* __restrict__ out, int Cout, int Cin,
                                                int taps, SplitPattern pat) {
  const int64_t total = (int64_t)Cin * taps * Cout;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(i % Cout);
    int64_t t = i / Cout;
    const int tap = (int)(t % taps);
    const int64_t ci = t / taps;
    bf16 pl[3];
    split3(w[((int64_t)co * Cin + ci) * taps + tap], pl);
    bf16* o = out + (ci * taps + tap) * (int64_t)pat.T * Cout + co;
#pragma unroll
    for (int j = 0; j < 6; ++j)
      if (j < pat.T) o[(int64_t)j * Cout] = pl[pat.b[j]];
  }
}

// dz = g masked by the ReLU of the BatchNorm output: MASK 0 none, 1 (y*scale + shift) > 0, 3 bit of the mask bytes
template <int MASK>
__device__ __forceinline__ float bwd_mask(float g, float y, const uint8_t* mask, int64_t e, float sc, float sh) {
  if (MASK == 1) return (y * sc + sh) > 0.f ? g : 0.f;
  if (MASK == 3) return ((__ldg(mask + (e >> 3)) >> (e & 7)) & 1u) ? g : 0.f;
  return g;
}

// part[block][0:C] = sum dz, part[block][C:2C] = sum dz * xhat over this block's rows (fp64); layout of stats_f32_kernel
template <int MASK>
__global__ void bn_bwd_reduce_f32_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                         const uint8_t* __restrict__ mask, const float* __restrict__ scale,
                                         const float* __restrict__ shift, const float* __restrict__ mean,
                                         const float* __restrict__ invstd, double* __restrict__ part, int64_t M, int C,
                                         int CT, int64_t rows_per_block) {
  const int col = blockIdx.y * CT + (int)(threadIdx.x % CT);
  const int rlane = (int)(threadIdx.x / CT);
  const int lanes = (int)(blockDim.x / CT);
  const int64_t r0 = blockIdx.x * rows_per_block;
  int64_t r1 = r0 + rows_per_block;
  if (r1 > M) r1 = M;
  double s = 0.0, q = 0.0;
  if (col < C) {
    const float sc = MASK == 1 ? scale[col] : 0.f, sh = MASK == 1 ? shift[col] : 0.f;
    const double mu = (double)mean[col], is = (double)invstd[col];
    for (int64_t r = r0 + rlane; r < r1; r += lanes) {
      const int64_t e = r * C + col;
      const float yv = y[e];
      const double dz = (double)bwd_mask<MASK>(g[e], yv, mask, e, sc, sh);
      s += dz;
      q += dz * (((double)yv - mu) * is);
    }
  }
  __shared__ double sh[2][256];
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = q;
  __syncthreads();
  if (rlane == 0 && col < C) {
    for (int l = 1; l < lanes; ++l) {
      s += sh[0][l * CT + (threadIdx.x % CT)];
      q += sh[1][l * CT + (threadIdx.x % CT)];
    }
    part[(int64_t)blockIdx.x * 2 * C + col] = s;
    part[(int64_t)blockIdx.x * 2 * C + C + col] = q;
  }
}

// 8 fp32 values of one row -> their T activation-pattern planes at base (plane stride C elements)
__device__ __forceinline__ void store_planes8(bf16* base, int C, const float (&o)[8], const SplitPattern& pat) {
  bf16 pl[8][3];
#pragma unroll
  for (int e = 0; e < 8; ++e) split3(o[e], pl[e]);
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    if (j < pat.T) {
      const int a = pat.a[j];
      uint4 q;
      __nv_bfloat162 h0 = __halves2bfloat162(pl[0][a], pl[1][a]), h1 = __halves2bfloat162(pl[2][a], pl[3][a]);
      __nv_bfloat162 h2 = __halves2bfloat162(pl[4][a], pl[5][a]), h3 = __halves2bfloat162(pl[6][a], pl[7][a]);
      q.x = *reinterpret_cast<uint32_t*>(&h0);
      q.y = *reinterpret_cast<uint32_t*>(&h1);
      q.z = *reinterpret_cast<uint32_t*>(&h2);
      q.w = *reinterpret_cast<uint32_t*>(&h3);
      *reinterpret_cast<uint4*>(base + (int64_t)j * C) = q;
    }
  }
}

// dy = gamma*invstd*(dz - s1/n - xhat*s2/n) on fp32 [M, C] -> planes (bf16 [M, T*C]) and / or fp32 dy; optional fp32
// dz (the residual branch's gradient).  Block 0 adds the rank-local sums to dgamma / dbeta: plain read-modify-write,
// the lanes of one layer are launched one after another on one stream.  One thread per 8 consecutive channels.
template <int MASK>
__global__ void bn_bwd_apply_f32_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                        const uint8_t* __restrict__ mask, const float* __restrict__ scale,
                                        const float* __restrict__ shift, const float* __restrict__ mean,
                                        const float* __restrict__ invstd, const float* __restrict__ gamma,
                                        const double* __restrict__ s12, double inv_count, bf16* __restrict__ planes,
                                        float* __restrict__ dy32, float* __restrict__ dz_out, int64_t nvec, int C,
                                        SplitPattern pat, const double* __restrict__ s12_local,
                                        float* __restrict__ dgamma, float* __restrict__ dbeta) {
  if (blockIdx.x == 0 && dgamma != nullptr) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      dgamma[c] += (float)s12_local[C + c];
      dbeta[c] += (float)s12_local[c];
    }
  }
  const int groups = C >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int gi = (int)(i % groups);
    const int64_t m = i / groups;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(g) + 2 * i);
    const float4 g1 = __ldg(reinterpret_cast<const float4*>(g) + 2 * i + 1);
    const float4 y0 = __ldg(reinterpret_cast<const float4*>(y) + 2 * i);
    const float4 y1 = __ldg(reinterpret_cast<const float4*>(y) + 2 * i + 1);
    const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float yv[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
    float dz[8], o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = gi * 8 + e;
      const float sc = MASK == 1 ? __ldg(scale + c) : 0.f, sh = MASK == 1 ? __ldg(shift + c) : 0.f;
      dz[e] = bwd_mask<MASK>(gv[e], yv[e], mask, 8 * i + e, sc, sh);
      const float is = __ldg(invstd + c);
      const float xhat = (yv[e] - __ldg(mean + c)) * is;
      const float k1 = (float)(s12[c] * inv_count), k2 = (float)(s12[C + c] * inv_count);
      o[e] = __ldg(gamma + c) * is * (dz[e] - k1 - xhat * k2);
    }
    if (planes != nullptr) store_planes8(planes + m * (int64_t)pat.T * C + gi * 8, C, o, pat);
    if (dy32 != nullptr) {
      reinterpret_cast<float4*>(dy32)[2 * i] = make_float4(o[0], o[1], o[2], o[3]);
      reinterpret_cast<float4*>(dy32)[2 * i + 1] = make_float4(o[4], o[5], o[6], o[7]);
    }
    if (dz_out != nullptr) {
      reinterpret_cast<float4*>(dz_out)[2 * i] = make_float4(dz[0], dz[1], dz[2], dz[3]);
      reinterpret_cast<float4*>(dz_out)[2 * i + 1] = make_float4(dz[4], dz[5], dz[6], dz[7]);
    }
  }
}

// max-pool backward over fp32 NHWC with the window positions maxpool_f32 wrote: every input pixel gathers the
// gradients of the windows that chose it (fixed order, no atomics)
__global__ void maxpool_bwd_f32_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ idx,
                                       float* __restrict__ dx, int N, int H, int W, int C, int Ho, int Wo, int k, int s,
                                       int p) {
  const int64_t total = (int64_t)N * H * W * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    int64_t t = i / C;
    const int iw = (int)(t % W); t /= W;
    const int ih = (int)(t % H);
    const int n = (int)(t / H);
    float acc = 0.f;
    for (int kh = (ih + p) % s; kh < k; kh += s) {
      const int oh = (ih + p - kh) / s;
      if (oh < 0 || oh >= Ho) continue;
      for (int kw = (iw + p) % s; kw < k; kw += s) {
        const int ow = (iw + p - kw) / s;
        if (ow < 0 || ow >= Wo) continue;
        const int64_t o = (((int64_t)n * Ho + oh) * Wo + ow) * C + c;
        if ((int)idx[o] == kh * k + kw) acc += dy[o];
      }
    }
    dx[i] = acc;
  }
}

// dx[n, r, c] = (ga[n, c] + gb[n, c]) / HW   (either gradient may be absent)
__global__ void avgpool_bwd_f32_kernel(const float* __restrict__ ga, const float* __restrict__ gb,
                                       float* __restrict__ dx, int N, int HW, int C) {
  const int64_t total = (int64_t)N * HW * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t n = i / ((int64_t)HW * C);
    const float a = ga != nullptr ? ga[n * C + c] : 0.f;
    const float b = gb != nullptr ? gb[n * C + c] : 0.f;
    dx[i] = (ga != nullptr && gb != nullptr ? a + b : (ga != nullptr ? a : b)) / (float)HW;
  }
}

}  // namespace byol

extern "C" int byol_prep_weight_dgrad_planes(const float* w, void* out, int Cout, int Cin, int taps, int T,
                                             cudaStream_t stream) {
  BYOL_CHECK_ARG(w && out && Cout > 0 && Cin > 0 && taps > 0, "byol_prep_weight_dgrad_planes: bad args");
  BYOL_CHECK_T(T);
  prep_weight_dgrad_planes_kernel<<<grid_for((int64_t)Cin * taps * Cout, 256), 256, 0, stream>>>(
      w, (bf16*)out, Cout, Cin, taps, make_pattern(T));
  return check_launch("prep_weight_dgrad_planes_kernel");
}

// s12 (fp64 [2C], accumulated): += [sum dz, sum dz * xhat] over the rows of g / y (fp32 [M, C])
extern "C" int byol_bn_bwd_reduce_f32(const float* g, const float* y, const void* mask, const float* scale,
                                      const float* shift, const float* mean, const float* invstd, double* s12,
                                      int64_t M, int C, int mask_mode, cudaStream_t stream) {
  BYOL_CHECK_ARG(g && y && mean && invstd && s12 && M > 0 && C > 0, "byol_bn_bwd_reduce_f32: bad args");
  BYOL_CHECK_ARG((mask_mode == 0) || (mask_mode == 1 && scale && shift) || (mask_mode == 3 && mask),
                 "byol_bn_bwd_reduce_f32: bad mask_mode %d", mask_mode);
  int CT = 1;
  while (CT < C && CT < 256) CT <<= 1;
  const int lanes = 256 / CT;
  int64_t rows_per_block = (M + 132 * 4 - 1) / (132 * 4);
  if (rows_per_block < 4 * lanes) rows_per_block = 4 * lanes;
  dim3 grid((unsigned)((M + rows_per_block - 1) / rows_per_block), (unsigned)((C + CT - 1) / CT));
  Fix128* scratch = fix_scratch(stream, ((int64_t)grid.x * C * 2 + 2) / 3);
  if (scratch == nullptr) return -2;
  double* part = reinterpret_cast<double*>(scratch);
  const uint8_t* mk = (const uint8_t*)mask;
  if (mask_mode == 0)
    bn_bwd_reduce_f32_kernel<0><<<grid, 256, 0, stream>>>(g, y, mk, scale, shift, mean, invstd, part, M, C, CT, rows_per_block);
  else if (mask_mode == 1)
    bn_bwd_reduce_f32_kernel<1><<<grid, 256, 0, stream>>>(g, y, mk, scale, shift, mean, invstd, part, M, C, CT, rows_per_block);
  else
    bn_bwd_reduce_f32_kernel<3><<<grid, 256, 0, stream>>>(g, y, mk, scale, shift, mean, invstd, part, M, C, CT, rows_per_block);
  if (check_launch("bn_bwd_reduce_f32_kernel") != 0) return -100;
  stats_f32_sum_kernel<<<(2 * C + 255) / 256, 256, 0, stream>>>(part, s12, (int)grid.x, 2 * C);
  return fix_done(stream, check_launch("stats_f32_sum_kernel"));
}

// s12: global (cross-rank) sums over `count` rows; s12_local (optional, default s12): this rank's sums for dgamma/dbeta
extern "C" int byol_bn_bwd_apply_f32(const float* g, const float* y, const void* mask, const float* scale,
                                     const float* shift, const float* mean, const float* invstd, const float* gamma,
                                     const double* s12, const double* s12_local, double count, void* planes,
                                     float* dy32, float* dz_out, float* dgamma, float* dbeta, int64_t M, int C,
                                     int mask_mode, int T, cudaStream_t stream) {
  BYOL_CHECK_ARG(g && y && mean && invstd && gamma && s12 && count > 0 && M > 0 && C % 8 == 0 && (planes || dy32),
                 "byol_bn_bwd_apply_f32: bad args");
  BYOL_CHECK_ARG((mask_mode == 0) || (mask_mode == 1 && scale && shift) || (mask_mode == 3 && mask),
                 "byol_bn_bwd_apply_f32: bad mask_mode %d", mask_mode);
  BYOL_CHECK_ARG((dgamma == nullptr) == (dbeta == nullptr), "byol_bn_bwd_apply_f32: need dgamma and dbeta or neither");
  BYOL_CHECK_T(T);
  if (s12_local == nullptr) s12_local = s12;
  const int64_t nvec = M * C / 8;
  const uint8_t* mk = (const uint8_t*)mask;
  const SplitPattern pat = make_pattern(T);
  const int grid = grid_for(nvec, 256);
  if (mask_mode == 0)
    bn_bwd_apply_f32_kernel<0><<<grid, 256, 0, stream>>>(g, y, mk, scale, shift, mean, invstd, gamma, s12, 1.0 / count,
                                                         (bf16*)planes, dy32, dz_out, nvec, C, pat, s12_local, dgamma, dbeta);
  else if (mask_mode == 1)
    bn_bwd_apply_f32_kernel<1><<<grid, 256, 0, stream>>>(g, y, mk, scale, shift, mean, invstd, gamma, s12, 1.0 / count,
                                                         (bf16*)planes, dy32, dz_out, nvec, C, pat, s12_local, dgamma, dbeta);
  else
    bn_bwd_apply_f32_kernel<3><<<grid, 256, 0, stream>>>(g, y, mk, scale, shift, mean, invstd, gamma, s12, 1.0 / count,
                                                         (bf16*)planes, dy32, dz_out, nvec, C, pat, s12_local, dgamma, dbeta);
  return check_launch("bn_bwd_apply_f32_kernel");
}

extern "C" int byol_maxpool_bwd_f32(const float* dy, const void* idx, float* dx, int N, int H, int W, int C, int k,
                                    int s, int p, cudaStream_t stream) {
  BYOL_CHECK_ARG(dy && idx && dx && N > 0 && C > 0 && k * k <= 255 && s > 0, "byol_maxpool_bwd_f32: bad args");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
  maxpool_bwd_f32_kernel<<<grid_for((int64_t)N * H * W * C, 256), 256, 0, stream>>>(dy, (const uint8_t*)idx, dx, N, H,
                                                                                     W, C, Ho, Wo, k, s, p);
  return check_launch("maxpool_bwd_f32_kernel");
}

extern "C" int byol_avgpool_bwd_f32(const float* ga, const float* gb, float* dx, int N, int HW, int C,
                                    cudaStream_t stream) {
  BYOL_CHECK_ARG((ga || gb) && dx && N > 0 && HW > 0 && C > 0, "byol_avgpool_bwd_f32: bad args");
  avgpool_bwd_f32_kernel<<<grid_for((int64_t)N * HW * C, 256), 256, 0, stream>>>(ga, gb, dx, N, HW, C);
  return check_launch("avgpool_bwd_f32_kernel");
}
