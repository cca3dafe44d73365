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

__device__ __forceinline__ void split3(float x, bf16 (&pl)[3]) {
  pl[0] = __float2bfloat16_rn(x);
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
    int bi = 0;
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
