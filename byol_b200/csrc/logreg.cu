// byol_b200 — transfer linear evaluation: H L2-regularised multinomial logistic regressions over the same fp32
// features, minimised together by full-batch L-BFGS (byol_b200/logreg.py drives the solver from the host).
//
// Head h minimises f_h(W, b) = (1/N) sum_i CE(softmax(W x_i + b), y_i) + (l2_h / 2) ||W||_F^2.  Its weights are rows
// h * Cp .. h * Cp + Cp - 1 of one fp32 [H * Cp, D] matrix (Cp = C rounded up to a multiple of 8; the padding rows stay
// zero), followed in the same buffer by the [H, Cp] biases: the layout of LinearHeads (linear_eval.py).  The logits of
// every head come from one split-operand GEMM (T = 6 planes, fp32-accurate; csrc/split.cu) and the weight gradient
// from one split-operand wgrad.  This file holds the kernels around them:
//
//   logreg_ce_kernel        per (row, head) segment of the fp32 logits: softmax cross-entropy, (softmax - onehot) / N
//                           as the six activation-pattern bf16 planes the wgrad reads, the bias gradient and the loss
//                           (fixed point); or, in evaluation mode, top-1 hits per (head, class)
//   logreg_grad_kernel      (a) g += l2_h W; per-head ||g||_inf and ||W||^2 of the evaluated point
//   logreg_dots_kernel      (b) up to 8 per-head dot products u_k . v_k in one pass, fp64
//   logreg_accept_kernel    x, g <- the accepted trial point and its gradient; s = x' - x and y = g' - g into the
//                           history with their s.y and y.y
//   logreg_commit_kernel    keeps (s, y) when s.y > 1e-10 y.y: rho, gamma and the ring of the last m pairs
//   logreg_twoloop_kernel   (c) one step of the two-loop recursion, d = -H g
//   logreg_trial_kernel     (d) x' = x + t_h d for the heads still searching
//
// Every per-head reduction is fp64 over a fixed slicing of the head's own vector (vec_blocks: slices of 16384 elements),
// summed in a fixed order, so a head's results do not depend on H or on the heads beside it, and a run gives the same
// bits every time.  Each vector kernel takes the per-head mode array and a bit mask of the modes it acts on: a head
// whose mode is not in the mask is not read or written (a stopped head's parameters are never written again).
#include <math.h>

#include "common.cuh"

namespace byol {

static constexpr int LR_WARPS = 8;
static constexpr int LR_ROWS = 64;             // rows per cross-entropy block (8 per warp)
static constexpr int VEC_THREADS = 256;
static constexpr int64_t VEC_SLICE = 16384;    // head-vector elements per block
static constexpr int MAX_DOTS = 8;

// one head's parameter vector: element e < Cp * D is weight h * Cp * D + e, the rest are its Cp biases
struct VecGeom {
  int H, Cp;
  int64_t nw;      // Cp * D
  int64_t L;       // nw + Cp
  int64_t P;       // H * L: the whole buffer
  int nb;          // blocks per head
};

static inline VecGeom make_geom(int H, int Cp, int D) {
  VecGeom g;
  g.H = H; g.Cp = Cp;
  g.nw = (int64_t)Cp * D;
  g.L = g.nw + Cp;
  g.P = (int64_t)H * g.L;
  g.nb = (int)((g.L + VEC_SLICE - 1) / VEC_SLICE);
  return g;
}

__device__ __forceinline__ int64_t vidx(const VecGeom& g, int h, int64_t e) {
  return e < g.nw ? (int64_t)h * g.nw + e : (int64_t)g.H * g.nw + (int64_t)h * g.Cp + (e - g.nw);
}

__device__ __forceinline__ bool head_on(const int* mode, int mask, int h) { return (mask >> mode[h]) & 1; }

// fixed-order block reductions (tree over the 256 threads); every thread returns the total
__device__ double block_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = VEC_THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// NaN-propagating max of non-negative values
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || b != b) ? NAN : fmax(a, b); }

__device__ double block_max(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = VEC_THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] = nan_max(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// sum of a head's nb partials, in block order
__device__ __forceinline__ double part_sum(const double* p, int nb) {
  double s = 0.0;
  for (int i = 0; i < nb; ++i) s += p[i];
  return s;
}

__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ uint4 pack8(const bf16 (&p)[8]) {
  uint4 q;
  __nv_bfloat162 h0 = __halves2bfloat162(p[0], p[1]), h1 = __halves2bfloat162(p[2], p[3]);
  __nv_bfloat162 h2 = __halves2bfloat162(p[4], p[5]), h3 = __halves2bfloat162(p[6], p[7]);
  q.x = *reinterpret_cast<uint32_t*>(&h0);
  q.y = *reinterpret_cast<uint32_t*>(&h1);
  q.z = *reinterpret_cast<uint32_t*>(&h2);
  q.w = *reinterpret_cast<uint32_t*>(&h3);
  return q;
}

// ---------------------------------------------------------------------------------------------------------------------
// Cross-entropy of the fp32 logits [B, H * Cp] (row pitch ld): block (x, h) handles rows 64x .. 64x + 63 of head h, one
// warp per row at a time, lane l owning the 8-column chunks l, l + 32, ... .  The loss and its gradient are those of
// linprobe_ce_kernel (csrc/linear_eval.cu): with m the segment's maximum, xl the label's logit, e = exp(xl - m) and s
// the sum of exp(v - m) over the other real columns, loss = log1p(s / e) when xl - m > -1, (m - xl) + log(s + e)
// otherwise; g = exp(v - m) / (s + e) / N, and -s / (s + e) / N at the label, in fp32.
//
// Fit mode (planes != nullptr): g is split exactly into three bf16 values g0 + g1 + g2 (|g| <= 1, so no saturation
// case) and stored as the T = 6 activation-pattern planes (g0, g0, g1, g1, g0, g2) of byol_split_planes, plane j of
// column n at j * H * Cp + n of the row; padding columns and rows whose label is outside [0, C) store zeros.  Each lane
// adds its columns' g to an fp64 per-warp row sum in shared memory (lane-exclusive columns, rows in order); the block
// adds the 8 warp sums in warp order and hands each column's total to a fixed-point accumulator (bias_acc [H * Cp]), and
// each row loss to loss_acc [H].  Both are order-independent, so the bias gradient and the loss have the same bits in
// every launch.
// Evaluation mode (class_hits != nullptr): class_hits [H, Cp] += the rows of each label whose logit has rank 0 (no
// other real logit larger or NaN; a NaN label logit is a miss, linprobe_ce_kernel's rule); class_count [Cp] += the
// rows of each label (head 0 counts them).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LR_WARPS * 32)
logreg_ce_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels, int B, int H, int C,
                 int Cp, float fn, bf16* __restrict__ planes, Fix128* __restrict__ loss_acc,
                 Fix128* __restrict__ bias_acc, unsigned long long* __restrict__ class_hits,
                 unsigned long long* __restrict__ class_count) {
  extern __shared__ double s_db[];                      // [LR_WARPS][Cp] when planes != nullptr
  __shared__ unsigned long long s_words[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.y;
  const int64_t HC = (int64_t)H * Cp;
  const int chunks = Cp >> 3;
  if (threadIdx.x == 0) { s_words[0] = 0ull; s_words[1] = 0ull; }
  if (planes != nullptr)
    for (int i = threadIdx.x; i < LR_WARPS * Cp; i += LR_WARPS * 32) s_db[i] = 0.0;
  __syncthreads();
  for (int k = warp; k < LR_ROWS; k += LR_WARPS) {
    const int r = blockIdx.x * LR_ROWS + k;
    if (r >= B) break;
    const float* __restrict__ x = logits + (int64_t)r * ld + (int64_t)h * Cp;
    const int64_t lab64 = labels[r];
    const bool lab_ok = lab64 >= 0 && lab64 < C;
    const int lab = lab_ok ? (int)lab64 : -1;
    float mx = -INFINITY;
    for (int j = lane; j < chunks; j += 32) {
      float v[8];
      load8(x + 8 * j, v);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (8 * j + i < C) mx = fmaxf(mx, v[i]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float xl = lab_ok ? __ldg(x + lab) : NAN;
    float so = 0.f;
    int gt = 0;
    for (int j = lane; j < chunks; j += 32) {
      float v[8];
      load8(x + 8 * j, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = 8 * j + i;
        if (c < C && c != lab) {
          so += expf(v[i] - mx);
          gt += v[i] <= xl ? 0 : 1;
        }
      }
    }
    so = warp_sum(so);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gt += __shfl_xor_sync(0xffffffffu, gt, o);
    const float el = expf(xl - mx);
    const float se = so + el;
    if (planes != nullptr) {
      bf16* __restrict__ d = planes + (int64_t)r * 6 * HC + (int64_t)h * Cp;
      double* __restrict__ acc = s_db + warp * Cp;
      for (int j = lane; j < chunks; j += 32) {
        float v[8];
        load8(x + 8 * j, v);
        bf16 p0[8], p1[8], p2[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = 8 * j + i;
          const float g = c >= C || !lab_ok ? 0.f : (c == lab ? -so / se : expf(v[i] - mx) / se) / fn;
          p0[i] = __float2bfloat16_rn(g);
          const float r1 = g - __bfloat162float(p0[i]);        // exact
          p1[i] = __float2bfloat16_rn(r1);
          p2[i] = __float2bfloat16_rn(r1 - __bfloat162float(p1[i]));
          acc[8 * j + i] += (double)g;
        }
        const uint4 q0 = pack8(p0), q1 = pack8(p1), q2 = pack8(p2);
        uint4* o = reinterpret_cast<uint4*>(d + 8 * j);
        const int64_t ps = HC / 8;                              // plane stride in uint4
        o[0] = q0; o[ps] = q0; o[2 * ps] = q1; o[3 * ps] = q1; o[4 * ps] = q0; o[5 * ps] = q2;
      }
    }
    if (lane == 0 && lab_ok) {
      if (loss_acc != nullptr) {
        const float loss = xl - mx > -1.f ? log1pf(so / el) : (mx - xl) + logf(se);
        fix_add_local(loss_acc + h, s_words, (double)loss);
      }
      if (class_hits != nullptr) {
        if (!isnan(xl) && gt < 1) atomicAdd(class_hits + (int64_t)h * Cp + lab, 1ull);
        if (h == 0) atomicAdd(class_count + lab, 1ull);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && loss_acc != nullptr) fix_add_words(loss_acc + h, s_words[0], (long long)s_words[1]);
  if (planes != nullptr && bias_acc != nullptr) {
    for (int c = threadIdx.x; c < C; c += LR_WARPS * 32) {
      double s = 0.0;
      for (int w = 0; w < LR_WARPS; ++w) s += s_db[w * Cp + c];
      fix_add(bias_acc + (int64_t)h * Cp + c, s);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// (a) The gradient of the evaluated point xt: gW += l2_h * W (fp32, each operation rounded on its own), gb = the fixed-
// point bias sums; part[h][blk] = (max |g|, sum W^2) over the block's slice; block 0 writes the head's loss sum.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(VEC_THREADS)
logreg_grad_kernel(const float* __restrict__ xt, float* __restrict__ gt, const Fix128* __restrict__ loss_acc,
                   const Fix128* __restrict__ bias_acc, const double* __restrict__ l2, const int* __restrict__ mode,
                   int mask, VecGeom G, double* __restrict__ part, double* __restrict__ loss, int ldo) {
  __shared__ double sh[VEC_THREADS];
  const int h = blockIdx.y, blk = blockIdx.x;
  if (!head_on(mode, mask, h)) return;
  const float lam = (float)l2[h];
  const int64_t e0 = (int64_t)blk * VEC_SLICE, e1 = min(G.L, e0 + VEC_SLICE);
  double mx = 0.0, w2 = 0.0;
  for (int64_t e = e0 + threadIdx.x; e < e1; e += VEC_THREADS) {
    const int64_t i = vidx(G, h, e);
    float g;
    if (e < G.nw) {
      const float w = xt[i];
      g = __fadd_rn(gt[i], __fmul_rn(lam, w));
      w2 += (double)w * (double)w;
    } else {
      g = (float)fix_value(bias_acc[(int64_t)h * G.Cp + (e - G.nw)]);
    }
    gt[i] = g;
    mx = nan_max(mx, fabs((double)g));
  }
  mx = block_max(mx, sh);
  w2 = block_sum(w2, sh);
  if (threadIdx.x == 0) {
    part[((int64_t)h * G.nb + blk) * 2] = mx;
    part[((int64_t)h * G.nb + blk) * 2 + 1] = w2;
    if (blk == 0) loss[(int64_t)h * ldo] = fix_value(loss_acc[h]);
  }
}

// out[h * ldo + k] = sum (or max, for the k whose bit is set in max_bits) of part[h][0 .. nb)[k], in block order
__global__ void logreg_head_sum_kernel(const double* __restrict__ part, int nb, int K, int max_bits,
                                       const int* __restrict__ mode, int mask, int H, double* __restrict__ out,
                                       int ldo) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H || !head_on(mode, mask, h)) return;
  for (int k = 0; k < K; ++k) {
    double s = 0.0;
    for (int b = 0; b < nb; ++b) {
      const double v = part[((int64_t)h * nb + b) * K + k];
      s = (max_bits >> k) & 1 ? nan_max(s, v) : s + v;
    }
    out[(int64_t)h * ldo + k] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// (b) part[h][blk][k] = the fp64 sum of u_k[i] * v_k[i] over the block's slice of head h, k < K (products of two fp32
// values are exact in fp64; each thread sums its elements in order, the block in a fixed tree)
// ---------------------------------------------------------------------------------------------------------------------
struct DotPtrs { const float* u[MAX_DOTS]; const float* v[MAX_DOTS]; };

__global__ void __launch_bounds__(VEC_THREADS)
logreg_dots_kernel(DotPtrs p, int K, const int* __restrict__ mode, int mask, VecGeom G, double* __restrict__ part) {
  __shared__ double sh[VEC_THREADS];
  const int h = blockIdx.y, blk = blockIdx.x;
  if (!head_on(mode, mask, h)) return;
  const int64_t e0 = (int64_t)blk * VEC_SLICE, e1 = min(G.L, e0 + VEC_SLICE);
  double acc[MAX_DOTS];
#pragma unroll
  for (int k = 0; k < MAX_DOTS; ++k) acc[k] = 0.0;
  for (int64_t e = e0 + threadIdx.x; e < e1; e += VEC_THREADS) {
    const int64_t i = vidx(G, h, e);
#pragma unroll
    for (int k = 0; k < MAX_DOTS; ++k)
      if (k < K) acc[k] += (double)__ldg(p.u[k] + i) * (double)__ldg(p.v[k] + i);
  }
#pragma unroll
  for (int k = 0; k < MAX_DOTS; ++k) {
    if (k < K) {
      const double s = block_sum(acc[k], sh);
      if (threadIdx.x == 0) part[((int64_t)h * G.nb + blk) * K + k] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Accepting a trial point.  hist[h] = (start, len): the stored pairs are ring slots start .. start + len - 1 (mod m + 1,
// oldest first); the next pair goes to slot (start + len) % (m + 1), which never holds a stored pair.
//   mode 2 / 4 (accept): s = xt - x, y = gt - g into that slot, x = xt, g = gt; part[h][blk] = (s.y, y.y)
//   mode 3 (the starting point, no pair): x = xt, g = gt
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(VEC_THREADS)
logreg_accept_kernel(float* __restrict__ x, const float* __restrict__ xt, float* __restrict__ g,
                     const float* __restrict__ gt, float* __restrict__ S, float* __restrict__ Y,
                     const int* __restrict__ hist, const int* __restrict__ mode, int mask, int m, VecGeom G,
                     double* __restrict__ part) {
  __shared__ double sh[VEC_THREADS];
  const int h = blockIdx.y, blk = blockIdx.x;
  if (!head_on(mode, mask, h)) return;
  const bool pair = mode[h] != 3;
  const int64_t slot = (hist[2 * h] + hist[2 * h + 1]) % (m + 1);
  float* __restrict__ s_out = S + slot * G.P;
  float* __restrict__ y_out = Y + slot * G.P;
  const int64_t e0 = (int64_t)blk * VEC_SLICE, e1 = min(G.L, e0 + VEC_SLICE);
  double sy = 0.0, yy = 0.0;
  for (int64_t e = e0 + threadIdx.x; e < e1; e += VEC_THREADS) {
    const int64_t i = vidx(G, h, e);
    const float xn = xt[i], gn = gt[i];
    if (pair) {
      const float s = __fsub_rn(xn, x[i]), y = __fsub_rn(gn, g[i]);
      s_out[i] = s;
      y_out[i] = y;
      sy += (double)s * (double)y;
      yy += (double)y * (double)y;
    }
    x[i] = xn;
    g[i] = gn;
  }
  if (!pair) return;
  sy = block_sum(sy, sh);
  yy = block_sum(yy, sh);
  if (threadIdx.x == 0) {
    part[((int64_t)h * G.nb + blk) * 2] = sy;
    part[((int64_t)h * G.nb + blk) * 2 + 1] = yy;
  }
}

// One thread per head of mode 2: the new pair is kept when s.y > 1e-10 y.y (rho = 1 / s.y, gamma = s.y / y.y); with m
// pairs stored already the oldest one is dropped.  Otherwise the history is left as it was.
__global__ void logreg_commit_kernel(const double* __restrict__ part, int nb, int* __restrict__ hist,
                                     double* __restrict__ rho, double* __restrict__ gamma,
                                     const int* __restrict__ mode, int H, int m) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H || mode[h] != 2) return;
  double sy = 0.0, yy = 0.0;
  for (int b = 0; b < nb; ++b) {
    sy += part[((int64_t)h * nb + b) * 2];
    yy += part[((int64_t)h * nb + b) * 2 + 1];
  }
  if (!(sy > 1e-10 * yy)) return;
  int start = hist[2 * h], len = hist[2 * h + 1];
  const int slot = (start + len) % (m + 1);
  rho[(int64_t)h * (m + 1) + slot] = 1.0 / sy;
  gamma[h] = sy / yy;
  if (len < m) ++len;
  else start = (start + 1) % (m + 1);
  hist[2 * h] = start;
  hist[2 * h + 1] = len;
}

// ---------------------------------------------------------------------------------------------------------------------
// (c) The two-loop recursion d = -H_k g, in place in d, one launch per step (the step's dot product needs every block
// of the head, so it is summed by the next launch).  With len stored pairs, newest index i = 0 .. len - 1 is ring slot
// (start + len - 1 - i) % (m + 1):
//   phase 0, step i = 0 .. len:  i = 0: q = g (and part4 = g.g);  i > 0: alpha_{i-1} = rho_{i-1} s_{i-1}.q (the sum of
//                                the previous step's partials), q -= alpha_{i-1} y_{i-1};  i < len: partial s_i.q
//   phase 1, step k = 0 .. len (oldest first, slot (start + k) % (m + 1)):  k = 0: r = gamma q, gamma = s.y / y.y of the
//                                newest pair, or 1 / ||g||_2 without pairs;  k > 0: beta = rho y.r (previous partials),
//                                r += (alpha - beta) s;  k < len: partial y_k.r;  k = len: d = -r
// Each step reads one s and one y at most, so each loop reads each history vector once.  Scalars are fp64, vectors fp32
// (each operation rounded on its own).  Partials: part + (slot_k * H + h) * nb, slots 0-1 (phase 0, by step parity),
// 2-3 (phase 1) and 4 (g.g).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(VEC_THREADS)
logreg_twoloop_kernel(int phase, int step, const float* __restrict__ g, float* __restrict__ d,
                      const float* __restrict__ S, const float* __restrict__ Y, const int* __restrict__ hist,
                      const double* __restrict__ rho, const double* __restrict__ gamma, double* __restrict__ alpha,
                      double* __restrict__ part, const int* __restrict__ mode, int mask, int m, VecGeom G) {
  __shared__ double sh[VEC_THREADS];
  const int h = blockIdx.y, blk = blockIdx.x;
  if (!head_on(mode, mask, h)) return;
  const int start = hist[2 * h], len = hist[2 * h + 1], M1 = m + 1;
  if (step > len) return;
  auto pslot = [&](int k) { return part + ((int64_t)k * G.H + h) * G.nb; };
  const int64_t e0 = (int64_t)blk * VEC_SLICE, e1 = min(G.L, e0 + VEC_SLICE);
  double acc = 0.0, acc2 = 0.0;
  if (phase == 0) {
    const float* s_cur = step < len ? S + (int64_t)((start + len - 1 - step) % M1) * G.P : nullptr;
    const float* y_prev = nullptr;
    float af = 0.f;
    if (step > 0) {
      const int sl = (start + len - step) % M1;                 // newest index step - 1
      const double a = rho[(int64_t)h * M1 + sl] * part_sum(pslot((step - 1) & 1), G.nb);
      if (blk == 0 && threadIdx.x == 0) alpha[(int64_t)h * M1 + step - 1] = a;
      af = (float)a;
      y_prev = Y + (int64_t)sl * G.P;
    }
    for (int64_t e = e0 + threadIdx.x; e < e1; e += VEC_THREADS) {
      const int64_t i = vidx(G, h, e);
      const float q = step == 0 ? g[i] : __fsub_rn(d[i], __fmul_rn(af, y_prev[i]));
      d[i] = q;
      if (s_cur != nullptr) acc += (double)s_cur[i] * (double)q;
      if (step == 0) acc2 += (double)q * (double)q;
    }
    if (s_cur != nullptr) {
      acc = block_sum(acc, sh);
      if (threadIdx.x == 0) pslot(step & 1)[blk] = acc;
    }
    if (step == 0) {
      acc2 = block_sum(acc2, sh);
      if (threadIdx.x == 0) pslot(4)[blk] = acc2;
    }
    return;
  }
  const float* y_cur = step < len ? Y + (int64_t)((start + step) % M1) * G.P : nullptr;
  const float* s_prev = nullptr;
  float cf = 0.f;
  if (step == 0) {
    cf = (float)(len > 0 ? gamma[h] : 1.0 / sqrt(part_sum(pslot(4), G.nb)));
  } else {
    const int sl = (start + step - 1) % M1;                     // newest index len - step
    const double beta = rho[(int64_t)h * M1 + sl] * part_sum(pslot(2 + ((step - 1) & 1)), G.nb);
    cf = (float)(alpha[(int64_t)h * M1 + len - step] - beta);
    s_prev = S + (int64_t)sl * G.P;
  }
  for (int64_t e = e0 + threadIdx.x; e < e1; e += VEC_THREADS) {
    const int64_t i = vidx(G, h, e);
    const float r = step == 0 ? __fmul_rn(cf, d[i]) : __fadd_rn(d[i], __fmul_rn(cf, s_prev[i]));
    d[i] = step == len ? -r : r;
    if (y_cur != nullptr) acc += (double)y_cur[i] * (double)r;
  }
  if (y_cur != nullptr) {
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) pslot(2 + (step & 1))[blk] = acc;
  }
}

// (d) xt = x + fp32(t_h) * d for the heads in the mask
__global__ void __launch_bounds__(VEC_THREADS)
logreg_trial_kernel(const float* __restrict__ x, const float* __restrict__ d, float* __restrict__ xt,
                    const double* __restrict__ t, const int* __restrict__ mode, int mask, VecGeom G) {
  const int h = blockIdx.y, blk = blockIdx.x;
  if (!head_on(mode, mask, h)) return;
  const float tf = (float)t[h];
  const int64_t e0 = (int64_t)blk * VEC_SLICE, e1 = min(G.L, e0 + VEC_SLICE);
  for (int64_t e = e0 + threadIdx.x; e < e1; e += VEC_THREADS) {
    const int64_t i = vidx(G, h, e);
    xt[i] = __fadd_rn(x[i], __fmul_rn(tf, d[i]));
  }
}

}  // namespace byol

using namespace byol;

#define LOGREG_CHECK_SHAPE(what)                                                                                     \
  BYOL_CHECK_ARG(H > 0 && H <= 65535 && C >= 2 && C <= Cp && Cp % 8 == 0 && D > 0 && D % 4 == 0,                      \
                 what ": bad shape H=%d C=%d Cp=%d D=%d", H, C, Cp, D)

extern "C" int byol_logreg_vec_blocks(int Cp, int D) { return make_geom(1, Cp, D).nb; }

extern "C" int byol_logreg_ce(const float* logits, int64_t ld, const int64_t* labels, int B, int H, int C, int Cp,
                              double n_total, void* planes, void* loss_acc, void* bias_acc, long long* class_hits,
                              long long* class_count, cudaStream_t stream) {
  BYOL_CHECK_ARG(logits && labels, "byol_logreg_ce: null pointer");
  BYOL_CHECK_ARG((planes && loss_acc && bias_acc && !class_hits && !class_count) ||
                     (!planes && !loss_acc && !bias_acc && class_hits && class_count),
                 "byol_logreg_ce: give planes, loss_acc and bias_acc (fit) or class_hits and class_count (evaluation)");
  BYOL_CHECK_ARG(B > 0 && H > 0 && H <= 65535 && C >= 2 && C <= Cp && Cp % 8 == 0 && (int64_t)H * Cp <= 0x7fffffffll,
                 "byol_logreg_ce: bad shape B=%d H=%d C=%d Cp=%d", B, H, C, Cp);
  BYOL_CHECK_ARG(ld >= (int64_t)H * Cp && ld % 4 == 0 && ((uintptr_t)logits & 15) == 0,
                 "byol_logreg_ce: logits need 16-byte aligned rows with pitch ld=%lld >= H*Cp", (long long)ld);
  BYOL_CHECK_ARG(((uintptr_t)planes & 15) == 0 && n_total >= 1.0, "byol_logreg_ce: planes must be 16-byte aligned");
  const int smem = planes != nullptr ? LR_WARPS * Cp * (int)sizeof(double) : 0;
  BYOL_CHECK_ARG(smem <= 200 * 1024, "byol_logreg_ce: C=%d is too many classes", C);
  if (smem > 48 * 1024 && smem_opt_in((const void*)logreg_ce_kernel, smem, "logreg_ce_kernel") != 0) return -2;
  const dim3 grid((unsigned)((B + LR_ROWS - 1) / LR_ROWS), (unsigned)H);
  logreg_ce_kernel<<<grid, LR_WARPS * 32, smem, stream>>>(logits, ld, labels, B, H, C, Cp, (float)n_total,
                                                          (bf16*)planes, (Fix128*)loss_acc, (Fix128*)bias_acc,
                                                          (unsigned long long*)class_hits,
                                                          (unsigned long long*)class_count);
  return check_launch("logreg_ce_kernel");
}

extern "C" int byol_logreg_grad(const float* xt, float* gt, const void* loss_acc, const void* bias_acc,
                                const double* l2, const int* mode, int mask, int H, int C, int Cp, int D, double* part,
                                double* out, int ldo, cudaStream_t stream) {
  BYOL_CHECK_ARG(xt && gt && loss_acc && bias_acc && l2 && mode && part && out && ldo >= 3, "byol_logreg_grad: bad args");
  LOGREG_CHECK_SHAPE("byol_logreg_grad");
  const VecGeom G = make_geom(H, Cp, D);
  // out[h * ldo + 0] = the loss sum (block 0 of each head writes it), [1] = max |g|, [2] = ||W||^2
  logreg_grad_kernel<<<dim3((unsigned)G.nb, (unsigned)H), VEC_THREADS, 0, stream>>>(
      xt, gt, (const Fix128*)loss_acc, (const Fix128*)bias_acc, l2, mode, mask, G, part, out, ldo);
  if (check_launch("logreg_grad_kernel") != 0) return -100;
  logreg_head_sum_kernel<<<(H + 127) / 128, 128, 0, stream>>>(part, G.nb, 2, 1, mode, mask, H, out + 1, ldo);
  return check_launch("logreg_head_sum_kernel");
}

extern "C" int byol_logreg_dots(const void* const* u, const void* const* v, int K, const int* mode, int mask, int H,
                                int C, int Cp, int D, double* part, double* out, int ldo, cudaStream_t stream) {
  BYOL_CHECK_ARG(u && v && mode && part && out && K >= 1 && K <= MAX_DOTS && ldo >= K, "byol_logreg_dots: bad args");
  LOGREG_CHECK_SHAPE("byol_logreg_dots");
  DotPtrs p;
  for (int k = 0; k < MAX_DOTS; ++k) {
    p.u[k] = k < K ? (const float*)u[k] : nullptr;
    p.v[k] = k < K ? (const float*)v[k] : nullptr;
    BYOL_CHECK_ARG(k >= K || (p.u[k] && p.v[k]), "byol_logreg_dots: null vector %d", k);
  }
  const VecGeom G = make_geom(H, Cp, D);
  logreg_dots_kernel<<<dim3((unsigned)G.nb, (unsigned)H), VEC_THREADS, 0, stream>>>(p, K, mode, mask, G, part);
  if (check_launch("logreg_dots_kernel") != 0) return -100;
  logreg_head_sum_kernel<<<(H + 127) / 128, 128, 0, stream>>>(part, G.nb, K, 0, mode, mask, H, out, ldo);
  return check_launch("logreg_head_sum_kernel");
}

extern "C" int byol_logreg_accept(float* x, const float* xt, float* g, const float* gt, float* S, float* Y, int* hist,
                                  double* rho, double* gamma, const int* mode, int m, int H, int C, int Cp, int D,
                                  double* part, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && xt && g && gt && S && Y && hist && rho && gamma && mode && part && m >= 1,
                 "byol_logreg_accept: bad args");
  LOGREG_CHECK_SHAPE("byol_logreg_accept");
  const VecGeom G = make_geom(H, Cp, D);
  // modes 2, 3, 4 (accept with a pair, the starting point, accept and stop)
  logreg_accept_kernel<<<dim3((unsigned)G.nb, (unsigned)H), VEC_THREADS, 0, stream>>>(x, xt, g, gt, S, Y, hist, mode,
                                                                                     (1 << 2) | (1 << 3) | (1 << 4), m,
                                                                                     G, part);
  if (check_launch("logreg_accept_kernel") != 0) return -100;
  logreg_commit_kernel<<<(H + 127) / 128, 128, 0, stream>>>(part, G.nb, hist, rho, gamma, mode, H, m);
  return check_launch("logreg_commit_kernel");
}

extern "C" int byol_logreg_twoloop(const float* g, float* d, const float* S, const float* Y, const int* hist,
                                   const double* rho, const double* gamma, double* alpha, double* part, const int* mode,
                                   int mask, int m, int H, int C, int Cp, int D, cudaStream_t stream) {
  BYOL_CHECK_ARG(g && d && S && Y && hist && rho && gamma && alpha && part && mode && m >= 1,
                 "byol_logreg_twoloop: bad args");
  LOGREG_CHECK_SHAPE("byol_logreg_twoloop");
  const VecGeom G = make_geom(H, Cp, D);
  const dim3 grid((unsigned)G.nb, (unsigned)H);
  for (int phase = 0; phase < 2; ++phase)
    for (int step = 0; step <= m; ++step) {
      logreg_twoloop_kernel<<<grid, VEC_THREADS, 0, stream>>>(phase, step, g, d, S, Y, hist, rho, gamma, alpha, part,
                                                              mode, mask, m, G);
      if (check_launch("logreg_twoloop_kernel") != 0) return -100;
    }
  return 0;
}

extern "C" int byol_logreg_trial(const float* x, const float* d, float* xt, const double* t, const int* mode, int mask,
                                 int H, int C, int Cp, int D, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && d && xt && t && mode, "byol_logreg_trial: bad args");
  LOGREG_CHECK_SHAPE("byol_logreg_trial");
  const VecGeom G = make_geom(H, Cp, D);
  logreg_trial_kernel<<<dim3((unsigned)G.nb, (unsigned)H), VEC_THREADS, 0, stream>>>(x, d, xt, t, mode, mask, G);
  return check_launch("logreg_trial_kernel");
}
