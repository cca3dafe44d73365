// byol_b200 — BYOL objective, target-network EMA and LARS + SGD-momentum kernels (fp32, HBM-bound).
//
//   byol_loss_fwd / bwd : /root/reference/objective.py:6-25 (regression_loss with WHOLE-MATRIX Frobenius
//                         norms, no per-row normalisation, rank-local; symmetric sum, mean over rows)
//   byol_ema_update     : /root/reference/main.py:159-162 (CosEMA.forward: mean = (1-d)*x + d*mean as three
//                         separately rounded fp32 ops; bit-exact => no FMA contraction)
//   byol_lars_*         : /root/reference/optimizers/lars.py:84-127 (apply_adaptive_lrs + wrapped SGD step,
//                         torch.optim.SGD momentum=0.9, dampening 0, no nesterov, weight decay folded by LARS)
//   byol_sgd_nesterov_step : Nesterov SGD over the same chunk tables (fine-tuning, byol_b200/finetune.py)
#include "common.cuh"

namespace byol {

// ---------------------------------------------------------------------------------------------
// loss
// sums[0] = |q1|^2  sums[1] = |q2|^2  sums[2] = |z1|^2  sums[3] = |z2|^2  sums[4] = <q1,z2>  sums[5] = <q2,z1>
// Every block writes its six fp32 partial sums to its own fp64 slots, part[k * gridDim.x + block]; the finalize kernel
// adds them in block order.  The result is deterministic and its precision relative, so the loss is invariant under
// power-of-two scaling of its inputs at any scale (a fixed-point accumulator's absolute resolution would not be: with
// predictions or targets of RMS ~1e-5 it would cost the loss whole fp32 ulps).
// ---------------------------------------------------------------------------------------------
__global__ void loss_fwd_partial_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                        const float* __restrict__ z1, const float* __restrict__ z2,
                                        double* __restrict__ part, int64_t n4) {
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(q1) + i);
    const float4 b = __ldg(reinterpret_cast<const float4*>(q2) + i);
    const float4 c = __ldg(reinterpret_cast<const float4*>(z1) + i);
    const float4 d = __ldg(reinterpret_cast<const float4*>(z2) + i);
    acc[0] += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
    acc[1] += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
    acc[2] += c.x * c.x + c.y * c.y + c.z * c.z + c.w * c.w;
    acc[3] += d.x * d.x + d.y * d.y + d.z * d.z + d.w * d.w;
    acc[4] += a.x * d.x + a.y * d.y + a.z * d.z + a.w * d.w;
    acc[5] += b.x * c.x + b.y * c.y + b.z * c.z + b.w * c.w;
  }
  __shared__ float sh[6][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    float v = warp_sum(acc[k]);
    if (lane == 0) sh[k][warp] = v;
  }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      float v = lane < nw ? sh[k][lane] : 0.f;
      v = warp_sum(v);
      if (lane == 0) part[k * gridDim.x + blockIdx.x] = (double)v;
    }
  }
}

// loss = -2/b * ( <q1,z2>/(|q1||z2|) + <q2,z1>/(|q2||z1|) );  also stores fp32 copies of the six sums.
// Thread k < 6 adds the nb block partials of sum k in block order and zeroes them (the slots live in the stream's
// scratch, which its users leave zeroed).
__global__ void loss_finalize_kernel(double* __restrict__ part, int nb, float* __restrict__ loss,
                                     float* __restrict__ saved, int rows) {
  __shared__ float v[6];
  if (threadIdx.x < 6) {
    double s = 0.0;
    for (int b = 0; b < nb; ++b) {
      s += part[threadIdx.x * nb + b];
      part[threadIdx.x * nb + b] = 0.0;
    }
    v[threadIdx.x] = (float)s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float nq1 = sqrtf(v[0]), nq2 = sqrtf(v[1]);
    const float nz1 = sqrtf(v[2]), nz2 = sqrtf(v[3]);
    const float s12 = v[4], s21 = v[5];
    const float l = (-2.f * s12 / (nq1 * nz2) + -2.f * s21 / (nq2 * nz1)) / (float)rows;
    loss[0] = l;
    saved[0] = nq1; saved[1] = nq2; saved[2] = nz1; saved[3] = nz2; saved[4] = s12; saved[5] = s21;
  }
}

// d loss / d q1 = go * (-2/b) * ( z2/(|q1||z2|) - <q1,z2> q1 / (|q1|^3 |z2|) ), same for q2 with z1
__global__ void loss_bwd_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                const float* __restrict__ z1, const float* __restrict__ z2,
                                const float* __restrict__ saved, const float* __restrict__ grad_out,
                                float* __restrict__ dq1, float* __restrict__ dq2, int64_t n4, int rows) {
  const float go = grad_out != nullptr ? grad_out[0] : 1.f;
  const float nq1 = saved[0], nq2 = saved[1], nz1 = saved[2], nz2 = saved[3], s12 = saved[4], s21 = saved[5];
  const float k = go * -2.f / (float)rows;
  const float a1 = k / (nq1 * nz2), b1 = -k * s12 / (nq1 * nq1 * nq1 * nz2);
  const float a2 = k / (nq2 * nz1), b2 = -k * s21 / (nq2 * nq2 * nq2 * nz1);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(q1) + i);
    const float4 b = __ldg(reinterpret_cast<const float4*>(q2) + i);
    const float4 c = __ldg(reinterpret_cast<const float4*>(z1) + i);
    const float4 d = __ldg(reinterpret_cast<const float4*>(z2) + i);
    reinterpret_cast<float4*>(dq1)[i] =
        make_float4(a1 * d.x + b1 * a.x, a1 * d.y + b1 * a.y, a1 * d.z + b1 * a.z, a1 * d.w + b1 * a.w);
    reinterpret_cast<float4*>(dq2)[i] =
        make_float4(a2 * c.x + b2 * b.x, a2 * c.y + b2 * b.y, a2 * c.z + b2 * b.z, a2 * c.w + b2 * b.w);
  }
}

// ---------------------------------------------------------------------------------------------
// The BYOL paper's loss: per-sample L2-normalised predictions and targets.
//   r(x) = max(sum x^2, eps)^(-1/2) (eps = 1e-12 under the square root), x^ = r(x) x,
//   l(q, z) = sum_d (q^_d - z^_d)^2,  L = (1/B) sum_i [ l(q1_i, z2_i) + l(q2_i, z1_i) ].
// A row whose sum of squares is NaN or +inf (a NaN or inf element, or a finite row whose squares overflow) gets
// r = NaN, so its loss and its gradient are NaN instead of those of a zero row.
// Every fp32 operation is written as an intrinsic or fmaf, so the compiler contracts nothing and the arithmetic is
// exactly what the source says.
// ---------------------------------------------------------------------------------------------
constexpr float kPaperLossEps = 1e-12f;
constexpr int kRowsPerBlock = 8;   // one warp per sample, 256 threads

__device__ __forceinline__ float add_squares(const float4 v, float s) {
  s = fmaf(v.x, v.x, s);
  s = fmaf(v.y, v.y, s);
  s = fmaf(v.z, v.z, s);
  return fmaf(v.w, v.w, s);
}

__device__ __forceinline__ float row_rnorm(float s) {
  return s < INFINITY ? __fdiv_rn(1.f, __fsqrt_rn(fmaxf(s, kPaperLossEps))) : __int_as_float(0x7fffffff);
}

// u = q^ - z^ for one element; l += u^2, p += q^ u
__device__ __forceinline__ void pair_terms(float q, float z, float rq, float rz, float& l, float& p) {
  const float qh = __fmul_rn(rq, q);
  const float u = __fsub_rn(qh, __fmul_rn(rz, z));
  l = fmaf(u, u, l);
  p = fmaf(qh, u, p);
}

__device__ __forceinline__ void pair_terms4(const float4 q, const float4 z, float rq, float rz, float& l, float& p) {
  pair_terms(q.x, z.x, rq, rz, l, p);
  pair_terms(q.y, z.y, rq, rz, l, p);
  pair_terms(q.z, z.z, rq, rz, l, p);
  pair_terms(q.w, z.w, rq, rz, l, p);
}

// Warp w of block b takes sample i = 8b + w, both of its pairs (q1_i, z2_i) and (q2_i, z1_i).  Lane l sums the float4s
// l, l + 32, ... of each row in order (x, y, z, w by fmaf), then a butterfly over the 32 lanes.  Pass 1 gives the
// sums of squares, pass 2 re-reads the rows (from L1) for l and q^.u.  saved[8 i ..] = r(q1), r(z2), c12, l12, r(q2),
// r(z1), c21, l21 with c = q^.u when sum q^2 > eps and 0 when the row is clamped.  part[b] = the fp64 sum, in warp
// order, of (double)l12 + (double)l21 over the block's samples.
__global__ void __launch_bounds__(256)
loss_rows_fwd_kernel(const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ z1,
                     const float* __restrict__ z2, int rows, int d4, float* __restrict__ saved,
                     double* __restrict__ part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = blockIdx.x * kRowsPerBlock + warp;
  double lrow = 0.0;
  if (row < rows) {
    const int64_t off = (int64_t)row * d4;
    const float4* __restrict__ a4 = reinterpret_cast<const float4*>(q1) + off;
    const float4* __restrict__ b4 = reinterpret_cast<const float4*>(z2) + off;
    const float4* __restrict__ c4 = reinterpret_cast<const float4*>(q2) + off;
    const float4* __restrict__ d4p = reinterpret_cast<const float4*>(z1) + off;
    float sq1 = 0.f, sz2 = 0.f, sq2 = 0.f, sz1 = 0.f;
    for (int j = lane; j < d4; j += 32) {
      sq1 = add_squares(__ldg(a4 + j), sq1);
      sz2 = add_squares(__ldg(b4 + j), sz2);
      sq2 = add_squares(__ldg(c4 + j), sq2);
      sz1 = add_squares(__ldg(d4p + j), sz1);
    }
    sq1 = warp_sum(sq1); sz2 = warp_sum(sz2); sq2 = warp_sum(sq2); sz1 = warp_sum(sz1);
    const float rq1 = row_rnorm(sq1), rz2 = row_rnorm(sz2), rq2 = row_rnorm(sq2), rz1 = row_rnorm(sz1);
    float l12 = 0.f, p12 = 0.f, l21 = 0.f, p21 = 0.f;
    for (int j = lane; j < d4; j += 32) {
      pair_terms4(__ldg(a4 + j), __ldg(b4 + j), rq1, rz2, l12, p12);
      pair_terms4(__ldg(c4 + j), __ldg(d4p + j), rq2, rz1, l21, p21);
    }
    l12 = warp_sum(l12); p12 = warp_sum(p12); l21 = warp_sum(l21); p21 = warp_sum(p21);
    if (lane == 0) {
      float4* s = reinterpret_cast<float4*>(saved + (int64_t)row * 8);
      s[0] = make_float4(rq1, rz2, sq1 > kPaperLossEps ? p12 : 0.f, l12);
      s[1] = make_float4(rq2, rz1, sq2 > kPaperLossEps ? p21 : 0.f, l21);
    }
    lrow = (double)l12 + (double)l21;
  }
  __shared__ double sh[kRowsPerBlock];
  if (lane == 0) sh[warp] = lrow;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kRowsPerBlock; ++w) s += sh[w];
    part[blockIdx.x] = s;
  }
}

// loss = (float)(S / rows), S the fp64 sum of the nb block slots: lane l adds slots l, l + 32, ... in order (and zeroes
// them: they live in the stream's scratch, which its users leave zeroed), then a butterfly over the lanes.
__global__ void loss_rows_finalize_kernel(double* __restrict__ part, int nb, int rows, float* __restrict__ loss) {
  const int lane = threadIdx.x;
  double s = 0.0;
  for (int b = lane; b < nb; b += 32) {
    s += part[b];
    part[b] = 0.0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) loss[0] = (float)(s / (double)rows);
}

// dq = a * (u - c q^) per element, a = fl(fl(2 go / rows) * r(q)), u = q^ - z^ recomputed from q, z and the saved
// r(q), r(z); the inner term is one fmaf(-c, q^, u).  One pass over q and z, no atomics.
__device__ __forceinline__ float pair_grad(float q, float z, float rq, float rz, float c, float a) {
  const float qh = __fmul_rn(rq, q);
  const float u = __fsub_rn(qh, __fmul_rn(rz, z));
  return __fmul_rn(a, fmaf(-c, qh, u));
}

__device__ __forceinline__ float4 pair_grad4(const float4 q, const float4 z, float rq, float rz, float c, float a) {
  return make_float4(pair_grad(q.x, z.x, rq, rz, c, a), pair_grad(q.y, z.y, rq, rz, c, a),
                     pair_grad(q.z, z.z, rq, rz, c, a), pair_grad(q.w, z.w, rq, rz, c, a));
}

__global__ void __launch_bounds__(256)
loss_rows_bwd_kernel(const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ z1,
                     const float* __restrict__ z2, const float* __restrict__ saved,
                     const float* __restrict__ grad_out, float* __restrict__ dq1, float* __restrict__ dq2,
                     int64_t n4, int d4, int rows) {
  const float go = grad_out != nullptr ? grad_out[0] : 1.f;
  const float k = __fdiv_rn(__fmul_rn(go, 2.f), (float)rows);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4* s = reinterpret_cast<const float4*>(saved + (i / d4) * 8);
    const float4 s12 = __ldg(s), s21 = __ldg(s + 1);
    reinterpret_cast<float4*>(dq1)[i] = pair_grad4(__ldg(reinterpret_cast<const float4*>(q1) + i),
                                                   __ldg(reinterpret_cast<const float4*>(z2) + i), s12.x, s12.y, s12.z,
                                                   __fmul_rn(k, s12.x));
    reinterpret_cast<float4*>(dq2)[i] = pair_grad4(__ldg(reinterpret_cast<const float4*>(q2) + i),
                                                   __ldg(reinterpret_cast<const float4*>(z1) + i), s21.x, s21.y, s21.z,
                                                   __fmul_rn(k, s21.x));
  }
}

// ---------------------------------------------------------------------------------------------
// EMA:  mean[i] = fl(fl(a*x[i]) + fl(d*mean[i]))   a = fp32(1-decay), d = fp32(decay)
// float4-vectorised; 12 B/param of HBM traffic.
// ---------------------------------------------------------------------------------------------
__global__ void ema_kernel(const float* __restrict__ x, float* __restrict__ mean, float a, float d, int64_t n) {
  const int64_t n4 = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + i);
    float4 mv = reinterpret_cast<float4*>(mean)[i];
    mv.x = __fadd_rn(__fmul_rn(a, xv.x), __fmul_rn(d, mv.x));
    mv.y = __fadd_rn(__fmul_rn(a, xv.y), __fmul_rn(d, mv.y));
    mv.z = __fadd_rn(__fmul_rn(a, xv.z), __fmul_rn(d, mv.z));
    mv.w = __fadd_rn(__fmul_rn(a, xv.w), __fmul_rn(d, mv.w));
    reinterpret_cast<float4*>(mean)[i] = mv;
  }
  // tail (n not a multiple of 4)
  for (int64_t i = (n4 << 2) + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
    mean[i] = __fadd_rn(__fmul_rn(a, x[i]), __fmul_rn(d, mean[i]));
}

// ---------------------------------------------------------------------------------------------
// Multi-tensor LARS + SGD momentum.
// Tensors are described by device pointer tables p_ptrs/g_ptrs/m_ptrs[t]; work is split by a chunk table:
// chunk j covers elements [chunk_start[j], chunk_start[j] + chunk_len[j]) of tensor chunk_tensor[j]; the chunks of
// tensor t are the contiguous range [tensor_first_chunk[t], tensor_first_chunk[t + 1]).
// Per tensor t: wd[t], lr[t], ignore[t] (1 = bias/BN: weight decay only if wd>0, no LARS scaling).
// Pass 1: partial[2j] = |p|^2, partial[2j+1] = |g + wd*p|^2 over chunk j (fp64, plain stores: NO atomics, so the
// norms - and with them the updates - are bit-identical on every data-parallel replica, main.py:440).
// Pass 2: every block re-adds its tensor's partials in chunk order (fixed tree) and applies the update.
// Both passes use 16-byte vector accesses when p / g / momentum share a 16-byte phase (always true for the engine's
// flat buffers); otherwise a scalar loop.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool aligned16(const void* a, const void* b, const void* c) {
  return ((((uintptr_t)a) | ((uintptr_t)b) | ((uintptr_t)c)) & 15u) == 0;
}

__global__ void __launch_bounds__(256)
lars_norms_kernel(const uint64_t* __restrict__ p_ptrs, const uint64_t* __restrict__ g_ptrs,
                  const int64_t* __restrict__ chunk_start, const int* __restrict__ chunk_len,
                  const int* __restrict__ chunk_tensor, const float* __restrict__ wd,
                  const int* __restrict__ ignore, double* __restrict__ partial) {
  const int j = blockIdx.x;
  const int t = chunk_tensor[j];
  if (ignore[t]) return;   // norms unused for ignored tensors
  const float* __restrict__ p = reinterpret_cast<const float*>(p_ptrs[t]) + chunk_start[j];
  const float* __restrict__ g = reinterpret_cast<const float*>(g_ptrs[t]) + chunk_start[j];
  const int len = chunk_len[j];
  const float w = wd[t];
  float ap = 0.f, ag = 0.f;
  int done = 0;
  if (aligned16(p, g, nullptr)) {
    const int n4 = len >> 2;
    const float4* __restrict__ p4 = reinterpret_cast<const float4*>(p);
    const float4* __restrict__ g4 = reinterpret_cast<const float4*>(g);
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
      const float4 pv = __ldg(p4 + i);
      float4 gv = __ldg(g4 + i);
      if (w > 0.f) { gv.x += w * pv.x; gv.y += w * pv.y; gv.z += w * pv.z; gv.w += w * pv.w; }
      ap += pv.x * pv.x + pv.y * pv.y + pv.z * pv.z + pv.w * pv.w;
      ag += gv.x * gv.x + gv.y * gv.y + gv.z * gv.z + gv.w * gv.w;
    }
    done = n4 << 2;
  }
  for (int i = done + threadIdx.x; i < len; i += blockDim.x) {
    const float pv = p[i];
    float gv = g[i];
    if (w > 0.f) gv = gv + w * pv;
    ap += pv * pv;
    ag += gv * gv;
  }
  __shared__ float sh[2][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  ap = warp_sum(ap);
  ag = warp_sum(ag);
  if (lane == 0) { sh[0][warp] = ap; sh[1][warp] = ag; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    float a = lane < nw ? sh[0][lane] : 0.f;
    float b = lane < nw ? sh[1][lane] : 0.f;
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) {
      partial[2 * j] = (double)a;
      partial[2 * j + 1] = (double)b;
    }
  }
}

// The elementwise part of a chunk update, shared by the LARS and the Nesterov-SGD kernels: `rule` updates element i
// of the chunk (vec: the four elements 4i .. 4i + 3 as float4, when p / g / momentum share a 16-byte phase; scalar:
// element i), one thread per element (group), block-strided.
template <class Rule, class G>
__device__ __forceinline__ void update_chunk(float* __restrict__ p, G* __restrict__ g, float* __restrict__ mom, int len,
                                             const Rule& rule) {
  int done = 0;
  if (aligned16(p, g, mom)) {
    const int n4 = len >> 2;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) rule.vec(p, g, mom, i);
    done = n4 << 2;
  }
  for (int i = done + threadIdx.x; i < len; i += blockDim.x) rule.scalar(p, g, mom, i);
}

// LARS-scaled SGD with momentum (torch.optim.SGD, momentum without nesterov; mom may be null: no momentum)
struct LarsRule {
  float w, ratio, rate, momentum;
  int first_step;
  __device__ __forceinline__ void vec(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ mom,
                                      int i) const {
    float4* __restrict__ p4 = reinterpret_cast<float4*>(p);
    const float4* __restrict__ g4 = reinterpret_cast<const float4*>(g);
    float4* __restrict__ m4 = reinterpret_cast<float4*>(mom);
    float4 pv = p4[i];
    float4 gv = __ldg(g4 + i);
    if (w > 0.f) { gv.x += w * pv.x; gv.y += w * pv.y; gv.z += w * pv.z; gv.w += w * pv.w; }
    gv.x *= ratio; gv.y *= ratio; gv.z *= ratio; gv.w *= ratio;
    float4 b = gv;
    if (mom != nullptr) {
      if (!first_step) {
        const float4 mv = m4[i];
        b.x = momentum * mv.x + gv.x; b.y = momentum * mv.y + gv.y;
        b.z = momentum * mv.z + gv.z; b.w = momentum * mv.w + gv.w;
      }
      m4[i] = b;
    }
    pv.x -= rate * b.x; pv.y -= rate * b.y; pv.z -= rate * b.z; pv.w -= rate * b.w;
    p4[i] = pv;
  }
  __device__ __forceinline__ void scalar(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ mom,
                                         int i) const {
    const float pv = p[i];
    float gv = g[i];
    if (w > 0.f) gv = gv + w * pv;
    gv = gv * ratio;
    float b = gv;
    if (mom != nullptr) {
      b = first_step ? gv : momentum * mom[i] + gv;
      mom[i] = b;
    }
    p[i] = pv - rate * b;
  }
};

__global__ void __launch_bounds__(256)
lars_update_kernel(const uint64_t* __restrict__ p_ptrs, const uint64_t* __restrict__ g_ptrs,
                   const uint64_t* __restrict__ m_ptrs, const int64_t* __restrict__ chunk_start,
                   const int* __restrict__ chunk_len, const int* __restrict__ chunk_tensor,
                   const int* __restrict__ tensor_first_chunk, const float* __restrict__ wd,
                   const float* __restrict__ lr, const int* __restrict__ ignore,
                   const double* __restrict__ partial, float trust_coef, float eps, float momentum,
                   int first_step) {
  const int j = blockIdx.x;
  const int t = chunk_tensor[j];
  float* __restrict__ p = reinterpret_cast<float*>(p_ptrs[t]) + chunk_start[j];
  const float* __restrict__ g = reinterpret_cast<const float*>(g_ptrs[t]) + chunk_start[j];
  float* __restrict__ mom = m_ptrs != nullptr ? reinterpret_cast<float*>(m_ptrs[t]) + chunk_start[j] : nullptr;
  const int len = chunk_len[j];
  const float w = wd[t];
  const float rate = lr[t];
  __shared__ float s_ratio;
  if (threadIdx.x < 32) {
    float ratio = 1.f;
    if (!ignore[t]) {
      // fixed-order sum of the tensor's chunk partials: lane l takes chunks l, l + 32, ...; then a shuffle tree
      double sp = 0.0, sg = 0.0;
      for (int c = tensor_first_chunk[t] + (int)threadIdx.x; c < tensor_first_chunk[t + 1]; c += 32) {
        sp += partial[2 * c];
        sg += partial[2 * c + 1];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        sp += __shfl_xor_sync(0xffffffffu, sp, o);
        sg += __shfl_xor_sync(0xffffffffu, sg, o);
      }
      const float pn = sqrtf((float)sp);
      const float gn = sqrtf((float)sg);
      if (pn > 0.f && gn > 0.f) ratio = trust_coef * pn / (gn + eps);
    }
    if (threadIdx.x == 0) s_ratio = ratio;
  }
  __syncthreads();
  update_chunk(p, g, mom, len, LarsRule{w, s_ratio, rate, momentum, first_step});
}

// Nesterov SGD (torch.optim.SGD(nesterov=True, dampening=0)) in torch's order with every fp32 operation rounded on its
// own (nesterov_update, common.cuh); the gradient is zeroed as it is read, for the next backward pass to accumulate on.
struct NesterovRule {
  float rate, decay, momentum;
  __device__ __forceinline__ void vec(float* __restrict__ p, float* __restrict__ g, float* __restrict__ mom,
                                      int i) const {
    float4* __restrict__ p4 = reinterpret_cast<float4*>(p);
    float4* __restrict__ g4 = reinterpret_cast<float4*>(g);
    float4* __restrict__ m4 = reinterpret_cast<float4*>(mom);
    float4 pv = p4[i], gv = g4[i], mv = m4[i];
    nesterov_update(pv.x, mv.x, gv.x, rate, decay, momentum);
    nesterov_update(pv.y, mv.y, gv.y, rate, decay, momentum);
    nesterov_update(pv.z, mv.z, gv.z, rate, decay, momentum);
    nesterov_update(pv.w, mv.w, gv.w, rate, decay, momentum);
    p4[i] = pv;
    m4[i] = mv;
    g4[i] = gv;
  }
  __device__ __forceinline__ void scalar(float* __restrict__ p, float* __restrict__ g, float* __restrict__ mom,
                                         int i) const {
    nesterov_update(p[i], mom[i], g[i], rate, decay, momentum);
  }
};

__global__ void __launch_bounds__(256)
sgd_nesterov_kernel(const uint64_t* __restrict__ p_ptrs, const uint64_t* __restrict__ g_ptrs,
                    const uint64_t* __restrict__ m_ptrs, const int64_t* __restrict__ chunk_start,
                    const int* __restrict__ chunk_len, const int* __restrict__ chunk_tensor,
                    const float* __restrict__ wd, const float* __restrict__ lr, float lr_scale, float momentum) {
  const int j = blockIdx.x;
  const int t = chunk_tensor[j];
  float* __restrict__ p = reinterpret_cast<float*>(p_ptrs[t]) + chunk_start[j];
  float* __restrict__ g = reinterpret_cast<float*>(g_ptrs[t]) + chunk_start[j];
  float* __restrict__ mom = reinterpret_cast<float*>(m_ptrs[t]) + chunk_start[j];
  update_chunk(p, g, mom, chunk_len[j], NesterovRule{__fmul_rn(lr[t], lr_scale), wd[t], momentum});
}

// ---------------------------------------------------------------------------------------------
// Linear-probe objective: softmax cross-entropy (mean over rows) + top-1 / top-5 accuracy of fp32 logits [R, C]
// (/root/reference/main.py:596-598: F.cross_entropy + helpers.metrics.topk on the [2b, 1000] classifier output).
// One warp per row: max, log-sum-exp, the label's logit and its rank.  The rank is the number of other columns whose
// logit is not <= the label's (linprobe_ce_kernel's rule): for finite logits the strictly larger ones, and a NaN
// column ranks above the label; the label is in the top k iff rank < k.  A row whose label logit is NaN, or whose
// label (compared as int64) is outside [0, C), is a miss for every k; the latter's loss is +inf.  Row results go to a
// scratch array; the last block to finish (ticket counter) adds them up in row order, so the three outputs are
// deterministic.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ce_topk_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, int LR, int R, int C, int ld,
                   float* __restrict__ row_lse, float* __restrict__ row_loss, int* __restrict__ row_rank,
                   unsigned int* __restrict__ ticket, float* __restrict__ out /* [3] loss, top1 %, top5 % */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = blockIdx.x * (blockDim.x >> 5) + warp;
  if (r < R) {
    const float* __restrict__ x = logits + (int64_t)r * ld;
    const int64_t lab64 = labels[r % LR];   // LR < R: the label vector repeats (two views per sample)
    const bool lab_ok = lab64 >= 0 && lab64 < C;
    const int lab = lab_ok ? (int)lab64 : -1;
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, x[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float xl = lab_ok ? x[lab] : -INFINITY;
    float se = 0.f;
    int gt = 0;
    for (int c = lane; c < C; c += 32) {
      const float v = x[c];
      se += expf(v - mx);
      gt += (c != lab && !(v <= xl)) ? 1 : 0;
    }
    se = warp_sum(se);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gt += __shfl_xor_sync(0xffffffffu, gt, o);
    if (lane == 0) {
      const float lse = mx + logf(se);
      row_lse[r] = lse;
      row_loss[r] = lse - xl;
      row_rank[r] = lab_ok && !isnan(xl) ? gt : 0x7fffffff;   // a miss for every k
    }
  }
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();
  // fixed-order reduction over rows: thread i takes rows i, i + 256, ...; then a fixed shared-memory tree
  double l = 0.0;
  int t1 = 0, t5 = 0;
  for (int i = threadIdx.x; i < R; i += blockDim.x) {
    l += (double)__ldcg(row_loss + i);
    const int rk = __ldcg(row_rank + i);
    t1 += rk < 1;
    t5 += rk < 5;
  }
  __shared__ double sl[256];
  __shared__ int s1[256], s5[256];
  sl[threadIdx.x] = l; s1[threadIdx.x] = t1; s5[threadIdx.x] = t5;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) {
      sl[threadIdx.x] += sl[threadIdx.x + o];
      s1[threadIdx.x] += s1[threadIdx.x + o];
      s5[threadIdx.x] += s5[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = (float)(sl[0] / (double)R);
    out[1] = 100.f * (float)s1[0] / (float)R;
    out[2] = 100.f * (float)s5[0] / (float)R;
    *ticket = 0u;   // ready for the next launch
  }
}

// dlogits[r, c] = go / R * (softmax(x_r)[c] - [c == label_r])
__global__ void __launch_bounds__(256)
ce_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, int LR,
              const float* __restrict__ row_lse, const float* __restrict__ grad_out, int R, int C, int ld,
              float* __restrict__ dlogits, int ldd) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = blockIdx.x * (blockDim.x >> 5) + warp;
  if (r >= R) return;
  const float k = (grad_out != nullptr ? grad_out[0] : 1.f) / (float)R;
  const float* __restrict__ x = logits + (int64_t)r * ld;
  float* __restrict__ d = dlogits + (int64_t)r * ldd;
  const float lse = row_lse[r];
  const int64_t lab64 = labels[r % LR];
  const int lab = lab64 >= 0 && lab64 < C ? (int)lab64 : -1;   // out of range: no one-hot term
  for (int c = lane; c < C; c += 32) d[c] = k * (expf(x[c] - lse) - (c == lab ? 1.f : 0.f));
}

static inline int grid_for(int64_t n, int block, int max_blocks = 132 * 16) {
  int64_t b = (n + block - 1) / block;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace byol

using namespace byol;

// q1,q2,z1,z2: [rows, dim] fp32 contiguous (rows*dim % 4 == 0).  workspace: 6 doubles (zeroed here).
// loss: 1 float.  saved: 6 floats consumed by byol_loss_bwd.  The per-block partial sums (6 x at most 132 doubles) live
// in the stream's zeroed scratch (fix_scratch, whose accumulators are three 8-byte words each, so zero bits read as
// 0.0); `workspace` is part of the ABI but no longer used.
extern "C" int byol_loss_fwd(const float* q1, const float* q2, const float* z1, const float* z2, int rows, int dim,
                             double* workspace, float* loss, float* saved, cudaStream_t stream) {
  BYOL_CHECK_ARG(q1 && q2 && z1 && z2 && workspace && loss && saved, "byol_loss_fwd: null pointer");
  const int64_t n = (int64_t)rows * dim;
  BYOL_CHECK_ARG(rows > 0 && dim > 0 && n % 4 == 0, "byol_loss_fwd: rows*dim must be a positive multiple of 4");
  constexpr int kMaxBlocks = 132;
  static_assert(sizeof(Fix128) == 3 * sizeof(double), "the partial slots are carved from the Fix128 scratch");
  Fix128* scratch = fix_scratch(stream, 2 * kMaxBlocks);   // 6 * kMaxBlocks doubles
  if (scratch == nullptr) return -2;
  double* part = reinterpret_cast<double*>(scratch);
  const int nb = grid_for(n / 4, 256, kMaxBlocks);
  loss_fwd_partial_kernel<<<nb, 256, 0, stream>>>(q1, q2, z1, z2, part, n / 4);
  loss_finalize_kernel<<<1, 32, 0, stream>>>(part, nb, loss, saved, rows);
  return fix_done(stream, check_launch("loss_fwd kernels"));
}

extern "C" int byol_loss_bwd(const float* q1, const float* q2, const float* z1, const float* z2, const float* saved,
                             const float* grad_out, float* dq1, float* dq2, int rows, int dim, cudaStream_t stream) {
  BYOL_CHECK_ARG(q1 && q2 && z1 && z2 && saved && dq1 && dq2, "byol_loss_bwd: null pointer");
  const int64_t n = (int64_t)rows * dim;
  BYOL_CHECK_ARG(rows > 0 && dim > 0 && n % 4 == 0, "byol_loss_bwd: rows*dim must be a positive multiple of 4");
  loss_bwd_kernel<<<grid_for(n / 4, 256, 132 * 4), 256, 0, stream>>>(q1, q2, z1, z2, saved, grad_out, dq1, dq2,
                                                                    n / 4, rows);
  return check_launch("loss_bwd_kernel");
}

static inline bool aligned16_host(const void* p) { return ((uintptr_t)p & 15u) == 0; }

// The paper's loss.  q1,q2,z1,z2: [rows, dim] fp32 contiguous, 16-byte aligned, dim a positive multiple of 4.
// loss: 1 float; saved: [rows, 8] floats (16-byte aligned) consumed by byol_loss_rows_bwd.  The per-block fp64 slots
// (one per 8 rows) live in the stream's zeroed scratch, as byol_loss_fwd's do; the grid depends on rows alone.
extern "C" int byol_loss_rows_fwd(const float* q1, const float* q2, const float* z1, const float* z2, int rows,
                                  int dim, float* loss, float* saved, cudaStream_t stream) {
  BYOL_CHECK_ARG(q1 && q2 && z1 && z2 && loss && saved, "byol_loss_rows_fwd: null pointer");
  BYOL_CHECK_ARG(rows > 0 && dim > 0 && dim % 4 == 0,
                 "byol_loss_rows_fwd: need rows >= 1 and dim a positive multiple of 4 (rows=%d dim=%d)", rows, dim);
  BYOL_CHECK_ARG(aligned16_host(q1) && aligned16_host(q2) && aligned16_host(z1) && aligned16_host(z2) &&
                     aligned16_host(saved),
                 "byol_loss_rows_fwd: q1, q2, z1, z2 and saved must be 16-byte aligned");
  const int nb = (rows + kRowsPerBlock - 1) / kRowsPerBlock;
  static_assert(sizeof(Fix128) == 3 * sizeof(double), "the block slots are carved from the Fix128 scratch");
  Fix128* scratch = fix_scratch(stream, (nb + 2) / 3);
  if (scratch == nullptr) return -2;
  double* part = reinterpret_cast<double*>(scratch);
  loss_rows_fwd_kernel<<<nb, 32 * kRowsPerBlock, 0, stream>>>(q1, q2, z1, z2, rows, dim / 4, saved, part);
  loss_rows_finalize_kernel<<<1, 32, 0, stream>>>(part, nb, rows, loss);
  return fix_done(stream, check_launch("loss_rows_fwd kernels"));
}

// dq1, dq2: [rows, dim] fp32 (16-byte aligned); grad_out: 1 float or null (1).
extern "C" int byol_loss_rows_bwd(const float* q1, const float* q2, const float* z1, const float* z2,
                                  const float* saved, const float* grad_out, float* dq1, float* dq2, int rows, int dim,
                                  cudaStream_t stream) {
  BYOL_CHECK_ARG(q1 && q2 && z1 && z2 && saved && dq1 && dq2, "byol_loss_rows_bwd: null pointer");
  BYOL_CHECK_ARG(rows > 0 && dim > 0 && dim % 4 == 0,
                 "byol_loss_rows_bwd: need rows >= 1 and dim a positive multiple of 4 (rows=%d dim=%d)", rows, dim);
  BYOL_CHECK_ARG(aligned16_host(q1) && aligned16_host(q2) && aligned16_host(z1) && aligned16_host(z2) &&
                     aligned16_host(saved) && aligned16_host(dq1) && aligned16_host(dq2),
                 "byol_loss_rows_bwd: every array must be 16-byte aligned");
  const int64_t n4 = (int64_t)rows * (dim / 4);
  loss_rows_bwd_kernel<<<grid_for(n4, 256, 132 * 4), 256, 0, stream>>>(q1, q2, z1, z2, saved, grad_out, dq1, dq2,
                                                                       n4, dim / 4, rows);
  return check_launch("loss_rows_bwd_kernel");
}

// mean = fl(fl(one_minus_decay*x) + fl(decay*mean)), elementwise over n fp32 values
extern "C" int byol_ema_update(const float* x, float* mean, float one_minus_decay, float decay, int64_t n,
                               cudaStream_t stream) {
  BYOL_CHECK_ARG(x && mean && n > 0, "byol_ema_update: bad args");
  BYOL_CHECK_ARG(((uintptr_t)x % 16 == 0) && ((uintptr_t)mean % 16 == 0), "byol_ema_update: pointers must be 16-byte aligned");
  ema_kernel<<<grid_for(n / 4 + 1, 256, 132 * 8), 256, 0, stream>>>(x, mean, one_minus_decay, decay, n);
  return check_launch("ema_kernel");
}

// p_ptrs/g_ptrs/m_ptrs: device arrays of num_tensors fp32 pointers (m_ptrs may be null: no momentum).
// tensor_first_chunk: [num_tensors + 1]; partial: 2 * num_chunks doubles of scratch.
extern "C" int byol_lars_sgd_step(const void* p_ptrs, const void* g_ptrs, const void* m_ptrs,
                                  const int64_t* chunk_start, const int* chunk_len, const int* chunk_tensor,
                                  int num_chunks, const int* tensor_first_chunk, const float* wd, const float* lr,
                                  const int* ignore, int num_tensors, double* partial, float trust_coef, float eps,
                                  float momentum, int first_step, cudaStream_t stream) {
  BYOL_CHECK_ARG(p_ptrs && g_ptrs && chunk_start && chunk_len && chunk_tensor && tensor_first_chunk && wd && lr &&
                     ignore && partial,
                 "byol_lars_sgd_step: null pointer");
  BYOL_CHECK_ARG(num_chunks > 0 && num_tensors > 0, "byol_lars_sgd_step: empty");
  lars_norms_kernel<<<num_chunks, 256, 0, stream>>>((const uint64_t*)p_ptrs, (const uint64_t*)g_ptrs, chunk_start,
                                                   chunk_len, chunk_tensor, wd, ignore, partial);
  lars_update_kernel<<<num_chunks, 256, 0, stream>>>((const uint64_t*)p_ptrs, (const uint64_t*)g_ptrs,
                                                    (const uint64_t*)m_ptrs, chunk_start, chunk_len, chunk_tensor,
                                                    tensor_first_chunk, wd, lr, ignore, partial, trust_coef, eps,
                                                    momentum, first_step);
  return check_launch("lars kernels");
}

// The chunk tables of byol_lars_sgd_step (m_ptrs required); lr = fp32(lr[t] * lr_scale) per tensor.
extern "C" int byol_sgd_nesterov_step(const void* p_ptrs, const void* g_ptrs, const void* m_ptrs,
                                      const int64_t* chunk_start, const int* chunk_len, const int* chunk_tensor,
                                      int num_chunks, const float* wd, const float* lr, float lr_scale, float momentum,
                                      cudaStream_t stream) {
  BYOL_CHECK_ARG(p_ptrs && g_ptrs && m_ptrs && chunk_start && chunk_len && chunk_tensor && wd && lr,
                 "byol_sgd_nesterov_step: null pointer");
  BYOL_CHECK_ARG(num_chunks > 0, "byol_sgd_nesterov_step: empty");
  sgd_nesterov_kernel<<<num_chunks, 256, 0, stream>>>((const uint64_t*)p_ptrs, (const uint64_t*)g_ptrs,
                                                     (const uint64_t*)m_ptrs, chunk_start, chunk_len, chunk_tensor,
                                                     wd, lr, lr_scale, momentum);
  return check_launch("sgd_nesterov_kernel");
}

// logits: fp32 [R, C] with row pitch ld; labels: int64 [label_rows], row r uses labels[r % label_rows].  row_lse / row_loss: R floats, row_rank: R ints,
// ticket: one zero-initialised uint32 (the kernel resets it).  out: [loss (mean), top-1 %, top-5 %].
extern "C" int byol_ce_topk_fwd(const float* logits, const int64_t* labels, int label_rows, int R, int C, int ld, float* row_lse,
                                float* row_loss, int* row_rank, unsigned int* ticket, float* out,
                                cudaStream_t stream) {
  BYOL_CHECK_ARG(logits && labels && row_lse && row_loss && row_rank && ticket && out, "byol_ce_topk_fwd: null pointer");
  BYOL_CHECK_ARG(R > 0 && C > 0 && ld >= C, "byol_ce_topk_fwd: bad shape R=%d C=%d ld=%d", R, C, ld);
  BYOL_CHECK_ARG(label_rows > 0 && R % label_rows == 0, "byol_ce_topk_fwd: %d labels do not tile %d rows", label_rows, R);
  ce_topk_fwd_kernel<<<(R + 7) / 8, 256, 0, stream>>>(logits, labels, label_rows, R, C, ld, row_lse, row_loss, row_rank, ticket,
                                                      out);
  return check_launch("ce_topk_fwd_kernel");
}

extern "C" int byol_ce_bwd(const float* logits, const int64_t* labels, int label_rows, const float* row_lse, const float* grad_out,
                           int R, int C, int ld, float* dlogits, int ldd, cudaStream_t stream) {
  BYOL_CHECK_ARG(logits && labels && row_lse && dlogits, "byol_ce_bwd: null pointer");
  BYOL_CHECK_ARG(R > 0 && C > 0 && ld >= C && ldd >= C && label_rows > 0 && R % label_rows == 0, "byol_ce_bwd: bad shape");
  ce_bwd_kernel<<<(R + 7) / 8, 256, 0, stream>>>(logits, labels, label_rows, row_lse, grad_out, R, C, ld, dlogits, ldd);
  return check_launch("ce_bwd_kernel");
}
