// byol_b200 — BYOL objective, target-network EMA and LARS + SGD-momentum kernels (fp32, HBM-bound).
//
//   byol_loss_fwd / bwd : /root/reference/objective.py:6-25 (regression_loss with WHOLE-MATRIX Frobenius
//                         norms, no per-row normalisation, rank-local; symmetric sum, mean over rows)
//   byol_ema_update     : /root/reference/main.py:159-162 (CosEMA.forward: mean = (1-d)*x + d*mean as three
//                         separately rounded fp32 ops; bit-exact => no FMA contraction)
//   byol_lars_*         : /root/reference/optimizers/lars.py:84-127 (apply_adaptive_lrs + wrapped SGD step,
//                         torch.optim.SGD momentum=0.9, dampening 0, no nesterov, weight decay folded by LARS)
#include "common.cuh"

namespace byol {

// ---------------------------------------------------------------------------------------------
// loss
// sums[0] = |q1|^2  sums[1] = |q2|^2  sums[2] = |z1|^2  sums[3] = |z2|^2  sums[4] = <q1,z2>  sums[5] = <q2,z1>
// ---------------------------------------------------------------------------------------------
__global__ void loss_fwd_partial_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                        const float* __restrict__ z1, const float* __restrict__ z2,
                                        Fix128* __restrict__ sums, int64_t n4) {
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
      if (lane == 0) fix_add(sums + k, v);   // fixed point: order-independent
    }
  }
}

// loss = -2/b * ( <q1,z2>/(|q1||z2|) + <q2,z1>/(|q2||z1|) );  also stores fp32 copies of the six sums
__global__ void loss_finalize_kernel(Fix128* __restrict__ sums, float* __restrict__ loss,
                                     float* __restrict__ saved, int rows) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    float v[6];
    for (int k = 0; k < 6; ++k) {
      v[k] = (float)fix_value(sums[k]);
      sums[k] = Fix128{0ull, 0ll, 0.0};   // the scratch is left zeroed (fix_scratch)
    }
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
  const float ratio = s_ratio;
  int done = 0;
  if (aligned16(p, g, mom)) {
    const int n4 = len >> 2;
    float4* __restrict__ p4 = reinterpret_cast<float4*>(p);
    const float4* __restrict__ g4 = reinterpret_cast<const float4*>(g);
    float4* __restrict__ m4 = reinterpret_cast<float4*>(mom);
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
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
    done = n4 << 2;
  }
  for (int i = done + threadIdx.x; i < len; i += blockDim.x) {
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
}

// ---------------------------------------------------------------------------------------------
// Linear-probe objective: softmax cross-entropy (mean over rows) + top-1 / top-5 accuracy of fp32 logits [R, C]
// (/root/reference/main.py:596-598: F.cross_entropy + helpers.metrics.topk on the [2b, 1000] classifier output).
// One warp per row: max, log-sum-exp, the label's logit and its rank (= number of strictly larger logits: the
// label is in the top k iff rank < k).  Row results go to a scratch array; the last block to finish (ticket
// counter) adds them up in row order, so the three outputs are deterministic.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ce_topk_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, int LR, int R, int C, int ld,
                   float* __restrict__ row_lse, float* __restrict__ row_loss, int* __restrict__ row_rank,
                   unsigned int* __restrict__ ticket, float* __restrict__ out /* [3] loss, top1 %, top5 % */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = blockIdx.x * (blockDim.x >> 5) + warp;
  if (r < R) {
    const float* __restrict__ x = logits + (int64_t)r * ld;
    const int lab = (int)labels[r % LR];   // LR < R: the label vector repeats (two views per sample)
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, x[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float xl = (lab >= 0 && lab < C) ? x[lab] : -INFINITY;
    float se = 0.f;
    int gt = 0;
    for (int c = lane; c < C; c += 32) {
      const float v = x[c];
      se += expf(v - mx);
      gt += (v > xl) ? 1 : 0;
    }
    se = warp_sum(se);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gt += __shfl_xor_sync(0xffffffffu, gt, o);
    if (lane == 0) {
      const float lse = mx + logf(se);
      row_lse[r] = lse;
      row_loss[r] = lse - xl;
      row_rank[r] = gt;
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
  const int lab = (int)labels[r % LR];
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
// loss: 1 float.  saved: 6 floats consumed by byol_loss_bwd.  The six sums are accumulated in fixed point in the
// stream's scratch (fix_scratch); `workspace` is part of the ABI but no longer used.
extern "C" int byol_loss_fwd(const float* q1, const float* q2, const float* z1, const float* z2, int rows, int dim,
                             double* workspace, float* loss, float* saved, cudaStream_t stream) {
  BYOL_CHECK_ARG(q1 && q2 && z1 && z2 && workspace && loss && saved, "byol_loss_fwd: null pointer");
  const int64_t n = (int64_t)rows * dim;
  BYOL_CHECK_ARG(rows > 0 && dim > 0 && n % 4 == 0, "byol_loss_fwd: rows*dim must be a positive multiple of 4");
  Fix128* sums = fix_scratch(stream, 6);
  if (sums == nullptr) return -2;
  loss_fwd_partial_kernel<<<grid_for(n / 4, 256, 132), 256, 0, stream>>>(q1, q2, z1, z2, sums, n / 4);
  loss_finalize_kernel<<<1, 32, 0, stream>>>(sums, loss, saved, rows);
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
