// byol_b200 — linear evaluation of frozen features: H linear classifiers (one per learning-rate / weight-decay pair)
// trained together with Nesterov SGD on the same bf16 features.
//
// The heads' weights are one [H * Cp, D] matrix (Cp = the class count C rounded up to a multiple of 8; rows c >= C of
// each head are zero padding), so the logits of all heads come from one tensor-core GEMM (byol_conv_igemm as a linear
// layer) and the weight gradient from one fixed-point wgrad.  This file holds the two kernels around them:
//
//   byol_linprobe_ce   per (row, head) segment of the fp32 logits: softmax cross-entropy, the label's rank, and
//                      optionally the bf16 gradient (softmax - onehot) / B of the segment
//   byol_linprobe_sgd  the Nesterov-SGD update of every head's weights and biases, the bf16 GEMM copy of the updated
//                      weights, and the gradient buffers zeroed for the next step
//
// The existing probe kernels (ce_topk_fwd / ce_bwd, csrc/optim.cu) handle one head per launch, keep an fp32 gradient
// and reduce through a single ticket; the H heads here would take 3H launches and an fp32 [B, H * C] intermediate.
#include <math.h>

#include "common.cuh"

namespace byol {

static constexpr int CE_WARPS = 8;
static constexpr int SGD_THREADS = 128;

// ---------------------------------------------------------------------------------------------------------------------
// Cross-entropy: block (x, h) handles rows 8x .. 8x + 7 of head h, one warp per row.  Lane l owns the 8-column chunks
// l, l + 32, ... of the segment (two float4 loads, one 16-byte bf16 store).  With m the segment's maximum, xl the
// label's logit, e = exp(xl - m) and s = the sum of exp(v - m) over the other columns:
//   loss = -log softmax[label] = log1p(s / e)          when xl - m > -1 (no cancellation as the loss goes to 0)
//                              = (m - xl) + log(s + e)  otherwise (the loss is >= 1)
//   grad = exp(v - m) / (s + e) / B,  and -s / (s + e) / B at the label (softmax - 1 without cancellation)
// The rank is the number of other columns whose logit is not <= the label's: for finite logits the strictly larger
// ones, and a NaN column ranks above the label; the label is in the top k iff rank < k.  A row whose label logit is
// NaN is a miss for every k, so diverged features or weights can not score hits.  ce_topk_fwd_kernel (csrc/optim.cu)
// ranks by the same rule.  A row whose label is outside [0, C) is ignored here: no loss, no hit, and a zero gradient
// (ce_topk_fwd_kernel counts it as a miss with loss +inf).  Per-head loss sums go to
// fixed-point accumulators and hit counts to integer counters, both order-independent, so every launch gives the
// same bits.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__global__ void __launch_bounds__(CE_WARPS * 32)
linprobe_ce_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels, int B, int C,
                   int Cp, bf16* __restrict__ dlogits, int64_t ldd, Fix128* __restrict__ loss_acc,
                   unsigned long long* __restrict__ hits) {
  __shared__ unsigned long long s_words[2];
  __shared__ unsigned int s_hit[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.y;
  const int r = blockIdx.x * CE_WARPS + warp;
  if (threadIdx.x == 0) {
    s_words[0] = 0ull; s_words[1] = 0ull;
    s_hit[0] = 0u; s_hit[1] = 0u;
  }
  __syncthreads();
  if (r < B) {
    const float* __restrict__ x = logits + (int64_t)r * ld + (int64_t)h * Cp;
    const int64_t lab64 = labels[r];
    const bool lab_ok = lab64 >= 0 && lab64 < C;
    const int lab = lab_ok ? (int)lab64 : -1;
    const int chunks = Cp >> 3;
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
        if (c < C) {
          if (c != lab) {
            so += expf(v[i] - mx);
            gt += v[i] <= xl ? 0 : 1;
          }
        }
      }
    }
    so = warp_sum(so);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gt += __shfl_xor_sync(0xffffffffu, gt, o);
    const float el = expf(xl - mx);
    const float se = so + el;
    if (dlogits != nullptr) {
      const float fb = (float)B;
      bf16* __restrict__ d = dlogits + (int64_t)r * ldd + (int64_t)h * Cp;
      for (int j = lane; j < chunks; j += 32) {
        float v[8];
        load8(x + 8 * j, v);
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 8; i += 2) {
          float g[2];
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int c = 8 * j + i + k;
            g[k] = c >= C || !lab_ok ? 0.f : (c == lab ? -so / se : expf(v[i + k] - mx) / se) / fb;
          }
          w[i >> 1] = pack_bf16x2(g[0], g[1]);
        }
        *reinterpret_cast<uint4*>(d + 8 * j) = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
    if (lane == 0 && lab_ok) {
      if (loss_acc != nullptr) {
        const float loss = xl - mx > -1.f ? log1pf(so / el) : (mx - xl) + logf(se);
        fix_add_local(loss_acc + h, s_words, (double)loss);
      }
      if (!isnan(xl)) {
        if (gt < 1) atomicAdd(&s_hit[0], 1u);
        if (gt < 5) atomicAdd(&s_hit[1], 1u);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (loss_acc != nullptr) fix_add_words(loss_acc + h, s_words[0], (long long)s_words[1]);
    if (hits != nullptr) {
      if (s_hit[0]) atomicAdd(hits + 2 * h, (unsigned long long)s_hit[0]);
      if (s_hit[1]) atomicAdd(hits + 2 * h + 1, (unsigned long long)s_hit[1]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Nesterov SGD, torch.optim.SGD(nesterov=True, dampening=0)'s order with every operation rounded on its own (no FMA
// contraction, as ema_kernel; nesterov_update, common.cuh):
//   g = dW + wd * w;   buf = mu * buf + g;   d = g + mu * buf;   w = w - lr * d
// The momentum starts at zero, so the first step gives buf = g, torch's first step.  One block per weight row (h, c):
// the row's D weights as float4, then its bias by thread 0.  The same pass writes bf16(w) (round to nearest even) to
// the GEMM copy and zeroes dW and db, so the next wgrad / column sum accumulate onto zero.  Padding rows c >= C are
// never read or written.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SGD_THREADS)
linprobe_sgd_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ m, bf16* __restrict__ wb,
                    const float* __restrict__ lr, const float* __restrict__ wd, float lr_scale, float mu, int H, int C,
                    int Cp, int D) {
  const int64_t rows = (int64_t)H * Cp;
  const int d4 = D >> 2;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const int h = (int)(row / Cp);
    if (row - (int64_t)h * Cp >= C) continue;          // padding row (block-uniform)
    const float rate = __fmul_rn(lr[h], lr_scale), decay = wd[h];
    float4* __restrict__ w4 = reinterpret_cast<float4*>(w + row * D);
    float4* __restrict__ g4 = reinterpret_cast<float4*>(g + row * D);
    float4* __restrict__ m4 = reinterpret_cast<float4*>(m + row * D);
    uint2* __restrict__ b4 = reinterpret_cast<uint2*>(wb + row * D);
    for (int j = threadIdx.x; j < d4; j += SGD_THREADS) {
      float4 wv = w4[j], gv = g4[j], mv = m4[j];
      nesterov_update(wv.x, mv.x, gv.x, rate, decay, mu);
      nesterov_update(wv.y, mv.y, gv.y, rate, decay, mu);
      nesterov_update(wv.z, mv.z, gv.z, rate, decay, mu);
      nesterov_update(wv.w, mv.w, gv.w, rate, decay, mu);
      w4[j] = wv;
      m4[j] = mv;
      g4[j] = gv;
      b4[j] = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
    }
    if (threadIdx.x == 0) {
      const int64_t bi = rows * D + row;                 // the biases [H, Cp] follow the weights
      nesterov_update(w[bi], m[bi], g[bi], rate, decay, mu);
    }
  }
}

}  // namespace byol

using namespace byol;

extern "C" int byol_linprobe_ce(const float* logits, int64_t ld, const int64_t* labels, int B, int H, int C, int Cp,
                                void* dlogits, float* loss_sum, long long* hits, cudaStream_t stream) {
  BYOL_CHECK_ARG(logits && labels, "byol_linprobe_ce: null pointer");
  BYOL_CHECK_ARG(dlogits || loss_sum || hits, "byol_linprobe_ce: no output");
  BYOL_CHECK_ARG(B > 0 && H > 0 && H <= 65535 && C >= 2 && C <= Cp && Cp % 8 == 0 && (int64_t)H * Cp <= 0x7fffffffll,
                 "byol_linprobe_ce: bad shape B=%d H=%d C=%d Cp=%d", B, H, C, Cp);
  BYOL_CHECK_ARG(ld >= (int64_t)H * Cp && ld % 4 == 0 && ((uintptr_t)logits & 15) == 0,
                 "byol_linprobe_ce: logits need 16-byte aligned rows with pitch ld=%lld >= H*Cp", (long long)ld);
  BYOL_CHECK_ARG(((uintptr_t)dlogits & 15) == 0, "byol_linprobe_ce: dlogits must be 16-byte aligned");
  Fix128* acc = nullptr;
  if (loss_sum != nullptr) {
    acc = fix_scratch(stream, H);
    if (acc == nullptr) return -2;
  }
  const dim3 grid((unsigned)((B + CE_WARPS - 1) / CE_WARPS), (unsigned)H);
  linprobe_ce_kernel<<<grid, CE_WARPS * 32, 0, stream>>>(logits, ld, labels, B, C, Cp, (bf16*)dlogits,
                                                          (int64_t)H * Cp, acc, (unsigned long long*)hits);
  const int rc = check_launch("linprobe_ce_kernel");
  if (acc == nullptr) return rc;
  return fix_done(stream, rc != 0 ? rc : fix_flush(acc, loss_sum, H, stream));
}

extern "C" int byol_linprobe_sgd(float* params, float* grads, float* momentum_buf, void* weight_bf16, const float* lr,
                                 const float* wd, float lr_scale, float momentum, int H, int C, int Cp, int D,
                                 cudaStream_t stream) {
  BYOL_CHECK_ARG(params && grads && momentum_buf && weight_bf16 && lr && wd, "byol_linprobe_sgd: null pointer");
  BYOL_CHECK_ARG(H > 0 && C >= 1 && C <= Cp && Cp % 8 == 0 && D > 0 && D % 4 == 0,
                 "byol_linprobe_sgd: bad shape H=%d C=%d Cp=%d D=%d", H, C, Cp, D);
  BYOL_CHECK_ARG(((((uintptr_t)params) | ((uintptr_t)grads) | ((uintptr_t)momentum_buf)) & 15) == 0 &&
                     ((uintptr_t)weight_bf16 & 7) == 0,
                 "byol_linprobe_sgd: params / grads / momentum must be 16-byte aligned, the bf16 copy 8-byte aligned");
  const int64_t rows = (int64_t)H * Cp;
  int64_t blocks = (int64_t)device_sm_count() * 16;
  if (blocks > rows) blocks = rows;
  linprobe_sgd_kernel<<<(int)blocks, SGD_THREADS, 0, stream>>>(params, grads, momentum_buf, (bf16*)weight_bf16, lr, wd,
                                                               lr_scale, momentum, H, C, Cp, D);
  return check_launch("linprobe_sgd_kernel");
}
