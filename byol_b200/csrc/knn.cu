// byol_b200 — weighted k-nearest-neighbour evaluation of frozen features (Wu et al. 2018; k = 20, T = 0.07 as in DINO).
//
// The bank holds L2-normalised bf16 features of the training split, the queries those of the test split; the cosine
// similarities of a chunk of queries against a chunk of the bank come from the tensor-core GEMM (byol_conv_igemm as a
// linear layer: the bank rows are the [Cout][K] weight layout).  This file holds the three kernels around that GEMM:
//
//   byol_l2_normalize_rows  fp32 [R, D] -> L2-normalised bf16 rows (fixed-order fp32 norm per row)
//   byol_knn_topk           the k best entries of each query row of an fp32 similarity chunk, merged with the query's
//                           running list from earlier chunks
//   byol_knn_vote           w = exp(s / T) per neighbour, per-class sums, the top-5 classes
//
// Selection order.  Entries are ranked by similarity descending, then bank index ascending.  That order is total, so
// the running list after any sequence of chunks is exactly the first k entries of a full sort of the query's row:
// it does not depend on the chunk sizes, on the number of blocks or on the order in which blocks finish.  -0 ranks as
// +0 and NaN ranks below every number.  Each entry is one 64-bit key (an order-preserving map of the float in the
// high word, the complement of the bank index in the low word), unique per entry, and "the k best" is "the k largest
// keys".  A block per query row finds the k-th largest key by radix selection (11-bit digits, most significant
// first, one histogram pass over the row per digit until at most KT_SORT entries remain above the digits fixed so
// far), gathers those entries into shared memory and sorts them there.
#include <math.h>

#include "common.cuh"

namespace byol {

static constexpr int KT_THREADS = 512;
static constexpr int KT_DIGIT = 11;
static constexpr int KT_BINS = 1 << KT_DIGIT;
static constexpr int KT_SORT = 2048;     // entries gathered and sorted in shared memory
static constexpr int KT_MAX_K = 256;
static constexpr int VOTE_WARPS = 8;

// ---------------------------------------------------------------------------------------------------------------------
// L2 normalisation: one warp per row.  Lane l sums x[l], x[l + 32], ... in order, then a butterfly over the 32 lane
// sums; every step is fixed, so a row always gives the same bits.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void l2_normalize_rows_kernel(const float* __restrict__ x, bf16* __restrict__ y, int64_t R, int D,
                                         int64_t ldx) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); r < R; r += warps) {
    const float* xr = x + r * ldx;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float v = __ldg(xr + c);
      s = fmaf(v, v, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float inv = s > 0.f ? 1.f / sqrtf(s) : 0.f;    // a zero row stays zero
    bf16* yr = y + r * D;
    for (int c = lane; c < D; c += 32) yr[c] = __float2bfloat16_rn(__ldg(xr + c) * inv);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// top-k selection
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t order_key(float v) {
  uint32_t u = __float_as_uint(v);
  if ((u << 1) == 0u) u = 0u;                             // -0 -> +0
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0u;         // NaN: below -inf (whose key is 0x007fffff)
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

// every real entry has a key > 0 (its low word ~index is >= 2^31), so 0 pads the sort
__device__ __forceinline__ unsigned long long entry_key(float v, int index) {
  return ((unsigned long long)order_key(v) << 32) | (unsigned long long)(~(uint32_t)index);
}

// One block per query row.  sim: the row's Nc similarities (pitch ld); bank index of column j is n0 + j.  vals / idx:
// the row's running list (k slots, best first; index -1 marks an empty slot), read when merge != 0 and rewritten.
__global__ void __launch_bounds__(KT_THREADS, 2) knn_topk_kernel(const float* __restrict__ sim, int Nc, int64_t ld,
                                                              int n0, int k, int merge, float* vals, int* idx) {
  __shared__ unsigned int hist[KT_BINS];
  __shared__ unsigned long long keys[KT_SORT];
  __shared__ unsigned int part[KT_THREADS / 32];
  __shared__ unsigned int s_digit, s_greater, s_count, s_n;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = sim + (int64_t)blockIdx.x * ld;
  float* lv = vals + (int64_t)blockIdx.x * k;
  int* li = idx + (int64_t)blockIdx.x * k;

  // entries: the chunk's Nc columns and, with merge, the list's occupied slots
  if (tid == 0) s_n = 0;
  __syncthreads();
  if (merge)
    for (int s = tid; s < k; s += KT_THREADS)
      if (li[s] >= 0) atomicAdd(&s_n, 1u);
  __syncthreads();

  // radix selection: `prefix` holds the top `bits` bits of the k-th largest key; `above` entries have larger top
  // bits, `count` entries share them; above < k <= above + count
  unsigned long long prefix = 0ull;
  int bits = 0;
  unsigned int above = 0, count = (unsigned int)Nc + s_n;
  while (above + count > (unsigned int)KT_SORT) {
    const int width = 64 - bits < KT_DIGIT ? 64 - bits : KT_DIGIT;
    const int shift = 64 - bits - width;
    for (int b = tid; b < KT_BINS; b += KT_THREADS) hist[b] = 0u;
    __syncthreads();
    const unsigned int dmask = (1u << width) - 1u;
    for (int j = tid; j < Nc; j += KT_THREADS) {
      const unsigned long long key = entry_key(__ldg(row + j), n0 + j);
      if (bits == 0 || (key >> (64 - bits)) == prefix) atomicAdd(&hist[(unsigned int)(key >> shift) & dmask], 1u);
    }
    if (merge)
      for (int s = tid; s < k; s += KT_THREADS) {
        const int ix = li[s];
        if (ix < 0) continue;
        const unsigned long long key = entry_key(lv[s], ix);
        if (bits == 0 || (key >> (64 - bits)) == prefix) atomicAdd(&hist[(unsigned int)(key >> shift) & dmask], 1u);
      }
    __syncthreads();
    // the digit d with (entries in digits > d) < need <= (entries in digits >= d): thread t owns the four digits
    // counted down from the top, an exclusive scan gives the entries above them
    static_assert(KT_BINS == 4 * KT_THREADS, "four histogram bins per thread");
    const unsigned int* mine = hist + KT_BINS - 4 - 4 * tid;     // mine[3 - j]: the j-th digit counted from the top
    const unsigned int sum = mine[0] + mine[1] + mine[2] + mine[3];
    unsigned int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) part[warp] = incl;
    __syncthreads();
    unsigned int excl = incl - sum;
    for (int w = 0; w < warp; ++w) excl += part[w];
    const unsigned int need = (unsigned int)k - above;
    if (excl < need && need <= excl + sum) {
      unsigned int run = excl;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const unsigned int cj = mine[3 - j];
        if (run + cj >= need) {
          s_digit = (unsigned int)(KT_BINS - 1 - 4 * tid - j);
          s_greater = run;
          s_count = cj;
          break;
        }
        run += cj;
      }
    }
    __syncthreads();
    prefix = (prefix << width) | s_digit;
    bits += width;
    above += s_greater;
    count = s_count;
    __syncthreads();   // s_* and hist are rewritten by the next digit
  }

  // gather every entry whose top `bits` bits are >= prefix: exactly above + count <= KT_SORT of them
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int j = tid; j < Nc; j += KT_THREADS) {
    const unsigned long long key = entry_key(__ldg(row + j), n0 + j);
    if (bits == 0 || (key >> (64 - bits)) >= prefix) keys[atomicAdd(&s_n, 1u)] = key;
  }
  if (merge)
    for (int s = tid; s < k; s += KT_THREADS) {
      const int ix = li[s];
      if (ix < 0) continue;
      const unsigned long long key = entry_key(lv[s], ix);
      if (bits == 0 || (key >> (64 - bits)) >= prefix) keys[atomicAdd(&s_n, 1u)] = key;
    }
  __syncthreads();
  const int n = (int)s_n;
  int P = 32;
  while (P < n) P <<= 1;
  for (int i = n + tid; i < P; i += KT_THREADS) keys[i] = 0ull;
  __syncthreads();
  // bitonic sort, descending
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < P / 2; i += KT_THREADS) {
        const int pos = 2 * i - (i & (stride - 1));
        const unsigned long long a = keys[pos], b = keys[pos + stride];
        const bool desc = (pos & size) == 0;
        if ((a < b) == desc) {
          keys[pos] = b;
          keys[pos + stride] = a;
        }
      }
      __syncthreads();
    }
  for (int s = tid; s < k; s += KT_THREADS) {
    if (s < n) {
      const unsigned long long key = keys[s];
      lv[s] = key_value((uint32_t)(key >> 32));
      li[s] = (int)~(uint32_t)key;
    } else {
      lv[s] = -INFINITY;
      li[s] = -1;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// vote: one warp per query.  A class's score is the fp64 sum, in neighbour rank order, of the fp32 weights
// w = expf(s / T) of its neighbours; classes rank by score descending, then class index ascending (classes without a
// neighbour score 0).
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool class_before(double sa, int la, double sb, int lb) {
  return sa > sb || (sa == sb && la < lb);
}

__global__ void __launch_bounds__(VOTE_WARPS * 32) knn_vote_kernel(const float* __restrict__ vals,
                                                                   const int* __restrict__ idx,
                                                                   const int64_t* __restrict__ labels, int Q, int k,
                                                                   int C, float T, int* __restrict__ pred,
                                                                   float* __restrict__ pred_scores) {
  __shared__ float sw[VOTE_WARPS][KT_MAX_K];
  __shared__ int sl[VOTE_WARPS][KT_MAX_K];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t q = (int64_t)blockIdx.x * VOTE_WARPS + warp;
  if (q >= Q) return;
  float* w = sw[warp];
  int* l = sl[warp];
  for (int j = lane; j < k; j += 32) {
    const int i = idx[q * k + j];
    l[j] = i >= 0 ? (int)labels[i] : -1;
    w[j] = i >= 0 ? expf(vals[q * k + j] / T) : 0.f;
  }
  __syncwarp();
  // the first neighbour of each class carries the class's score; lane owns neighbours lane, lane + 32, ...
  constexpr int PER_LANE = KT_MAX_K / 32;
  double rs[PER_LANE];
  int rl[PER_LANE];
#pragma unroll
  for (int m = 0; m < PER_LANE; ++m) {
    const int j = lane + 32 * m;
    rl[m] = -1;
    rs[m] = 0.0;
    if (j >= k || l[j] < 0) continue;
    const int c = l[j];
    bool first = true;
    double s = 0.0;
    for (int i = 0; i < k; ++i) {
      if (l[i] != c) continue;
      if (i < j) { first = false; break; }
      s += (double)w[i];
    }
    if (first && s > 0.0) { rl[m] = c; rs[m] = s; }
  }
  __shared__ int s_chosen[VOTE_WARPS][5];
  __shared__ double s_chosen_s[VOTE_WARPS][5];
  int* chosen = s_chosen[warp];
  double* chosen_s = s_chosen_s[warp];
  int found = 0;
  for (; found < 5; ++found) {
    double bs = 0.0;
    int bl = -1;
#pragma unroll
    for (int m = 0; m < PER_LANE; ++m)
      if (rl[m] >= 0 && (bl < 0 || class_before(rs[m], rl[m], bs, bl))) { bs = rs[m]; bl = rl[m]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double os = __shfl_xor_sync(0xffffffffu, bs, o);
      const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
      if (ol >= 0 && (bl < 0 || class_before(os, ol, bs, bl))) { bs = os; bl = ol; }
    }
    if (bl < 0) break;                       // no class with a positive score left
    if (lane == 0) {
      chosen[found] = bl;
      chosen_s[found] = bs;
    }
#pragma unroll
    for (int m = 0; m < PER_LANE; ++m)
      if (rl[m] == bl) rl[m] = -1;
  }
  // the remaining places go to the lowest-index classes with score 0
  if (lane == 0) {
    int c = 0;
    for (int r = found; r < 5; ++r) {
      bool taken = true;
      while (c < C && taken) {
        taken = false;
        for (int t = 0; t < found; ++t) taken |= chosen[t] == c;
        if (taken) ++c;
      }
      chosen[r] = c < C ? c++ : -1;
      chosen_s[r] = 0.0;
    }
    for (int r = 0; r < 5; ++r) {
      pred[q * 5 + r] = chosen[r];
      if (pred_scores != nullptr) pred_scores[q * 5 + r] = (float)chosen_s[r];
    }
  }
}

}  // namespace byol

using namespace byol;

extern "C" int byol_l2_normalize_rows(const float* x, void* y, int64_t R, int D, int64_t ldx, cudaStream_t stream) {
  BYOL_CHECK_ARG(x && y, "byol_l2_normalize_rows: null pointer");
  BYOL_CHECK_ARG(R > 0 && D > 0 && ldx >= D, "byol_l2_normalize_rows: bad shape R=%lld D=%d ldx=%lld", (long long)R, D,
                 (long long)ldx);
  int64_t blocks = (R + 7) / 8;
  if (blocks > 132 * 32) blocks = 132 * 32;
  l2_normalize_rows_kernel<<<(int)blocks, 256, 0, stream>>>(x, (bf16*)y, R, D, ldx);
  return check_launch("l2_normalize_rows_kernel");
}

extern "C" int byol_knn_topk(const float* sim, int Q, int Nc, int64_t ld, int n0, int k, int merge, float* top_vals,
                             int* top_idx, cudaStream_t stream) {
  BYOL_CHECK_ARG(sim && top_vals && top_idx, "byol_knn_topk: null pointer");
  BYOL_CHECK_ARG(Q > 0 && Nc > 0 && ld >= Nc && n0 >= 0, "byol_knn_topk: bad shape Q=%d Nc=%d ld=%lld n0=%d", Q, Nc,
                 (long long)ld, n0);
  BYOL_CHECK_ARG((int64_t)n0 + Nc <= 0x7fffffffll, "byol_knn_topk: bank index n0 + Nc = %lld exceeds 2^31 - 1",
                 (long long)n0 + Nc);
  BYOL_CHECK_ARG(k >= 1 && k <= KT_MAX_K, "byol_knn_topk: k=%d outside [1, %d]", k, KT_MAX_K);
  knn_topk_kernel<<<Q, KT_THREADS, 0, stream>>>(sim, Nc, ld, n0, k, merge ? 1 : 0, top_vals, top_idx);
  return check_launch("knn_topk_kernel");
}

extern "C" int byol_knn_vote(const float* top_vals, const int* top_idx, const int64_t* bank_labels, int Q, int k,
                             int num_classes, float temperature, int* pred, float* pred_scores, cudaStream_t stream) {
  BYOL_CHECK_ARG(top_vals && top_idx && bank_labels && pred, "byol_knn_vote: null pointer");
  BYOL_CHECK_ARG(Q > 0 && k >= 1 && k <= KT_MAX_K && num_classes >= 1, "byol_knn_vote: bad args Q=%d k=%d classes=%d",
                 Q, k, num_classes);
  BYOL_CHECK_ARG(temperature > 0.f && isfinite(temperature), "byol_knn_vote: temperature %g must be positive",
                 (double)temperature);
  knn_vote_kernel<<<(Q + VOTE_WARPS - 1) / VOTE_WARPS, VOTE_WARPS * 32, 0, stream>>>(
      top_vals, top_idx, bank_labels, Q, k, num_classes, temperature, pred, pred_scores);
  return check_launch("knn_vote_kernel");
}
