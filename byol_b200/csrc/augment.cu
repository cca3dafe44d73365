// byol_b200 — on-device two-view augmentation (SURVEY.md §8 f4): the torchvision recipe the reference builds in
// /root/reference/main.py:386-397
//     RandomResizedCrop(R) -> RandomHorizontalFlip(0.5) -> RandomApply(ColorJitter(0.8s, 0.8s, 0.8s, 0.2s), 0.8)
//     -> RandomGrayscale(0.2) -> GaussianBlur(kernel 0.1 R, p 0.5)
// for a batch of decoded images already resident in HBM (fp32 NCHW in [0, 1]), so that real data can feed the step at
// > 20 k images/s/GPU without host-side PIL work.  Three kinds of kernels:
//   augment_params_kernel : per (sample, view) the random parameters (Philox counter RNG keyed by seed / step / sample)
//   augment_gray_mean_kernel + augment_apply_kernel : crop + bilinear resize + flip + colour ops in the sampled order
//       (adjust_contrast blends with the MEAN grey level of the image as it stands before that op, hence the small
//       reduction pass) + grayscale
//   augment_blur_kernel   : separable Gaussian with reflect padding, only for the samples that drew it
// The arithmetic follows torchvision.transforms.v2.functional (float tensors): tests/test_gpu_augment.py compares every
// stage with it on identical parameters.  The missing `datasets.utils.GaussianBlur` is taken as the SimCLR one
// (sigma ~ U(0.1, 2.0); kernel size made odd) — unpinned, like the rest of that submodule.
#include "common.cuh"

namespace byol {

static constexpr int AP = 16;   // floats per (sample, view) parameter record
// record layout: 0 top, 1 left, 2 crop_h, 3 crop_w, 4 flip, 5 jitter_on, 6..9 op order (0 brightness, 1 contrast,
// 2 saturation, 3 hue), 10 brightness, 11 contrast, 12 saturation, 13 hue, 14 gray_on, 15 blur sigma (0 = no blur)

// ---- Philox4x32-10 (counter based; no state to store) ----
__device__ __forceinline__ uint4 philox(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
struct Rng {
  uint2 key;
  uint4 ctr, buf;
  int have;
  __device__ Rng(uint64_t seed, uint64_t stream) : have(0) {
    key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    ctr = make_uint4(0u, 0u, (uint32_t)stream, (uint32_t)(stream >> 32));
  }
  __device__ float uniform() {      // [0, 1)
    if (have == 0) { buf = philox(ctr, key); ++ctr.x; have = 4; }
    const uint32_t v = have == 4 ? buf.x : have == 3 ? buf.y : have == 2 ? buf.z : buf.w;
    --have;
    return (float)(v >> 8) * (1.0f / 16777216.0f);
  }
};

__global__ void augment_params_kernel(float* __restrict__ params, int N, int Hs, int Ws, uint64_t seed, uint64_t step,
                                      float strength, float p_flip, float p_jitter, float p_gray, float p_blur) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // (sample, view)
  if (i >= 2 * N) return;
  Rng rng(seed, step * (uint64_t)(2 * N) + (uint64_t)i);
  float* q = params + (int64_t)i * AP;
  // RandomResizedCrop.get_params: scale (0.08, 1), ratio (3/4, 4/3), 10 attempts, then a centre crop
  const float area = (float)Hs * (float)Ws;
  const float lr0 = logf(3.f / 4.f), lr1 = logf(4.f / 3.f);
  int top = 0, left = 0, ch = Hs, cw = Ws;
  bool found = false;
  for (int a = 0; a < 10; ++a) {
    const float target = area * (0.08f + 0.92f * rng.uniform());
    const float ar = expf(lr0 + (lr1 - lr0) * rng.uniform());
    const int w = (int)rintf(sqrtf(target * ar)), h = (int)rintf(sqrtf(target / ar));
    const float u1 = rng.uniform(), u2 = rng.uniform();
    if (!found && w > 0 && w <= Ws && h > 0 && h <= Hs) {
      top = min((int)(u1 * (float)(Hs - h + 1)), Hs - h);
      left = min((int)(u2 * (float)(Ws - w + 1)), Ws - w);
      ch = h; cw = w;
      found = true;
    }
  }
  if (!found) {
    const float in_ratio = (float)Ws / (float)Hs;
    if (in_ratio < 3.f / 4.f) { cw = Ws; ch = (int)rintf((float)cw / (3.f / 4.f)); }
    else if (in_ratio > 4.f / 3.f) { ch = Hs; cw = (int)rintf((float)ch * (4.f / 3.f)); }
    else { cw = Ws; ch = Hs; }
    ch = min(ch, Hs); cw = min(cw, Ws);
    top = (Hs - ch) / 2;
    left = (Ws - cw) / 2;
  }
  q[0] = (float)top; q[1] = (float)left; q[2] = (float)ch; q[3] = (float)cw;
  q[4] = rng.uniform() < p_flip ? 1.f : 0.f;
  q[5] = rng.uniform() < p_jitter ? 1.f : 0.f;
  // random permutation of the four colour ops (Fisher-Yates)
  int ord[4] = {0, 1, 2, 3};
  for (int k = 3; k > 0; --k) {
    const int j = min((int)(rng.uniform() * (float)(k + 1)), k);
    const int t = ord[k]; ord[k] = ord[j]; ord[j] = t;
  }
  for (int k = 0; k < 4; ++k) q[6 + k] = (float)ord[k];
  const float b = 0.8f * strength, c = 0.8f * strength, s = 0.8f * strength, hh = 0.2f * strength;
  q[10] = fmaxf(0.f, 1.f - b) + (1.f + b - fmaxf(0.f, 1.f - b)) * rng.uniform();
  q[11] = fmaxf(0.f, 1.f - c) + (1.f + c - fmaxf(0.f, 1.f - c)) * rng.uniform();
  q[12] = fmaxf(0.f, 1.f - s) + (1.f + s - fmaxf(0.f, 1.f - s)) * rng.uniform();
  q[13] = -hh + 2.f * hh * rng.uniform();
  q[14] = rng.uniform() < p_gray ? 1.f : 0.f;
  const float sigma = 0.1f + 1.9f * rng.uniform();
  q[15] = rng.uniform() < p_blur ? sigma : 0.f;
}

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }
__device__ __forceinline__ float gray_of(float r, float g, float b) { return 0.2989f * r + 0.587f * g + 0.114f * b; }

// crop + bilinear resize + horizontal flip: output pixel (y, x) of sample n.  Antialiased like
// torch.nn.functional.interpolate(mode="bilinear", antialias=True) / PIL: a triangle filter whose support grows with the
// down-scaling factor (for up-scaling it degenerates to plain bilinear, align_corners = False).
struct AxisTaps { int lo, n; float center, invscale, total; };
__device__ __forceinline__ AxisTaps axis_taps(int o, int in_size, int out_size) {
  AxisTaps t;
  const float scale = (float)in_size / (float)out_size;
  t.center = scale * ((float)o + 0.5f);
  const float support = scale >= 1.f ? scale : 1.f;
  t.invscale = scale >= 1.f ? 1.f / scale : 1.f;
  t.lo = max((int)(t.center - support + 0.5f), 0);
  t.n = min((int)(t.center + support + 0.5f), in_size) - t.lo;
  t.total = 0.f;
  for (int j = 0; j < t.n; ++j) {
    const float x = fabsf(((float)(j + t.lo) - t.center + 0.5f) * t.invscale);
    t.total += x < 1.f ? 1.f - x : 0.f;
  }
  return t;
}
__device__ __forceinline__ float tap_w(const AxisTaps& t, int j) {
  const float x = fabsf(((float)(j + t.lo) - t.center + 0.5f) * t.invscale);
  return (x < 1.f ? 1.f - x : 0.f) / t.total;
}
__device__ __forceinline__ void sample_crop(const float* __restrict__ src, int Hs, int Ws, const float* q, int R, int y,
                                            int x, float& r, float& g, float& b) {
  const int top = (int)q[0], left = (int)q[1], ch = (int)q[2], cw = (int)q[3];
  const int xx = q[4] != 0.f ? (R - 1 - x) : x;
  const AxisTaps ty = axis_taps(y, ch, R), tx = axis_taps(xx, cw, R);
  const int64_t plane = (int64_t)Hs * Ws;
  float v[3] = {0.f, 0.f, 0.f};
  for (int jy = 0; jy < ty.n; ++jy) {
    const float wy = tap_w(ty, jy);
    const float* row = src + (int64_t)(top + ty.lo + jy) * Ws + left + tx.lo;
    float h[3] = {0.f, 0.f, 0.f};
    for (int jx = 0; jx < tx.n; ++jx) {
      const float wx = tap_w(tx, jx);
#pragma unroll
      for (int c = 0; c < 3; ++c) h[c] += wx * __ldg(row + jx + c * plane);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] += wy * h[c];
  }
  r = v[0]; g = v[1]; b = v[2];
}

// torchvision _rgb2hsv / _hsv2rgb on one pixel, hue shifted by `dh` (in turns)
__device__ __forceinline__ void hue_shift(float& r, float& g, float& b, float dh) {
  const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
  const bool eqc = maxc == minc;
  const float cr = maxc - minc;
  const float ones = 1.f;
  const float s = cr / (eqc ? ones : maxc);
  const float crd = eqc ? ones : cr;
  const float rc = (maxc - r) / crd, gc = (maxc - g) / crd, bc = (maxc - b) / crd;
  const float hr = (maxc == r) ? (bc - gc) : 0.f;
  const float hg = ((maxc == g) && (maxc != r)) ? (2.f + rc - bc) : 0.f;
  const float hb = ((maxc != g) && (maxc != r)) ? (4.f + gc - rc) : 0.f;
  float h = fmodf((hr + hg + hb) / 6.f + 1.f, 1.f);
  h = fmodf(h + dh, 1.f);
  if (h < 0.f) h += 1.f;
  const float v = maxc;
  const float i6 = floorf(h * 6.f);
  const float f = h * 6.f - i6;
  const int i = ((int)i6) % 6;
  const float p = clamp01(v * (1.f - s)), qv = clamp01(v * (1.f - s * f)), t = clamp01(v * (1.f - s * (1.f - f)));
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = qv; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = qv; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = qv; break;
  }
}

// colour ops of the record in their sampled order, stopping BEFORE op `stop_at` (4 = run all); `mean_gray` is the image's
// mean grey level at the moment adjust_contrast runs
__device__ __forceinline__ void colour_ops(const float* q, float& r, float& g, float& b, int stop_at, float mean_gray) {
  if (q[5] == 0.f) return;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int op = (int)q[6 + k];
    if (op == stop_at) return;
    if (op == 0) {
      const float f = q[10];
      r = clamp01(r * f); g = clamp01(g * f); b = clamp01(b * f);
    } else if (op == 1) {
      const float f = q[11], m = (1.f - f) * mean_gray;
      r = clamp01(f * r + m); g = clamp01(f * g + m); b = clamp01(f * b + m);
    } else if (op == 2) {
      const float f = q[12], m = (1.f - f) * gray_of(r, g, b);
      r = clamp01(f * r + m); g = clamp01(f * g + m); b = clamp01(f * b + m);
    } else {
      hue_shift(r, g, b, q[13]);
    }
  }
}

// mean grey level per (sample, view) of the image as it stands right before adjust_contrast (sum in fp32 per block,
// blocks combined in fixed point); skipped (mean unused) when the jitter is off
__global__ void augment_gray_mean_kernel(const float* __restrict__ src, const float* __restrict__ params,
                                         Fix128* __restrict__ gray_sum, int N, int Hs, int Ws, int R) {
  const int sv = blockIdx.y;                      // sample * 2 + view... laid out view-major: sv = view * N + n
  const int n = sv % N;
  const float* q = params + (int64_t)sv * AP;
  if (q[5] == 0.f) return;
  float acc = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R * R; i += gridDim.x * blockDim.x) {
    float r, g, b;
    sample_crop(src + (int64_t)n * 3 * Hs * Ws, Hs, Ws, q, R, i / R, i % R, r, g, b);
    colour_ops(q, r, g, b, 1, 0.f);
    acc += gray_of(r, g, b);
  }
  acc = warp_sum(acc);
  __shared__ float sh[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    float v = lane < (int)(blockDim.x >> 5) ? sh[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) fix_add(gray_sum + sv, v);   // fixed point: order-independent
  }
}

// out[view][n, c, y, x] (fp32 NCHW): crop / resize / flip, colour jitter, grayscale
__global__ void augment_apply_kernel(const float* __restrict__ src, const float* __restrict__ params,
                                     const Fix128* __restrict__ gray_sum, float* __restrict__ out, int N, int Hs, int Ws,
                                     int R) {
  const int sv = blockIdx.y;
  const int n = sv % N;
  const float* q = params + (int64_t)sv * AP;
  const float mean_gray = (float)(fix_value(gray_sum[sv]) / (double)(R * R));
  float* o = out + (int64_t)sv * 3 * R * R;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R * R; i += gridDim.x * blockDim.x) {
    float r, g, b;
    sample_crop(src + (int64_t)n * 3 * Hs * Ws, Hs, Ws, q, R, i / R, i % R, r, g, b);
    colour_ops(q, r, g, b, 4, mean_gray);
    if (q[14] != 0.f) { const float gr = gray_of(r, g, b); r = gr; g = gr; b = gr; }
    o[i] = r; o[R * R + i] = g; o[2 * R * R + i] = b;
  }
}

// one pass of the separable Gaussian (reflect padding); horizontal = 1: along x, else along y.  Samples without blur
// are copied.  dst and src must differ.
__global__ void augment_blur_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                    const float* __restrict__ params, int R, int ksize, int horizontal) {
  const int sv = blockIdx.y;
  const float sigma = params[(int64_t)sv * AP + 15];
  const float* s = src + (int64_t)sv * 3 * R * R;
  float* d = dst + (int64_t)sv * 3 * R * R;
  const int half = ksize / 2;
  float wsum = 0.f;
  if (sigma > 0.f)
    for (int k = -half; k <= half; ++k) wsum += expf(-0.5f * (float)(k * k) / (sigma * sigma));
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 3 * R * R; i += gridDim.x * blockDim.x) {
    if (sigma <= 0.f) { d[i] = s[i]; continue; }
    const int c = i / (R * R), rem = i % (R * R), y = rem / R, x = rem % R;
    const float* pl = s + (int64_t)c * R * R;
    float acc = 0.f;
    for (int k = -half; k <= half; ++k) {
      int t = (horizontal ? x : y) + k;
      if (t < 0) t = -t;                        // reflect (no edge repeat), like torch's F.pad(mode="reflect")
      if (t >= R) t = 2 * (R - 1) - t;
      const float w = expf(-0.5f * (float)(k * k) / (sigma * sigma));
      acc += w * (horizontal ? pl[y * R + t] : pl[t * R + x]);
    }
    d[i] = acc / wsum;
  }
}

}  // namespace byol

using namespace byol;

extern "C" int byol_augment_record_floats(void) { return AP; }

// params: [2, N, 16] fp32 (view-major).  strength = color_jitter_strength (main.py:390-393).
extern "C" int byol_augment_params(float* params, int N, int Hs, int Ws, uint64_t seed, uint64_t step, float strength,
                                   float p_flip, float p_jitter, float p_gray, float p_blur, cudaStream_t stream) {
  BYOL_CHECK_ARG(params && N > 0 && Hs > 0 && Ws > 0, "byol_augment_params: bad args");
  augment_params_kernel<<<(2 * N + 127) / 128, 128, 0, stream>>>(params, N, Hs, Ws, seed, step, strength, p_flip,
                                                                p_jitter, p_gray, p_blur);
  return check_launch("augment_params_kernel");
}

// src: fp32 NCHW [N, 3, Hs, Ws] in [0, 1]; out: fp32 [2, N, 3, R, R] (view 1 | view 2); tmp: same size as out (blur);
// gray_sum: part of the ABI, no longer used (the per-view sums live in the stream's fix_scratch); ksize: odd Gaussian kernel size (0 = no blur stage).
extern "C" int byol_augment_apply(const float* src, const float* params, float* out, float* tmp, double* gray_sum,
                                  int N, int Hs, int Ws, int R, int ksize, cudaStream_t stream) {
  BYOL_CHECK_ARG(src && params && out && gray_sum && N > 0 && R > 0, "byol_augment_apply: bad args");
  BYOL_CHECK_ARG(ksize == 0 || (ksize % 2 == 1 && ksize < 2 * R - 1 && tmp != nullptr), "byol_augment_apply: bad ksize %d", ksize);
  Fix128* gsum = fix_scratch(stream, 2 * (int64_t)N);
  if (gsum == nullptr) return -2;
  int bx = (R * R + 255) / 256;
  if (bx > 64) bx = 64;
  dim3 grid((unsigned)bx, (unsigned)(2 * N));
  augment_gray_mean_kernel<<<grid, 256, 0, stream>>>(src, params, gsum, N, Hs, Ws, R);
  augment_apply_kernel<<<grid, 256, 0, stream>>>(src, params, gsum, out, N, Hs, Ws, R);
  // every block of augment_apply_kernel read the sums: leave the scratch zeroed (fix_scratch)
  if (cudaMemsetAsync(gsum, 0, 2 * (size_t)N * sizeof(Fix128), stream) != cudaSuccess) {
    set_last_error("byol_augment_apply: memset failed");
    return -2;
  }
  if (ksize > 0) {
    augment_blur_kernel<<<grid, 256, 0, stream>>>(out, tmp, params, R, ksize, 1);
    augment_blur_kernel<<<grid, 256, 0, stream>>>(tmp, out, params, R, ksize, 0);
  }
  return fix_done(stream, check_launch("augment kernels"));
}
