// byol_b200 — on-device two-view augmentation (SURVEY.md §8 f4): the torchvision recipe the reference builds in
// /root/reference/main.py:386-397
//     RandomResizedCrop(R) -> RandomHorizontalFlip(0.5) -> RandomApply(ColorJitter(0.8s, 0.8s, 0.8s, 0.2s), 0.8)
//     -> RandomGrayscale(0.2) -> GaussianBlur(kernel 0.1 R, p 0.5)
// and the BYOL paper's (Grill et al. 2020, Appendix B): bicubic crop resize, ColorJitter(0.4s, 0.4s, 0.2s, 0.1s),
// blur p 1.0 / 0.1 and solarize p 0.0 / 0.2 on view 1 / view 2 (AugRecipe; the records say which transform they are)
// for a batch of decoded images already resident in HBM, so that real data can feed the step without host-side PIL
// work.  Two kinds of input: one fp32 NCHW batch in [0, 1] of equal-sized images, or a table of uint8 CHW images of
// any sizes, as a GPU JPEG decoder returns them (read as v / 255; the arithmetic after that is the same).  Three kinds of kernels:
//   augment_params_kernel : per (sample, view) the random parameters (Philox counter RNG keyed by seed / step / sample)
//   augment_gray_mean_kernel + augment_apply_kernel : crop + bilinear or bicubic resize (or resize + window, for the
//       evaluation transforms' records) + flip + colour ops in the
//       sampled order (adjust_contrast blends with the MEAN grey level of the image as it stands before that op, hence
//       the small reduction pass) + grayscale (+ solarize, for the samples the blur does not reach)
//   augment_blur_kernel   : separable Gaussian with reflect padding, only for the samples that drew it (+ solarize on
//       the blurred value in the second pass)
// The arithmetic follows torchvision.transforms.v2.functional (float tensors): tests/test_gpu_augment.py compares every
// stage with it on identical parameters.  The missing `datasets.utils.GaussianBlur` is taken as the SimCLR one
// (sigma ~ U(0.1, 2.0); kernel size made odd) — unpinned, like the rest of that submodule.
#include "common.cuh"
#include "../../include/byol_b200.h"

namespace byol {

static constexpr int AP = 16;   // floats per (sample, view) parameter record
// record layout: 0 top, 1 left, 2 crop_h, 3 crop_w, 4 flip, 5 jitter_on, 6..9 op order (0 brightness, 1 contrast,
// 2 saturation, 3 hue), 10 brightness, 11 contrast, 12 saturation, 13 hue, 14 flag word, 15 blur sigma (0 = no blur).
// Flag word bits: grayscale, solarize, bicubic resampling, window.  The reference recipe sets only the grayscale bit,
// so its records hold 0 or 1 there, as before the word had other bits.  A window record (bit 3, made on the host for
// the evaluation transforms) reads floats 0-3 as (top, left, Sh, Sw): the R x R window at (top, left) of the whole
// image resized to Sh x Sw, i.e. a resize followed by a crop, where a crop record (bit 3 clear) crops, then resizes.
static constexpr int FLAG_GRAY = 1, FLAG_SOLARIZE = 2, FLAG_BICUBIC = 4, FLAG_WINDOW = 8;

// what the sampler draws from: colour-jitter factors (multiplied by color_jitter_strength, as ColorJitter(0.8s, ...)),
// the switches' probabilities, per view where the recipe makes the views differ
struct AugRecipe {
  float jitter[4];          // brightness, contrast, saturation, hue
  float p_flip, p_jitter, p_gray;
  float p_blur[2], p_solarize[2];
  int bicubic;
};

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

// one (sample, view) record for an Hs x Ws source image, drawn from `rng`
__device__ __forceinline__ void sample_record(float* q, Rng& rng, int Hs, int Ws, float strength, const AugRecipe& rc,
                                              int view) {
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
  q[4] = rng.uniform() < rc.p_flip ? 1.f : 0.f;
  q[5] = rng.uniform() < rc.p_jitter ? 1.f : 0.f;
  // random permutation of the four colour ops (Fisher-Yates)
  int ord[4] = {0, 1, 2, 3};
  for (int k = 3; k > 0; --k) {
    const int j = min((int)(rng.uniform() * (float)(k + 1)), k);
    const int t = ord[k]; ord[k] = ord[j]; ord[j] = t;
  }
  for (int k = 0; k < 4; ++k) q[6 + k] = (float)ord[k];
  const float b = rc.jitter[0] * strength, c = rc.jitter[1] * strength, s = rc.jitter[2] * strength,
              hh = rc.jitter[3] * strength;
  q[10] = fmaxf(0.f, 1.f - b) + (1.f + b - fmaxf(0.f, 1.f - b)) * rng.uniform();
  q[11] = fmaxf(0.f, 1.f - c) + (1.f + c - fmaxf(0.f, 1.f - c)) * rng.uniform();
  q[12] = fmaxf(0.f, 1.f - s) + (1.f + s - fmaxf(0.f, 1.f - s)) * rng.uniform();
  q[13] = -hh + 2.f * hh * rng.uniform();
  const bool gray = rng.uniform() < rc.p_gray;
  const float sigma = 0.1f + 1.9f * rng.uniform();
  q[15] = rng.uniform() < (view ? rc.p_blur[1] : rc.p_blur[0]) ? sigma : 0.f;
  // drawn after every other switch, so that the records of recipes without solarization keep their draws
  const bool solarize = rng.uniform() < (view ? rc.p_solarize[1] : rc.p_solarize[0]);
  q[14] = (float)((gray ? FLAG_GRAY : 0) | (solarize ? FLAG_SOLARIZE : 0) | (rc.bicubic ? FLAG_BICUBIC : 0));
}

// the reference recipe as the scalar-argument entry points describe it
__host__ __device__ inline AugRecipe reference_recipe(float p_flip, float p_jitter, float p_gray, float p_blur) {
  return AugRecipe{{0.8f, 0.8f, 0.8f, 0.2f}, p_flip, p_jitter, p_gray, {p_blur, p_blur}, {0.f, 0.f}, 0};
}

__global__ void augment_params_kernel(float* __restrict__ params, int N, int Hs, int Ws, uint64_t seed, uint64_t step,
                                      float strength, AugRecipe rc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // view * N + sample
  if (i >= 2 * N) return;
  Rng rng(seed, step * (uint64_t)(2 * N) + (uint64_t)i);
  sample_record(params + (int64_t)i * AP, rng, Hs, Ws, strength, rc, i / N);
}

// records for samples [n0, n0 + n) of a batch of N images of their own sizes (hw: int32 [n, 2], rows H, W).  The
// stream of (view, sample) is the one augment_params_kernel gives it for an N-image batch, so a batch sampled in
// chunks gets the same records as one call, and equal sizes with n0 = 0, n = N reproduce augment_params_kernel.
// params: [2, n, AP], view-major over the chunk.
__global__ void augment_params_ragged_kernel(float* __restrict__ params, const int* __restrict__ hw, int n, int n0,
                                             int N, uint64_t seed, uint64_t step, float strength, AugRecipe rc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;      // view * n + j
  if (i >= 2 * n) return;
  const int view = i / n, j = i % n;
  Rng rng(seed, step * (uint64_t)(2 * N) + (uint64_t)view * (uint64_t)N + (uint64_t)(n0 + j));
  sample_record(params + (int64_t)i * AP, rng, hw[2 * j], hw[2 * j + 1], strength, rc, view);
}

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }
__device__ __forceinline__ float gray_of(float r, float g, float b) { return 0.2989f * r + 0.587f * g + 0.114f * b; }

// crop + resize + horizontal flip: output pixel (y, x) of sample n.  Antialiased like
// torch.nn.functional.interpolate(mode="bilinear" / "bicubic", antialias=True) / PIL: a filter whose support grows with
// the down-scaling factor (for up-scaling it degenerates to plain bilinear / bicubic, align_corners = False).
//   Triangle: 1 - |x| on |x| < 1 (bilinear).
//   Cubic: Keys' cubic convolution with a = -0.5 (what interpolate uses with antialias=True, as PIL) on |x| < 2.  It
//   overshoots: a resized value can leave [0, 1] by a fraction of the local contrast (resample() clamps it).
struct Triangle {
  static __device__ __forceinline__ float support(float scale) { return scale >= 1.f ? scale : 1.f; }
  static __device__ __forceinline__ float weight(float x) { return x < 1.f ? 1.f - x : 0.f; }
};
struct Cubic {
  static __device__ __forceinline__ float support(float scale) { return scale >= 1.f ? 2.f * scale : 2.f; }
  static __device__ __forceinline__ float weight(float x) {
    const float a = -0.5f;
    if (x < 1.f) return ((a + 2.f) * x - (a + 3.f)) * x * x + 1.f;
    if (x < 2.f) return ((a * x - 5.f * a) * x + 8.f * a) * x - 4.f * a;
    return 0.f;
  }
};
struct AxisTaps { int lo, n; float center, invscale, total; };
template <typename F>
__device__ __forceinline__ AxisTaps axis_taps(int o, int in_size, int out_size) {
  AxisTaps t;
  const float scale = (float)in_size / (float)out_size;
  t.center = scale * ((float)o + 0.5f);
  const float support = F::support(scale);
  t.invscale = scale >= 1.f ? 1.f / scale : 1.f;
  t.lo = max((int)(t.center - support + 0.5f), 0);
  t.n = min((int)(t.center + support + 0.5f), in_size) - t.lo;
  t.total = 0.f;
  for (int j = 0; j < t.n; ++j) {
    const float x = fabsf(((float)(j + t.lo) - t.center + 0.5f) * t.invscale);
    t.total += F::weight(x);
  }
  return t;
}
template <typename F>
__device__ __forceinline__ float tap_w(const AxisTaps& t, int j) {
  const float x = fabsf(((float)(j + t.lo) - t.center + 0.5f) * t.invscale);
  return F::weight(x) / t.total;
}
// a source value in [0, 1]: fp32 images are read as they are, uint8 ones as v / 255
__device__ __forceinline__ float load_px(const float* p) { return __ldg(p); }
__device__ __forceinline__ float load_px(const uint8_t* p) { return (float)__ldg(p) / 255.f; }

// A crop record resizes the box (top, left, h, w) to R x R: output pixel (y, x) has the taps of (y, x) over the box,
// which is where they stop.  A window record's output pixel (y, x) is pixel (y + top, x + left) of the whole image
// resized to (Sh, Sw): its taps run over the whole image, also outside the window.  Flip mirrors the output.
template <typename F, typename T>
__device__ __forceinline__ void sample_crop(const T* __restrict__ src, int Hs, int Ws, const float* q, int flags, int R,
                                            int y, int x, float& r, float& g, float& b) {
  const int top = (int)q[0], left = (int)q[1], qh = (int)q[2], qw = (int)q[3];
  const int xx = q[4] != 0.f ? (R - 1 - x) : x;
  const bool window = flags & FLAG_WINDOW;
  const AxisTaps ty = axis_taps<F>(window ? y + top : y, window ? Hs : qh, window ? qh : R),
                 tx = axis_taps<F>(window ? xx + left : xx, window ? Ws : qw, window ? qw : R);
  const int y0 = window ? 0 : top, x0 = window ? 0 : left;
  const int64_t plane = (int64_t)Hs * Ws;
  float v[3] = {0.f, 0.f, 0.f};
  for (int jy = 0; jy < ty.n; ++jy) {
    const float wy = tap_w<F>(ty, jy);
    const T* row = src + (int64_t)(y0 + ty.lo + jy) * Ws + x0 + tx.lo;
    float h[3] = {0.f, 0.f, 0.f};
    for (int jx = 0; jx < tx.n; ++jx) {
      const float wx = tap_w<F>(tx, jx);
#pragma unroll
      for (int c = 0; c < 3; ++c) h[c] += wx * load_px(row + jx + c * plane);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] += wy * h[c];
  }
  r = v[0]; g = v[1]; b = v[2];
}

// the record's crop + resize (or resize + window): bicubic values are clamped to [0, 1] before any colour op, as a
// uint8 / PIL pipeline stores them (colour ops on an overshooting value would leave [0, 1], and solarize would turn it
// negative)
template <typename T>
__device__ __forceinline__ void resample(const T* __restrict__ src, int Hs, int Ws, const float* q, int flags, int R,
                                         int y, int x, float& r, float& g, float& b) {
  if (flags & FLAG_BICUBIC) {
    sample_crop<Cubic>(src, Hs, Ws, q, flags, R, y, x, r, g, b);
    r = clamp01(r); g = clamp01(g); b = clamp01(b);
  } else {
    sample_crop<Triangle>(src, Hs, Ws, q, flags, R, y, x, r, g, b);
  }
}
// torchvision solarize(x, 0.5) on float input
__device__ __forceinline__ float solarize(float v) { return v >= 0.5f ? 1.f - v : v; }

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

// where sample n's image is and how large: one fp32 [N, 3, Hs, Ws] batch, or a table of per-image uint8 [3, H, W]
// tensors with their sizes (hw: int32 [N, 2])
struct DenseSrc {
  using T = float;
  const float* p;
  int Hs, Ws;
  __device__ const float* image(int n, int& h, int& w) const { h = Hs; w = Ws; return p + (int64_t)n * 3 * Hs * Ws; }
};
struct RaggedSrc {
  using T = uint8_t;
  const uint8_t* const* p;
  const int* hw;
  __device__ const uint8_t* image(int n, int& h, int& w) const { h = hw[2 * n]; w = hw[2 * n + 1]; return p[n]; }
};

// mean grey level per (sample, view) of the image as it stands right before adjust_contrast (sum in fp32 per block,
// blocks combined in fixed point); skipped (mean unused) when the jitter is off
template <typename Src>
__global__ void augment_gray_mean_kernel(Src src, const float* __restrict__ params, Fix128* __restrict__ gray_sum,
                                         int N, int R) {
  const int sv = blockIdx.y;                      // sample * 2 + view... laid out view-major: sv = view * N + n
  const int n = sv % N;
  const float* q = params + (int64_t)sv * AP;
  if (q[5] == 0.f) return;
  const int flags = (int)q[14];
  int Hs, Ws;
  const typename Src::T* img = src.image(n, Hs, Ws);
  float acc = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R * R; i += gridDim.x * blockDim.x) {
    float r, g, b;
    resample(img, Hs, Ws, q, flags, R, i / R, i % R, r, g, b);
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

// out[view][n, c, y, x] (fp32 NCHW): crop / resize / flip, colour jitter, grayscale, and solarize when the blur stage
// (blur_on) will not blur this sample (augment_blur_kernel solarizes the blurred ones).  At most 64 registers, so that
// four 256-thread blocks fit on an SM
template <typename Src>
__global__ void __launch_bounds__(256, 4)
augment_apply_kernel(Src src, const float* __restrict__ params, const Fix128* __restrict__ gray_sum,
                     float* __restrict__ out, int N, int R, int blur_on) {
  const int sv = blockIdx.y;
  const int n = sv % N;
  const float* q = params + (int64_t)sv * AP;
  const float mean_gray = (float)(fix_value(gray_sum[sv]) / (double)(R * R));
  const int flags = (int)q[14];
  const bool solarize_here = (flags & FLAG_SOLARIZE) && !(blur_on && q[15] > 0.f);
  float* o = out + (int64_t)sv * 3 * R * R;
  int Hs, Ws;
  const typename Src::T* img = src.image(n, Hs, Ws);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R * R; i += gridDim.x * blockDim.x) {
    float r, g, b;
    resample(img, Hs, Ws, q, flags, R, i / R, i % R, r, g, b);
    colour_ops(q, r, g, b, 4, mean_gray);
    if (flags & FLAG_GRAY) { const float gr = gray_of(r, g, b); r = gr; g = gr; b = gr; }
    if (solarize_here) { r = solarize(r); g = solarize(g); b = solarize(b); }
    o[i] = r; o[R * R + i] = g; o[2 * R * R + i] = b;
  }
}

// one pass of the separable Gaussian (reflect padding); horizontal = 1: along x, else along y, then the record's
// solarize.  Samples without blur are copied (augment_apply_kernel solarized them).  dst and src must differ.
__global__ void augment_blur_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                    const float* __restrict__ params, int R, int ksize, int horizontal) {
  const int sv = blockIdx.y;
  const float sigma = params[(int64_t)sv * AP + 15];
  const bool solarize_here = !horizontal && ((int)params[(int64_t)sv * AP + 14] & FLAG_SOLARIZE);
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
    const float v = acc / wsum;
    d[i] = solarize_here ? solarize(v) : v;
  }
}

}  // namespace byol

using namespace byol;

extern "C" int byol_augment_record_floats(void) { return AP; }

static AugRecipe recipe_of(const byol_augment_recipe_t& r) {
  return AugRecipe{{r.jitter[0], r.jitter[1], r.jitter[2], r.jitter[3]}, r.p_flip, r.p_jitter, r.p_gray,
                   {r.p_blur[0], r.p_blur[1]}, {r.p_solarize[0], r.p_solarize[1]}, r.bicubic ? 1 : 0};
}

static int bad_recipe(const byol_augment_recipe_t* r) {
  if (r == nullptr) return 1;
  const float ps[7] = {r->p_flip, r->p_jitter, r->p_gray, r->p_blur[0], r->p_blur[1], r->p_solarize[0],
                       r->p_solarize[1]};
  for (float p : ps)
    if (!(p >= 0.f && p <= 1.f)) return 1;
  for (float j : r->jitter)
    if (!(j >= 0.f)) return 1;
  return 0;
}

// params: [2, N, 16] fp32 (view-major).  strength = color_jitter_strength (main.py:390-393).
extern "C" int byol_augment_params(float* params, int N, int Hs, int Ws, uint64_t seed, uint64_t step, float strength,
                                   float p_flip, float p_jitter, float p_gray, float p_blur, cudaStream_t stream) {
  BYOL_CHECK_ARG(params && N > 0 && Hs > 0 && Ws > 0, "byol_augment_params: bad args");
  augment_params_kernel<<<(2 * N + 127) / 128, 128, 0, stream>>>(params, N, Hs, Ws, seed, step, strength,
                                                                reference_recipe(p_flip, p_jitter, p_gray, p_blur));
  return check_launch("augment_params_kernel");
}

// byol_augment_params with the recipe spelled out (per-view blur / solarize, jitter factors, bicubic resampling)
extern "C" int byol_augment_params_recipe(float* params, int N, int Hs, int Ws, uint64_t seed, uint64_t step,
                                          float strength, const byol_augment_recipe_t* recipe, cudaStream_t stream) {
  BYOL_CHECK_ARG(params && N > 0 && Hs > 0 && Ws > 0, "byol_augment_params_recipe: bad args");
  BYOL_CHECK_ARG(!bad_recipe(recipe), "byol_augment_params_recipe: bad recipe");
  augment_params_kernel<<<(2 * N + 127) / 128, 128, 0, stream>>>(params, N, Hs, Ws, seed, step, strength,
                                                                recipe_of(*recipe));
  return check_launch("augment_params_kernel");
}

// the gray-mean, apply and blur passes over any source (DenseSrc / RaggedSrc)
template <typename Src>
static int augment_apply_launch(Src src, const float* params, float* out, float* tmp, int N, int R, int ksize,
                                cudaStream_t stream, const char* what) {
  Fix128* gsum = fix_scratch(stream, 2 * (int64_t)N);
  if (gsum == nullptr) return -2;
  int bx = (R * R + 255) / 256;
  if (bx > 64) bx = 64;
  dim3 grid((unsigned)bx, (unsigned)(2 * N));
  augment_gray_mean_kernel<<<grid, 256, 0, stream>>>(src, params, gsum, N, R);
  augment_apply_kernel<<<grid, 256, 0, stream>>>(src, params, gsum, out, N, R, ksize > 0 ? 1 : 0);
  // every block of augment_apply_kernel read the sums: leave the scratch zeroed (fix_scratch)
  if (cudaMemsetAsync(gsum, 0, 2 * (size_t)N * sizeof(Fix128), stream) != cudaSuccess) {
    set_last_error("%s: memset failed", what);
    return -2;
  }
  if (ksize > 0) {
    augment_blur_kernel<<<grid, 256, 0, stream>>>(out, tmp, params, R, ksize, 1);
    augment_blur_kernel<<<grid, 256, 0, stream>>>(tmp, out, params, R, ksize, 0);
  }
  return fix_done(stream, check_launch("augment kernels"));
}

// src: fp32 NCHW [N, 3, Hs, Ws] in [0, 1]; out: fp32 [2, N, 3, R, R] (view 1 | view 2); tmp: same size as out (blur);
// gray_sum: part of the ABI, no longer used (the per-view sums live in the stream's fix_scratch); ksize: odd Gaussian kernel size (0 = no blur stage).
extern "C" int byol_augment_apply(const float* src, const float* params, float* out, float* tmp, double* gray_sum,
                                  int N, int Hs, int Ws, int R, int ksize, cudaStream_t stream) {
  BYOL_CHECK_ARG(src && params && out && gray_sum && N > 0 && R > 0, "byol_augment_apply: bad args");
  BYOL_CHECK_ARG(ksize == 0 || (ksize % 2 == 1 && ksize < 2 * R - 1 && tmp != nullptr), "byol_augment_apply: bad ksize %d", ksize);
  return augment_apply_launch(DenseSrc{src, Hs, Ws}, params, out, tmp, N, R, ksize, stream, "byol_augment_apply");
}

// Mixed-size batches.  hw: device int32 [n, 2] (H, W of each image); params: [2, n, 16] records for samples
// [n0, n0 + n) of an N-image batch (see augment_params_ragged_kernel).
extern "C" int byol_augment_params_ragged(float* params, const int* hw, int n, int n0, int N, uint64_t seed,
                                          uint64_t step, float strength, float p_flip, float p_jitter, float p_gray,
                                          float p_blur, cudaStream_t stream) {
  BYOL_CHECK_ARG(params && hw, "byol_augment_params_ragged: null pointer");
  BYOL_CHECK_ARG(n > 0 && n0 >= 0 && N > 0 && n0 <= N - n, "byol_augment_params_ragged: bad chunk n %d n0 %d N %d",
                 n, n0, N);
  augment_params_ragged_kernel<<<(2 * n + 127) / 128, 128, 0, stream>>>(
      params, hw, n, n0, N, seed, step, strength, reference_recipe(p_flip, p_jitter, p_gray, p_blur));
  return check_launch("augment_params_ragged_kernel");
}

// byol_augment_params_ragged with the recipe spelled out (see byol_augment_params_recipe)
extern "C" int byol_augment_params_ragged_recipe(float* params, const int* hw, int n, int n0, int N, uint64_t seed,
                                                 uint64_t step, float strength, const byol_augment_recipe_t* recipe,
                                                 cudaStream_t stream) {
  BYOL_CHECK_ARG(params && hw, "byol_augment_params_ragged_recipe: null pointer");
  BYOL_CHECK_ARG(n > 0 && n0 >= 0 && N > 0 && n0 <= N - n,
                 "byol_augment_params_ragged_recipe: bad chunk n %d n0 %d N %d", n, n0, N);
  BYOL_CHECK_ARG(!bad_recipe(recipe), "byol_augment_params_ragged_recipe: bad recipe");
  augment_params_ragged_kernel<<<(2 * n + 127) / 128, 128, 0, stream>>>(params, hw, n, n0, N, seed, step, strength,
                                                                       recipe_of(*recipe));
  return check_launch("augment_params_ragged_kernel");
}

// srcs: device table of N pointers to uint8 CHW [3, H_i, W_i] images (values v read as v / 255); hw: device int32
// [N, 2]; the rest as byol_augment_apply.
extern "C" int byol_augment_apply_ragged(const uint8_t* const* srcs, const int* hw, const float* params, float* out,
                                         float* tmp, int N, int R, int ksize, cudaStream_t stream) {
  BYOL_CHECK_ARG(srcs && hw && params && out, "byol_augment_apply_ragged: null pointer");
  BYOL_CHECK_ARG(N > 0 && 2 * (int64_t)N <= 65535 && R > 0, "byol_augment_apply_ragged: bad N %d or R %d", N, R);
  BYOL_CHECK_ARG(ksize == 0 || (ksize % 2 == 1 && ksize < 2 * R - 1 && tmp != nullptr),
                 "byol_augment_apply_ragged: bad ksize %d", ksize);
  return augment_apply_launch(RaggedSrc{srcs, hw}, params, out, tmp, N, R, ksize, stream, "byol_augment_apply_ragged");
}
