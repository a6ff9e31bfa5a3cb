// Image augmentations of vision/data_augmentations.py (serl_b200.vision.data_augmentations): the random crop (edge-padded
// shift), colour jitter, horizontal flip, Gaussian blur and solarize, with the reference's key derivations on the device.
//
// Reference (relative to serl_launcher/serl_launcher):
//   vision/data_augmentations.py:7-36     random_crop / batched_random_crop: split(rng, n)[i], randint((2,), 0, 2p + 1), edge pad,
//                                         dynamic_slice
//   vision/data_augmentations.py:39-42    _maybe_apply: uniform(rng) <= apply_prob
//   vision/data_augmentations.py:62-105   _gaussian_blur_single_image / _random_gaussian_blur: radius int(kernel_size / 2),
//                                         normalised Gaussian taps, depthwise conv along W then H, SAME zero padding
//   vision/data_augmentations.py:108-186  rgb_to_hsv / hsv_to_rgb (the TF kernels) and the four adjustments
//   vision/data_augmentations.py:224-302  color_transform: keys, decisions, jitter order, clip after every op, grayscale
//   vision/data_augmentations.py:305-309  random_flip: uniform(split(rng)[1]) <= 0.5, flip along W
//   vision/data_augmentations.py:336-340  solarize
// Restated in oracle/augment.py.  Every random draw is jax's float32 construction with each operation rounded on its own
// (__fmul_rn / __fadd_rn: no contraction), so decisions and drawn parameters equal the oracle's bit for bit.
#include "common.cuh"
#include "serl_b200.h"

namespace serl {

constexpr int kAugThreads = 256;
constexpr int kCropUnits = 2;                // crop units (16-byte chunks or elements) per thread
constexpr int kEltItems = 16;                // flip / solarize elements per thread
constexpr int kColorThreads = 512;
constexpr int kBlurRows = 32;                // output rows of a blur tile
constexpr int kBlurCols = 256;               // floats of a row (x * C + c) per blur tile, one per thread

// Image i's key: keys[2i], keys[2i + 1] (one key per image, jax.vmap's form), or split(keys[0:2], split_n)[i] when split_n > 0.
__device__ inline u32x2 image_key(const uint32_t* keys, int split_n, int i) {
  if (split_n > 0) return jax_split_at(u32x2{keys[0], keys[1]}, (uint32_t)split_n, (uint32_t)i);
  return u32x2{keys[2 * i], keys[2 * i + 1]};
}

// jax.random.uniform(key, (), float32, lo, hi) = max(lo, f * (hi - lo) + lo), f = bitcast(bits >> 9 | 0x3f800000) - 1.
__device__ inline float jax_uniform(u32x2 key, float lo, float hi) {
  const float f = bits_to_uniform01(jax_random_bits_at(key, 1u, 0u));
  return fmaxf(lo, __fadd_rn(__fmul_rn(f, __fsub_rn(hi, lo)), lo));
}

__device__ inline float clip01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// jnp.remainder for float32: the sign of the divisor.
__device__ inline float jrem(float a, float b) {
  float r = fmodf(a, b);
  if (r != 0.f && ((r < 0.f) != (b < 0.f))) r += b;
  return r;
}

// ---- crop ------------------------------------------------------------------------------------------------------------------
// Output pixel (y, x) of image i = input pixel (clamp(y + cy - p, 0, H - 1), clamp(x + cx - p, 0, W - 1)): jnp.pad(mode="edge")
// followed by dynamic_slice at (cy, cx), without the padded copy.  A pure copy, so the result is bit-exact by construction.
struct CropArgs {
  const uint8_t* src;
  uint8_t* dst;
  const uint32_t* keys;
  int split_n, H, W, pix_bytes, pad, blocks_per_image;
};

__device__ inline void crop_offsets_cta(const CropArgs& a, int img, int* s_dy, int* s_sx) {
  if (threadIdx.x == 0) {
    int cy, cx;
    jax_randint2(image_key(a.keys, a.split_n, img), (uint32_t)(2 * a.pad + 1), &cy, &cx);
    *s_dy = cy - a.pad; *s_sx = cx - a.pad;
  }
  __syncthreads();
}

// Rows of 16-byte multiples with 16-byte-aligned buffers: one 16-byte store per unit.  An interior chunk is the source row shifted
// by sx pixels, read as aligned words and funnel-shifted into place; a chunk that reaches past either edge gathers its bytes.
__global__ void __launch_bounds__(kAugThreads) crop_wide_kernel(const CropArgs a) {
  pdl_prologue();
  __shared__ int s_dy, s_sx;
  const int img = blockIdx.x / a.blocks_per_image, blk = blockIdx.x - img * a.blocks_per_image;
  crop_offsets_cta(a, img, &s_dy, &s_sx);
  const int row_bytes = a.W * a.pix_bytes, cpr = row_bytes >> 4, units = a.H * cpr;
  const int shift = s_sx * a.pix_bytes;
  const size_t frame = (size_t)a.H * row_bytes;
  const uint8_t* src = a.src + (size_t)img * frame;
  uint8_t* dst = a.dst + (size_t)img * frame;
  const int q0 = blk * kAugThreads * kCropUnits;
  const int q1 = min(q0 + kAugThreads * kCropUnits, units);
  for (int q = q0 + threadIdx.x; q < q1; q += kAugThreads) {
    const int y = q / cpr, b0 = (q - y * cpr) * 16;
    const uint8_t* srow = src + (size_t)min(max(y + s_dy, 0), a.H - 1) * row_bytes;
    const int a0 = b0 + shift;
    uint4 v;
    if (a0 >= 0 && a0 + 16 <= row_bytes) {
      const uint32_t* s32 = reinterpret_cast<const uint32_t*>(srow) + (a0 >> 2);
      const int bs = (a0 & 3) * 8;
      const uint32_t w0 = __ldg(s32), w1 = __ldg(s32 + 1), w2 = __ldg(s32 + 2), w3 = __ldg(s32 + 3);
      const uint32_t w4 = bs ? __ldg(s32 + 4) : 0u;     // word 4 starts inside the row only when the chunk is misaligned
      v.x = __funnelshift_r(w0, w1, bs); v.y = __funnelshift_r(w1, w2, bs);
      v.z = __funnelshift_r(w2, w3, bs); v.w = __funnelshift_r(w3, w4, bs);
    } else {
      uint32_t o[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int b = 0; b < 16; ++b) {
        const int ob = b0 + b, x = ob / a.pix_bytes, within = ob - x * a.pix_bytes;
        const int xs = min(max(x + s_sx, 0), a.W - 1);
        o[b >> 2] |= (uint32_t)srow[xs * a.pix_bytes + within] << ((b & 3) * 8);
      }
      v = make_uint4(o[0], o[1], o[2], o[3]);
    }
    *reinterpret_cast<uint4*>(dst + (size_t)y * row_bytes + b0) = v;
  }
}

// Any other row: units of U bytes (the widest of 8, 4, 2, 1 that divides the pixel and both buffers' alignment), upp per pixel.
template <typename U>
__global__ void __launch_bounds__(kAugThreads) crop_unit_kernel(const CropArgs a) {
  pdl_prologue();
  __shared__ int s_dy, s_sx;
  const int img = blockIdx.x / a.blocks_per_image, blk = blockIdx.x - img * a.blocks_per_image;
  crop_offsets_cta(a, img, &s_dy, &s_sx);
  const int upp = a.pix_bytes / (int)sizeof(U), upr = a.W * upp, units = a.H * upr;
  const U* src = reinterpret_cast<const U*>(a.src) + (size_t)img * units;
  U* dst = reinterpret_cast<U*>(a.dst) + (size_t)img * units;
  const int q0 = blk * kAugThreads * kCropUnits;
  const int q1 = min(q0 + kAugThreads * kCropUnits, units);
  for (int q = q0 + threadIdx.x; q < q1; q += kAugThreads) {
    const int y = q / upr, r = q - y * upr, x = r / upp, u = r - x * upp;
    const int ys = min(max(y + s_dy, 0), a.H - 1), xs = min(max(x + s_sx, 0), a.W - 1);
    dst[q] = src[(size_t)ys * upr + xs * upp + u];
  }
}

// ---- colour jitter ---------------------------------------------------------------------------------------------------------
// One CTA per image.  The ops run in the drawn order on each pixel in registers; contrast needs each channel's mean over the image
// of the values that reach it, so when contrast runs the CTA first sweeps the image through the ops before it and sums per
// channel in float64 (fixed pixel-to-thread assignment, fixed shuffle tree, warps added in order: bitwise repeatable), then sweeps
// again through every op.  One launch; the second read of an image is mostly L2 hits.
struct ColorArgs {
  const float* src;
  float* dst;
  const uint32_t* keys;
  float* draws;          // nullable: SERL_COLOR_DRAWS floats per image
  int HW;
  serl_color_desc d;
};

__device__ inline void rgb_to_hsv(float r, float g, float b, float& h, float& s, float& v) {
  const float vv = fmaxf(fmaxf(r, g), b);
  const float range = vv - fminf(fminf(r, g), b);
  s = vv > 0.f ? range / vv : 0.f;
  const float norm = range != 0.f ? 1.f / (6.f * range) : 1e9f;
  const float hr = norm * (g - b), hg = norm * (b - r) + 2.f / 6.f, hb = norm * (r - g) + 4.f / 6.f;
  float hue = r == vv ? hr : (g == vv ? hg : hb);
  hue = range > 0.f ? hue : 0.f;
  h = hue < 0.f ? hue + 1.f : hue;
  v = vv;
}

__device__ inline void hsv_to_rgb(float h, float s, float v, float& r, float& g, float& b) {
  const float c = s * v, m = v - c;
  const float dh = jrem(h, 1.f) * 6.f;
  const float x = c * (1.f - fabsf(jrem(dh, 2.f) - 1.f));
  const int hc = (int)floorf(dh);
  r = ((hc == 0 || hc == 5) ? c : (hc == 1 || hc == 4) ? x : 0.f) + m;
  g = ((hc == 1 || hc == 2) ? c : (hc == 0 || hc == 3) ? x : 0.f) + m;
  b = ((hc == 3 || hc == 4) ? c : (hc == 2 || hc == 5) ? x : 0.f) + m;
}

// Op `op` (0 brightness, 1 contrast, 2 saturation, 3 hue) with its drawn parameter, then the clip to [0, 1].
__device__ inline void color_op(int op, float p, const float* mean, float& r, float& g, float& b) {
  if (op == 0) {
    r += p; g += p; b += p;
  } else if (op == 1) {
    r = p * (r - mean[0]) + mean[0]; g = p * (g - mean[1]) + mean[1]; b = p * (b - mean[2]) + mean[2];
  } else {
    float h, s, v;
    rgb_to_hsv(r, g, b, h, s, v);
    if (op == 2) s = clip01(s * p);
    else h = jrem(h + p, 1.f);
    hsv_to_rgb(h, s, v, r, g, b);
  }
  r = clip01(r); g = clip01(g); b = clip01(b);
}

__global__ void __launch_bounds__(kColorThreads) color_kernel(const ColorArgs a) {
  pdl_prologue();
  __shared__ int s_ops[4], s_nops, s_pc, s_gray;
  __shared__ float s_par[4], s_mean[3];
  __shared__ double s_red[kColorThreads / 32][3];
  const int img = blockIdx.x;
  if (threadIdx.x == 0) {
    const u32x2 rng = image_key(a.keys, 0, img);
    const u32x2 apply_rng = jax_split_at(rng, 2, 0), tr = jax_split_at(rng, 2, 1);
    u32x2 k[7];                                                  // perm, brightness, contrast, saturation, hue, jitter, grayscale
#pragma unroll
    for (int j = 0; j < 7; ++j) k[j] = jax_split_at(tr, 7, j);
    const bool apply = jax_uniform(apply_rng, 0.f, 1.f) <= a.d.apply_prob;
    const bool gray = jax_uniform(k[6], 0.f, 1.f) <= a.d.gray_prob;
    const bool jitter = jax_uniform(k[5], 0.f, 1.f) <= a.d.jitter_prob;
    float par[4];
#pragma unroll
    for (int op = 0; op < 4; ++op) par[op] = jax_uniform(k[1 + op], a.d.lo[op], a.d.hi[op]);
    int order[4] = {0, 1, 2, 3};
    if (a.d.shuffle) {                                           // permutation(perm_rng, arange(4)): one round of jax's _shuffle
      const u32x2 sub = jax_split_at(k[0], 2, 1);
      uint32_t bits[4];
#pragma unroll
      for (int m = 0; m < 4; ++m) bits[m] = jax_random_bits_at(sub, 4u, (uint32_t)m);
#pragma unroll
      for (int m = 0; m < 4; ++m) {                              // stable sort by the bits
        int rank = 0;
        for (int j = 0; j < 4; ++j) rank += (bits[j] < bits[m]) || (bits[j] == bits[m] && j < m);
        order[rank] = m;
      }
    }
    int nops = 0, pc = -1;
    for (int pos = 0; pos < 4; ++pos) {
      const int op = order[pos];
      if (apply && jitter && ((a.d.enabled >> op) & 1)) {
        if (op == 1) pc = nops;
        s_ops[nops] = op; s_par[nops] = par[op]; ++nops;
      }
    }
    s_nops = nops; s_pc = pc; s_gray = apply && gray;
    if (a.draws) {
      float* o = a.draws + (size_t)img * SERL_COLOR_DRAWS;
      o[0] = apply; o[1] = jitter; o[2] = gray;
      for (int j = 0; j < 4; ++j) { o[3 + j] = (float)order[j]; o[7 + j] = par[j]; }
      o[11] = 0.f;
    }
  }
  __syncthreads();
  const int nops = s_nops, pc = s_pc;
  const float* src = a.src + (size_t)img * a.HW * 3;
  float* dst = a.dst + (size_t)img * a.HW * 3;
  if (pc >= 0) {
    double acc[3] = {0.0, 0.0, 0.0};
    for (int p = threadIdx.x; p < a.HW; p += kColorThreads) {
      float r = __ldg(src + 3 * p), g = __ldg(src + 3 * p + 1), b = __ldg(src + 3 * p + 2);
      for (int j = 0; j < pc; ++j) color_op(s_ops[j], s_par[j], nullptr, r, g, b);
      acc[0] += r; acc[1] += g; acc[2] += b;
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
      if (l == 0) s_red[w][c] = acc[c];
    }
    __syncthreads();
    if (threadIdx.x < 3) {
      double t = 0.0;
      for (int j = 0; j < kColorThreads / 32; ++j) t += s_red[j][threadIdx.x];
      s_mean[threadIdx.x] = (float)(t / (double)a.HW);
    }
    __syncthreads();
  }
  const float mean[3] = {s_mean[0], s_mean[1], s_mean[2]};
  const bool gray = s_gray;
  for (int p = threadIdx.x; p < a.HW; p += kColorThreads) {
    float r = __ldg(src + 3 * p), g = __ldg(src + 3 * p + 1), b = __ldg(src + 3 * p + 2);
    for (int j = 0; j < nops; ++j) color_op(s_ops[j], s_par[j], mean, r, g, b);
    if (gray) { const float y = 0.2989f * r + 0.5870f * g + 0.1140f * b; r = g = b = y; }
    dst[3 * p] = clip01(r); dst[3 * p + 1] = clip01(g); dst[3 * p + 2] = clip01(b);
  }
}

// ---- Gaussian blur ---------------------------------------------------------------------------------------------------------
// A CTA owns kBlurRows output rows x kBlurCols floats of the row (flattened x * C + c, one per thread) of one image: the
// horizontal pass fills a shared buffer with its kBlurRows + 2 radius input rows (zeros outside the image: SAME padding of the
// intermediate), the vertical pass reads it.  One launch; taps summed in index order.
struct BlurArgs {
  const float* src;
  float* dst;
  const uint32_t* keys;
  float* draws;          // nullable: apply, sigma per image
  int H, W, C, radius, tiles_x, tiles_y;
  float sigma_lo, sigma_hi, apply_prob;
};

__global__ void __launch_bounds__(kBlurCols) blur_kernel(const BlurArgs a) {
  pdl_prologue();
  extern __shared__ float hbuf[];                                // (kBlurRows + 2 radius) x kBlurCols
  __shared__ float s_w[2 * SERL_BLUR_MAX_RADIUS + 1];
  __shared__ int s_apply;
  __shared__ float s_sigma;
  const int tiles = a.tiles_x * a.tiles_y;
  const int img = blockIdx.x / tiles, t = blockIdx.x - img * tiles;
  const int ty = t / a.tiles_x, tx = t - ty * a.tiles_x;
  const int r = a.radius, taps = 2 * r + 1, WC = a.W * a.C;
  if (threadIdx.x == 0) {
    const u32x2 rng = image_key(a.keys, 0, img);
    const u32x2 apply_rng = jax_split_at(rng, 2, 0), tr = jax_split_at(rng, 2, 1);
    s_apply = jax_uniform(apply_rng, 0.f, 1.f) <= a.apply_prob;
    s_sigma = jax_uniform(jax_split_at(tr, 1, 0), a.sigma_lo, a.sigma_hi);
    if (a.draws && t == 0) { a.draws[2 * img] = (float)s_apply; a.draws[2 * img + 1] = s_sigma; }
  }
  __syncthreads();
  const int y0 = ty * kBlurRows, rows = min(kBlurRows, a.H - y0);
  const int col = tx * kBlurCols + threadIdx.x;
  const bool live = col < WC;
  const float* src = a.src + (size_t)img * a.H * WC;
  float* dst = a.dst + (size_t)img * a.H * WC;
  if (!s_apply) {
    if (live)
      for (int i = 0; i < rows; ++i) dst[(size_t)(y0 + i) * WC + col] = __ldg(src + (size_t)(y0 + i) * WC + col);
    return;
  }
  if (threadIdx.x < taps) {
    const float x = (float)((int)threadIdx.x - r), sg = s_sigma;
    s_w[threadIdx.x] = expf(-(x * x) / (2.f * (sg * sg)));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
    for (int k = 0; k < taps; ++k) sum += s_w[k];
    s_sigma = sum;                                               // reused as the taps' sum
  }
  __syncthreads();
  if (threadIdx.x < taps) s_w[threadIdx.x] = s_w[threadIdx.x] / s_sigma;
  __syncthreads();
  const int x = live ? col / a.C : 0, c = col - x * a.C;
  const int k_lo = max(0, r - x), k_hi = min(taps, a.W + r - x); // taps whose column lies inside the row
  for (int j = 0; j < rows + 2 * r; ++j) {
    const int yy = y0 - r + j;
    float v = 0.f;
    if (live && yy >= 0 && yy < a.H) {
      const float* srow = src + (size_t)yy * WC + c;
      for (int k = k_lo; k < k_hi; ++k) v = fmaf(s_w[k], __ldg(srow + (size_t)(x + k - r) * a.C), v);
    }
    hbuf[j * kBlurCols + threadIdx.x] = v;
  }
  __syncthreads();
  if (!live) return;
  for (int i = 0; i < rows; ++i) {
    float v = 0.f;
    for (int k = 0; k < taps; ++k) v = fmaf(s_w[k], hbuf[(i + k) * kBlurCols + threadIdx.x], v);
    dst[(size_t)(y0 + i) * WC + col] = v;
  }
}

// ---- flip and solarize -----------------------------------------------------------------------------------------------------
// Elementwise over CTAs of kAugThreads * kEltItems elements of one image; thread 0 draws the image's decision.
struct EltArgs {
  const float* src;
  float* dst;
  const uint32_t* keys;
  int H, W, C, blocks_per_image;
  float threshold, apply_prob;
};

template <bool kFlip>
__global__ void __launch_bounds__(kAugThreads) elementwise_kernel(const EltArgs a) {
  pdl_prologue();
  __shared__ int s_on;
  const int img = blockIdx.x / a.blocks_per_image, blk = blockIdx.x - img * a.blocks_per_image;
  if (threadIdx.x == 0) {
    const u32x2 rng = image_key(a.keys, 0, img);
    s_on = kFlip ? jax_uniform(jax_split_at(rng, 2, 1), 0.f, 1.f) <= 0.5f : jax_uniform(rng, 0.f, 1.f) <= a.apply_prob;
  }
  __syncthreads();
  const bool on = s_on;
  const int WC = a.W * a.C, n = a.H * WC;
  const float* src = a.src + (size_t)img * n;
  float* dst = a.dst + (size_t)img * n;
  const int e0 = blk * kAugThreads * kEltItems + threadIdx.x, e1 = min(blk * kAugThreads * kEltItems + kAugThreads * kEltItems, n);
#pragma unroll 4
  for (int e = e0; e < e1; e += kAugThreads) {
    if constexpr (kFlip) {
      int s = e;
      if (on) { const int y = e / WC, rx = e - y * WC, x = rx / a.C; s = y * WC + (a.W - 1 - x) * a.C + (rx - x * a.C); }
      dst[e] = __ldg(src + s);
    } else {
      const float v = __ldg(src + e);
      dst[e] = (on && !(v < a.threshold)) ? 1.f - v : v;
    }
  }
}

static int check_images(const char* fn, const void* src, const void* dst, const void* keys, int n, int H, int W, int C) {
  if (!src || !dst || !keys || n < 1 || H < 1 || W < 1 || C < 1 || (long long)H * W * C > 0x7fffffffLL) {
    set_last_error("%s: invalid arguments (n=%d H=%d W=%d C=%d)", fn, n, H, W, C);
    return SERL_ERR_INVALID;
  }
  return SERL_OK;
}

static int grid_or_error(const char* fn, long long blocks, int* out) {
  if (blocks > 0x7fffffffLL) { set_last_error("%s: %lld CTAs exceed the grid", fn, blocks); return SERL_ERR_INVALID; }
  *out = (int)blocks;
  return SERL_OK;
}

}  // namespace serl

using namespace serl;

extern "C" int serl_aug_crop(const void* src, void* dst, const uint32_t* keys, int split_n, int n, int H, int W, int pix_bytes,
                             int padding, void* stream) {
  if (int e = check_images("serl_aug_crop", src, dst, keys, n, H, W, pix_bytes)) return e;
  if (padding < 0 || split_n < 0 || (split_n > 0 && split_n != n)) {
    set_last_error("serl_aug_crop: invalid padding %d or split %d of %d images", padding, split_n, n);
    return SERL_ERR_INVALID;
  }
  CropArgs a{static_cast<const uint8_t*>(src), static_cast<uint8_t*>(dst), keys, split_n, H, W, pix_bytes, padding, 0};
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uintptr_t align = reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst);
  const long long row_bytes = (long long)W * pix_bytes;
  const int per_cta = kAugThreads * kCropUnits;
  int grid = 0;
  if (row_bytes % 16 == 0 && align % 16 == 0) {
    a.blocks_per_image = ceil_div(H * (int)(row_bytes / 16), per_cta);
    if (int e = grid_or_error("serl_aug_crop", (long long)n * a.blocks_per_image, &grid)) return e;
    launch_k(crop_wide_kernel, dim3(grid), dim3(kAugThreads), 0, st, a);
    return check_launch("crop_wide_kernel");
  }
  int u = 8;
  while (u > 1 && (pix_bytes % u != 0 || align % u != 0)) u >>= 1;
  a.blocks_per_image = ceil_div(H * W * (pix_bytes / u), per_cta);
  if (int e = grid_or_error("serl_aug_crop", (long long)n * a.blocks_per_image, &grid)) return e;
  switch (u) {
    case 8: launch_k(crop_unit_kernel<uint64_t>, dim3(grid), dim3(kAugThreads), 0, st, a); break;
    case 4: launch_k(crop_unit_kernel<uint32_t>, dim3(grid), dim3(kAugThreads), 0, st, a); break;
    case 2: launch_k(crop_unit_kernel<uint16_t>, dim3(grid), dim3(kAugThreads), 0, st, a); break;
    default: launch_k(crop_unit_kernel<uint8_t>, dim3(grid), dim3(kAugThreads), 0, st, a); break;
  }
  return check_launch("crop_unit_kernel");
}

extern "C" int serl_aug_color(const float* src, float* dst, const uint32_t* keys, float* draws, int n, int H, int W,
                              const serl_color_desc* desc, void* stream) {
  if (int e = check_images("serl_aug_color", src, dst, keys, n, H, W, 3)) return e;
  if (!desc) { set_last_error("serl_aug_color: no descriptor"); return SERL_ERR_INVALID; }
  ColorArgs a{src, dst, keys, draws, H * W, *desc};
  launch_k(color_kernel, dim3(n), dim3(kColorThreads), 0, static_cast<cudaStream_t>(stream), a);
  return check_launch("color_kernel");
}

extern "C" int serl_aug_blur(const float* src, float* dst, const uint32_t* keys, float* draws, int n, int H, int W, int C, int radius,
                             float sigma_min, float sigma_max, float apply_prob, void* stream) {
  if (int e = check_images("serl_aug_blur", src, dst, keys, n, H, W, C)) return e;
  if (radius < 0 || radius > SERL_BLUR_MAX_RADIUS) {
    set_last_error("serl_aug_blur: radius %d outside [0, %d]", radius, SERL_BLUR_MAX_RADIUS);
    return SERL_ERR_INVALID;
  }
  BlurArgs a{src, dst, keys, draws, H, W, C, radius, ceil_div(W * C, kBlurCols), ceil_div(H, kBlurRows), sigma_min, sigma_max, apply_prob};
  int grid = 0;
  if (int e = grid_or_error("serl_aug_blur", (long long)n * a.tiles_x * a.tiles_y, &grid)) return e;
  const size_t smem = sizeof(float) * (size_t)(kBlurRows + 2 * radius) * kBlurCols;
  if (cudaFuncSetAttribute(blur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return check_launch("cudaFuncSetAttribute(blur_kernel)");
  launch_k(blur_kernel, dim3(grid), dim3(kBlurCols), smem, static_cast<cudaStream_t>(stream), a);
  return check_launch("blur_kernel");
}

static int elementwise_launch(bool flip, const char* fn, const float* src, float* dst, const uint32_t* keys, int n, int H, int W, int C,
                              float threshold, float apply_prob, void* stream) {
  if (int e = check_images(fn, src, dst, keys, n, H, W, C)) return e;
  EltArgs a{src, dst, keys, H, W, C, ceil_div(H * W * C, kAugThreads * kEltItems), threshold, apply_prob};
  int grid = 0;
  if (int e = grid_or_error(fn, (long long)n * a.blocks_per_image, &grid)) return e;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (flip) launch_k(elementwise_kernel<true>, dim3(grid), dim3(kAugThreads), 0, st, a);
  else launch_k(elementwise_kernel<false>, dim3(grid), dim3(kAugThreads), 0, st, a);
  return check_launch(flip ? "elementwise_kernel<true>" : "elementwise_kernel<false>");
}

extern "C" int serl_aug_flip(const float* src, float* dst, const uint32_t* keys, int n, int H, int W, int C, void* stream) {
  return elementwise_launch(true, "serl_aug_flip", src, dst, keys, n, H, W, C, 0.f, 0.f, stream);
}

extern "C" int serl_aug_solarize(const float* src, float* dst, const uint32_t* keys, int n, int H, int W, int C, float threshold,
                                 float apply_prob, void* stream) {
  return elementwise_launch(false, "serl_aug_solarize", src, dst, keys, n, H, W, C, threshold, apply_prob, stream);
}
