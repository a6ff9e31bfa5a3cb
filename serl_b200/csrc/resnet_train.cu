// DrQ's trainable ResNet-10 encoder (encoder_type="resnet": vision/resnet_v1.py:129-286 with pre_pooling=False): the
// convolutions' forward, input gradient (dgrad) and weight gradient (wgrad) at any (kh, kw, stride, pad), the GroupNorm and
// 3x3/2 max-pool backward passes, and the stem's normalised input copy.
//
// Convolutions: one implicit GEMM per mode over NHWC fp32 maps with Ci % 4 == 0 (the stem's 3-channel image is staged as a
// normalised, zero-padded 4-channel copy by rn_stem_prep_kernel), weights (kh, kw, Cw, Co) with Cw <= Ci (Cw = 3 for the stem):
//   fwd    C[(n,oy,ox), co]  = sum_{(ky,kx,ci)} x[n, s oy - pad + ky, s ox - pad + kx, ci] W[ky,kx,ci,co]
//   dgrad  C[(n,iy,ix), ci]  = sum_{(ky,kx,co)} dz[n, (iy + pad - ky) / s, (ix + pad - kx) / s, co] W[ky,kx,ci,co]
//          run per parity class (iy % s, ix % s) = blockIdx.z over the taps with (i + pad - k) % s == 0 only: a stride-2
//          dgrad multiplies no structural zeros (the 1x1/2 projection's odd-parity classes have no tap and write zeros)
//   wgrad  C[(ky,kx,ci), co] = sum_{(n,oy,ox)} x[n, s oy - pad + ky, s ox - pad + kx, ci] dz[n,oy,ox,co]
//          in fixed split-K ranges of pixels, summed in split order by rn_wgrad_reduce_kernel
// Every operand element comes in 16-byte groups of 4 consecutive channels (one tap), copied by cp.async with zero-fill at the
// image borders and the GEMM edges into a 4-stage ring of raw fp32 tiles (128 x 32 of A, 32 x 64 of B), so three k-blocks
// of loads stay in flight while one is consumed.  Two consumers of the same ring, chosen per call (`tc`):
//   * tc = 0 (fp32 build, 1e-5 parity): CUDA-core FMAs from the raw tiles, 8 x 4 outputs per thread, k in order;
//   * tc = 1 (fp16 / bf16 builds): each raw tile is split into hi = rna_tf32(x), lo = x - hi in K-major 128B-swizzled operand
//     tiles and accumulated as lo*hi + hi*lo + hi*hi by wgmma m64n64k8 tf32 (as gemm_tf32x3.cu): fp32-class products, fp32
//     masters and fp32 activations.  Row-major raw tiles are written in the operand tiles' swizzle already, so their split
//     is element-wise.
// No atomics anywhere: two launches are bitwise equal.
#include "common.cuh"
#include "gemm_common.cuh"
#include "wgmma.cuh"
#include "serl_b200.h"

namespace serl {
namespace rconv {

enum Mode { FWD = 0, DGRAD = 1, WGRAD = 2 };
constexpr int TM = 128, TN = 64, TK = 32, STAGES = 4;
constexpr int RAW_A = TM * TK * 4, RAW_B = TN * TK * 4, RAW_STAGE = RAW_A + RAW_B;
constexpr int OP_A = TM * 128, OP_B = TN * 128, OP_STAGE = 2 * OP_A + 2 * OP_B;     // hi + lo of both operands
constexpr int SMEM_TC = 2 * OP_STAGE + STAGES * RAW_STAGE + 1024;
constexpr int SMEM_CC = STAGES * RAW_STAGE + 1024;
constexpr int WGRAD_CTAS = 2 * 132;        // wgrad split-K target: about two CTAs per SM

struct Args {
  const float* x;       // conv input (N,H,W,Ci)                        fwd, wgrad
  const float* w;       // (kh,kw,Cw,Co)                                fwd, dgrad
  const float* dz;      // gradient of the conv output (N,Ho,Wo,Co)     dgrad, wgrad
  float* out;           // fwd (N,Ho,Wo,Co) | dgrad (N,H,W,Ci) | wgrad partials (splits, kh*kw*Ci, Co)
  int N, H, W, Ci, Cw, Ho, Wo, Co, kh, kw, stride, pad;
  int accumulate;       // dgrad: out += result
  int k_split;          // wgrad: pixels per split (multiple of TK)
};

__device__ __forceinline__ void cp16(uint32_t dst, const float* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
// byte offset of element group (r, c) (c = k / 4) of a row-major 32-wide tile in the 128B swizzle (wgmma.cuh)
__device__ __forceinline__ int sw_off(int r, int c) { return r * 128 + ((c ^ (r & 7)) << 4); }

// Per-CTA problem geometry of one mode
struct Geo {
  int M, NC, kbeg, kend;
  int py, px, ky0, kx0, nkx;      // dgrad: parity class and its tap lattice
  int Hq, Wq;                      // dgrad: rows per parity class
};

template <int kMode>
__device__ __forceinline__ Geo geometry(const Args& a) {
  Geo g{};
  if (kMode == FWD) {
    g.M = a.N * a.Ho * a.Wo; g.NC = a.Co; g.kbeg = 0; g.kend = a.kh * a.kw * a.Ci;
  } else if (kMode == DGRAD) {
    const int s = a.stride;
    g.py = blockIdx.z / s; g.px = blockIdx.z - g.py * s;
    g.ky0 = (g.py + a.pad) % s; g.kx0 = (g.px + a.pad) % s;
    const int nky = g.ky0 < a.kh ? (a.kh - g.ky0 + s - 1) / s : 0;
    g.nkx = g.kx0 < a.kw ? (a.kw - g.kx0 + s - 1) / s : 0;
    g.Hq = a.H / s; g.Wq = a.W / s;
    g.M = a.N * g.Hq * g.Wq; g.NC = a.Ci; g.kbeg = 0; g.kend = nky * g.nkx * a.Co;
  } else {
    g.M = a.kh * a.kw * a.Ci; g.NC = a.Co;
    const int K = a.N * a.Ho * a.Wo;
    g.kbeg = blockIdx.z * a.k_split; g.kend = min(K, g.kbeg + a.k_split);
  }
  return g;
}

template <int kMode>
__device__ __forceinline__ void store_out(const Args& a, const Geo& g, int m, int n, float v) {
  if (m >= g.M || n >= g.NC) return;
  if (kMode == FWD) {
    a.out[(size_t)m * a.Co + n] = v;
  } else if (kMode == DGRAD) {
    const int HWq = g.Hq * g.Wq, b = m / HWq, r = m - b * HWq, qy = r / g.Wq, qx = r - qy * g.Wq;
    float* o = a.out + (((size_t)b * a.H + qy * a.stride + g.py) * a.W + qx * a.stride + g.px) * a.Ci + n;
    *o = a.accumulate ? *o + v : v;
  } else {
    a.out[((size_t)blockIdx.z * g.M + m) * a.Co + n] = v;
  }
}

template <int kMode, bool kTC>
__global__ void __launch_bounds__(256, kTC ? 1 : 2) rconv_kernel(const Args a) {
  pdl_prologue();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sRaw = smem + (kTC ? 2 * OP_STAGE : 0);
  const int tid = threadIdx.x;
  const Geo g = geometry<kMode>(a);
  const int m0 = blockIdx.x * TM, n0 = blockIdx.y * TN;
  const int nk = g.kend > g.kbeg ? ceil_div(g.kend - g.kbeg, TK) : 0;

  // A: fwd / dgrad row-major (swizzled) - thread's rows (tid >> 3) + 32 i, channel group tid & 7; wgrad k-major [k][128] -
  // thread's rows 4 (tid & 31) .. + 3, pixels (tid >> 5) + 8 i
  int rb[4], ry[4], rx[4];                 // fwd: (image, s oy - pad, s ox - pad); dgrad: (image, iy, ix); -1: no row
  int wtap_y = 0, wtap_x = 0, wci = 0;     // wgrad: the thread's rows' tap and first channel
  bool wrow = false;
  if (kMode != WGRAD) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + (tid >> 3) + 32 * i;
      rb[i] = -1; ry[i] = rx[i] = 0;
      if (m < g.M) {
        if (kMode == FWD) {
          const int HWo = a.Ho * a.Wo, b = m / HWo, r = m - b * HWo, oy = r / a.Wo, ox = r - oy * a.Wo;
          rb[i] = b; ry[i] = oy * a.stride - a.pad; rx[i] = ox * a.stride - a.pad;
        } else {
          const int HWq = g.Hq * g.Wq, b = m / HWq, r = m - b * HWq, qy = r / g.Wq, qx = r - qy * g.Wq;
          rb[i] = b; ry[i] = qy * a.stride + g.py; rx[i] = qx * a.stride + g.px;
        }
      }
    }
  } else {
    const int m = m0 + 4 * (tid & 31);
    wrow = m < g.M;
    if (wrow) {
      const int tap = m / a.Ci;
      wci = m - tap * a.Ci; wtap_y = tap / a.kw; wtap_x = tap - wtap_y * a.kw;
    }
  }

  auto issue = [&](int kt) {
    const uint32_t dA = t_smem(sRaw + (kt % STAGES) * RAW_STAGE), dB = dA + RAW_A;
    const int k0 = g.kbeg + kt * TK;
    if (kMode != WGRAD) {
      const int c = tid & 7, k = k0 + 4 * c;
      const int C = kMode == FWD ? a.Ci : a.Co;
      const int tap = k / C, ch = k - tap * C;
      int ky, kx;
      if (kMode == FWD) { ky = tap / a.kw; kx = tap - ky * a.kw; }
      else { const int jy = g.nkx ? tap / g.nkx : 0; ky = g.ky0 + a.stride * jy; kx = g.kx0 + a.stride * (tap - jy * g.nkx); }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = (tid >> 3) + 32 * i;
        const float* src = nullptr;
        if (rb[i] >= 0 && k < g.kend) {
          if (kMode == FWD) {
            const int iy = ry[i] + ky, ix = rx[i] + kx;
            if (iy >= 0 && iy < a.H && ix >= 0 && ix < a.W) src = a.x + (((size_t)rb[i] * a.H + iy) * a.W + ix) * a.Ci + ch;
          } else {
            const int ty = ry[i] + a.pad - ky, tx = rx[i] + a.pad - kx;      // multiples of s by the parity class
            if (ty >= 0 && tx >= 0 && ty < a.Ho * a.stride && tx < a.Wo * a.stride)
              src = a.dz + (((size_t)rb[i] * a.Ho + ty / a.stride) * a.Wo + tx / a.stride) * a.Co + ch;
          }
        }
        cp16(dA + sw_off(r, c), src ? src : a.out, src != nullptr);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = (tid >> 5) + 8 * i, p = k0 + kk;
        const float* src = nullptr;
        if (wrow && p < g.kend) {
          const int HWo = a.Ho * a.Wo, b = p / HWo, r = p - b * HWo, oy = r / a.Wo, ox = r - oy * a.Wo;
          const int iy = oy * a.stride - a.pad + wtap_y, ix = ox * a.stride - a.pad + wtap_x;
          if (iy >= 0 && iy < a.H && ix >= 0 && ix < a.W) src = a.x + (((size_t)b * a.H + iy) * a.W + ix) * a.Ci + wci;
        }
        cp16(dA + kk * (TM * 4) + (tid & 31) * 16, src ? src : a.out, src != nullptr);
      }
    }
    // B: fwd / wgrad k-major [k][64]; dgrad row-major (swizzled) [ci][32]
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int it = tid + 256 * i;
      const float* src = nullptr;
      if (kMode == DGRAD) {
        const int r = it >> 3, c = it & 7, k = k0 + 4 * c, ci = n0 + r;
        if (k < g.kend && ci < a.Ci) {
          const int tap = k / a.Co, co = k - tap * a.Co, jy = tap / g.nkx;
          const int ky = g.ky0 + a.stride * jy, kx = g.kx0 + a.stride * (tap - jy * g.nkx);
          src = a.w + ((size_t)(ky * a.kw + kx) * a.Ci + ci) * a.Co + co;
        }
        cp16(dB + sw_off(r, c), src ? src : a.out, src != nullptr);
      } else {
        const int kk = it >> 4, c = it & 15, k = k0 + kk, co = n0 + 4 * c;
        if (k < g.kend && co < a.Co) {
          if (kMode == FWD) {
            const int tap = k / a.Ci, ci = k - tap * a.Ci;
            if (ci < a.Cw) src = a.w + ((size_t)tap * a.Cw + ci) * a.Co + co;
          } else {
            src = a.dz + (size_t)k * a.Co + co;
          }
        }
        cp16(dB + kk * (TN * 4) + c * 16, src ? src : a.out, src != nullptr);
      }
    }
  };

#pragma unroll
  for (int st = 0; st < STAGES - 1; ++st) {
    if (st < nk) issue(st);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }

  if constexpr (kTC) {
    const int warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int kt = 0; kt < nk; ++kt) {
      asm volatile("cp.async.wait_group %0;" ::"n"(STAGES - 2) : "memory");
      __syncthreads();             // raw stage kt landed; the MMAs of k-block kt - 2 (operand stage kt & 1) are retired
      if (kt + STAGES - 1 < nk) issue(kt + STAGES - 1);
      asm volatile("cp.async.commit_group;" ::: "memory");
      uint8_t* op = smem + (kt & 1) * OP_STAGE;
      const uint8_t* raw = sRaw + (kt % STAGES) * RAW_STAGE;
      if (kMode == WGRAD) {
        t_convert<TM>(reinterpret_cast<const float*>(raw), op, op + OP_A, true, tid);
      } else {
#pragma unroll
        for (int i = 0; i < TM * 8 / 256; ++i) {
          const int off = (tid + 256 * i) * 16;
          const float4 v = *reinterpret_cast<const float4*>(raw + off);
          float4 h, l;
          t_split(v.x, h.x, l.x); t_split(v.y, h.y, l.y); t_split(v.z, h.z, l.z); t_split(v.w, h.w, l.w);
          *reinterpret_cast<float4*>(op + off) = h;
          *reinterpret_cast<float4*>(op + OP_A + off) = l;
        }
      }
      if (kMode == DGRAD) {
#pragma unroll
        for (int i = 0; i < TN * 8 / 256; ++i) {
          const int off = (tid + 256 * i) * 16;
          const float4 v = *reinterpret_cast<const float4*>(raw + RAW_A + off);
          float4 h, l;
          t_split(v.x, h.x, l.x); t_split(v.y, h.y, l.y); t_split(v.z, h.z, l.z); t_split(v.w, h.w, l.w);
          *reinterpret_cast<float4*>(op + 2 * OP_A + off) = h;
          *reinterpret_cast<float4*>(op + 2 * OP_A + OP_B + off) = l;
        }
      } else {
        t_convert<TN>(reinterpret_cast<const float*>(raw + RAW_A), op + 2 * OP_A, op + 2 * OP_A + OP_B, true, tid);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // generic-proxy stores -> tensor-core reads
      __syncthreads();
      const uint64_t a_hi = wg_desc(t_smem(op) + wg * 8192), a_lo = wg_desc(t_smem(op + OP_A) + wg * 8192);
      const uint64_t b_hi = wg_desc(t_smem(op + 2 * OP_A)), b_lo = wg_desc(t_smem(op + 2 * OP_A + OP_B));
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
      for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
#pragma unroll
      for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, a_hi + 2 * k, b_hi + 2 * k, 1u);
      wg_commit();
      wg_wait<1>();
    }
    wg_wait<0>();
    asm volatile("cp.async.wait_all;" ::: "memory");
    // accumulator fragments (wgmma.cuh): rows 16 (warp % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) store_out<kMode>(a, g, m, n0 + 8 * j + 2 * (lane & 3) + e, acc[4 * j + 2 * h + e]);
    }
  } else {
    const int tx = tid & 15, ty = tid >> 4;            // rows ty + 16 i, columns tx + 16 j
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int kt = 0; kt < nk; ++kt) {
      asm volatile("cp.async.wait_group %0;" ::"n"(STAGES - 2) : "memory");
      __syncthreads();             // raw stage kt landed; every thread is done with the stage the next issue overwrites
      if (kt + STAGES - 1 < nk) issue(kt + STAGES - 1);
      asm volatile("cp.async.commit_group;" ::: "memory");
      const float* rA = reinterpret_cast<const float*>(sRaw + (kt % STAGES) * RAW_STAGE);
      const float* rB = rA + TM * TK;
#pragma unroll 4
      for (int k = 0; k < TK; ++k) {
        float av[8], bv[4];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = ty + 16 * i;
          av[i] = kMode == WGRAD ? rA[k * TM + r] : rA[r * 32 + ((((k >> 2) ^ (r & 7))) << 2) + (k & 3)];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int n = tx + 16 * j;
          bv[j] = kMode == DGRAD ? rB[n * 32 + ((((k >> 2) ^ (n & 7))) << 2) + (k & 3)] : rB[k * TN + n];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) store_out<kMode>(a, g, m0 + ty + 16 * i, n0 + tx + 16 * j, acc[i][j]);
  }
}

// dw[(tap, ci < Cw), co] = sum over the splits, in split order, of the partials' row (tap, ci) (tap * Ci + ci)
__global__ void __launch_bounds__(256) rn_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, int taps, int Ci,
                                                              int Cw, int Co, int splits) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= taps * Cw * Co) return;
  const int co = i % Co, r = i / Co, ci = r % Cw, tap = r / Cw;
  const size_t M = (size_t)taps * Ci, src = ((size_t)tap * Ci + ci) * Co + co;
  float s = 0.f;
  for (int z = 0; z < splits; ++z) s += part[(size_t)z * M * Co + src];
  dw[i] = s;
}

// (N,H,W,3) uint8 -> (N,H,W,4) fp32: (x / 255 - mean) / std per channel (resnet_v1.py:222-224, the same expression as
// trunk_fp32.cu's on-load normalisation), channel 3 zero
__global__ void rn_stem_prep_kernel(const uint8_t* __restrict__ x, float* __restrict__ y, long long pixels) {
  pdl_prologue();
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < pixels; p += (long long)gridDim.x * blockDim.x) {
    float4 o;
    o.x = ((float)x[3 * p] / 255.0f - mean[0]) / stdv[0];
    o.y = ((float)x[3 * p + 1] / 255.0f - mean[1]) / stdv[1];
    o.z = ((float)x[3 * p + 2] / 255.0f - mean[2]) / stdv[2];
    o.w = 0.f;
    reinterpret_cast<float4*>(y)[p] = o;
  }
}

// (N,H,W,Ci) uint8 -> (N,H,W,Cp) fp32, Cp = Ci rounded up to a multiple of 4: rn_stem_prep_kernel's normalisation of channel c by
// the statistics of c mod 3 (a stack of T RGB frames on the channel axis, Ci = 3T), channels Ci .. Cp-1 zero.  One thread per
// output float.
__global__ void rn_stem_prep_stacked_kernel(const uint8_t* __restrict__ x, float* __restrict__ y, long long pixels, int Ci, int Cp) {
  pdl_prologue();
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < pixels * Cp; e += (long long)gridDim.x * blockDim.x) {
    const long long p = e / Cp;
    const int c = (int)(e - p * Cp), c3 = c % 3;
    const float mean = c3 == 0 ? 0.485f : (c3 == 1 ? 0.456f : 0.406f), stdv = c3 == 0 ? 0.229f : (c3 == 1 ? 0.224f : 0.225f);
    y[e] = c < Ci ? ((float)x[p * Ci + c] / 255.0f - mean) / stdv : 0.f;
  }
}

// dp = dy gated by y > 0 (y == nullptr: no ReLU) and xhat = (x - mean) * rstd of one channel quad
__device__ __forceinline__ void gn_grad_in(const float* x, const float* dy, const float* y, size_t off, float mean, float rstd, float4& dp,
                                           float4& xh) {
  const float4 v = *reinterpret_cast<const float4*>(x + off);
  dp = *reinterpret_cast<const float4*>(dy + off);
  if (y) {
    const float4 o = *reinterpret_cast<const float4*>(y + off);
    dp.x = o.x > 0.f ? dp.x : 0.f; dp.y = o.y > 0.f ? dp.y : 0.f; dp.z = o.z > 0.f ? dp.z : 0.f; dp.w = o.w > 0.f ? dp.w : 0.f;
  }
  xh = make_float4((v.x - mean) * rstd, (v.y - mean) * rstd, (v.z - mean) * rstd, (v.w - mean) * rstd);
}

// GroupNorm statistics of the forward (trunk_fp32.cu groupnorm_f32_kernel): its loop, thread count and reduction, so mean and
// rstd are bitwise the forward's.  stats[(n G + g) 2 + {0, 1}] = (mean, rstd).  grid (G, N), 512 threads.
__global__ void __launch_bounds__(512) rn_groupnorm_stats_kernel(const float* __restrict__ x, float* __restrict__ stats, int HW, int C,
                                                                 int G, float eps) {
  pdl_prologue();
  __shared__ float red[64];
  const int g = blockIdx.x, n = blockIdx.y;
  const int Cg = C / G, q = Cg >> 2;
  const float* xb = x + (size_t)n * HW * C + g * Cg;
  const int total = HW * q;
  float s = 0.f, ss = 0.f;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    int p = e / q, c4 = e - p * q;
    float4 v = *reinterpret_cast<const float4*>(xb + (size_t)p * C + c4 * 4);
    s += (v.x + v.y) + (v.z + v.w);
    ss += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  block_sum2(s, ss, red);
  if (threadIdx.x == 0) {
    const float cnt = (float)HW * (float)Cg;
    const float mean = s / cnt;
    const float var = fmaxf(ss / cnt - mean * mean, 0.f);
    stats[((size_t)n * G + g) * 2] = mean;
    stats[((size_t)n * G + g) * 2 + 1] = rsqrtf(var + eps);
  }
}

// GroupNorm backward, one CTA per (group, image), 512 threads, from the forward's statistics (rn_groupnorm_stats_kernel):
//   y = [relu](xhat * scale + bias [+ residual]),  xhat = (x - mean) * rstd
//   dp = dy * (y > 0) (relu' = 0 at 0), or dy;  dres = dp;  g = dp * scale
//   dx = rstd (g - sum(g) / n - xhat sum(g xhat) / n)     (sums over the (image, group): block_sum2, a fixed order)
//   partials[image][c] = sum_p dp xhat (dscale), partials[N + image][c] = sum_p dp (dbias), each over the image's pixels
//   in a fixed order (thread-strided, then the threads that share the channel in thread order)
// The first T = (512 / q) q threads walk the group's (pixel, quad) elements with stride T, a multiple of q, so each keeps one
// channel quad; when q does not divide 512 the other threads hold no element and add zeros to the block sums.
__global__ void __launch_bounds__(512) rn_groupnorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                               const float* __restrict__ dy, const float* __restrict__ scale,
                                                               const float* __restrict__ stats, float* __restrict__ dx,
                                                               float* __restrict__ dres, float* __restrict__ partials, int N, int HW,
                                                               int C, int G, int relu) {
  pdl_prologue();
  __shared__ float red[64];
  __shared__ __align__(16) float part[2][512 * 4];
  const int grp = blockIdx.x, n = blockIdx.y;
  const int Cg = C / G, q = Cg >> 2;
  const size_t base = (size_t)n * HW * C + grp * Cg;
  const float* xb = x + base;
  const int total = HW * q;
  const float cnt = (float)HW * (float)Cg;
  const float mean = stats[((size_t)n * G + grp) * 2], rstd = stats[((size_t)n * G + grp) * 2 + 1];

  const int T = ((int)blockDim.x / q) * q, c4 = threadIdx.x % q;          // q <= 128: T > 384
  const bool walks = (int)threadIdx.x < T;
  const float4 sc = *reinterpret_cast<const float4*>(scale + grp * Cg + c4 * 4);
  float s1 = 0.f, s2 = 0.f;
  float4 dg = make_float4(0.f, 0.f, 0.f, 0.f), db = dg;
  for (int e = walks ? threadIdx.x : total; e < total; e += T) {
    const int p = e / q;
    float4 dp, xh;
    gn_grad_in(xb, dy + base, relu ? y + base : nullptr, (size_t)p * C + c4 * 4, mean, rstd, dp, xh);
    const float4 gg = make_float4(dp.x * sc.x, dp.y * sc.y, dp.z * sc.z, dp.w * sc.w);
    s1 += (gg.x + gg.y) + (gg.z + gg.w);
    s2 += (gg.x * xh.x + gg.y * xh.y) + (gg.z * xh.z + gg.w * xh.w);
    dg.x += dp.x * xh.x; dg.y += dp.y * xh.y; dg.z += dp.z * xh.z; dg.w += dp.w * xh.w;
    db.x += dp.x; db.y += dp.y; db.z += dp.z; db.w += dp.w;
  }
  reinterpret_cast<float4*>(part[0])[threadIdx.x] = dg;
  reinterpret_cast<float4*>(part[1])[threadIdx.x] = db;
  block_sum2(s1, s2, red);                             // (its leading __syncthreads also publishes part)
  __syncthreads();
  if (threadIdx.x < Cg) {
    const int cc = threadIdx.x, cq = cc >> 2, comp = cc & 3;
    float a0 = 0.f, a1 = 0.f;
    for (int t = cq; t < T; t += q) {
      a0 += part[0][4 * t + comp];
      a1 += part[1][4 * t + comp];
    }
    partials[(size_t)n * C + grp * Cg + cc] = a0;
    partials[(size_t)(N + n) * C + grp * Cg + cc] = a1;
  }
  const float m1 = s1 / cnt, m2 = s2 / cnt;
  for (int e = walks ? threadIdx.x : total; e < total; e += T) {
    const int p = e / q;
    const size_t off = (size_t)p * C + c4 * 4;
    float4 dp, xh;
    gn_grad_in(xb, dy + base, relu ? y + base : nullptr, off, mean, rstd, dp, xh);
    float4 o;
    o.x = rstd * (dp.x * sc.x - m1 - xh.x * m2); o.y = rstd * (dp.y * sc.y - m1 - xh.y * m2);
    o.z = rstd * (dp.z * sc.z - m1 - xh.z * m2); o.w = rstd * (dp.w * sc.w - m1 - xh.w * m2);
    *reinterpret_cast<float4*>(dx + base + off) = o;
    if (dres) *reinterpret_cast<float4*>(dres + base + off) = dp;
  }
}

// dscale[c] = sum_n partials[n][c], dbias[c] = sum_n partials[N + n][c], in image order
__global__ void rn_groupnorm_param_reduce_kernel(const float* __restrict__ partials, float* __restrict__ dscale, float* __restrict__ dbias,
                                                 int N, int C) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * C) return;
  const int which = i / C, c = i - which * C;
  const float* p = partials + (size_t)which * N * C + c;
  float s = 0.f;
  for (int n = 0; n < N; ++n) s += p[(size_t)n * C];
  (which ? dbias : dscale)[c] = s;
}

// max_pool 3x3 / stride 2 SAME backward as a gather: input pixel (iy, ix) sums, over the windows that contain it in (oy, ox)
// order, the output gradients of the windows whose first maximal element (row-major window order; XLA select_and_scatter
// with `ge`) it is.  The windows' maxima are recomputed from the saved input x.  pad_y / pad_x: each axis's low SAME pad.
__global__ void rn_maxpool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, int N, int H,
                                      int W, int C, int Ho, int Wo, int pad_y, int pad_x) {
  pdl_prologue();
  const long long total = (long long)N * H * W * C;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    long long r = e / C;
    const int ix = (int)(r % W); r /= W;
    const int iy = (int)(r % H);
    const int n = (int)(r / H);
    const float* xn = x + (size_t)n * H * W * C + c;
    float acc = 0.f;
    const int oy_lo = max(0, (iy + pad_y - 1) / 2), oy_hi = min(Ho - 1, (iy + pad_y) / 2);
    const int ox_lo = max(0, (ix + pad_x - 1) / 2), ox_hi = min(Wo - 1, (ix + pad_x) / 2);
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      const int y0 = 2 * oy - pad_y;
      if (iy < y0 || iy > y0 + 2) continue;
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        const int x0 = 2 * ox - pad_x;
        if (ix < x0 || ix > x0 + 2) continue;
        int by = -1, bx = -1;
        float best = 0.f;
        for (int dh = 0; dh < 3; ++dh) {
          const int hy = y0 + dh;
          if (hy < 0 || hy >= H) continue;
          for (int dw = 0; dw < 3; ++dw) {
            const int wx = x0 + dw;
            if (wx < 0 || wx >= W) continue;
            const float v = xn[((size_t)hy * W + wx) * C];
            if (by < 0 || v > best) { best = v; by = hy; bx = wx; }
          }
        }
        if (by == iy && bx == ix) acc += dy[(((size_t)n * Ho + oy) * Wo + ox) * C + c];
      }
    }
    dx[e] = acc;
  }
}

struct Shape {
  int Ho, Wo;
};

inline Shape out_shape(int H, int W, int kh, int kw, int stride, int pad_lo, int pad_hi) {
  return {(H + pad_lo + pad_hi - kh) / stride + 1, (W + pad_lo + pad_hi - kw) / stride + 1};
}

inline bool conv_ok(int N, int H, int W, int Ci, int Cw, int Co, int kh, int kw, int stride, int pad_lo, int pad_hi) {
  if (N < 1 || H < 1 || W < 1 || Ci < 4 || Ci % 4 || Cw < 1 || Cw > Ci || Co < 4 || Co % 4 || kh < 1 || kw < 1 || stride < 1 ||
      pad_lo < 0 || pad_hi < 0 || pad_lo >= kh || pad_lo >= kw)
    return false;
  const Shape o = out_shape(H, W, kh, kw, stride, pad_lo, pad_hi);
  return o.Ho >= 1 && o.Wo >= 1;
}

// split count of a wgrad (a function of the shape only, so the summation order is fixed)
inline int wgrad_splits(int N, int Ho, int Wo, int Ci, int Co, int kh, int kw) {
  const long long K = (long long)N * Ho * Wo;
  const int tiles = ceil_div(kh * kw * Ci, TM) * ceil_div(Co, TN);
  long long s = WGRAD_CTAS / tiles;
  s = std::min(s, K / (4 * TK));
  return (int)std::max(1LL, s);
}

}  // namespace rconv
}  // namespace serl

using namespace serl;
using namespace serl::rconv;

template <int kMode>
static int launch_conv(int tc, dim3 grid, cudaStream_t st, const Args& a, const char* name) {
  if (tc) {
    static bool attr_done = false;
    if (!attr_done) {
      if (cudaFuncSetAttribute(rconv_kernel<kMode, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TC) != cudaSuccess) {
        set_last_error("%s: cannot reserve %d bytes of shared memory", name, SMEM_TC);
        return SERL_ERR_CUDA;
      }
      attr_done = true;
    }
    launch_k(rconv_kernel<kMode, true>, grid, 256, SMEM_TC, st, a);
  } else {
    static bool attr_done = false;
    if (!attr_done) {
      if (cudaFuncSetAttribute(rconv_kernel<kMode, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CC) != cudaSuccess) {
        set_last_error("%s: cannot reserve %d bytes of shared memory", name, SMEM_CC);
        return SERL_ERR_CUDA;
      }
      attr_done = true;
    }
    launch_k(rconv_kernel<kMode, false>, grid, 256, SMEM_CC, st, a);
  }
  return check_launch(name);
}

static Args make_args(int N, int H, int W, int Ci, int Cw, int Co, int kh, int kw, int stride, int pad_lo, int pad_hi) {
  Args a{};
  a.N = N; a.H = H; a.W = W; a.Ci = Ci; a.Cw = Cw; a.Co = Co; a.kh = kh; a.kw = kw; a.stride = stride; a.pad = pad_lo;
  const Shape o = out_shape(H, W, kh, kw, stride, pad_lo, pad_hi);
  a.Ho = o.Ho; a.Wo = o.Wo;
  return a;
}

extern "C" int serl_rconv_fwd(const float* x, const float* w, float* y, int N, int H, int W, int Ci, int Cw, int Co, int kh, int kw,
                              int stride, int pad_lo, int pad_hi, int tc, void* stream) {
  if (!conv_ok(N, H, W, Ci, Cw, Co, kh, kw, stride, pad_lo, pad_hi)) {
    set_last_error("serl_rconv_fwd: unsupported shape (N=%d H=%d W=%d Ci=%d Cw=%d Co=%d k=%dx%d s=%d pad=%d,%d)", N, H, W, Ci, Cw, Co,
                   kh, kw, stride, pad_lo, pad_hi);
    return SERL_ERR_UNSUPPORTED;
  }
  Args a = make_args(N, H, W, Ci, Cw, Co, kh, kw, stride, pad_lo, pad_hi);
  a.x = x; a.w = w; a.out = y;
  const long long M = (long long)N * a.Ho * a.Wo;
  return launch_conv<FWD>(tc, dim3((unsigned)ceil_div_ll(M, TM), ceil_div(Co, TN), 1), static_cast<cudaStream_t>(stream), a,
                          "rconv_kernel<fwd>");
}

extern "C" int serl_rconv_dgrad(const float* dz, const float* w, float* dx, int N, int H, int W, int Ci, int Co, int kh, int kw, int stride,
                                int pad_lo, int pad_hi, int accumulate, int tc, void* stream) {
  if (!conv_ok(N, H, W, Ci, Ci, Co, kh, kw, stride, pad_lo, pad_hi) || H % stride || W % stride) {
    set_last_error("serl_rconv_dgrad: unsupported shape (N=%d H=%d W=%d Ci=%d Co=%d k=%dx%d s=%d pad=%d,%d)", N, H, W, Ci, Co, kh, kw,
                   stride, pad_lo, pad_hi);
    return SERL_ERR_UNSUPPORTED;
  }
  Args a = make_args(N, H, W, Ci, Ci, Co, kh, kw, stride, pad_lo, pad_hi);
  a.dz = dz; a.w = w; a.out = dx; a.accumulate = accumulate;
  const long long M = (long long)N * (H / stride) * (W / stride);
  return launch_conv<DGRAD>(tc, dim3((unsigned)ceil_div_ll(M, TM), ceil_div(Ci, TN), stride * stride), static_cast<cudaStream_t>(stream),
                            a, "rconv_kernel<dgrad>");
}

extern "C" int serl_rconv_wgrad_workspace(int N, int H, int W, int Ci, int Co, int kh, int kw, int stride, int pad_lo, int pad_hi,
                                          long long* floats) {
  if (!floats || !conv_ok(N, H, W, Ci, Ci, Co, kh, kw, stride, pad_lo, pad_hi)) {
    set_last_error("serl_rconv_wgrad_workspace: unsupported shape");
    return SERL_ERR_UNSUPPORTED;
  }
  const Shape o = out_shape(H, W, kh, kw, stride, pad_lo, pad_hi);
  const long long K = (long long)N * o.Ho * o.Wo;
  const int splits = wgrad_splits(N, o.Ho, o.Wo, Ci, Co, kh, kw);
  const long long ks = ceil_div_ll(ceil_div_ll(K, splits), TK) * TK;
  *floats = ceil_div_ll(K, ks) * kh * kw * Ci * Co;
  return SERL_OK;
}

extern "C" int serl_rconv_wgrad(const float* x, const float* dz, float* dw, float* workspace, long long workspace_bytes, int N, int H, int W,
                                int Ci, int Cw, int Co, int kh, int kw, int stride, int pad_lo, int pad_hi, int tc, void* stream) {
  if (!conv_ok(N, H, W, Ci, Cw, Co, kh, kw, stride, pad_lo, pad_hi)) {
    set_last_error("serl_rconv_wgrad: unsupported shape (N=%d H=%d W=%d Ci=%d Cw=%d Co=%d k=%dx%d s=%d pad=%d,%d)", N, H, W, Ci, Cw, Co,
                   kh, kw, stride, pad_lo, pad_hi);
    return SERL_ERR_UNSUPPORTED;
  }
  Args a = make_args(N, H, W, Ci, Cw, Co, kh, kw, stride, pad_lo, pad_hi);
  a.x = x; a.dz = dz; a.out = workspace;
  const long long K = (long long)N * a.Ho * a.Wo;
  const int splits = wgrad_splits(N, a.Ho, a.Wo, Ci, Co, kh, kw);
  a.k_split = (int)(ceil_div_ll(ceil_div_ll(K, splits), TK) * TK);
  const int z = (int)ceil_div_ll(K, a.k_split);
  const int M = kh * kw * Ci;
  if ((long long)z * M * Co * 4 > workspace_bytes) {
    set_last_error("serl_rconv_wgrad: workspace of %lld bytes < %lld", workspace_bytes, (long long)z * M * Co * 4);
    return SERL_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = launch_conv<WGRAD>(tc, dim3(ceil_div(M, TM), ceil_div(Co, TN), z), st, a, "rconv_kernel<wgrad>")) return rc;
  launch_k(rn_wgrad_reduce_kernel, ceil_div(kh * kw * Cw * Co, 256), 256, 0, st, workspace, dw, kh * kw, Ci, Cw, Co, z);
  return check_launch("rn_wgrad_reduce_kernel");
}

extern "C" int serl_rconv_stem_prep(const uint8_t* x, float* y, int N, int H, int W, void* stream) {
  const long long pixels = (long long)N * H * W;
  int blocks = (int)std::min(ceil_div_ll(pixels, 256), 132LL * 16);
  launch_k(rn_stem_prep_kernel, std::max(blocks, 1), 256, 0, static_cast<cudaStream_t>(stream), x, y, pixels);
  return check_launch("rn_stem_prep_kernel");
}

extern "C" int serl_rconv_stem_prep_stacked(const uint8_t* x, float* y, int N, int H, int W, int Ci, void* stream) {
  if (N < 1 || H < 1 || W < 1 || Ci < 1) {
    set_last_error("serl_rconv_stem_prep_stacked: invalid shape (N=%d H=%d W=%d Ci=%d)", N, H, W, Ci);
    return SERL_ERR_INVALID;
  }
  const long long elems = (long long)N * H * W * ((Ci + 3) / 4 * 4);
  int blocks = (int)std::min(ceil_div_ll(elems, 256), 132LL * 16);
  launch_k(rn_stem_prep_stacked_kernel, std::max(blocks, 1), 256, 0, static_cast<cudaStream_t>(stream), x, y, (long long)N * H * W, Ci,
           (Ci + 3) / 4 * 4);
  return check_launch("rn_stem_prep_stacked_kernel");
}

extern "C" int serl_groupnorm_bwd_nhwc(const float* x, const float* y, const float* dy, const float* scale, float* dx, float* dres,
                                       float* dscale, float* dbias, float* workspace, int N, int HW, int C, int groups, float eps, int relu,
                                       void* stream) {
  if (N < 1 || groups < 1 || C % groups || (C / groups) % 4 || C / groups > 512 || (relu && !y)) {
    set_last_error("serl_groupnorm_bwd_nhwc: unsupported arguments (N=%d C=%d G=%d relu=%d)", N, C, groups, relu);
    return SERL_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* partials = workspace;                                   // (2N, C), then the (N, G, 2) statistics
  float* stats = workspace + (size_t)2 * N * C;
  launch_k(rn_groupnorm_stats_kernel, dim3(groups, N), 512, 0, st, x, stats, HW, C, groups, eps);
  if (int rc = check_launch("rn_groupnorm_stats_kernel")) return rc;
  launch_k(rn_groupnorm_bwd_kernel, dim3(groups, N), 512, 0, st, x, y, dy, scale, (const float*)stats, dx, dres, partials, N, HW, C, groups,
           relu);
  if (int rc = check_launch("rn_groupnorm_bwd_kernel")) return rc;
  launch_k(rn_groupnorm_param_reduce_kernel, ceil_div(2 * C, 256), 256, 0, st, (const float*)partials, dscale, dbias, N, C);
  return check_launch("rn_groupnorm_param_reduce_kernel");
}

extern "C" int serl_maxpool3x3s2_bwd_nhwc(const float* x, const float* dy, float* dx, int N, int H, int W, int C, void* stream) {
  if (N < 1 || H < 1 || W < 1 || C < 1) {
    set_last_error("serl_maxpool3x3s2_bwd_nhwc: invalid shape");
    return SERL_ERR_INVALID;
  }
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;                 // XLA SAME per axis, as serl_maxpool3x3s2_nhwc_f32
  const int pad_y = std::max((Ho - 1) * 2 + 3 - H, 0) / 2, pad_x = std::max((Wo - 1) * 2 + 3 - W, 0) / 2;
  const long long total = (long long)N * H * W * C;
  const int blocks = (int)std::min(ceil_div_ll(total, 256), 132LL * 16);
  launch_k(rn_maxpool_bwd_kernel, blocks, 256, 0, static_cast<cudaStream_t>(stream), x, dy, dx, N, H, W, C, Ho, Wo, pad_y, pad_x);
  return check_launch("rn_maxpool_bwd_kernel");
}
