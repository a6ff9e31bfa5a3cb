// DrQ's trainable "small" pixel encoder (reference vision/small_encoders.py:9-55 as agents/continuous/drq.py:137-152 builds
// it): four 3x3 / stride-2 VALID convolutions with bias and ReLU on x = uint8 / 255, then the mean over the last map.
//
// Forward, input gradient (dgrad) and weight + bias gradient (wgrad) are one CUDA-core implicit GEMM (fp32 operands, fp32
// accumulation: the same arithmetic in every build) that differs only in how the A / B operands are gathered and in the
// epilogue:
//   fwd    C[(n,oy,ox), co]   = sum_{(ky,kx,ci)} x[n, 2oy+ky, 2ox+kx, ci] W[ky,kx,ci,co]        -> relu(C + b)
//   dgrad  C[(n,iy,ix), ci]   = sum_{(ky,kx,co)} dz[n, (iy-ky)/2, (ix-kx)/2, co] W[ky,kx,ci,co]  -> C * (x > 0)
//          (terms whose (iy-ky) or (ix-kx) is odd or out of range are zero)
//   wgrad  C[(ky,kx,ci), co]  = sum_{(n,oy,ox)} x[n, 2oy+ky, 2ox+kx, ci] dz[n,oy,ox,co], plus one extra row of ones that
//          gives the bias gradient; split-K partials, reduced in a fixed order by a second kernel.
// dz is the gradient of the pre-activation; dgrad's epilogue applies the previous layer's ReLU mask (its output x > 0, which
// is jax's relu' = 0 at 0), so its result is the previous layer's dz.  No atomics anywhere: two runs are bitwise equal.
//
// Two implementations of the same three GEMMs, chosen per call (`tc`):
//   * sconv_gemm_kernel: CUDA-core FMAs, 64x64 tiles - the fp32 (1e-5 parity) build;
//   * sconv_tc_kernel: Hopper tensor cores (wgmma m64n64k8 tf32), 128x64 tiles, one warpgroup per 64 rows - the fp16 / bf16
//     builds.  Operands are gathered straight from global memory into K-major 128B-swizzled shared tiles, each fp32 value split
//     as hi = rna_tf32(x), lo = x - hi, and accumulated as lo*hi + hi*lo + hi*hi ("3xTF32", as gemm_tf32x3.cu): fp32-class
//     products at tensor-core rate.  The weights are read from the fp32 masters the optimizer writes, so there is no 16-bit
//     copy to repack inside the step, and the activations and gradients stay fp32.
#include "common.cuh"
#include "gemm_common.cuh"
#include "wgmma.cuh"
#include "serl_b200.h"

namespace serl {
namespace sconv {

constexpr int BM = 64, BN = 64, BK = 16;
enum Mode { FWD = 0, DGRAD = 1, WGRAD = 2 };

struct Args {
  const void* x;        // layer input (N,H,W,Ci): uint8 (layer 0, scaled by 1/255) or fp32
  const float* w;       // (3,3,Ci,Co)
  const float* bias;    // (Co,)              fwd
  const float* dz;      // (N,Ho,Wo,Co)       dgrad, wgrad
  float* out;           // fwd (N,Ho,Wo,Co) | dgrad (N,H,W,Ci) | wgrad partials (splits, 9Ci+1, Co)
  int N, H, W, Ci, Ho, Wo, Co;
  int k_split;          // wgrad: K range of one split (multiple of BK)
};

template <bool kU8>
__device__ __forceinline__ float load_x(const Args& a, size_t off) {
  if (kU8) return (float)static_cast<const uint8_t*>(a.x)[off] / 255.0f;
  return static_cast<const float*>(a.x)[off];
}

template <int kMode, bool kU8>
__global__ void __launch_bounds__(256) sconv_gemm_kernel(const Args a) {
  pdl_prologue();
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const int HoWo = a.Ho * a.Wo;
  const int M = kMode == FWD ? a.N * HoWo : kMode == DGRAD ? a.N * a.H * a.W : 9 * a.Ci + 1;
  const int Nc = kMode == DGRAD ? a.Ci : a.Co;
  const int Kfull = kMode == FWD ? 9 * a.Ci : kMode == DGRAD ? 9 * a.Co : a.N * HoWo;
  const int kbeg = kMode == WGRAD ? blockIdx.z * a.k_split : 0;
  const int kend = kMode == WGRAD ? min(Kfull, kbeg + a.k_split) : Kfull;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int tx = tid & 15, ty = tid >> 4;
  const int nk = (kend - kbeg + BK - 1) / BK;

  // A loads: row am (fixed per thread), k = k0 + ak + e
  const int am = tid & 63, ak = (tid >> 6) * 4;
  const int gm = m0 + am;
  const bool mvalid = gm < M;
  // per-row decode
  size_t xbase = 0;                 // fwd: x offset of the window's top-left tap
  int rn = 0, ry = 0, rx = 0;       // dgrad: (n, iy, ix)
  int wtap_off = 0, wci = 0;        // wgrad: tap offset (ky*W+kx)*Ci + ci within an image, ci
  if (mvalid) {
    if (kMode == FWD) {
      const int n = gm / HoWo, r = gm - n * HoWo, oy = r / a.Wo, ox = r - oy * a.Wo;
      xbase = (((size_t)n * a.H + 2 * oy) * a.W + 2 * ox) * a.Ci;
    } else if (kMode == DGRAD) {
      rn = gm / (a.H * a.W); const int r = gm - rn * a.H * a.W; ry = r / a.W; rx = r - ry * a.W;
    } else if (gm < 9 * a.Ci) {
      const int tap = gm / a.Ci; wci = gm - tap * a.Ci;
      wtap_off = ((tap / 3) * a.W + tap % 3) * a.Ci + wci;
    }
  }
  // B loads: row bk, columns bn + e
  const int bk = tid >> 4, bn = (tid & 15) * 4;

  float ra[4], rb[4];
  auto gload = [&](int kt) {
    const int k0 = kbeg + kt * BK;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = k0 + ak + e;
      float v = 0.f;
      if (mvalid && k < kend) {
        if (kMode == FWD) {
          const int tap = k / a.Ci, ci = k - tap * a.Ci;
          v = load_x<kU8>(a, xbase + ((size_t)(tap / 3) * a.W + tap % 3) * a.Ci + ci);
        } else if (kMode == DGRAD) {
          const int tap = k / a.Co, co = k - tap * a.Co;
          const int dy = ry - tap / 3, dx = rx - tap % 3;
          if (dy >= 0 && dx >= 0 && !(dy & 1) && !(dx & 1) && (dy >> 1) < a.Ho && (dx >> 1) < a.Wo)
            v = a.dz[(((size_t)rn * a.Ho + (dy >> 1)) * a.Wo + (dx >> 1)) * a.Co + co];
        } else {
          if (gm == 9 * a.Ci) {
            v = 1.f;
          } else {
            const int n = k / HoWo, r = k - n * HoWo, oy = r / a.Wo, ox = r - oy * a.Wo;
            v = load_x<kU8>(a, (((size_t)n * a.H + 2 * oy) * a.W + 2 * ox) * a.Ci + wtap_off);
          }
        }
      }
      ra[e] = v;
    }
    const int kb = k0 + bk;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int n = n0 + bn + e;
      float v = 0.f;
      if (kb < kend && n < Nc) {
        if (kMode == FWD) v = a.w[(size_t)kb * a.Co + n];
        else if (kMode == DGRAD) { const int tap = kb / a.Co, co = kb - tap * a.Co; v = a.w[((size_t)tap * a.Ci + n) * a.Co + co]; }
        else v = a.dz[(size_t)kb * a.Co + n];
      }
      rb[e] = v;
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int e = 0; e < 4; ++e) As[buf][ak + e][am] = ra[e];
    *reinterpret_cast<float4*>(&Bs[buf][bk][bn]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  if (nk > 0) { gload(0); sstore(0); }
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 av = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      float4 bv = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    if (kt + 1 < nk) sstore(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= Nc) continue;
      if (kMode == FWD) {
        a.out[(size_t)m * Nc + n] = fmaxf(acc[i][j] + a.bias[n], 0.f);
      } else if (kMode == DGRAD) {
        const size_t o = (size_t)m * Nc + n;
        a.out[o] = static_cast<const float*>(a.x)[o] > 0.f ? acc[i][j] : 0.f;
      } else {
        a.out[((size_t)blockIdx.z * M + m) * Nc + n] = acc[i][j];
      }
    }
  }
}

// A(m, k) and B(k, n) of the three GEMMs (see the header comment), zero outside [0, M) x [kbeg, kend) / [kbeg, kend) x [0, Nc).
template <int kMode, bool kU8>
__device__ __forceinline__ float tc_load_a(const Args& a, int m, int k, int M, int kend) {
  if (m >= M || k >= kend) return 0.f;
  const int HoWo = a.Ho * a.Wo;
  if (kMode == FWD) {
    const int n = m / HoWo, r = m - n * HoWo, oy = r / a.Wo, ox = r - oy * a.Wo;
    const int tap = k / a.Ci, ci = k - tap * a.Ci;
    return load_x<kU8>(a, (((size_t)n * a.H + 2 * oy + tap / 3) * a.W + 2 * ox + tap % 3) * a.Ci + ci);
  } else if (kMode == DGRAD) {
    const int HW = a.H * a.W, n = m / HW, r = m - n * HW, iy = r / a.W, ix = r - iy * a.W;
    const int tap = k / a.Co, co = k - tap * a.Co;
    const int dy = iy - tap / 3, dx = ix - tap % 3;
    if (dy < 0 || dx < 0 || (dy & 1) || (dx & 1) || (dy >> 1) >= a.Ho || (dx >> 1) >= a.Wo) return 0.f;
    return a.dz[(((size_t)n * a.Ho + (dy >> 1)) * a.Wo + (dx >> 1)) * a.Co + co];
  } else {
    if (m == 9 * a.Ci) return 1.f;
    const int tap = m / a.Ci, ci = m - tap * a.Ci;
    const int n = k / HoWo, r = k - n * HoWo, oy = r / a.Wo, ox = r - oy * a.Wo;
    return load_x<kU8>(a, (((size_t)n * a.H + 2 * oy + tap / 3) * a.W + 2 * ox + tap % 3) * a.Ci + ci);
  }
}

template <int kMode>
__device__ __forceinline__ float tc_load_b(const Args& a, int k, int n, int Nc, int kend) {
  if (n >= Nc || k >= kend) return 0.f;
  if (kMode == FWD) return a.w[(size_t)k * a.Co + n];
  if (kMode == DGRAD) { const int tap = k / a.Co, co = k - tap * a.Co; return a.w[((size_t)tap * a.Ci + n) * a.Co + co]; }
  return a.dz[(size_t)k * a.Co + n];
}

constexpr int TC_M = 128, TC_N = 64, TC_K = 32;
constexpr int TC_A = TC_M * 128, TC_B = TC_N * 128;            // one K-major 128B-swizzled tile (32 fp32 per row)
constexpr int TC_SMEM = 2 * TC_A + 2 * TC_B + 1024;             // hi + lo of both operands, + alignment

// element (r, k) of a K-major 128B-swizzled tile (gemm_common.cuh::t_convert's layout)
__device__ __forceinline__ void tc_put(uint8_t* hi, uint8_t* lo, int r, int k, float v) {
  float h, l;
  t_split(v, h, l);
  const int off = r * 128 + ((((k >> 2) ^ (r & 7))) << 4) + (k & 3) * 4;
  *reinterpret_cast<float*>(hi + off) = h;
  *reinterpret_cast<float*>(lo + off) = l;
}

template <int kMode, bool kU8>
__global__ void __launch_bounds__(256) sconv_tc_kernel(const Args a) {
  pdl_prologue();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *sAh = smem, *sAl = smem + TC_A, *sBh = smem + 2 * TC_A, *sBl = smem + 2 * TC_A + TC_B;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int HoWo = a.Ho * a.Wo;
  const int M = kMode == FWD ? a.N * HoWo : kMode == DGRAD ? a.N * a.H * a.W : 9 * a.Ci + 1;
  const int Nc = kMode == DGRAD ? a.Ci : a.Co;
  const int Kfull = kMode == FWD ? 9 * a.Ci : kMode == DGRAD ? 9 * a.Co : a.N * HoWo;
  const int kbeg = kMode == WGRAD ? blockIdx.z * a.k_split : 0;
  const int kend = kMode == WGRAD ? min(Kfull, kbeg + a.k_split) : Kfull;
  const int m0 = blockIdx.x * TC_M, n0 = blockIdx.y * TC_N;
  constexpr int RA = TC_M * TC_K / 256;                // A elements per thread and k-block
  // fwd / dgrad: thread t gathers column k = t % 32 of rows t / 32 + 8 i; the rows' decode is done once here
  int rbase[RA], ryx[RA];
  if (kMode != WGRAD) {
#pragma unroll
    for (int i = 0; i < RA; ++i) {
      const int m = m0 + (tid >> 5) + 8 * i;
      rbase[i] = -1; ryx[i] = 0;
      if (m < M) {
        if (kMode == FWD) {
          const int n = m / HoWo, r = m - n * HoWo, oy = r / a.Wo, ox = r - oy * a.Wo;
          rbase[i] = ((n * a.H + 2 * oy) * a.W + 2 * ox) * a.Ci;
        } else {
          const int HW = a.H * a.W, n = m / HW, r = m - n * HW, iy = r / a.W, ix = r - iy * a.W;
          rbase[i] = n * HoWo; ryx[i] = (iy << 16) | ix;
        }
      }
    }
  }
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  for (int k0 = kbeg; k0 < kend; k0 += TC_K) {
    __syncthreads();                                   // every warpgroup has retired the previous k-block's MMAs
    // consecutive threads take the operand's contiguous index: k for fwd / dgrad A (channels), m for wgrad A (channels)
    if (kMode == WGRAD) {
#pragma unroll 4
      for (int i = 0; i < RA; ++i) {
        const int it = tid + 256 * i, r = it & 127, k = it >> 7;
        tc_put(sAh, sAl, r, k, tc_load_a<kMode, kU8>(a, m0 + r, k0 + k, M, kend));
      }
    } else {
      const int kk = tid & 31, k = k0 + kk;
      const int C = kMode == FWD ? a.Ci : a.Co;
      const int tap = k / C, c = k - tap * C, ky = tap / 3, kx = tap - 3 * ky;
      const int toff = (ky * a.W + kx) * a.Ci + c;     // fwd: offset of (ky, kx, ci) from the window's top-left
#pragma unroll
      for (int i = 0; i < RA; ++i) {
        float v = 0.f;
        if (rbase[i] >= 0 && k < kend) {
          if (kMode == FWD) {
            v = load_x<kU8>(a, (size_t)rbase[i] + toff);
          } else {
            const int dy = (ryx[i] >> 16) - ky, dx = (ryx[i] & 0xffff) - kx;
            if (dy >= 0 && dx >= 0 && !(dy & 1) && !(dx & 1) && (dy >> 1) < a.Ho && (dx >> 1) < a.Wo)
              v = a.dz[((size_t)rbase[i] + (dy >> 1) * a.Wo + (dx >> 1)) * a.Co + c];
          }
        }
        tc_put(sAh, sAl, (tid >> 5) + 8 * i, kk, v);
      }
    }
#pragma unroll 4
    for (int i = 0; i < TC_N * TC_K / 256; ++i) {
      const int it = tid + 256 * i;
      const int n = kMode == DGRAD ? (it >> 5) : (it & 63), k = kMode == DGRAD ? (it & 31) : (it >> 6);
      tc_put(sBh, sBl, n, k, tc_load_b<kMode>(a, k0 + k, n0 + n, Nc, kend));
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> tensor-core reads
    __syncthreads();
    const uint64_t ah = wg_desc(t_smem(sAh) + wg * 8192), al = wg_desc(t_smem(sAl) + wg * 8192);
    const uint64_t bh = wg_desc(t_smem(sBh)), bl = wg_desc(t_smem(sBl));
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, al + 2 * k, bh + 2 * k, 1u);
#pragma unroll
    for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, ah + 2 * k, bl + 2 * k, 1u);
#pragma unroll
    for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, ah + 2 * k, bh + 2 * k, 1u);
    wg_commit();
    wg_wait<0>();
  }
  // epilogue from the accumulator fragments (wgmma.cuh): rows 16 (warp % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + 8 * j + 2 * (lane & 3) + e;
        if (n >= Nc) continue;
        const float v = acc[4 * j + 2 * h + e];
        if (kMode == FWD) {
          a.out[(size_t)m * Nc + n] = fmaxf(v + a.bias[n], 0.f);
        } else if (kMode == DGRAD) {
          const size_t o = (size_t)m * Nc + n;
          a.out[o] = static_cast<const float*>(a.x)[o] > 0.f ? v : 0.f;
        } else {
          a.out[((size_t)blockIdx.z * M + m) * Nc + n] = v;
        }
      }
    }
  }
}

// dw[m][co] (m < 9Ci) and db[co] (row 9Ci) = sum over the splits, in split order.
__global__ void __launch_bounds__(256) sconv_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw,
                                                                 float* __restrict__ db, int M, int Co, int splits) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * Co) return;
  float s = 0.f;
  for (int z = 0; z < splits; ++z) s += part[(size_t)z * M * Co + i];
  const int m = i / Co;
  if (m < M - 1) dw[i] = s;
  else db[i - m * Co] = s;
}

// out[n][c] = mean_p y[n][p][c]
__global__ void __launch_bounds__(256) sconv_mean_fwd_kernel(const float* __restrict__ y, float* __restrict__ out, int N, int P, int C) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  const float* p = y + (size_t)n * P * C + c;
  float s = 0.f;
  for (int k = 0; k < P; ++k) s += p[(size_t)k * C];
  out[i] = s / (float)P;
}

// dz[n][p][c] = dout[n][c] / P where y[n][p][c] > 0, else 0
__global__ void __launch_bounds__(256) sconv_mean_bwd_kernel(const float* __restrict__ dout, int ld, const float* __restrict__ y,
                                                             float* __restrict__ dz, int N, int P, int C) {
  pdl_prologue();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)N * P * C) return;
  const int c = (int)(i % C);
  const size_t n = i / ((size_t)P * C);
  dz[i] = y[i] > 0.f ? dout[n * ld + c] / (float)P : 0.f;
}

inline bool shape_ok(int N, int H, int W, int Ci, int Co) {
  return N >= 1 && H >= 3 && W >= 3 && Ci >= 1 && Co >= 4 && Co % 4 == 0;
}

}  // namespace sconv
}  // namespace serl

using namespace serl;
using namespace serl::sconv;

// the CUDA-core kernel (tc == 0) or the tensor-core one on a (rows / tile) x (Nc / 64) x z grid
template <int kMode, bool kU8>
static void launch_gemm(int tc, long long M, int Nc, int z, cudaStream_t st, const Args& a) {
  if (tc) {
    static bool attr_done = false;
    if (!attr_done) {
      cudaFuncSetAttribute(sconv_tc_kernel<kMode, kU8>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
      attr_done = true;
    }
    launch_k(sconv_tc_kernel<kMode, kU8>, dim3((unsigned)ceil_div_ll(M, TC_M), ceil_div(Nc, TC_N), z), 256, TC_SMEM, st, a);
  } else {
    launch_k(sconv_gemm_kernel<kMode, kU8>, dim3((unsigned)ceil_div_ll(M, BM), ceil_div(Nc, BN), z), 256, 0, st, a);
  }
}

static Args make_args(const void* x, int N, int H, int W, int Ci, int Co) {
  Args a{};
  a.x = x; a.N = N; a.H = H; a.W = W; a.Ci = Ci; a.Co = Co;
  a.Ho = (H - 3) / 2 + 1; a.Wo = (W - 3) / 2 + 1;
  return a;
}

extern "C" int serl_sconv_fwd(const void* x, int x_is_u8, const float* w, const float* bias, float* y, int N, int H, int W, int Ci,
                              int Co, int tc, void* stream) {
  if (!shape_ok(N, H, W, Ci, Co)) {
    set_last_error("serl_sconv_fwd: unsupported shape (N=%d H=%d W=%d Ci=%d Co=%d)", N, H, W, Ci, Co);
    return SERL_ERR_UNSUPPORTED;
  }
  Args a = make_args(x, N, H, W, Ci, Co);
  a.w = w; a.bias = bias; a.out = y;
  const long long M = (long long)N * a.Ho * a.Wo;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (x_is_u8) launch_gemm<FWD, true>(tc, M, Co, 1, st, a);
  else launch_gemm<FWD, false>(tc, M, Co, 1, st, a);
  return check_launch("sconv fwd");
}

extern "C" int serl_sconv_dgrad(const float* dz, const float* w, const float* x, float* dx, int N, int H, int W, int Ci, int Co,
                                int tc, void* stream) {
  if (!shape_ok(N, H, W, Ci, Co) || Ci % 4 != 0) {
    set_last_error("serl_sconv_dgrad: unsupported shape (N=%d H=%d W=%d Ci=%d Co=%d)", N, H, W, Ci, Co);
    return SERL_ERR_UNSUPPORTED;
  }
  Args a = make_args(x, N, H, W, Ci, Co);
  a.w = w; a.dz = dz; a.out = dx;
  const long long M = (long long)N * H * W;
  launch_gemm<DGRAD, false>(tc, M, Ci, 1, static_cast<cudaStream_t>(stream), a);
  return check_launch("sconv dgrad");
}

extern "C" int serl_sconv_wgrad(const void* x, int x_is_u8, const float* dz, float* dw, float* db, float* workspace,
                                long long workspace_bytes, int splits, int N, int H, int W, int Ci, int Co, int tc, void* stream) {
  if (!shape_ok(N, H, W, Ci, Co) || splits < 1) {
    set_last_error("serl_sconv_wgrad: unsupported shape (N=%d H=%d W=%d Ci=%d Co=%d splits=%d)", N, H, W, Ci, Co, splits);
    return SERL_ERR_UNSUPPORTED;
  }
  Args a = make_args(x, N, H, W, Ci, Co);
  a.dz = dz; a.out = workspace;
  const int M = 9 * Ci + 1, K = N * a.Ho * a.Wo;
  a.k_split = ceil_div(ceil_div(K, splits), BK) * BK;
  const int z = ceil_div(K, a.k_split);
  if ((long long)z * M * Co * 4 > workspace_bytes) {
    set_last_error("serl_sconv_wgrad: workspace of %lld bytes < %lld", workspace_bytes, (long long)z * M * Co * 4);
    return SERL_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (x_is_u8) launch_gemm<WGRAD, true>(tc, M, Co, z, st, a);
  else launch_gemm<WGRAD, false>(tc, M, Co, z, st, a);
  int rc = check_launch("sconv wgrad");
  if (rc) return rc;
  launch_k(sconv_wgrad_reduce_kernel, ceil_div(M * Co, 256), 256, 0, st, workspace, dw, db, M, Co, z);
  return check_launch("sconv_wgrad_reduce_kernel");
}

extern "C" int serl_sconv_mean_fwd(const float* y, float* out, int N, int P, int C, void* stream) {
  launch_k(sconv_mean_fwd_kernel, ceil_div(N * C, 256), 256, 0, static_cast<cudaStream_t>(stream), y, out, N, P, C);
  return check_launch("sconv_mean_fwd_kernel");
}

extern "C" int serl_sconv_mean_bwd(const float* dout, int ld, const float* y, float* dz, int N, int P, int C, void* stream) {
  const long long total = (long long)N * P * C;
  launch_k(sconv_mean_bwd_kernel, (unsigned)ceil_div_ll(total, 256), 256, 0, static_cast<cudaStream_t>(stream), dout, ld, y, dz, N, P, C);
  return check_launch("sconv_mean_bwd_kernel");
}
