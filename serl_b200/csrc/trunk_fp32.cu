// Frozen ResNet-10 trunk, fp32 build (CUDA-core implicit GEMM): the 1e-5 parity path.
// The 16-bit tensor-core (wgmma) build of the same layers lives in conv_tcgen05.cu.
//
// Replaces (reference, relative to serl_launcher/serl_launcher) vision/resnet_v1.py:217-286
// (ResNetEncoder.__call__ with pre_pooling=True) and :129-156 (ResNetBlock); XLA SAME-padding and
// GroupNorm statistics as restated in oracle/drq.py::trunk_forward.
#include "common.cuh"
#include "serl_b200.h"

namespace serl {

constexpr int BM = 64, BN = 64, BK = 16;

struct ConvArgs {
  const void* x;        // (N,Hi,Wi,Ci) fp32, or uint8 when kU8
  const float* w;       // (kh,kw,Ci,Co) HWIO
  float* y;             // (N,Ho,Wo,Co)
  int N, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad;   // pad = low padding (high side implied by bounds)
  float mean[3], stdv[3];      // kU8: (x/255 - mean) / std per channel (ci % 3), resnet_v1.py:222-224
};

// A operand element (m, k): m -> (n, ho, wo), k -> (r, s, ci).
template <bool kU8>
__device__ inline float conv_load_a(const ConvArgs& a, int n, int hb, int wb, int k, int K) {
  if (k >= K) return 0.f;
  int ci = k % a.Ci; int rs = k / a.Ci; int s = rs % a.kw; int r = rs / a.kw;
  int hi = hb + r, wi = wb + s;
  if (hi < 0 || hi >= a.Hi || wi < 0 || wi >= a.Wi) return 0.f;
  size_t off = (((size_t)n * a.Hi + hi) * a.Wi + wi) * a.Ci + ci;
  if (kU8) {
    float v = (float)static_cast<const uint8_t*>(a.x)[off];
    int c3 = ci % 3;
    return (v / 255.0f - a.mean[c3]) / a.stdv[c3];
  }
  return static_cast<const float*>(a.x)[off];
}

// kVec: Ci % 16 == 0 (a BK slice is one tap, contiguous channels) -> float4 gathers.
template <bool kVec, bool kU8>
__global__ void __launch_bounds__(256) conv_igemm_f32_kernel(const ConvArgs a) {
  pdl_prologue();
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN];
  const int tid = threadIdx.x;
  const int M = a.N * a.Ho * a.Wo, K = a.kh * a.kw * a.Ci;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int tx = tid & 15, ty = tid >> 4;
  const int nk = ceil_div(K, BK);

  // A-load mapping
  int am, ak;                                 // vec: row am, k-quad ak (4 floats); scalar: row am = tid & 63, ak = tid >> 6 (4 k's)
  if (kVec) { am = tid >> 2; ak = (tid & 3) * 4; } else { am = tid & 63; ak = (tid >> 6) * 4; }
  const int gm = m0 + am;
  int an = 0, hb = 0, wb = 0;
  const bool mvalid = gm < M;
  if (mvalid) {
    an = gm / (a.Ho * a.Wo); int rem = gm - an * a.Ho * a.Wo; int ho = rem / a.Wo; int wo = rem - ho * a.Wo;
    hb = ho * a.stride - a.pad; wb = wo * a.stride - a.pad;
  }
  // B-load mapping: row bk = tid >> 4, col quad (tid & 15) * 4
  const int bk = tid >> 4, bn = (tid & 15) * 4;

  float ra[4], rb[4];
  auto gload = [&](int kt) {
    const int k0 = kt * BK;
    if (kVec) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (mvalid) {
        int k = k0 + ak; int ci = k % a.Ci; int rs = k / a.Ci; int s = rs % a.kw; int r = rs / a.kw;
        int hi = hb + r, wi = wb + s;
        if (hi >= 0 && hi < a.Hi && wi >= 0 && wi < a.Wi)
          v = *reinterpret_cast<const float4*>(static_cast<const float*>(a.x) +
                                               (((size_t)an * a.Hi + hi) * a.Wi + wi) * a.Ci + ci);
      }
      ra[0] = v.x; ra[1] = v.y; ra[2] = v.z; ra[3] = v.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) ra[e] = mvalid ? conv_load_a<kU8>(a, an, hb, wb, k0 + ak + e, K) : 0.f;
    }
    const int kb = k0 + bk;
    if (kb < K) {
      float4 v = *reinterpret_cast<const float4*>(a.w + (size_t)kb * a.Co + n0 + bn);
      rb[0] = v.x; rb[1] = v.y; rb[2] = v.z; rb[3] = v.w;
    } else { rb[0] = rb[1] = rb[2] = rb[3] = 0.f; }
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

  gload(0); sstore(0); __syncthreads();
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
    if (m < M)
      *reinterpret_cast<float4*>(a.y + (size_t)m * a.Co + n0 + tx * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  }
}

// GroupNorm over (H, W, C/G) per sample with flax statistics (var = E[x^2] - E[x]^2, clipped at 0),
// optional residual add and ReLU.  In-place safe (y may alias x).  grid (G, N).
__global__ void __launch_bounds__(512) groupnorm_f32_kernel(const float* x, float* y,
                                                            const float* __restrict__ scale, const float* __restrict__ bias,
                                                            const float* residual, int HW, int C, int G, float eps, int relu) {
  pdl_prologue();
  __shared__ float red[64];
  const int g = blockIdx.x, n = blockIdx.y;
  const int Cg = C / G, q = Cg >> 2;                       // float4 per pixel in this group
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
  const float cnt = (float)HW * (float)Cg;
  const float mean = s / cnt;
  const float var = fmaxf(ss / cnt - mean * mean, 0.f);
  const float rstd = rsqrtf(var + eps);
  float* yb = y + (size_t)n * HW * C + g * Cg;
  const float* rbp = residual ? residual + (size_t)n * HW * C + g * Cg : nullptr;
  for (int e = threadIdx.x; e < total; e += blockDim.x) {
    int p = e / q, c4 = e - p * q;
    size_t off = (size_t)p * C + c4 * 4;
    float4 v = *reinterpret_cast<const float4*>(xb + off);
    float4 sc = *reinterpret_cast<const float4*>(scale + g * Cg + c4 * 4);
    float4 bi = *reinterpret_cast<const float4*>(bias + g * Cg + c4 * 4);
    float4 o;
    o.x = (v.x - mean) * rstd * sc.x + bi.x; o.y = (v.y - mean) * rstd * sc.y + bi.y;
    o.z = (v.z - mean) * rstd * sc.z + bi.z; o.w = (v.w - mean) * rstd * sc.w + bi.w;
    if (rbp) { float4 r = *reinterpret_cast<const float4*>(rbp + off); o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w; }
    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    *reinterpret_cast<float4*>(yb + off) = o;
  }
}

// max_pool 3x3 stride 2, XLA SAME per axis (pad low 0 / high 1 on even sizes, 1 / 1 on odd ones, -inf padding).
__global__ void maxpool3x3s2_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int Hi, int Wi, int C,
                                        int Ho, int Wo, int pad_y, int pad_x) {
  pdl_prologue();
  const int c4n = C >> 2;
  size_t total = (size_t)N * Ho * Wo * c4n;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    int c4 = (int)(e % c4n); size_t r = e / c4n;
    int wo = (int)(r % Wo); r /= Wo; int ho = (int)(r % Ho); int n = (int)(r / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int dh = 0; dh < 3; ++dh) {
      int hi = ho * 2 - pad_y + dh; if (hi < 0 || hi >= Hi) continue;
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        int wi = wo * 2 - pad_x + dw; if (wi < 0 || wi >= Wi) continue;
        float4 v = *reinterpret_cast<const float4*>(x + (((size_t)n * Hi + hi) * Wi + wi) * C + c4 * 4);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    *reinterpret_cast<float4*>(y + (((size_t)n * Ho + ho) * Wo + wo) * C + c4 * 4) = m;
  }
}

}  // namespace serl

using namespace serl;

extern "C" int serl_conv2d_nhwc_f32(const void* x, int x_is_u8, const float* w, float* y, int N, int Hi, int Wi, int Ci,
                                    int Co, int kh, int kw, int stride, int pad_lo, int pad_hi, void* stream) {
  if (N < 1 || Co % BN != 0 || Ci < 1 || stride < 1) {
    set_last_error("serl_conv2d_nhwc_f32: unsupported shape (N=%d Ci=%d Co=%d)", N, Ci, Co);
    return SERL_ERR_UNSUPPORTED;
  }
  ConvArgs a{};
  a.x = x; a.w = w; a.y = y; a.N = N; a.Hi = Hi; a.Wi = Wi; a.Ci = Ci; a.Co = Co; a.kh = kh; a.kw = kw;
  a.stride = stride; a.pad = pad_lo;
  a.Ho = (Hi + pad_lo + pad_hi - kh) / stride + 1;
  a.Wo = (Wi + pad_lo + pad_hi - kw) / stride + 1;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  long long M = (long long)N * a.Ho * a.Wo;
  dim3 grid((unsigned)ceil_div_ll(M, BM), Co / BN);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (x_is_u8) launch_k(conv_igemm_f32_kernel<false, true>, grid, 256, 0, st, a);
  else if (Ci % 16 == 0) launch_k(conv_igemm_f32_kernel<true, false>, grid, 256, 0, st, a);
  else launch_k(conv_igemm_f32_kernel<false, false>, grid, 256, 0, st, a);
  return check_launch("conv_igemm_f32_kernel");
}

extern "C" int serl_groupnorm_nhwc_f32(const float* x, float* y, const float* scale, const float* bias,
                                       const float* residual, int N, int HW, int C, int groups, float eps, int relu,
                                       void* stream) {
  if (C % groups != 0 || (C / groups) % 4 != 0) {
    set_last_error("serl_groupnorm_nhwc_f32: C/groups must be a multiple of 4 (C=%d G=%d)", C, groups);
    return SERL_ERR_UNSUPPORTED;
  }
  dim3 grid(groups, N);
  launch_k(groupnorm_f32_kernel, grid, 512, 0, static_cast<cudaStream_t>(stream), x, y, scale, bias, residual, HW, C, groups, eps, relu);
  return check_launch("groupnorm_f32_kernel");
}

extern "C" int serl_maxpool3x3s2_nhwc_f32(const float* x, float* y, int N, int Hi, int Wi, int C, void* stream) {
  if (C % 4 != 0) { set_last_error("serl_maxpool3x3s2_nhwc_f32: C %% 4 != 0"); return SERL_ERR_UNSUPPORTED; }
  int Ho = (Hi + 1) / 2, Wo = (Wi + 1) / 2;
  const int pad_y = std::max((Ho - 1) * 2 + 3 - Hi, 0) / 2, pad_x = std::max((Wo - 1) * 2 + 3 - Wi, 0) / 2;   // low pads
  size_t total = (size_t)N * Ho * Wo * (C / 4);
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
  launch_k(maxpool3x3s2_f32_kernel, blocks, 256, 0, static_cast<cudaStream_t>(stream), x, y, N, Hi, Wi, C, Ho, Wo, pad_y, pad_x);
  return check_launch("maxpool3x3s2_f32_kernel");
}
