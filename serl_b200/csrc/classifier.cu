// Binary reward classifier head (fp32): the layers BinaryClassifier adds on top of the encoder heads, and the loss of
// examples/*/train_reward_classifier.py.
//
// Reference (relative to serl_launcher/serl_launcher):
//   networks/reward_classifier.py:16-28   Dense(256) -> Dropout(0.1) -> LayerNorm(eps 1e-6, fast variance) -> relu -> Dense(1)
//   examples/async_cable_route_drq/train_reward_classifier.py:121-137
//                                         loss = mean(sigmoid_binary_cross_entropy(logits, labels)),
//                                         accuracy = mean((sigmoid(logits_eval) >= 0.5) == labels)
//   vision/resnet_v1.py:352               Dropout(0.1) of the image heads: where(mask, x / keep, 0); its backward is dropout_bwd
// Restated in oracle/classifier.py.
#include "common.cuh"
#include "serl_b200.h"

namespace serl {

constexpr int kHeadD = 256;

// ---- LayerNorm + relu + Dense(256 -> 1) forward: warp per row, lane owns columns lane + 32 j ----------------------------
__global__ void __launch_bounds__(256) ln_relu_head_fwd_kernel(const float* __restrict__ z, const uint8_t* __restrict__ mask, float keep,
                                                               const float* __restrict__ scale, const float* __restrict__ bias,
                                                               const float* __restrict__ w, const float* __restrict__ b,
                                                               float* __restrict__ h, float* __restrict__ xhat, float* __restrict__ rstd_out,
                                                               float* __restrict__ logit, int R, float eps) {
  pdl_prologue();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= R) return;
  float v[8];
  float s = 0.f, ss = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const size_t e = (size_t)row * kHeadD + lane + 32 * j;
    float x = z[e];
    if (mask) x = mask[e] ? x / keep : 0.f;
    v[j] = x; s += x; ss += x * x;
  }
  s = warp_sum(s); ss = warp_sum(ss);
  const float mean = s / (float)kHeadD;                            // same statistics as ln_tanh_fwd_kernel (heads.cu)
  const float var = fmaxf(ss / (float)kHeadD - mean * mean, 0.f);
  const float rstd = rsqrtf(var + eps);
  float dot = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = lane + 32 * j;
    const float xh = (v[j] - mean) * rstd;
    const float hv = fmaxf(xh * scale[d] + bias[d], 0.f);
    dot = fmaf(hv, w[d], dot);
    if (h) h[(size_t)row * kHeadD + d] = hv;
    if (xhat) xhat[(size_t)row * kHeadD + d] = xh;
  }
  dot = warp_sum(dot);
  if (lane == 0) {
    logit[row] = dot + b[0];
    if (rstd_out) rstd_out[row] = rstd;
  }
}

// ---- backward: dh = dlogit * w (the Dense(1) input gradient), relu, LayerNorm, dropout ---------------------------------
// dy = dh * 1[h > 0];  dzd = rstd * (dy*scale - mean(dy*scale) - xhat * mean(dy*scale*xhat));  dz = where(mask, dzd / keep, 0)
__global__ void __launch_bounds__(256) ln_relu_head_bwd_kernel(const float* __restrict__ dlogit, const float* __restrict__ w,
                                                               const float* __restrict__ h, const float* __restrict__ xhat,
                                                               const float* __restrict__ rstd, const float* __restrict__ scale,
                                                               const uint8_t* __restrict__ mask, float keep, float* __restrict__ dy_out,
                                                               float* __restrict__ dz, int R) {
  pdl_prologue();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= R) return;
  const float dl = dlogit[row];
  float dy[8], xh[8];
  float m1 = 0.f, m2 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = lane + 32 * j;
    const size_t e = (size_t)row * kHeadD + d;
    dy[j] = h[e] > 0.f ? dl * w[d] : 0.f;
    xh[j] = xhat[e];
    const float dxh = dy[j] * scale[d];
    m1 += dxh; m2 += dxh * xh[j];
    if (dy_out) dy_out[e] = dy[j];
  }
  m1 = warp_sum(m1) / (float)kHeadD; m2 = warp_sum(m2) / (float)kHeadD;
  const float rs = rstd[row];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = lane + 32 * j;
    const size_t e = (size_t)row * kHeadD + d;
    const float g = rs * (dy[j] * scale[d] - m1 - xh[j] * m2);
    dz[e] = mask ? (mask[e] ? g / keep : 0.f) : g;
  }
}

// ---- sigmoid binary cross-entropy + accuracy: one CTA, fixed-order reduction (deterministic) ---------------------------
constexpr int kBceThreads = 256;

__global__ void __launch_bounds__(kBceThreads) bce_logits_loss_kernel(const float* __restrict__ x_train, const float* __restrict__ x_eval,
                                                                      const float* __restrict__ labels, float grad_scale,
                                                                      float* __restrict__ dlogit, float* __restrict__ info, int B) {
  pdl_prologue();
  __shared__ float rl[kBceThreads], ra[kBceThreads];
  float sl = 0.f, sa = 0.f;
  const float inv = 1.f / (float)B;
  for (int i = threadIdx.x; i < B; i += kBceThreads) {
    const float x = x_train[i], y = labels[i];
    // optax.sigmoid_binary_cross_entropy in the overflow-free form: max(x,0) - x*y + log1p(exp(-|x|))
    sl += fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
    const float sg = 1.f / (1.f + expf(-x));
    dlogit[i] = (sg - y) * grad_scale * inv;
    // (sigmoid(logits_eval) >= 0.5) == labels, with sigmoid rounded to fp32 first: tiny negative logits give exactly 0.5
    const float se = 1.f / (1.f + expf(-x_eval[i]));
    sa += ((se >= 0.5f ? 1.f : 0.f) == y) ? 1.f : 0.f;
  }
  rl[threadIdx.x] = sl; ra[threadIdx.x] = sa;
  __syncthreads();
  for (int o = kBceThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) { rl[threadIdx.x] += rl[threadIdx.x + o]; ra[threadIdx.x] += ra[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { info[0] = rl[0] * inv; info[1] = ra[0] * inv; }
}

// ---- Dropout backward in place: dx = mask ? dx / keep : 0 ----------------------------------------------------------------
__global__ void dropout_bwd_kernel(float* __restrict__ dx, const uint8_t* __restrict__ mask, float keep, int n) {
  pdl_prologue();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dx[i] = mask[i] ? dx[i] / keep : 0.f;
}

}  // namespace serl

using namespace serl;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int serl_layernorm_relu_head_fwd(const float* z, const uint8_t* mask, float keep, const float* scale, const float* bias,
                                            const float* w, const float* b, float* h, float* xhat, float* rstd, float* logit,
                                            int R, int D, float eps, void* stream) {
  if (!z || !scale || !bias || !w || !b || !logit || R < 1 || D != kHeadD || (mask && !(keep > 0.f))) {
    set_last_error("serl_layernorm_relu_head_fwd: invalid arguments (D must be %d)", kHeadD); return SERL_ERR_INVALID;
  }
  launch_k(ln_relu_head_fwd_kernel, ceil_div(R, 8), 256, 0, ST(stream), z, mask, keep, scale, bias, w, b, h, xhat, rstd, logit, R, eps);
  return check_launch("ln_relu_head_fwd_kernel");
}

extern "C" int serl_layernorm_relu_head_bwd(const float* dlogit, const float* w, const float* h, const float* xhat, const float* rstd,
                                            const float* scale, const uint8_t* mask, float keep, float* dy, float* dz, int R, int D,
                                            void* stream) {
  if (!dlogit || !w || !h || !xhat || !rstd || !scale || !dz || R < 1 || D != kHeadD || (mask && !(keep > 0.f))) {
    set_last_error("serl_layernorm_relu_head_bwd: invalid arguments (D must be %d)", kHeadD); return SERL_ERR_INVALID;
  }
  launch_k(ln_relu_head_bwd_kernel, ceil_div(R, 8), 256, 0, ST(stream), dlogit, w, h, xhat, rstd, scale, mask, keep, dy, dz, R);
  return check_launch("ln_relu_head_bwd_kernel");
}

extern "C" int serl_bce_logits_loss(const float* logits_train, const float* logits_eval, const float* labels, float grad_scale,
                                    float* dlogit, float* info, int B, void* stream) {
  if (!logits_train || !logits_eval || !labels || !dlogit || !info || B < 1) { set_last_error("serl_bce_logits_loss: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(bce_logits_loss_kernel, 1, kBceThreads, 0, ST(stream), logits_train, logits_eval, labels, grad_scale, dlogit, info, B);
  return check_launch("bce_logits_loss_kernel");
}

extern "C" int serl_dropout_bwd_f32(float* dx, const uint8_t* mask, float keep, int n, void* stream) {
  if (!dx || !mask || n < 0 || !(keep > 0.f)) { set_last_error("serl_dropout_bwd_f32: invalid arguments"); return SERL_ERR_INVALID; }
  if (n == 0) return SERL_OK;
  int blocks = ceil_div(n, 256); if (blocks > 1184) blocks = 1184;
  launch_k(dropout_bwd_kernel, blocks, 256, 0, ST(stream), dx, mask, keep, n);
  return check_launch("dropout_bwd_kernel");
}
