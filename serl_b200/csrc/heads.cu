// Trainable encoder-head / MLP element kernels (fp32): SpatialLearnedEmbeddings, Dropout,
// LayerNorm+tanh (forward and backward), column reductions for bias / scale gradients.
//
// Reference (relative to serl_launcher/serl_launcher):
//   vision/resnet_v1.py:81-116   SpatialLearnedEmbeddings: out[b, c*F+f] = sum_{h,w} feat[b,h,w,c] K[h,w,c,f]
//   vision/resnet_v1.py:352      nn.Dropout(0.1): where(mask, x / keep, 0)
//   vision/resnet_v1.py:371-374, common/encoding.py:65-70, networks/mlp.py:26-31
//                                Dense -> LayerNorm(eps 1e-6, var = E[x^2]-E[x]^2) -> tanh
// Restated in oracle/drq.py (encode, mlp2, layer_norm).
#include "common.cuh"
#include "serl_b200.h"

namespace serl {

// ---- SpatialLearnedEmbeddings forward: thread per (n, c), F == 8 --------------------------------
__global__ void sle_fwd_kernel(const float* __restrict__ feat, const float* __restrict__ kern,
                               const uint8_t* __restrict__ keep_mask, float keep, float* __restrict__ out,
                               int N, int P, int C, int ld_out) {
  pdl_prologue();
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * C) return;
  const int n = e / C, c = e - n * C;
  float acc[8];
#pragma unroll
  for (int f = 0; f < 8; ++f) acc[f] = 0.f;
  for (int p = 0; p < P; ++p) {
    const float v = feat[((size_t)n * P + p) * C + c];
    const float4 k0 = *reinterpret_cast<const float4*>(kern + ((size_t)p * C + c) * 8);
    const float4 k1 = *reinterpret_cast<const float4*>(kern + ((size_t)p * C + c) * 8 + 4);
    acc[0] = fmaf(v, k0.x, acc[0]); acc[1] = fmaf(v, k0.y, acc[1]); acc[2] = fmaf(v, k0.z, acc[2]); acc[3] = fmaf(v, k0.w, acc[3]);
    acc[4] = fmaf(v, k1.x, acc[4]); acc[5] = fmaf(v, k1.y, acc[5]); acc[6] = fmaf(v, k1.z, acc[6]); acc[7] = fmaf(v, k1.w, acc[7]);
  }
  if (keep_mask) {
    const uint8_t* mk = keep_mask + (size_t)n * C * 8 + c * 8;
#pragma unroll
    for (int f = 0; f < 8; ++f) acc[f] = mk[f] ? acc[f] / keep : 0.f;
  }
  float* o = out + (size_t)n * ld_out + c * 8;
  *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// ---- SLE kernel gradient: partial[chunk][p][c][f] = sum_{n in chunk} feat[n,p,c] * dout[n, c*8+f] ----
__global__ void sle_bwd_partial_kernel(const float* __restrict__ feat, const float* __restrict__ dout,
                                       float* __restrict__ partial, int N, int P, int C, int ld_dout, int chunks) {
  pdl_prologue();
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= P * C) return;
  const int p = e / C, c = e - p * C;
  const int ch = blockIdx.y;
  const int per = ceil_div(N, chunks);
  const int n0 = ch * per, n1 = min(N, n0 + per);
  float acc[8];
#pragma unroll
  for (int f = 0; f < 8; ++f) acc[f] = 0.f;
  for (int n = n0; n < n1; ++n) {
    const float v = feat[((size_t)n * P + p) * C + c];
    const float4 d0 = *reinterpret_cast<const float4*>(dout + (size_t)n * ld_dout + c * 8);
    const float4 d1 = *reinterpret_cast<const float4*>(dout + (size_t)n * ld_dout + c * 8 + 4);
    acc[0] = fmaf(v, d0.x, acc[0]); acc[1] = fmaf(v, d0.y, acc[1]); acc[2] = fmaf(v, d0.z, acc[2]); acc[3] = fmaf(v, d0.w, acc[3]);
    acc[4] = fmaf(v, d1.x, acc[4]); acc[5] = fmaf(v, d1.y, acc[5]); acc[6] = fmaf(v, d1.z, acc[6]); acc[7] = fmaf(v, d1.w, acc[7]);
  }
  float* o = partial + ((size_t)ch * P * C + e) * 8;
  *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// ---- out[g][d] = sum_{r < rows} x[(g*rows + r) * ld + d] --------------------------------------------------------
// block = 32 columns x 8 row-slices (coalesced 128-byte row reads), fixed-order tree over the slices: deterministic.
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, float* __restrict__ out, int groups, int rows, int D,
                                                     long long ld, int accumulate) {
  pdl_prologue();
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int cblocks = ceil_div(D, 32);
  const int g = blockIdx.x / cblocks, d = (blockIdx.x - g * cblocks) * 32 + cx;
  float s = 0.f;
  if (d < D) {
    const float* p = x + (size_t)g * rows * ld + d;
    for (int r = sl; r < rows; r += 8) s += p[(size_t)r * ld];
  }
  red[sl][cx] = s;
  __syncthreads();
  if (sl == 0 && d < D) {
    float t = red[0][cx];
#pragma unroll
    for (int k = 1; k < 8; ++k) t += red[k][cx];
    const size_t e = (size_t)g * D + d;
    out[e] = accumulate ? out[e] + t : t;
  }
}

// ---- MLP activations (networks/mlp.py:31; flax.linen / jax.nn definitions) ------------------------
// act_fwd: the activation of pre-activation y.  act_grad: its derivative at y (jax's: relu' = 0 and leaky_relu' = 1 at 0).
template <int kAct>
__device__ __forceinline__ float act_fwd(float y) {
  if constexpr (kAct == SERL_ACT_TANH) return tanhf(y);
  if constexpr (kAct == SERL_ACT_RELU) return fmaxf(y, 0.f);
  if constexpr (kAct == SERL_ACT_SWISH) return y / (1.f + expf(-y));
  if constexpr (kAct == SERL_ACT_LEAKY_RELU) return y >= 0.f ? y : 0.01f * y;
  if constexpr (kAct == SERL_ACT_GELU) return y * (0.5f * (1.f + tanhf(0.7978845608028654f * (y + 0.044715f * (y * y * y)))));
  return 0.f;
}
template <int kAct>
__device__ __forceinline__ float act_grad(float y) {
  if constexpr (kAct == SERL_ACT_TANH) { const float t = tanhf(y); return 1.f - t * t; }
  if constexpr (kAct == SERL_ACT_RELU) return y > 0.f ? 1.f : 0.f;
  if constexpr (kAct == SERL_ACT_SWISH) { const float s = 1.f / (1.f + expf(-y)); return s * (1.f + y * (1.f - s)); }
  if constexpr (kAct == SERL_ACT_LEAKY_RELU) return y >= 0.f ? 1.f : 0.01f;
  if constexpr (kAct == SERL_ACT_GELU) {
    const float k = 0.7978845608028654f, th = tanhf(k * (y + 0.044715f * (y * y * y)));
    return 0.5f * (1.f + th) + 0.5f * y * (1.f - th * th) * k * (1.f + 3.f * 0.044715f * y * y);
  }
  return 0.f;
}

// ---- [LayerNorm +] activation forward: warp per row ------------------------------------------------
// rows R = groups * rows_per_group; scale/bias of row r at (r / rows_per_group) * group_stride.  Without LayerNorm the row is
// activated as it is (z is the pre-activation the backward reads).  <TANH, true> is the launcher architecture's layer.
// kDrop: nn.Dropout ahead of the LayerNorm / activation (networks/mlp.py:26-31), z' = mask ? z * inv_keep : 0 with the (R, D) keep
// mask.  Without LayerNorm z' is written to zw (the callers pass z itself: each element is read once, then written by the same
// lane), so the backward's `pre` is the activation's real input.  Row r reads mask row r % mask_rows: a critic ensemble's E*B
// rows (member-major) share one (B, D) mask with mask_rows = B.
template <int kAct, bool kLN, bool kDrop = false>
__global__ void ln_act_fwd_kernel(const float* __restrict__ z, int ld_z, const float* __restrict__ scale,
                                  const float* __restrict__ bias, int rows_per_group, int group_stride,
                                  float* __restrict__ out, int ld_out, float* __restrict__ xhat, float* __restrict__ rstd_out,
                                  int R, int D, float eps, const uint8_t* __restrict__ mask, float inv_keep, float* zw, int mask_rows) {
  pdl_prologue();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= R) return;
  const float* zr = z + (size_t)row * ld_z;
  auto in = [&](int d) {
    float v = zr[d];
    if constexpr (kDrop) v = mask[(size_t)(row % mask_rows) * D + d] ? v * inv_keep : 0.f;
    return v;
  };
  if constexpr (!kLN) {
    for (int d = lane; d < D; d += 32) {
      const float v = in(d);
      if constexpr (kDrop) zw[(size_t)row * ld_z + d] = v;
      out[(size_t)row * ld_out + d] = act_fwd<kAct>(v);
    }
    return;
  }
  float s = 0.f, ss = 0.f;
  for (int d = lane; d < D; d += 32) { float v = in(d); s += v; ss += v * v; }
  s = warp_sum(s); ss = warp_sum(ss);
  const float mean = s / (float)D;
  const float var = fmaxf(ss / (float)D - mean * mean, 0.f);
  const float rstd = rsqrtf(var + eps);
  const int g = row / rows_per_group;
  const float* sc = scale + (size_t)g * group_stride;
  const float* bi = bias + (size_t)g * group_stride;
  for (int d = lane; d < D; d += 32) {
    const float xh = (in(d) - mean) * rstd;
    out[(size_t)row * ld_out + d] = act_fwd<kAct>(xh * sc[d] + bi[d]);
    if (xhat) xhat[(size_t)row * D + d] = xh;
  }
  if (rstd_out && lane == 0) rstd_out[row] = rstd;
}

// ---- [LayerNorm +] activation backward: warp per row -----------------------------------------------
// dy = dt * act'(y): tanh reads its output t (1 - t^2); the other activations need the pre-activation y, recomputed as
// xhat*scale + bias with LayerNorm and read from `pre` (the saved z) without.
// With LayerNorm: dz = rstd * (dy*scale - mean(dy*scale) - xhat * mean(dy*scale*xhat)), dy kept for the param grads.
// Without: dz = dy.  kDrop: dz *= mask ? inv_keep : 0 (the forward's dropout, same mask rows r % mask_rows).
template <int kAct, bool kLN, bool kDrop = false>
__global__ void ln_act_bwd_kernel(const float* __restrict__ dt, int ld_dt, const float* __restrict__ t, int ld_t,
                                  const float* __restrict__ pre, int ld_pre, const float* __restrict__ xhat, const float* __restrict__ rstd,
                                  const float* __restrict__ scale, const float* __restrict__ bias, int rows_per_group, int group_stride,
                                  float* __restrict__ dz, float* __restrict__ dy_out, int R, int D, const uint8_t* __restrict__ mask,
                                  float inv_keep, int mask_rows) {
  pdl_prologue();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= R) return;
  if constexpr (!kLN) {
    for (int d = lane; d < D; d += 32) {
      float g;
      if constexpr (kAct == SERL_ACT_TANH) { const float tv = t[(size_t)row * ld_t + d]; g = 1.f - tv * tv; }
      else g = act_grad<kAct>(pre[(size_t)row * ld_pre + d]);
      if constexpr (kDrop) g = mask[(size_t)(row % mask_rows) * D + d] ? g * inv_keep : 0.f;
      dz[(size_t)row * D + d] = dt[(size_t)row * ld_dt + d] * g;
    }
    return;
  }
  auto out = [&](int d, float v) {
    if constexpr (kDrop) v = mask[(size_t)(row % mask_rows) * D + d] ? v * inv_keep : 0.f;
    dz[(size_t)row * D + d] = v;
  };
  const float* sc = scale + (size_t)(row / rows_per_group) * group_stride;
  const float* bi = bias + (size_t)(row / rows_per_group) * group_stride;
  float m1 = 0.f, m2 = 0.f;
  for (int d = lane; d < D; d += 32) {
    float dy;
    if constexpr (kAct == SERL_ACT_TANH) {
      const float tv = t[(size_t)row * ld_t + d];
      dy = dt[(size_t)row * ld_dt + d] * (1.f - tv * tv);
    } else {
      dy = dt[(size_t)row * ld_dt + d] * act_grad<kAct>(xhat[(size_t)row * D + d] * sc[d] + bi[d]);
    }
    const float dxh = dy * sc[d];
    m1 += dxh; m2 += dxh * xhat[(size_t)row * D + d];
    dy_out[(size_t)row * D + d] = dy;
  }
  m1 = warp_sum(m1) / (float)D; m2 = warp_sum(m2) / (float)D;
  const float rs = rstd[row];
  for (int d = lane; d < D; d += 32) {
    const float dxh = dy_out[(size_t)row * D + d] * sc[d];
    out(d, rs * (dxh - m1 - xhat[(size_t)row * D + d] * m2));
  }
}

// ---- dscale[g][d] = sum_r dy*xhat ; dbias[g][d] = sum_r dy   (same 32 x 8 block shape as colsum) -----------------
__global__ void __launch_bounds__(256) ln_param_grad_kernel(const float* __restrict__ dy, const float* __restrict__ xhat,
                                                            float* __restrict__ dscale, float* __restrict__ dbias, int groups, int rows, int D) {
  pdl_prologue();
  __shared__ float ra[8][33], rb[8][33];
  const int cx = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int cblocks = ceil_div(D, 32);
  const int g = blockIdx.x / cblocks, d = (blockIdx.x - g * cblocks) * 32 + cx;
  float a = 0.f, b = 0.f;
  if (d < D) {
    for (int r = sl; r < rows; r += 8) {
      const size_t off = ((size_t)g * rows + r) * D + d;
      const float v = dy[off];
      a += v * xhat[off]; b += v;
    }
  }
  ra[sl][cx] = a; rb[sl][cx] = b;
  __syncthreads();
  if (sl == 0 && d < D) {
    float ta = ra[0][cx], tb = rb[0][cx];
#pragma unroll
    for (int k = 1; k < 8; ++k) { ta += ra[k][cx]; tb += rb[k][cx]; }
    dscale[(size_t)g * D + d] = ta; dbias[(size_t)g * D + d] = tb;
  }
}

// ---- strided 2-D copy (concat helper) -------------------------------------------------------------
__global__ void copy2d_kernel(const float* __restrict__ src, long long ld_src, float* __restrict__ dst, long long ld_dst, int R, int D) {
  pdl_prologue();
  const size_t total = (size_t)R * D;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / D), d = (int)(e - (size_t)r * D);
    dst[(size_t)r * ld_dst + d] = src[(size_t)r * ld_src + d];
  }
}

}  // namespace serl

using namespace serl;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int serl_sle_fwd(const float* feat, const float* kernel, const uint8_t* keep_mask, float keep, float* out,
                            int N, int P, int C, int F, int ld_out, void* stream) {
  if (F != 8 || (ld_out & 3)) { set_last_error("serl_sle_fwd: num_features must be 8 and ld_out %% 4 == 0"); return SERL_ERR_UNSUPPORTED; }
  launch_k(sle_fwd_kernel, ceil_div(N * C, 128), 128, 0, ST(stream), feat, kernel, keep_mask, keep, out, N, P, C, ld_out);
  return check_launch("sle_fwd_kernel");
}

extern "C" int serl_sle_bwd_kernel_grad(const float* feat, const float* dout, float* dkernel, float* workspace,
                                        size_t workspace_bytes, int N, int P, int C, int F, int ld_dout, void* stream) {
  if (F != 8 || (ld_dout & 3)) { set_last_error("serl_sle_bwd_kernel_grad: num_features must be 8"); return SERL_ERR_UNSUPPORTED; }
  int chunks = N >= 64 ? 16 : 1;
  const size_t per = (size_t)P * C * F * sizeof(float);
  while (chunks > 1 && per * chunks > workspace_bytes) chunks >>= 1;
  if (!workspace || per * chunks > workspace_bytes) { set_last_error("serl_sle_bwd_kernel_grad: workspace too small (%zu needed)", per); return SERL_ERR_INVALID; }
  dim3 grid(ceil_div(P * C, 128), chunks);
  launch_k(sle_bwd_partial_kernel, grid, 128, 0, ST(stream), feat, dout, workspace, N, P, C, ld_dout, chunks);
  if (int e = check_launch("sle_bwd_partial_kernel")) return e;
  const int D = P * C * F;
  launch_k(colsum_kernel, ceil_div(D, 32), 256, 0, ST(stream), workspace, dkernel, 1, chunks, D, D, 0);
  return check_launch("colsum_kernel(sle)");
}

extern "C" int serl_colsum_f32(const float* x, float* out, int groups, int rows, int D, long long ld, int accumulate, void* stream) {
  launch_k(colsum_kernel, groups * ceil_div(D, 32), 256, 0, ST(stream), x, out, groups, rows, D, ld, accumulate);
  return check_launch("colsum_kernel");
}

extern "C" int serl_layernorm_tanh_fwd(const float* z, int ld_z, const float* scale, const float* bias, int rows_per_group,
                                       int group_stride, float* out, int ld_out, float* xhat, float* rstd, int R, int D,
                                       float eps, void* stream) {
  launch_k(ln_act_fwd_kernel<SERL_ACT_TANH, true>, ceil_div(R, 8), 256, 0, ST(stream), z, ld_z, scale, bias, rows_per_group, group_stride,
           out, ld_out, xhat, rstd, R, D, eps, (const uint8_t*)nullptr, 1.f, (float*)nullptr, 1);
  return check_launch("ln_tanh_fwd_kernel");
}

extern "C" int serl_layernorm_tanh_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* xhat, const float* rstd,
                                       const float* scale, int rows_per_group, int group_stride, float* dz, float* dy,
                                       float* dscale, float* dbias, int R, int D, void* stream) {
  launch_k(ln_act_bwd_kernel<SERL_ACT_TANH, true>, ceil_div(R, 8), 256, 0, ST(stream), dt, ld_dt, t, ld_t, (const float*)nullptr, 0, xhat, rstd,
           scale, (const float*)nullptr, rows_per_group, group_stride, dz, dy, R, D, (const uint8_t*)nullptr, 1.f, 1);
  if (int e = check_launch("ln_tanh_bwd_kernel")) return e;
  if (dscale && dbias) {
    const int groups = R / rows_per_group;
    launch_k(ln_param_grad_kernel, groups * ceil_div(D, 32), 256, 0, ST(stream), dy, xhat, dscale, dbias, groups, rows_per_group, D);
    return check_launch("ln_param_grad_kernel");
  }
  return SERL_OK;
}

// one instantiation per (activation, LayerNorm, dropout) triple; the switch runs on the host
#define SERL_ACT_SWITCH(KERNEL, DROP)                                                                                        \
  switch (act) {                                                                                                             \
    case SERL_ACT_TANH: return layer_norm ? KERNEL<SERL_ACT_TANH, true, DROP> : KERNEL<SERL_ACT_TANH, false, DROP>;          \
    case SERL_ACT_RELU: return layer_norm ? KERNEL<SERL_ACT_RELU, true, DROP> : KERNEL<SERL_ACT_RELU, false, DROP>;          \
    case SERL_ACT_SWISH: return layer_norm ? KERNEL<SERL_ACT_SWISH, true, DROP> : KERNEL<SERL_ACT_SWISH, false, DROP>;       \
    case SERL_ACT_LEAKY_RELU:                                                                                                \
      return layer_norm ? KERNEL<SERL_ACT_LEAKY_RELU, true, DROP> : KERNEL<SERL_ACT_LEAKY_RELU, false, DROP>;               \
    case SERL_ACT_GELU: return layer_norm ? KERNEL<SERL_ACT_GELU, true, DROP> : KERNEL<SERL_ACT_GELU, false, DROP>;          \
    default: return nullptr;                                                                                                 \
  }
using LnActFwdFn = decltype(&ln_act_fwd_kernel<SERL_ACT_TANH, true>);
using LnActBwdFn = decltype(&ln_act_bwd_kernel<SERL_ACT_TANH, true>);
static LnActFwdFn ln_act_fwd_fn(int act, int layer_norm, bool drop) {
  if (drop) { SERL_ACT_SWITCH(ln_act_fwd_kernel, true) }
  SERL_ACT_SWITCH(ln_act_fwd_kernel, false)
}
static LnActBwdFn ln_act_bwd_fn(int act, int layer_norm, bool drop) {
  if (drop) { SERL_ACT_SWITCH(ln_act_bwd_kernel, true) }
  SERL_ACT_SWITCH(ln_act_bwd_kernel, false)
}
#undef SERL_ACT_SWITCH

extern "C" int serl_layernorm_act_fwd(const float* z, int ld_z, const float* scale, const float* bias, int rows_per_group,
                                      int group_stride, float* out, int ld_out, float* xhat, float* rstd, int R, int D,
                                      float eps, int act, int layer_norm, void* stream) {
  LnActFwdFn k = ln_act_fwd_fn(act, layer_norm, false);
  if (!k || (layer_norm && (!scale || !bias || rows_per_group < 1))) {
    set_last_error("serl_layernorm_act_fwd: unknown activation %d or LayerNorm without scale / bias", act); return SERL_ERR_INVALID;
  }
  launch_k(k, ceil_div(R, 8), 256, 0, ST(stream), z, ld_z, scale, bias, rows_per_group, group_stride, out, ld_out, xhat, rstd, R, D, eps,
           (const uint8_t*)nullptr, 1.f, (float*)nullptr, 1);
  return check_launch("ln_act_fwd_kernel");
}

// serl_layernorm_act_fwd with the layer's Dropout first: mask keep bytes (serl_dropout_mask_fill), inv_keep = 1 / keep; row r
// reads mask row r % mask_rows (mask_rows = R: one mask row per row; mask_rows = B: an E*B-row ensemble shares a (B, D) mask).
// Without LayerNorm the dropped-out z is written back to z (the backward's pre).
extern "C" int serl_ln_act_dropout_rows_fwd(float* z, int ld_z, const float* scale, const float* bias, int rows_per_group, int group_stride,
                                            const uint8_t* mask, int mask_rows, float inv_keep, float* out, int ld_out, float* xhat, float* rstd,
                                            int R, int D, float eps, int act, int layer_norm, void* stream) {
  LnActFwdFn k = ln_act_fwd_fn(act, layer_norm, true);
  if (!k || !z || !mask || !out || mask_rows < 1 || (layer_norm && (!scale || !bias || rows_per_group < 1))) {
    set_last_error("serl_ln_act_dropout_fwd: unknown activation %d, missing mask, mask_rows < 1 or LayerNorm without scale / bias", act);
    return SERL_ERR_INVALID;
  }
  launch_k(k, ceil_div(R, 8), 256, 0, ST(stream), (const float*)z, ld_z, scale, bias, rows_per_group, group_stride, out, ld_out, xhat, rstd,
           R, D, eps, mask, inv_keep, z, mask_rows);
  return check_launch("ln_act_dropout_fwd_kernel");
}

extern "C" int serl_ln_act_dropout_fwd(float* z, int ld_z, const float* scale, const float* bias, int rows_per_group, int group_stride,
                                       const uint8_t* mask, float inv_keep, float* out, int ld_out, float* xhat, float* rstd, int R, int D,
                                       float eps, int act, int layer_norm, void* stream) {
  return serl_ln_act_dropout_rows_fwd(z, ld_z, scale, bias, rows_per_group, group_stride, mask, R > 0 ? R : 1, inv_keep, out, ld_out, xhat,
                                      rstd, R, D, eps, act, layer_norm, stream);
}

extern "C" int serl_layernorm_act_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* pre, int ld_pre,
                                      const float* xhat, const float* rstd, const float* scale, const float* bias, int rows_per_group,
                                      int group_stride, float* dz, float* dy, int R, int D, int act, int layer_norm, void* stream) {
  LnActBwdFn k = ln_act_bwd_fn(act, layer_norm, false);
  const bool ok = layer_norm ? (xhat && rstd && scale && dy && rows_per_group >= 1 && (act == SERL_ACT_TANH ? t != nullptr : bias != nullptr))
                             : (act == SERL_ACT_TANH ? t != nullptr : pre != nullptr);
  if (!k || !ok || !dz) {
    set_last_error("serl_layernorm_act_bwd: unknown activation %d or missing operand", act); return SERL_ERR_INVALID;
  }
  launch_k(k, ceil_div(R, 8), 256, 0, ST(stream), dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride,
           dz, dy, R, D, (const uint8_t*)nullptr, 1.f, 1);
  return check_launch("ln_act_bwd_kernel");
}

// serl_layernorm_act_bwd of serl_ln_act_dropout_rows_fwd: dz leaves through the same mask rows, times inv_keep
extern "C" int serl_ln_act_dropout_rows_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* pre, int ld_pre,
                                            const float* xhat, const float* rstd, const float* scale, const float* bias, int rows_per_group,
                                            int group_stride, const uint8_t* mask, int mask_rows, float inv_keep, float* dz, float* dy, int R,
                                            int D, int act, int layer_norm, void* stream) {
  LnActBwdFn k = ln_act_bwd_fn(act, layer_norm, true);
  const bool ok = layer_norm ? (xhat && rstd && scale && dy && rows_per_group >= 1 && (act == SERL_ACT_TANH ? t != nullptr : bias != nullptr))
                             : (act == SERL_ACT_TANH ? t != nullptr : pre != nullptr);
  if (!k || !ok || !dz || !mask || mask_rows < 1) {
    set_last_error("serl_ln_act_dropout_bwd: unknown activation %d or missing operand", act); return SERL_ERR_INVALID;
  }
  launch_k(k, ceil_div(R, 8), 256, 0, ST(stream), dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride,
           dz, dy, R, D, mask, inv_keep, mask_rows);
  return check_launch("ln_act_dropout_bwd_kernel");
}

extern "C" int serl_ln_act_dropout_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* pre, int ld_pre,
                                       const float* xhat, const float* rstd, const float* scale, const float* bias, int rows_per_group,
                                       int group_stride, const uint8_t* mask, float inv_keep, float* dz, float* dy, int R, int D, int act,
                                       int layer_norm, void* stream) {
  return serl_ln_act_dropout_rows_bwd(dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride, mask,
                                      R > 0 ? R : 1, inv_keep, dz, dy, R, D, act, layer_norm, stream);
}

// the parameter-gradient half of serl_layernorm_tanh_bwd on its own (dy, xhat as that call left them): lets the caller put it
// on a side stream, off the dz -> next-layer chain
extern "C" int serl_layernorm_param_grad(const float* dy, const float* xhat, float* dscale, float* dbias, int rows_per_group, int R, int D,
                                         void* stream) {
  if (!dy || !xhat || !dscale || !dbias || rows_per_group < 1 || R % rows_per_group != 0) {
    set_last_error("serl_layernorm_param_grad: invalid arguments"); return SERL_ERR_INVALID;
  }
  const int groups = R / rows_per_group;
  launch_k(ln_param_grad_kernel, groups * ceil_div(D, 32), 256, 0, ST(stream), dy, xhat, dscale, dbias, groups, rows_per_group, D);
  return check_launch("ln_param_grad_kernel");
}

extern "C" int serl_copy2d_f32(const float* src, long long ld_src, float* dst, long long ld_dst, int R, int D, void* stream) {
  size_t total = (size_t)R * D;
  int blocks = (int)((total + 255) / 256); if (blocks > 1184) blocks = 1184; if (blocks < 1) blocks = 1;
  launch_k(copy2d_kernel, blocks, 256, 0, ST(stream), src, ld_src, dst, ld_dst, R, D);
  return check_launch("copy2d_kernel");
}

// ---- multi-action critic, first layer (networks/actor_critic_nets.py:33-46), forward only: warp per (member, state, candidate) row --
// z = P[e, b] + a[b, n] @ W_act[e] with P = enc @ W_enc + b0 from the GEMMs, so the encoder and its K = F contraction run once per
// state instead of once per candidate.  The candidate's A <= 32 action values are loaded one per lane and broadcast to registers;
// the k-sum runs in ascending k on top of P.  Then [LayerNorm +] activation exactly as ln_act_fwd_kernel (z re-read from memory).
namespace serl {
template <int kAct, bool kLN>
__global__ void critic_multi_action_kernel(const float* __restrict__ P, const float* __restrict__ actions, const float* __restrict__ w_act,
                                           long long w_act_z, const float* __restrict__ scale, const float* __restrict__ bias,
                                           float* __restrict__ z, float* __restrict__ out, int E, int B, int N, int A, int H, float eps) {
  pdl_prologue();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= E * B * N) return;                                     // whole warps leave together: the shuffles below are warp-uniform
  const int e = row / (B * N), bn = row - e * (B * N), b = bn / N;
  const float mine = lane < A ? actions[(size_t)bn * A + lane] : 0.f;
  float a[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) a[k] = __shfl_sync(0xffffffffu, mine, k);
  const float* p = P + ((size_t)e * B + b) * H;
  const float* w = w_act + (size_t)e * w_act_z;
  float* zr = z + (size_t)row * H;
  float* o = out + (size_t)row * H;
  float s = 0.f, ss = 0.f;
  for (int d = lane; d < H; d += 32) {
    float v = p[d];
#pragma unroll
    for (int k = 0; k < 32; ++k)
      if (k < A) v = fmaf(a[k], w[(size_t)k * H + d], v);
    zr[d] = v;
    if constexpr (kLN) { s += v; ss += v * v; } else { o[d] = act_fwd<kAct>(v); }
  }
  if constexpr (kLN) {
    s = warp_sum(s); ss = warp_sum(ss);
    const float mean = s / (float)H;
    const float var = fmaxf(ss / (float)H - mean * mean, 0.f);
    const float rstd = rsqrtf(var + eps);
    const float* sc = scale + (size_t)e * H;
    const float* bi = bias + (size_t)e * H;
    for (int d = lane; d < H; d += 32) o[d] = act_fwd<kAct>((zr[d] - mean) * rstd * sc[d] + bi[d]);
  }
}

using MultiActionFn = decltype(&critic_multi_action_kernel<SERL_ACT_TANH, true>);
static MultiActionFn multi_action_fn(int act, int layer_norm) {
  switch (act) {
    case SERL_ACT_TANH: return layer_norm ? critic_multi_action_kernel<SERL_ACT_TANH, true> : critic_multi_action_kernel<SERL_ACT_TANH, false>;
    case SERL_ACT_RELU: return layer_norm ? critic_multi_action_kernel<SERL_ACT_RELU, true> : critic_multi_action_kernel<SERL_ACT_RELU, false>;
    case SERL_ACT_SWISH: return layer_norm ? critic_multi_action_kernel<SERL_ACT_SWISH, true> : critic_multi_action_kernel<SERL_ACT_SWISH, false>;
    case SERL_ACT_LEAKY_RELU:
      return layer_norm ? critic_multi_action_kernel<SERL_ACT_LEAKY_RELU, true> : critic_multi_action_kernel<SERL_ACT_LEAKY_RELU, false>;
    case SERL_ACT_GELU: return layer_norm ? critic_multi_action_kernel<SERL_ACT_GELU, true> : critic_multi_action_kernel<SERL_ACT_GELU, false>;
    default: return nullptr;
  }
}
}  // namespace serl

extern "C" int serl_critic_multi_action_fwd(const float* P, const float* actions, const float* w_act, long long w_act_z, const float* scale,
                                            const float* bias, float* z, float* out, int E, int B, int N, int A, int H, float eps, int act,
                                            int layer_norm, void* stream) {
  MultiActionFn k = multi_action_fn(act, layer_norm);
  if (!k || !P || !actions || !w_act || !z || !out || (layer_norm && (!scale || !bias)) || E < 1 || B < 1 || N < 1 || A < 1 || A > 32 ||
      H < 1 || (long long)E * B * N > 0x7fffffffLL) {
    set_last_error("serl_critic_multi_action_fwd: unknown activation %d, missing operand or bad shape (E %d, B %d, N %d, A %d: need 1 <= A <= 32)",
                   act, E, B, N, A);
    return SERL_ERR_INVALID;
  }
  const int R = E * B * N;
  launch_k(k, ceil_div(R, 8), 256, 0, ST(stream), P, actions, w_act, w_act_z, scale, bias, z, out, E, B, N, A, H, eps);
  return check_launch("critic_multi_action_kernel");
}
