// VICE reward classifier (fp32): the kernels `VICEAgent.update_vice` adds on top of the shared trunk / SLE / GEMM kernels, and
// the reward relabelling of `update_critics` / `update_high_utd`.
//
// Reference (relative to serl_launcher/serl_launcher):
//   agents/continuous/vice.py:357-517   update_vice: mixup (lam ~ Beta(1,1) = U(0,1) here, one permutation of the 2B encoded
//                                       rows), label smoothing y*0.8 + 0.1, BCE, gradient penalty 10 * mean((|dy/dx| - 1)^2) on
//                                       eps*mix[i] + (1-eps)*mix[B+i], |g| = sqrt(sum(g^2 + 1e-6))
//   agents/continuous/vice.py:519-600   vice_reward = sigmoid(logit); rewards = (vice_reward >= 0.5) * 1.0
//   networks/mlp.py:17-32               Dense -> Dropout -> LayerNorm -> leaky_relu (slope 0.01) of the VICE MLP
//   vision/resnet_v1.py:324-376         SLE -> Dropout -> Dense(512) -> LayerNorm -> tanh of the VICE image heads
//
// The penalty's parameter gradient is taken as the reverse-mode gradient of the directional derivative
//   d/dtheta [ v . dy/dx ] = d/dtheta ydot,   ydot = J_x y(x; theta) v,   v = d gp / d g  (held constant),
// so the forward pass carries a tangent (z, zdot) through every layer (`tangent` rows of the LayerNorm kernels) and the backward
// pass carries two cotangents (zbar, zdotbar).  Rows are stacked: [0, 2B) mixup rows (BCE), [2B, 3B) penalty rows (primal),
// [3B, 4B) their tangents, so every weight gradient is ONE GEMM over 4B rows and every bias / scale gradient one column sum.
// Restated in tests/vice_oracle.py (float64 autograd with create_graph=True).
#include "common.cuh"
#include "serl_b200.h"

namespace serl {

constexpr int kViceMaxRows = 2048;           // 2B of one update_vice call (one CTA sorts them)
constexpr float kLeakySlope = 0.01f;         // flax nn.leaky_relu default

// ---- draws: lam = uniform(k0), perm = permutation(k1, N) (jax _shuffle: per round key, sub = split(key); stable sort of the rows
// by random_bits(sub, (N,))), eps = uniform(k_eps, (N/2,)).  One CTA per camera. ----------------------------------------------
__global__ void __launch_bounds__(512) vice_draws_kernel(const uint32_t* __restrict__ keys, int N, int rounds, float* __restrict__ lam,
                                                          int* __restrict__ perm, float* __restrict__ eps) {
  pdl_prologue();
  __shared__ uint32_t bits[kViceMaxRows];
  __shared__ int x[kViceMaxRows], nx[kViceMaxRows];
  const int cam = blockIdx.x;
  const uint32_t* k = keys + 6 * cam;
  const u32x2 k0{k[0], k[1]}, k_eps{k[4], k[5]};
  u32x2 key{k[2], k[3]};
  if (threadIdx.x == 0) lam[cam] = bits_to_uniform01(jax_random_bits_at(k0, 1u, 0u));
  for (int i = threadIdx.x; i < N / 2; i += blockDim.x) eps[(size_t)cam * (N / 2) + i] = bits_to_uniform01(jax_random_bits_at(k_eps, N / 2, i));
  for (int i = threadIdx.x; i < N; i += blockDim.x) x[i] = i;
  for (int r = 0; r < rounds; ++r) {
    const u32x2 sub = jax_split_at(key, 2, 1);
    key = jax_split_at(key, 2, 0);
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) bits[i] = jax_random_bits_at(sub, N, i);
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) {          // stable rank: smaller bits first, ties in row order
      const uint32_t b = bits[i];
      int rank = 0;
      for (int j = 0; j < N; ++j) rank += (bits[j] < b) || (bits[j] == b && j < i);
      nx[rank] = x[i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) x[i] = nx[i];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) perm[(size_t)cam * N + i] = x[i];
}

// ---- mixup + penalty interpolates: out rows [0, N) = lam f + (1 - lam) f[perm], rows [N, 3N/2) = eps mix[i] + (1 - eps) mix[N/2 + i]
__global__ void vice_mix_kernel(const float* __restrict__ feats, long long in_stride, const float* __restrict__ lam,
                                const int* __restrict__ perm, const float* __restrict__ eps, float* __restrict__ out, long long out_stride,
                                int ncams, int N, int D) {
  pdl_prologue();
  const int H = N / 2;
  const long long per = (long long)H * D, total = per * ncams;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int cam = (int)(e / per);
    const long long r = e - cam * per;
    const int i = (int)(r / D), d = (int)(r - (long long)i * D);
    const float* f = feats + cam * in_stride;
    const int* p = perm + (size_t)cam * N;
    const float l = lam[cam], l1 = 1.f - l;
    const float a = l * f[(size_t)i * D + d] + l1 * f[(size_t)p[i] * D + d];
    const float b = l * f[(size_t)(H + i) * D + d] + l1 * f[(size_t)p[H + i] * D + d];
    float* o = out + cam * out_stride;
    o[(size_t)i * D + d] = a;
    o[(size_t)(H + i) * D + d] = b;
    const float ep = eps[(size_t)cam * H + i];
    o[(size_t)(N + i) * D + d] = ep * a + (1.f - ep) * b;
  }
}

// ---- smoothed-label mixup BCE: y = [1]*N/2 + [0]*N/2 smoothed y*0.8 + 0.1, y_a = y, y_b = y[perm];
// loss = lam mean(bce(x, y_a)) + (1 - lam) mean(bce(x, y_b)); dlogit = grad_scale (sigmoid(x) - lam y_a - (1 - lam) y_b) / N.
// grad_scale (1/world under data parallelism) also scales info[0], so one SUM all-reduce of gradient + infos yields the mean.
__device__ __forceinline__ float vice_label(int i, int N) {
  const float y = i < N / 2 ? 1.f : 0.f;
  return __fadd_rn(__fmul_rn(y, 1.f - 0.2f), 0.5f * 0.2f);
}

__device__ __forceinline__ float bce_f(float x, float y) { return fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x))); }

__global__ void __launch_bounds__(256) vice_bce_kernel(const float* __restrict__ logits, const float* __restrict__ lam,
                                                       const int* __restrict__ perm, float grad_scale, float* __restrict__ dlogit,
                                                       float* __restrict__ info, int N) {
  pdl_prologue();
  __shared__ float ra[256], rb[256];
  const float l = lam[0];
  float sa = 0.f, sb = 0.f;
  const float inv = 1.f / (float)N;
  for (int i = threadIdx.x; i < N; i += 256) {
    const float x = logits[i], ya = vice_label(i, N), yb = vice_label(perm[i], N);
    sa += bce_f(x, ya); sb += bce_f(x, yb);
    const float sg = 1.f / (1.f + expf(-x));
    dlogit[i] = (l * (sg - ya) + (1.f - l) * (sg - yb)) * grad_scale * inv;
  }
  ra[threadIdx.x] = sa; rb[threadIdx.x] = sb;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { ra[threadIdx.x] += ra[threadIdx.x + o]; rb[threadIdx.x] += rb[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) info[0] = (l * (ra[0] * inv) + (1.f - l) * (rb[0] * inv)) * grad_scale;   // pre-scaled like the gradient
}

// ---- activations ----------------------------------------------------------------------------------------------------------
template <int ACT> struct Act;
template <> struct Act<SERL_ACT_TANH> {
  static __device__ __forceinline__ float f(float u) { return tanhf(u); }
  static __device__ __forceinline__ void d(float u, float& a1, float& a2) { const float t = tanhf(u); a1 = 1.f - t * t; a2 = -2.f * t * a1; }
};
template <> struct Act<SERL_ACT_LEAKY_RELU> {
  static __device__ __forceinline__ float f(float u) { return u >= 0.f ? u : kLeakySlope * u; }
  static __device__ __forceinline__ void d(float u, float& a1, float& a2) { a1 = u >= 0.f ? 1.f : kLeakySlope; a2 = 0.f; }
};

// ---- [dropout] -> LayerNorm (eps, fast variance) -> act [-> Dense(1)], warp per row, lane owns columns lane + 32 j ------------
// Primal rows r in [R0, R): z' = mask(z + pre_bias), xhat, rstd saved, y = act(u), logit = y . w + b.
// Tangent rows r in [R0, R) (tangent = 1): partner p = r - pair_off; zdot' = mask_p(zdot) is written back to z,
// xhatdot = rstd_p (zdot' - mean(zdot') - xhat_p mean(xhat_p zdot')), ydot = act'(u_p) scale xhatdot.
template <int ACT, int NV>
__global__ void __launch_bounds__(256) vice_ln_act_fwd_kernel(float* __restrict__ z, int ld_z, const float* __restrict__ pre_bias,
                                                              const uint8_t* __restrict__ mask, int ld_mask, float keep,
                                                              const float* __restrict__ scale, const float* __restrict__ bias,
                                                              float* __restrict__ y, int ld_y, float* __restrict__ xhat,
                                                              float* __restrict__ rstd, const float* __restrict__ hw,
                                                              const float* __restrict__ hb, float* __restrict__ logit, int R0, int R,
                                                              int pair_off, int tangent, float eps) {
  pdl_prologue();
  constexpr int D = NV * 32;
  const int r = R0 + blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  const int p = tangent ? r - pair_off : r;
  float v[NV], xh[NV];
  float s = 0.f, ss = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int d = lane + 32 * j;
    float x = z[(size_t)r * ld_z + d];
    if (!tangent && pre_bias) x += pre_bias[d];
    if (mask) x = mask[(size_t)p * ld_mask + d] ? x / keep : 0.f;
    v[j] = x;
    if (tangent) { z[(size_t)r * ld_z + d] = x; xh[j] = xhat[(size_t)p * D + d]; s += x; ss += x * xh[j]; }
    else { s += x; ss += x * x; }
  }
  s = warp_sum(s); ss = warp_sum(ss);
  float dot = 0.f;
  if (!tangent) {
    const float mean = s / (float)D;
    const float var = fmaxf(ss / (float)D - mean * mean, 0.f);
    const float rs = rsqrtf(var + eps);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int d = lane + 32 * j;
      const float x = (v[j] - mean) * rs;
      const float o = Act<ACT>::f(x * scale[d] + bias[d]);
      if (xhat) xhat[(size_t)r * D + d] = x;
      if (y) y[(size_t)r * ld_y + d] = o;
      if (hw) dot = fmaf(o, hw[d], dot);
    }
    if (lane == 0 && rstd) rstd[r] = rs;
  } else {
    const float m1 = s / (float)D, m2 = ss / (float)D, rs = rstd[p];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int d = lane + 32 * j;
      const float xd = rs * (v[j] - m1 - xh[j] * m2);
      float a1, a2;
      Act<ACT>::d(xh[j] * scale[d] + bias[d], a1, a2);
      const float o = a1 * scale[d] * xd;
      if (y) y[(size_t)r * ld_y + d] = o;
    }
  }
  if (hw && !tangent) {
    dot = warp_sum(dot);
    if (lane == 0) logit[r] = dot + hb[0];
  }
}

// ---- reverse of the above for primal rows r in [R0, R); rows r >= R - R_pair carry the tangent row r + R_pair --------------
// Cotangents: ybar from dy (or head: a_r w with a_r = dlogit[r] | dlogit_const), ydotbar from dy's tangent row (or head: tan_seed w).
//   ubar = a1 ybar + a2 udot ydotbar,  udotbar = a1 ydotbar,  dscale = xhat ubar + xhatdot udotbar,  dbias = ubar
//   zdotbar = r P (scale udotbar),  xhatbar = scale ubar - r (scale udotbar mean(xhat zdot') + zdot' mean(xhat scale udotbar)),
//   rbar = sum(scale udotbar xhatdot) / r,  zbar = r P xhatbar - r^2 xhat rbar / D,   P v = v - mean(v) - xhat mean(xhat v)
// then the dropout mask on zbar and zdotbar.  Head: dw_rows = a_r y_r + tan_seed ydot_r (column sums give the Dense(1) kernel grad).
template <int ACT, int NV>
__global__ void __launch_bounds__(256) vice_ln_act_bwd_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ dlogit,
                                                              float dlogit_const, const float* __restrict__ hw, float tan_seed,
                                                              const float* __restrict__ xhat, const float* __restrict__ rstd,
                                                              const float* __restrict__ z, int ld_z, const uint8_t* __restrict__ mask,
                                                              int ld_mask, float keep, const float* __restrict__ scale,
                                                              const float* __restrict__ bias, const float* __restrict__ y, int ld_y,
                                                              float* __restrict__ dz, int ld_dz, float* __restrict__ dscale_rows,
                                                              float* __restrict__ dbias_rows, float* __restrict__ dw_rows, int R0, int R,
                                                              int R_pair) {
  pdl_prologue();
  constexpr int D = NV * 32;
  const int r = R0 + blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  const bool pair = r >= R - R_pair;
  const int t = r + R_pair;
  const float rs = rstd[r];
  const float a = hw ? (dlogit ? dlogit[r] : dlogit_const) : 0.f;
  float xh[NV], zt[NV], yb[NV], ytb[NV];
  float mz = 0.f, mxz = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int d = lane + 32 * j;
    xh[j] = xhat[(size_t)r * D + d];
    yb[j] = hw ? a * hw[d] : (dy ? dy[(size_t)r * ld_dy + d] : 0.f);
    zt[j] = pair ? z[(size_t)t * ld_z + d] : 0.f;
    ytb[j] = pair ? (hw ? tan_seed * hw[d] : dy[(size_t)t * ld_dy + d]) : 0.f;
    mz += zt[j]; mxz += xh[j] * zt[j];
  }
  if (pair) { mz = warp_sum(mz) / (float)D; mxz = warp_sum(mxz) / (float)D; }
  float ub[NV], xdt[NV], xdb[NV];
  float m1 = 0.f, m2 = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int d = lane + 32 * j;
    float a1, a2;
    Act<ACT>::d(xh[j] * scale[d] + bias[d], a1, a2);
    xdt[j] = pair ? rs * (zt[j] - mz - xh[j] * mxz) : 0.f;
    const float udot = scale[d] * xdt[j];
    ub[j] = a1 * yb[j] + a2 * udot * ytb[j];
    const float udb = a1 * ytb[j];
    if (dscale_rows) dscale_rows[(size_t)r * D + d] = xh[j] * ub[j] + xdt[j] * udb;
    if (dbias_rows) dbias_rows[(size_t)r * D + d] = ub[j];
    if (dw_rows) dw_rows[(size_t)r * D + d] = a * y[(size_t)r * ld_y + d] + (pair ? tan_seed * y[(size_t)t * ld_y + d] : 0.f);
    xdb[j] = scale[d] * udb;
    m1 += xdb[j]; m2 += xh[j] * xdb[j];
  }
  float rb = 0.f;
  if (pair) {
    m1 = warp_sum(m1) / (float)D; m2 = warp_sum(m2) / (float)D;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int d = lane + 32 * j;
      float g = rs * (xdb[j] - m1 - xh[j] * m2);
      if (mask) g = mask[(size_t)r * ld_mask + d] ? g / keep : 0.f;
      dz[(size_t)t * ld_dz + d] = g;
      rb += xdb[j] * xdt[j];
    }
    rb = warp_sum(rb) / rs;
  }
  float xb[NV];
  float m3 = 0.f, m4 = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int d = lane + 32 * j;
    xb[j] = scale[d] * ub[j] - (pair ? rs * (xdb[j] * mxz + zt[j] * m2) : 0.f);
    m3 += xb[j]; m4 += xh[j] * xb[j];
  }
  m3 = warp_sum(m3) / (float)D; m4 = warp_sum(m4) / (float)D;
  const float cr = rs * rs * rb / (float)D;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int d = lane + 32 * j;
    float g = rs * (xb[j] - m3 - xh[j] * m4) - cr * xh[j];
    if (mask) g = mask[(size_t)r * ld_mask + d] ? g / keep : 0.f;
    dz[(size_t)r * ld_dz + d] = g;
  }
}

// ---- SLE input gradient: dx[r, p, c] = sum_f ds[r, c*F + f] k[p, c, f] -----------------------------------------------------
__global__ void vice_sle_input_grad_kernel(const float* __restrict__ ds, int ld_ds, const float* __restrict__ k, float* __restrict__ dx,
                                           int R, int P, int C) {
  pdl_prologue();
  const long long total = (long long)R * P * C;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / ((long long)P * C));
    const int pc = (int)(e - (long long)r * P * C), c = pc % C;
    const float4* kk = reinterpret_cast<const float4*>(k + (size_t)pc * 8);
    const float4* dd = reinterpret_cast<const float4*>(ds + (size_t)r * ld_ds + (size_t)c * 8);
    const float4 k0 = kk[0], k1 = kk[1], d0 = dd[0], d1 = dd[1];
    float s = d0.x * k0.x;
    s = fmaf(d0.y, k0.y, s); s = fmaf(d0.z, k0.z, s); s = fmaf(d0.w, k0.w, s);
    s = fmaf(d1.x, k1.x, s); s = fmaf(d1.y, k1.y, s); s = fmaf(d1.z, k1.z, s); s = fmaf(d1.w, k1.w, s);
    dx[e] = s;
  }
}

// ---- keep masks: (rows, n) = bernoulli(fold_in(key, fold), keep, (rows, n)), or one (n,) row broadcast to every row ----------
__global__ void vice_mask_fill_kernel(const uint32_t* __restrict__ key, int fold, float keep, uint8_t* __restrict__ out, int rows, int n,
                                      int broadcast) {
  pdl_prologue();
  const u32x2 k = jax_fold_in(u32x2{key[0], key[1]}, (uint32_t)fold);
  const long long total = (long long)rows * n;
  const uint32_t size = broadcast ? (uint32_t)n : (uint32_t)total;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const uint32_t j = broadcast ? (uint32_t)(e % n) : (uint32_t)e;
    out[e] = bits_to_uniform01(jax_random_bits_at(k, size, j)) < keep ? 1 : 0;
  }
}

// ---- penalty rows: block per (camera, row): |g| = sqrt(sum(g^2 + 1e-6)), v = coef (|g| - 1) / |g| g ------------------------
__global__ void __launch_bounds__(256) vice_gp_rows_kernel(const float* __restrict__ g, long long g_stride, float* __restrict__ v,
                                                           long long v_stride, float coef, float* __restrict__ norms, int B, int D) {
  pdl_prologue();
  __shared__ float red[256];
  const int cam = blockIdx.y, r = blockIdx.x;
  const float* gr = g + cam * g_stride + (size_t)r * D;
  float s = 0.f;
  for (int d = threadIdx.x; d < D; d += 256) s += gr[d] * gr[d] + 1e-6f;
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const float nrm = sqrtf(red[0]);
  const float c = coef * (nrm - 1.f) / nrm;
  float* vr = v + cam * v_stride + (size_t)r * D;
  for (int d = threadIdx.x; d < D; d += 256) vr[d] = c * gr[d];
  if (threadIdx.x == 0) norms[(size_t)cam * B + r] = nrm;
}

// info[0] = bce (in, already scaled); writes info[1] = s mean |g|, info[2] = s gp, gp = mean((|g| - 1)^2), info[3] = info[0] + 10 info[2]
// with s = info_scale (1/world under data parallelism, like the gradients).  One CTA.
__global__ void __launch_bounds__(256) vice_gp_finish_kernel(const float* __restrict__ norms, int M, float gp_weight, float info_scale,
                                                             float* __restrict__ info) {
  pdl_prologue();
  __shared__ float ra[256], rb[256];
  float sa = 0.f, sb = 0.f;
  for (int i = threadIdx.x; i < M; i += 256) { const float n = norms[i]; sa += n; sb += (n - 1.f) * (n - 1.f); }
  ra[threadIdx.x] = sa; rb[threadIdx.x] = sb;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { ra[threadIdx.x] += ra[threadIdx.x + o]; rb[threadIdx.x] += rb[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float gp = rb[0] / (float)M * info_scale;
    info[1] = ra[0] / (float)M * info_scale; info[2] = gp; info[3] = info[0] + gp_weight * gp;
  }
}

// ---- relabelling: rewards = (float)(sigmoid(logit) >= 0.5) with sigmoid in fp32 (threshold = 0: sigmoid); mean_out = mean.  One CTA. ---------
__global__ void __launch_bounds__(256) vice_reward_kernel(const float* __restrict__ logit, float* __restrict__ rewards,
                                                          float* __restrict__ mean_out, int B, int threshold) {
  pdl_prologue();
  __shared__ float red[256];
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += 256) {
    const float sg = 1.f / (1.f + expf(-logit[i]));
    const float r = threshold ? (sg >= 0.5f ? 1.f : 0.f) : sg;
    rewards[i] = r; s += r;
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0 && mean_out) mean_out[0] = red[0] / (float)B;
}

template <int NV>
static void launch_fwd(int act, dim3 g, cudaStream_t st, float* z, int ld_z, const float* pre_bias, const uint8_t* mask, int ld_mask,
                       float keep, const float* scale, const float* bias, float* y, int ld_y, float* xhat, float* rstd, const float* hw,
                       const float* hb, float* logit, int R0, int R, int pair_off, int tangent, float eps) {
  if (act == SERL_ACT_TANH)
    launch_k(vice_ln_act_fwd_kernel<SERL_ACT_TANH, NV>, g, 256, 0, st, z, ld_z, pre_bias, mask, ld_mask, keep, scale, bias, y, ld_y, xhat,
             rstd, hw, hb, logit, R0, R, pair_off, tangent, eps);
  else
    launch_k(vice_ln_act_fwd_kernel<SERL_ACT_LEAKY_RELU, NV>, g, 256, 0, st, z, ld_z, pre_bias, mask, ld_mask, keep, scale, bias, y, ld_y,
             xhat, rstd, hw, hb, logit, R0, R, pair_off, tangent, eps);
}

template <int NV>
static void launch_bwd(int act, dim3 g, cudaStream_t st, const float* dy, int ld_dy, const float* dlogit, float dlogit_const, const float* hw,
                       float tan_seed, const float* xhat, const float* rstd, const float* z, int ld_z, const uint8_t* mask, int ld_mask,
                       float keep, const float* scale, const float* bias, const float* y, int ld_y, float* dz, int ld_dz,
                       float* dscale_rows, float* dbias_rows, float* dw_rows, int R0, int R, int R_pair) {
  if (act == SERL_ACT_TANH)
    launch_k(vice_ln_act_bwd_kernel<SERL_ACT_TANH, NV>, g, 256, 0, st, dy, ld_dy, dlogit, dlogit_const, hw, tan_seed, xhat, rstd, z, ld_z,
             mask, ld_mask, keep, scale, bias, y, ld_y, dz, ld_dz, dscale_rows, dbias_rows, dw_rows, R0, R, R_pair);
  else
    launch_k(vice_ln_act_bwd_kernel<SERL_ACT_LEAKY_RELU, NV>, g, 256, 0, st, dy, ld_dy, dlogit, dlogit_const, hw, tan_seed, xhat, rstd, z,
             ld_z, mask, ld_mask, keep, scale, bias, y, ld_y, dz, ld_dz, dscale_rows, dbias_rows, dw_rows, R0, R, R_pair);
}

}  // namespace serl

using namespace serl;
#define ST(s) static_cast<cudaStream_t>(s)

static int grid_for(long long n) { long long b = (n + 255) / 256; return (int)(b > 2368 ? 2368 : (b < 1 ? 1 : b)); }

extern "C" int serl_vice_draws(const uint32_t* keys, int ncams, int N, int rounds, float* lam, int* perm, float* eps, void* stream) {
  if (!keys || !lam || !perm || !eps || ncams < 1 || N < 2 || N > kViceMaxRows || (N & 1) || rounds < 1) {
    set_last_error("serl_vice_draws: invalid arguments (2 <= N <= %d, N even)", kViceMaxRows); return SERL_ERR_INVALID;
  }
  launch_k(vice_draws_kernel, ncams, 512, 0, ST(stream), keys, N, rounds, lam, perm, eps);
  return check_launch("vice_draws_kernel");
}

extern "C" int serl_vice_mix(const float* feats, long long in_stride, const float* lam, const int* perm, const float* eps, float* out,
                             long long out_stride, int ncams, int N, int D, void* stream) {
  if (!feats || !lam || !perm || !eps || !out || ncams < 1 || N < 2 || (N & 1) || D < 1) { set_last_error("serl_vice_mix: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(vice_mix_kernel, grid_for((long long)ncams * (N / 2) * D), 256, 0, ST(stream), feats, in_stride, lam, perm, eps, out, out_stride,
           ncams, N, D);
  return check_launch("vice_mix_kernel");
}

extern "C" int serl_vice_bce(const float* logits, const float* lam, const int* perm, float grad_scale, float* dlogit, float* info, int N,
                             void* stream) {
  if (!logits || !lam || !perm || !dlogit || !info || N < 2) { set_last_error("serl_vice_bce: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(vice_bce_kernel, 1, 256, 0, ST(stream), logits, lam, perm, grad_scale, dlogit, info, N);
  return check_launch("vice_bce_kernel");
}

extern "C" int serl_vice_ln_act_fwd(float* z, int ld_z, const float* pre_bias, const uint8_t* mask, int ld_mask, float keep, const float* scale,
                                    const float* bias, float* y, int ld_y, float* xhat, float* rstd, const float* head_w, const float* head_b,
                                    float* logit, int R0, int R, int pair_off, int tangent, int D, int act, float eps, void* stream) {
  const bool ok_act = act == SERL_ACT_TANH || act == SERL_ACT_LEAKY_RELU;
  if (!z || !scale || !bias || !ok_act || (D != 256 && D != 512) || R0 < 0 || R <= R0 || (mask && !(keep > 0.f)) ||
      (head_w && (!head_b || !logit)) || (tangent && (!xhat || !rstd || pair_off < 1 || R0 < pair_off)) || (!tangent && !rstd)) {
    set_last_error("serl_vice_ln_act_fwd: invalid arguments (D 256 | 512, act tanh | leaky_relu)"); return SERL_ERR_INVALID;
  }
  const dim3 g(ceil_div(R - R0, 8));
  if (D == 256) launch_fwd<8>(act, g, ST(stream), z, ld_z, pre_bias, mask, ld_mask, keep, scale, bias, y, ld_y, xhat, rstd, head_w, head_b, logit, R0, R, pair_off, tangent, eps);
  else launch_fwd<16>(act, g, ST(stream), z, ld_z, pre_bias, mask, ld_mask, keep, scale, bias, y, ld_y, xhat, rstd, head_w, head_b, logit, R0, R, pair_off, tangent, eps);
  return check_launch("vice_ln_act_fwd_kernel");
}

extern "C" int serl_vice_ln_act_bwd(const float* dy, int ld_dy, const float* dlogit, float dlogit_const, const float* head_w, float tan_seed,
                                    const float* xhat, const float* rstd, const float* z, int ld_z, const uint8_t* mask, int ld_mask, float keep,
                                    const float* scale, const float* bias, const float* y, int ld_y, float* dz, int ld_dz, float* dscale_rows,
                                    float* dbias_rows, float* dw_rows, int R0, int R, int R_pair, int D, int act, void* stream) {
  const bool ok_act = act == SERL_ACT_TANH || act == SERL_ACT_LEAKY_RELU;
  if (!xhat || !rstd || !scale || !bias || !dz || !ok_act || (D != 256 && D != 512) || R0 < 0 || R <= R0 || R_pair < 0 ||
      R_pair > R - R0 || (mask && !(keep > 0.f)) || (!head_w && !dy) || (R_pair && !z) || (dw_rows && (!head_w || !y))) {
    set_last_error("serl_vice_ln_act_bwd: invalid arguments (D 256 | 512, act tanh | leaky_relu)"); return SERL_ERR_INVALID;
  }
  const dim3 g(ceil_div(R - R0, 8));
  if (D == 256) launch_bwd<8>(act, g, ST(stream), dy, ld_dy, dlogit, dlogit_const, head_w, tan_seed, xhat, rstd, z, ld_z, mask, ld_mask, keep, scale, bias, y, ld_y, dz, ld_dz, dscale_rows, dbias_rows, dw_rows, R0, R, R_pair);
  else launch_bwd<16>(act, g, ST(stream), dy, ld_dy, dlogit, dlogit_const, head_w, tan_seed, xhat, rstd, z, ld_z, mask, ld_mask, keep, scale, bias, y, ld_y, dz, ld_dz, dscale_rows, dbias_rows, dw_rows, R0, R, R_pair);
  return check_launch("vice_ln_act_bwd_kernel");
}

extern "C" int serl_vice_sle_input_grad(const float* ds, int ld_ds, const float* kernel, float* dx, int R, int P, int C, void* stream) {
  if (!ds || !kernel || !dx || R < 1 || P < 1 || C < 1 || (ld_ds & 3) || (reinterpret_cast<uintptr_t>(ds) & 15) || (reinterpret_cast<uintptr_t>(kernel) & 15)) {
    set_last_error("serl_vice_sle_input_grad: invalid arguments (16-byte aligned ds / kernel, ld_ds % 4 == 0)"); return SERL_ERR_INVALID;
  }
  launch_k(vice_sle_input_grad_kernel, grid_for((long long)R * P * C), 256, 0, ST(stream), ds, ld_ds, kernel, dx, R, P, C);
  return check_launch("vice_sle_input_grad_kernel");
}

extern "C" int serl_vice_mask_fill(const uint32_t* key, int fold, float keep, uint8_t* out, int rows, int n, int broadcast, void* stream) {
  if (!key || !out || rows < 1 || n < 1 || !(keep > 0.f)) { set_last_error("serl_vice_mask_fill: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(vice_mask_fill_kernel, grid_for((long long)rows * n), 256, 0, ST(stream), key, fold, keep, out, rows, n, broadcast);
  return check_launch("vice_mask_fill_kernel");
}

extern "C" int serl_vice_gp_rows(const float* g, long long g_stride, float* v, long long v_stride, float coef, float* norms, int ncams, int B,
                                 int D, void* stream) {
  if (!g || !v || !norms || ncams < 1 || B < 1 || D < 1) { set_last_error("serl_vice_gp_rows: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(vice_gp_rows_kernel, dim3(B, ncams), 256, 0, ST(stream), g, g_stride, v, v_stride, coef, norms, B, D);
  return check_launch("vice_gp_rows_kernel");
}

extern "C" int serl_vice_gp_finish(const float* norms, int M, float gp_weight, float info_scale, float* info, void* stream) {
  if (!norms || !info || M < 1) { set_last_error("serl_vice_gp_finish: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(vice_gp_finish_kernel, 1, 256, 0, ST(stream), norms, M, gp_weight, info_scale, info);
  return check_launch("vice_gp_finish_kernel");
}

extern "C" int serl_vice_reward(const float* logit, float* rewards, float* mean_out, int B, int threshold, void* stream) {
  if (!logit || !rewards || B < 1) { set_last_error("serl_vice_reward: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(vice_reward_kernel, 1, 256, 0, ST(stream), logit, rewards, mean_out, B, threshold);
  return check_launch("vice_reward_kernel");
}
