// Batched CUDA-core companions of the TF32 head GEMMs (tgemm.cu): the parts of the trainable heads that are reductions or
// element-wise, each as ONE launch over every problem of a step instead of one launch per (camera, pass, layer):
//   sle_fwd_multi     SpatialLearnedEmbeddings (+ Dropout) of several (features, kernel) pairs        (vision/resnet_v1.py:81-116, :352)
//   enc_finish        k-split partial sums of Dense(4096 -> 256) -> + bias -> LayerNorm -> tanh for several problems, and the
//                     proprio Dense(S -> 64) -> LayerNorm -> tanh (fan-in too small / unaligned for TMA)   (resnet_v1.py:371-374,
//                     common/encoding.py:55-70)
//   ln_tanh_bwd_multi LayerNorm + tanh backward for several problems; the upstream gradient may be the outer product
//                     dQ (x) w of the value head (networks/actor_critic_nets.py:64-72)
//   small_grads       every bias / LayerNorm scale / LayerNorm bias / value-head gradient of an MLP: column reductions over
//                     the rows of each ensemble member                                               (networks/mlp.py:22-31)
// Same arithmetic as the single-problem kernels in heads.cu (which the fp32 build keeps using).
#include "common.cuh"
#include "serl_b200.h"

namespace serl {

// ---- SpatialLearnedEmbeddings forward, P problems: thread per (n, c), F == 8 ------------------------------------------
struct SleMultiArgs { serl_sle_problem p[SERL_HEADS_MAX_PROBLEMS]; int P, N, Pp, C; float keep; };

__global__ void sle_fwd_multi_kernel(const __grid_constant__ SleMultiArgs a) {
  pdl_prologue();
  const serl_sle_problem& q = a.p[blockIdx.y];
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.N * a.C) return;
  const int n = e / a.C, c = e - n * a.C;
  float acc[8];
#pragma unroll
  for (int f = 0; f < 8; ++f) acc[f] = 0.f;
  for (int p = 0; p < a.Pp; ++p) {
    const float v = q.feat[((size_t)n * a.Pp + p) * a.C + c];
    const float4 k0 = *reinterpret_cast<const float4*>(q.kernel + ((size_t)p * a.C + c) * 8);
    const float4 k1 = *reinterpret_cast<const float4*>(q.kernel + ((size_t)p * a.C + c) * 8 + 4);
    acc[0] = fmaf(v, k0.x, acc[0]); acc[1] = fmaf(v, k0.y, acc[1]); acc[2] = fmaf(v, k0.z, acc[2]); acc[3] = fmaf(v, k0.w, acc[3]);
    acc[4] = fmaf(v, k1.x, acc[4]); acc[5] = fmaf(v, k1.y, acc[5]); acc[6] = fmaf(v, k1.z, acc[6]); acc[7] = fmaf(v, k1.w, acc[7]);
  }
  if (q.keep_mask) {
    const uint8_t* mk = q.keep_mask + (size_t)n * a.C * 8 + c * 8;
#pragma unroll
    for (int f = 0; f < 8; ++f) acc[f] = mk[f] ? acc[f] / a.keep : 0.f;
  }
  float* o = q.out + (size_t)n * q.ld_out + c * 8;
  *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// ---- SLE kernel gradient, P problems: partial[problem][chunk][p][c][f] = sum_{n in chunk} feat[n,p,c] * dout[n, c*8+f] ----------
struct SleBwdArgs { serl_sle_bwd_problem p[SERL_HEADS_MAX_PROBLEMS]; float* partial; int P, N, Pp, C, chunks; };

__global__ void sle_bwd_partial_multi_kernel(const __grid_constant__ SleBwdArgs a) {
  pdl_prologue();
  const serl_sle_bwd_problem& q = a.p[blockIdx.z];
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.Pp * a.C) return;
  const int p = e / a.C, c = e - p * a.C;
  const int ch = blockIdx.y;
  const int per = ceil_div(a.N, a.chunks);
  const int n0 = ch * per, n1 = min(a.N, n0 + per);
  float acc[8];
#pragma unroll
  for (int f = 0; f < 8; ++f) acc[f] = 0.f;
  for (int n = n0; n < n1; ++n) {
    const float v = q.feat[((size_t)n * a.Pp + p) * a.C + c];
    const float4 d0 = *reinterpret_cast<const float4*>(q.dout + (size_t)n * q.ld_dout + c * 8);
    const float4 d1 = *reinterpret_cast<const float4*>(q.dout + (size_t)n * q.ld_dout + c * 8 + 4);
    acc[0] = fmaf(v, d0.x, acc[0]); acc[1] = fmaf(v, d0.y, acc[1]); acc[2] = fmaf(v, d0.z, acc[2]); acc[3] = fmaf(v, d0.w, acc[3]);
    acc[4] = fmaf(v, d1.x, acc[4]); acc[5] = fmaf(v, d1.y, acc[5]); acc[6] = fmaf(v, d1.z, acc[6]); acc[7] = fmaf(v, d1.w, acc[7]);
  }
  float* o = a.partial + (((size_t)blockIdx.z * a.chunks + ch) * a.Pp * a.C + e) * 8;
  *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// dkernel[problem][d] = sum_chunk partial[problem][chunk][d]: thread per 4 elements, fixed order
__global__ void sle_bwd_reduce_multi_kernel(const __grid_constant__ SleBwdArgs a) {
  pdl_prologue();
  const serl_sle_bwd_problem& q = a.p[blockIdx.y];
  const size_t D4 = (size_t)a.Pp * a.C * 2;                         // float4 elements
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D4) return;
  const float4* src = reinterpret_cast<const float4*>(a.partial) + (size_t)blockIdx.y * a.chunks * D4 + i;
  float4 s = src[0];
  for (int ch = 1; ch < a.chunks; ++ch) { const float4 v = src[(size_t)ch * D4]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
  reinterpret_cast<float4*>(q.dkernel)[i] = s;
}

// ---- encoder finish: warp per row ---------------------------------------------------------------------------------------
struct EncFinishArgs { serl_enc_finish_problem p[SERL_HEADS_MAX_PROBLEMS]; int P, rows; float eps; };

__global__ void __launch_bounds__(256) enc_finish_kernel(const __grid_constant__ EncFinishArgs a) {
  pdl_prologue();
  const serl_enc_finish_problem& q = a.p[blockIdx.y];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= a.rows) return;
  const int D = q.D;                                              // 256 (image head) or 64 (proprio)
  float v[8];
  if (q.partials) {                                               // sum of the k-split partial products, fixed order
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    for (int s = 0; s < q.S; ++s) {
      const float* pr = q.partials + ((size_t)s * a.rows + row) * D;
#pragma unroll
      for (int j = 0; j < 8; ++j) if (lane + 32 * j < D) v[j] += pr[lane + 32 * j];
    }
  } else {                                                        // small dense: x (rows, K) @ w (K, D)
    const float* x = q.x + (size_t)row * q.ld_x;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    for (int k = 0; k < q.K; ++k) {
      const float xv = x[k];
#pragma unroll
      for (int j = 0; j < 8; ++j) if (lane + 32 * j < D) v[j] = fmaf(xv, q.w[(size_t)k * D + lane + 32 * j], v[j]);
    }
  }
  float s = 0.f, ss = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) if (lane + 32 * j < D) { v[j] += q.bias[lane + 32 * j]; s += v[j]; ss += v[j] * v[j]; }
  s = warp_sum(s); ss = warp_sum(ss);
  const float mean = s / (float)D;
  const float var = fmaxf(ss / (float)D - mean * mean, 0.f);
  const float rstd = rsqrtf(var + a.eps);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = lane + 32 * j;
    if (d < D) {
      const float xh = (v[j] - mean) * rstd;
      q.out[(size_t)row * q.ld_out + d] = tanhf(xh * q.ln_scale[d] + q.ln_bias[d]);
      if (q.xhat) q.xhat[(size_t)row * D + d] = xh;
    }
  }
  if (q.rstd && lane == 0) q.rstd[row] = rstd;
}

// ---- LayerNorm + tanh backward, P problems: warp per row (same formulas as ln_tanh_bwd_kernel, heads.cu) ----------------
struct LnBwdArgs { serl_ln_bwd_problem p[SERL_HEADS_MAX_PROBLEMS]; int P; };
// MLP Dropout ahead of the LayerNorm (serl_layernorm_tanh_bwd_multi_masked): row r of problem i reads mask row r % mask_rows
struct LnBwdMask { const uint8_t* mask[SERL_HEADS_MAX_PROBLEMS]; int mask_rows; float inv_keep; };

// kMask: dz *= mask ? inv_keep : 0 (dy, the LayerNorm parameter gradients' input, is not masked).  The instantiation without it is
// ln_tanh_bwd_multi_kernel, unchanged.
template <bool kMask>
__device__ __forceinline__ void ln_tanh_bwd_multi_body(const LnBwdArgs& a, const LnBwdMask& mk) {
  pdl_prologue();
  const serl_ln_bwd_problem& q = a.p[blockIdx.y];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= q.R) return;
  const int D = q.D, g = row / q.rows_per_group;
  const float* sc = q.scale + (size_t)g * q.group_stride;
  float dqv = 0.f;
  const float* hw = nullptr;
  if (q.dq) { dqv = q.dq[row]; hw = q.head_w + (size_t)g * q.head_w_stride; }
  float dy[8], xh[8];
  float m1 = 0.f, m2 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = lane + 32 * j;
    dy[j] = 0.f; xh[j] = 0.f;
    if (d < D) {
      const float tv = q.t[(size_t)row * q.ld_t + d];
      float dt;
      if (q.dq) dt = dqv * hw[d];
      else {
        dt = q.dt[(size_t)row * q.ld_dt + d];
        for (int pp = 1; pp < q.dt_parts; ++pp) dt += q.dt[(size_t)pp * q.dt_part_stride + (size_t)row * q.ld_dt + d];   // fixed order
      }
      if (q.dt2) dt += q.dt2[(size_t)row * q.ld_dt2 + d];
      dy[j] = dt * (1.f - tv * tv);
      xh[j] = q.xhat[(size_t)row * D + d];
      const float dxh = dy[j] * sc[d];
      m1 += dxh; m2 += dxh * xh[j];
      if (q.dy) q.dy[(size_t)row * D + d] = dy[j];
    }
  }
  m1 = warp_sum(m1) / (float)D; m2 = warp_sum(m2) / (float)D;
  const float rs = q.rstd[row];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int d = lane + 32 * j;
    if (d < D) {
      float v = rs * (dy[j] * sc[d] - m1 - xh[j] * m2);
      if constexpr (kMask) v = mk.mask[blockIdx.y][(size_t)(row % mk.mask_rows) * D + d] ? v * mk.inv_keep : 0.f;
      q.dz[(size_t)row * D + d] = v;
    }
  }
}

__global__ void __launch_bounds__(256) ln_tanh_bwd_multi_kernel(const __grid_constant__ LnBwdArgs a) {
  ln_tanh_bwd_multi_body<false>(a, LnBwdMask{});
}

__global__ void __launch_bounds__(256) ln_tanh_bwd_multi_mask_kernel(const __grid_constant__ LnBwdArgs a, const __grid_constant__ LnBwdMask mk) {
  ln_tanh_bwd_multi_body<true>(a, mk);
}

// ---- column reductions: block = 32 columns x 32 row-slices, four rows in flight per thread, fixed-order tree (deterministic) ----
struct SmallGradArgs { serl_small_grad_job j[SERL_SMALL_GRAD_MAX_JOBS]; int J; };

__global__ void __launch_bounds__(1024) small_grads_kernel(const __grid_constant__ SmallGradArgs a) {
  pdl_prologue();
  __shared__ float ra[32][33], rb[32][33];
  const serl_small_grad_job& q = a.j[blockIdx.z];
  const int cx = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const int g = blockIdx.y, d = blockIdx.x * 32 + cx;
  if (g >= q.groups || blockIdx.x * 32 >= q.D) return;            // uniform per block
  float sa = 0.f, sb = 0.f;
  if (d < q.D) {
    const float* xp = q.x + (size_t)g * q.rows * q.ld_x + d;
    if (q.kind == SERL_SMALL_GRAD_COLSUM) {
      int r = sl;
      for (; r + 96 < q.rows; r += 128) {
        const float x0 = xp[(size_t)r * q.ld_x], x1 = xp[(size_t)(r + 32) * q.ld_x], x2 = xp[(size_t)(r + 64) * q.ld_x], x3 = xp[(size_t)(r + 96) * q.ld_x];
        sa += x0; sa += x1; sa += x2; sa += x3;
      }
      for (; r < q.rows; r += 32) sa += xp[(size_t)r * q.ld_x];
    } else if (q.kind == SERL_SMALL_GRAD_LN) {
      const float* yp = q.y + (size_t)g * q.rows * q.ld_y + d;
      int r = sl;
      for (; r + 96 < q.rows; r += 128) {
        const float x0 = xp[(size_t)r * q.ld_x], x1 = xp[(size_t)(r + 32) * q.ld_x], x2 = xp[(size_t)(r + 64) * q.ld_x], x3 = xp[(size_t)(r + 96) * q.ld_x];
        const float y0 = yp[(size_t)r * q.ld_y], y1 = yp[(size_t)(r + 32) * q.ld_y], y2 = yp[(size_t)(r + 64) * q.ld_y], y3 = yp[(size_t)(r + 96) * q.ld_y];
        sa = fmaf(x0, y0, sa); sb += x0; sa = fmaf(x1, y1, sa); sb += x1; sa = fmaf(x2, y2, sa); sb += x2; sa = fmaf(x3, y3, sa); sb += x3;
      }
      for (; r < q.rows; r += 32) { const float x = xp[(size_t)r * q.ld_x]; sa = fmaf(x, yp[(size_t)r * q.ld_y], sa); sb += x; }
    } else {                                                      // SERL_SMALL_GRAD_HEAD: x = h (rows, D), y = dq (rows)
      const float* yp = q.y + (size_t)g * q.rows;
      int r = sl;
      for (; r + 96 < q.rows; r += 128) {
        const float x0 = xp[(size_t)r * q.ld_x], x1 = xp[(size_t)(r + 32) * q.ld_x], x2 = xp[(size_t)(r + 64) * q.ld_x], x3 = xp[(size_t)(r + 96) * q.ld_x];
        const float w0 = yp[r], w1 = yp[r + 32], w2 = yp[r + 64], w3 = yp[r + 96];
        sa = fmaf(x0, w0, sa); sb += w0; sa = fmaf(x1, w1, sa); sb += w1; sa = fmaf(x2, w2, sa); sb += w2; sa = fmaf(x3, w3, sa); sb += w3;
      }
      for (; r < q.rows; r += 32) { const float w = yp[r]; sa = fmaf(xp[(size_t)r * q.ld_x], w, sa); sb += w; }
    }
  }
  ra[sl][cx] = sa; rb[sl][cx] = sb;
  __syncthreads();
  if (sl == 0 && d < q.D) {
    float ta = ra[0][cx], tb = rb[0][cx];
#pragma unroll
    for (int k = 1; k < 32; ++k) { ta += ra[k][cx]; tb += rb[k][cx]; }
    q.out_a[(size_t)g * q.D + d] = ta;
    if (q.out_b && q.kind == SERL_SMALL_GRAD_LN) q.out_b[(size_t)g * q.D + d] = tb;
    if (q.out_b && q.kind == SERL_SMALL_GRAD_HEAD && d == 0) q.out_b[g] = tb;
  }
}

}  // namespace serl

using namespace serl;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int serl_sle_fwd_multi(const serl_sle_problem* problems, int num_problems, float keep, int N, int P, int C, int F, void* stream) {
  if (!problems || num_problems < 1 || num_problems > SERL_HEADS_MAX_PROBLEMS || F != 8) { set_last_error("serl_sle_fwd_multi: 1..%d problems, num_features 8", SERL_HEADS_MAX_PROBLEMS); return SERL_ERR_INVALID; }
  SleMultiArgs a{};
  for (int i = 0; i < num_problems; ++i) {
    a.p[i] = problems[i];
    if (!a.p[i].feat || !a.p[i].kernel || !a.p[i].out || (a.p[i].ld_out & 3)) { set_last_error("serl_sle_fwd_multi: problem %d invalid", i); return SERL_ERR_INVALID; }
  }
  a.P = num_problems; a.N = N; a.Pp = P; a.C = C; a.keep = keep;
  launch_k(sle_fwd_multi_kernel, dim3(ceil_div(N * C, 128), num_problems), 128, 0, ST(stream), a);
  return check_launch("sle_fwd_multi_kernel");
}

extern "C" int serl_sle_bwd_multi(const serl_sle_bwd_problem* problems, int num_problems, float* workspace, size_t workspace_bytes,
                                  int N, int P, int C, int F, void* stream) {
  if (!problems || num_problems < 1 || num_problems > SERL_HEADS_MAX_PROBLEMS || F != 8) { set_last_error("serl_sle_bwd_multi: 1..%d problems, num_features 8", SERL_HEADS_MAX_PROBLEMS); return SERL_ERR_INVALID; }
  SleBwdArgs a{};
  for (int i = 0; i < num_problems; ++i) {
    a.p[i] = problems[i];
    if (!a.p[i].feat || !a.p[i].dout || !a.p[i].dkernel || (a.p[i].ld_dout & 3) || (reinterpret_cast<uintptr_t>(a.p[i].dkernel) & 15)) {
      set_last_error("serl_sle_bwd_multi: problem %d invalid", i); return SERL_ERR_INVALID;
    }
  }
  int chunks = N >= 64 ? 16 : 1;
  const size_t per = (size_t)P * C * F * sizeof(float) * num_problems;
  while (chunks > 1 && per * chunks > workspace_bytes) chunks >>= 1;
  if (!workspace || per * chunks > workspace_bytes) { set_last_error("serl_sle_bwd_multi: workspace too small (%zu needed)", per); return SERL_ERR_INVALID; }
  a.partial = workspace; a.P = num_problems; a.N = N; a.Pp = P; a.C = C; a.chunks = chunks;
  launch_k(sle_bwd_partial_multi_kernel, dim3(ceil_div(P * C, 128), chunks, num_problems), 128, 0, ST(stream), a);
  if (int e = check_launch("sle_bwd_partial_multi_kernel")) return e;
  launch_k(sle_bwd_reduce_multi_kernel, dim3(ceil_div(P * C * 2, 256), num_problems), 256, 0, ST(stream), a);
  return check_launch("sle_bwd_reduce_multi_kernel");
}

extern "C" int serl_enc_finish(const serl_enc_finish_problem* problems, int num_problems, int rows, float eps, void* stream) {
  if (!problems || num_problems < 1 || num_problems > SERL_HEADS_MAX_PROBLEMS || rows < 1) { set_last_error("serl_enc_finish: 1..%d problems", SERL_HEADS_MAX_PROBLEMS); return SERL_ERR_INVALID; }
  EncFinishArgs a{};
  for (int i = 0; i < num_problems; ++i) {
    a.p[i] = problems[i];
    const serl_enc_finish_problem& q = a.p[i];
    if (!q.out || !q.bias || !q.ln_scale || !q.ln_bias || q.D < 1 || q.D > 256 || (!q.partials && (!q.x || !q.w || q.K < 1)) || (q.partials && q.S < 1)) {
      set_last_error("serl_enc_finish: problem %d invalid (D <= 256; partials + S, or x + w + K)", i); return SERL_ERR_INVALID;
    }
  }
  a.P = num_problems; a.rows = rows; a.eps = eps;
  launch_k(enc_finish_kernel, dim3(ceil_div(rows, 8), num_problems), 256, 0, ST(stream), a);
  return check_launch("enc_finish_kernel");
}

static int ln_bwd_multi_launch(const serl_ln_bwd_problem* problems, int num_problems, const uint8_t* const* masks, int mask_rows,
                               float inv_keep, void* stream) {
  if (!problems || num_problems < 1 || num_problems > SERL_HEADS_MAX_PROBLEMS) { set_last_error("serl_layernorm_tanh_bwd_multi: 1..%d problems", SERL_HEADS_MAX_PROBLEMS); return SERL_ERR_INVALID; }
  LnBwdArgs a{};
  int rmax = 0;
  for (int i = 0; i < num_problems; ++i) {
    a.p[i] = problems[i];
    const serl_ln_bwd_problem& q = a.p[i];
    if ((!q.dt && !q.dq) || (q.dq && !q.head_w) || !q.t || !q.xhat || !q.rstd || !q.scale || !q.dz || q.R < 1 || q.D < 1 || q.D > 256 || q.rows_per_group < 1) {
      set_last_error("serl_layernorm_tanh_bwd_multi: problem %d invalid", i); return SERL_ERR_INVALID;
    }
    rmax = q.R > rmax ? q.R : rmax;
  }
  a.P = num_problems;
  if (masks) {
    LnBwdMask mk{};
    if (mask_rows < 1 || !(inv_keep > 0.f)) { set_last_error("serl_layernorm_tanh_bwd_multi_masked: mask_rows >= 1 and inv_keep > 0 required"); return SERL_ERR_INVALID; }
    for (int i = 0; i < num_problems; ++i) {
      if (!masks[i]) { set_last_error("serl_layernorm_tanh_bwd_multi_masked: problem %d: mask required", i); return SERL_ERR_INVALID; }
      mk.mask[i] = masks[i];
    }
    mk.mask_rows = mask_rows; mk.inv_keep = inv_keep;
    launch_k(ln_tanh_bwd_multi_mask_kernel, dim3(ceil_div(rmax, 8), num_problems), 256, 0, ST(stream), a, mk);
    return check_launch("ln_tanh_bwd_multi_mask_kernel");
  }
  launch_k(ln_tanh_bwd_multi_kernel, dim3(ceil_div(rmax, 8), num_problems), 256, 0, ST(stream), a);
  return check_launch("ln_tanh_bwd_multi_kernel");
}

extern "C" int serl_layernorm_tanh_bwd_multi(const serl_ln_bwd_problem* problems, int num_problems, void* stream) {
  return ln_bwd_multi_launch(problems, num_problems, nullptr, 1, 1.f, stream);
}

extern "C" int serl_layernorm_tanh_bwd_multi_masked(const serl_ln_bwd_problem* problems, int num_problems, const uint8_t* const* masks,
                                                    int mask_rows, float inv_keep, void* stream) {
  if (!masks) { set_last_error("serl_layernorm_tanh_bwd_multi_masked: masks required"); return SERL_ERR_INVALID; }
  return ln_bwd_multi_launch(problems, num_problems, masks, mask_rows, inv_keep, stream);
}

extern "C" int serl_small_grads(const serl_small_grad_job* jobs, int num_jobs, void* stream) {
  if (!jobs || num_jobs < 1 || num_jobs > SERL_SMALL_GRAD_MAX_JOBS) { set_last_error("serl_small_grads: 1..%d jobs", SERL_SMALL_GRAD_MAX_JOBS); return SERL_ERR_INVALID; }
  SmallGradArgs a{};
  int gmax = 0, dmax = 0;
  for (int i = 0; i < num_jobs; ++i) {
    a.j[i] = jobs[i];
    const serl_small_grad_job& q = a.j[i];
    if (!q.x || !q.out_a || q.groups < 1 || q.rows < 1 || q.D < 1 || (q.kind != SERL_SMALL_GRAD_COLSUM && !q.y) || q.kind < 0 || q.kind > SERL_SMALL_GRAD_HEAD) {
      set_last_error("serl_small_grads: job %d invalid", i); return SERL_ERR_INVALID;
    }
    gmax = q.groups > gmax ? q.groups : gmax; dmax = q.D > dmax ? q.D : dmax;
  }
  a.J = num_jobs;
  launch_k(small_grads_kernel, dim3(ceil_div(dmax, 32), gmax, num_jobs), 1024, 0, ST(stream), a);
  return check_launch("small_grads_kernel");
}
