// SAC / DrQ loss-side kernels (fp32): JAX-compatible key schedule and random fills, tanh-Gaussian
// sample + log-prob, REDQ subsample-min TD target, the three losses with their analytic gradients,
// and the fused 3-optimizer Adam + polyak update.
//
// Reference (relative to serl_launcher/serl_launcher):
//   agents/continuous/sac.py:118-132   _compute_next_actions (policy forward, sample_and_log_prob)
//   agents/continuous/sac.py:134-191   critic_loss_fn   (subsample with replacement, min, TD target, MSE)
//   agents/continuous/sac.py:193-221   policy_loss_fn   (mean over the ensemble, -mean(q - alpha*logp))
//   agents/continuous/sac.py:223-234   temperature_loss_fn + networks/lagrange.py:9-78
//   agents/continuous/sac.py:243-299   update: key split order, rng bookkeeping
//   agents/continuous/drq.py:307-308   augmentation key split
//   networks/actor_critic_nets.py:178-272   Policy / TanhMultivariateNormalDiag
//   common/common.py:124-168           target_update, apply_gradients (3 Adam txs, all tick every call)
//   common/optimizers.py:6-56          Adam + warmup schedule
// Restated in oracle/drq.py (derive_update_randomness, tanh_normal_sample_logp, update, adam_tx_update).
#include <cstdio>

#include "common.cuh"
#include "serl_b200.h"

namespace serl {

// ---------------------------------------------------------------------------------------------
// Key schedule.  keys[] slots (2 words each): see SERL_KEY_* in serl_b200.h.
// ---------------------------------------------------------------------------------------------
__global__ void rng_schedule_kernel(uint32_t* rng, uint32_t* keys, int do_aug, int do_update) {
  pdl_prologue();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  u32x2 r{rng[0], rng[1]};
  auto put = [&](int slot, u32x2 k) { keys[2 * slot] = k.x; keys[2 * slot + 1] = k.y; };
  if (do_aug) {                                     // drq.py:307-308: rng, obs_rng, next_obs_rng = split(rng, 3)
    put(SERL_KEY_CROP_OBS, jax_split_at(r, 3, 1));
    put(SERL_KEY_CROP_NEXT, jax_split_at(r, 3, 2));
    r = jax_split_at(r, 3, 0);
  }
  if (do_update) {                                  // common.py:198-200: new_rng, actor, critic, temperature = split(rng, 4)
    const u32x2 k_actor = jax_split_at(r, 4, 1), k_critic = jax_split_at(r, 4, 2), k_temp = jax_split_at(r, 4, 3);
    const u32x2 c1 = jax_split_at(k_critic, 2, 0);  // sac.py:137  rng, next_action_sample_key = split(rng)
    put(SERL_KEY_CRITIC_NEXT, jax_split_at(k_critic, 2, 1));
    put(SERL_KEY_CRITIC_SUBSAMPLE, jax_split_at(c1, 2, 1));   // sac.py:152
    put(SERL_KEY_ACTOR_DROPOUT, jax_split_at(k_actor, 4, 1)); // sac.py:197  rng, policy_rng, sample_rng, critic_rng
    put(SERL_KEY_ACTOR_SAMPLE, jax_split_at(k_actor, 4, 2));
    put(SERL_KEY_TEMP_NEXT, jax_split_at(k_temp, 2, 1));      // sac.py:224
    r = jax_split_at(r, 2, 0);                      // sac.py:288  rng, _ = split(self.state.rng)
  }
  rng[0] = r.x; rng[1] = r.y;
}

// The critic-MLP dropout keys of one update (SERL_KEY_MLP_*), from the state rng BEFORE rng_schedule_kernel advances it (same
// do_aug): c1 = split(k_critic)[0] keys the target critic (sac.py:141-145: forward_target_critic's default train=True), c2 =
// split(c1)[0] the online critic when critic_subsample_size is set (sac.py:152,174-176; c1 otherwise), and the actor loss's
// critic_rng = split(k_actor, 4)[3] its critic forward (sac.py:197,203-207).  A separate launch, so rng_schedule_kernel and the
// agents without MLP dropout stay as they are.
__host__ __device__ inline void mlp_dropout_keys(u32x2 r, int do_aug, uint32_t* keys) {
  auto put = [&](int slot, u32x2 k) { keys[2 * slot] = k.x; keys[2 * slot + 1] = k.y; };
  if (do_aug) r = jax_split_at(r, 3, 0);
  const u32x2 k_actor = jax_split_at(r, 4, 1), k_critic = jax_split_at(r, 4, 2);
  const u32x2 c1 = jax_split_at(k_critic, 2, 0);
  put(SERL_KEY_MLP_CRITIC_TARGET, c1);
  put(SERL_KEY_MLP_CRITIC_SUBSAMPLED, jax_split_at(c1, 2, 0));
  put(SERL_KEY_MLP_ACTOR_CRITIC, jax_split_at(k_actor, 4, 3));
}

__global__ void mlp_dropout_keys_kernel(const uint32_t* rng, uint32_t* keys, int do_aug) {
  pdl_prologue();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  mlp_dropout_keys(u32x2{rng[0], rng[1]}, do_aug, keys);
}

// BCAgent.update's key chain: new_rng, k = split(rng) (common.py:198-200 with one loss); dropout key = split(k)[1] (bc.py:47);
// rng <- new_rng.  On the device so that a step needs no host round trip for its key and can be replayed from a CUDA graph.
__host__ __device__ inline void bc_key_chain(uint32_t* rng, uint32_t* key) {
  const u32x2 r{rng[0], rng[1]};
  const u32x2 drop = jax_split_at(jax_split_at(r, 2, 1), 2, 1), next = jax_split_at(r, 2, 0);
  key[0] = drop.x; key[1] = drop.y;
  rng[0] = next.x; rng[1] = next.y;
}

__global__ void bc_key_chain_kernel(uint32_t* rng, uint32_t* key) {
  pdl_prologue();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  bc_key_chain(rng, key);
}

__global__ void normal_fill_kernel(const uint32_t* key, float* out, int n) {
  pdl_prologue();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) out[j] = bits_to_normal(jax_random_bits_at(u32x2{key[0], key[1]}, (uint32_t)n, (uint32_t)j));
}

// keep-mask of camera `fold`: bernoulli(fold_in(key, fold), keep, (n,)) (repo spec, oracle/drq.py::_dropout_masks)
__global__ void dropout_mask_kernel(const uint32_t* key, uint32_t fold, float keep, uint8_t* mask, int n) {
  pdl_prologue();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const u32x2 k = jax_fold_in(u32x2{key[0], key[1]}, fold);
  mask[j] = bits_to_uniform01(jax_random_bits_at(k, (uint32_t)n, (uint32_t)j)) < keep ? 1 : 0;
}

// jax.random.randint(key, (n,), 0, ensemble) (sac.py:152-158): k1, k2 = split(key); element j combines word j of
// random_bits(k1, (n,)) and random_bits(k2, (n,)) exactly like jax_randint2 does for n = 2.
__global__ void subsample_idx_kernel(const uint32_t* key, int ensemble, int32_t* out, int n) {
  pdl_prologue();
  const int j = threadIdx.x;
  if (blockIdx.x != 0 || j >= n) return;
  const u32x2 k{key[0], key[1]};
  const uint32_t span = (uint32_t)ensemble;
  const uint32_t hb = jax_random_bits_at(jax_split_at(k, 2, 0), (uint32_t)n, (uint32_t)j);
  const uint32_t lb = jax_random_bits_at(jax_split_at(k, 2, 1), (uint32_t)n, (uint32_t)j);
  uint32_t mult = 65536u % span; mult = (mult * mult) % span;
  out[j] = (int)(((hb % span) * mult + (lb % span)) % span);
}

// ---------------------------------------------------------------------------------------------
// tanh-Gaussian: std = clip(exp(log_std), lo, hi); u = mu + std*eps; a = tanh(u);
// logp = sum_i [-0.5 z^2 - log std - 0.5 log 2pi] - sum_i 2 (log 2 - u - softplus(-2u)),  z = (u - mu)/std
// ---------------------------------------------------------------------------------------------
__device__ inline float softplusf(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// unclipped std of the std head's output x (SERL_STD_*; "uniform" is exp of the broadcast log_stds leaf, "fixed" the broadcast
// constant std itself)
template <int kStd>
__device__ __forceinline__ float raw_std(float x) {
  if constexpr (kStd == SERL_STD_SOFTPLUS) return softplusf(x);
  if constexpr (kStd == SERL_STD_FIXED) return x;
  return expf(x);
}

template <int kStd>
__global__ void tanh_gaussian_fwd_kernel(const float* __restrict__ mu, const float* __restrict__ log_std, int ld_ls,
                                         const float* __restrict__ eps, float std_min, float std_max,
                                         float* __restrict__ act, int ld_act, float* __restrict__ logp,
                                         float* __restrict__ u_out, float* __restrict__ std_out, int B, int A, int deterministic) {
  pdl_prologue();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float lp = 0.f;
  for (int i = 0; i < A; ++i) {
    const float m = mu[b * A + i];
    const float sd = fminf(fmaxf(raw_std<kStd>(log_std[b * ld_ls + i]), std_min), std_max);
    const float e = deterministic ? 0.f : eps[b * A + i];
    const float u = m + sd * e;
    const float z = (u - m) / sd;
    lp += -0.5f * z * z - logf(sd) - 0.918938533204672742f;
    lp -= 2.f * (0.693147180559945309f - u - softplusf(-2.f * u));
    act[(size_t)b * ld_act + i] = tanhf(u);
    if (u_out) u_out[b * A + i] = u;
    if (std_out) std_out[b * A + i] = sd;
  }
  if (logp) logp[b] = lp;
}

// ---------------------------------------------------------------------------------------------
// TD target + critic loss.  One CTA; E*B is a few thousand.
//   y_b = r_b + gamma * mask_b * min_j Q'[sub_j, b]  (- alpha * logp'_b if backup_entropy)
//   loss = mean_{e,b} (Q[e,b] - y_b)^2 ; dQ[e,b] = 2 (Q - y) / (E*B) * grad_scale
// info[0..2] = {critic_loss, mean Q, mean y} * grad_scale: grad_scale = 1/world under data parallelism, so that the ONE
// SUM all-reduce that carries the gradients also turns the per-rank infos into their mean (jax.lax.pmean(grads_and_aux),
// common.py:213-214); 1 otherwise.  Same convention in actor_loss_kernel / temperature_loss_kernel.
// kWeighted (prioritized replay, serl_critic_loss_weighted): row b's terms carry its importance weight w_b,
//   loss = sum_{e,b} w_b (Q - y)^2 / (E*B) ; dQ[e,b] = 2 w_b (Q - y) / (E*B) * grad_scale,
// and delta_b = (sum_e |Q[e,b] - y_b|, e ascending) / E is the row's TD error.  w_b * d is formed first, so w = 1 gives the
// unweighted kernel's bits.
// ---------------------------------------------------------------------------------------------
template <bool kWeighted>
__device__ __forceinline__ void critic_loss_body(const float* __restrict__ q, const float* __restrict__ q_next,
                                                 const int32_t* __restrict__ sub, int n_sub,
                                                 const float* __restrict__ rewards, const float* __restrict__ masks,
                                                 const float* __restrict__ logp_next, const float* __restrict__ lagrange,
                                                 int backup_entropy, float gamma, float grad_scale,
                                                 float* __restrict__ target_q, float* __restrict__ dq,
                                                 float* __restrict__ info, int E, int B,
                                                 const float* __restrict__ w, float* __restrict__ delta) {
  pdl_prologue();
  __shared__ float red[64];
  float sl = 0.f, sq = 0.f, sy = 0.f, dummy = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float mn;
    if (n_sub > 0) {
      mn = q_next[(size_t)sub[0] * B + b];
      for (int j = 1; j < n_sub; ++j) mn = fminf(mn, q_next[(size_t)sub[j] * B + b]);
    } else {
      mn = q_next[b];
      for (int e = 1; e < E; ++e) mn = fminf(mn, q_next[(size_t)e * B + b]);
    }
    float y = rewards[b] + gamma * masks[b] * mn;
    if (backup_entropy) y -= softplusf(lagrange[0]) * logp_next[b];
    target_q[b] = y;
    sy += y;
    if constexpr (kWeighted) {
      const float wb = w[b];
      float sabs = 0.f;
      for (int e = 0; e < E; ++e) {
        const float d = __fsub_rn(q[(size_t)e * B + b], y);
        const float wd = __fmul_rn(wb, d);
        sl += wd * d; sq += q[(size_t)e * B + b];
        dq[(size_t)e * B + b] = 2.f * wd / (float)(E * B) * grad_scale;
        sabs = __fadd_rn(sabs, fabsf(d));
      }
      delta[b] = __fdiv_rn(sabs, (float)E);
    } else {
      for (int e = 0; e < E; ++e) {
        const float d = q[(size_t)e * B + b] - y;
        sl += d * d; sq += q[(size_t)e * B + b];
        dq[(size_t)e * B + b] = 2.f * d / (float)(E * B) * grad_scale;
      }
    }
  }
  block_sum2(sl, sq, red);
  block_sum2(sy, dummy, red);
  if (threadIdx.x == 0) { info[0] = grad_scale * sl / (float)(E * B); info[1] = grad_scale * sq / (float)(E * B); info[2] = grad_scale * sy / (float)B; }
}

__global__ void __launch_bounds__(1024) critic_loss_kernel(const float* __restrict__ q, const float* __restrict__ q_next,
                                                           const int32_t* __restrict__ sub, int n_sub,
                                                           const float* __restrict__ rewards, const float* __restrict__ masks,
                                                           const float* __restrict__ logp_next, const float* __restrict__ lagrange,
                                                           int backup_entropy, float gamma, float grad_scale,
                                                           float* __restrict__ target_q, float* __restrict__ dq,
                                                           float* __restrict__ info, int E, int B) {
  critic_loss_body<false>(q, q_next, sub, n_sub, rewards, masks, logp_next, lagrange, backup_entropy, gamma, grad_scale, target_q, dq,
                          info, E, B, nullptr, nullptr);
}

__global__ void __launch_bounds__(1024) critic_loss_weighted_kernel(const float* __restrict__ q, const float* __restrict__ q_next,
                                                                    const int32_t* __restrict__ sub, int n_sub,
                                                                    const float* __restrict__ rewards, const float* __restrict__ masks,
                                                                    const float* __restrict__ logp_next, const float* __restrict__ lagrange,
                                                                    int backup_entropy, float gamma, float grad_scale,
                                                                    float* __restrict__ target_q, float* __restrict__ dq,
                                                                    float* __restrict__ info, int E, int B,
                                                                    const float* __restrict__ w, float* __restrict__ delta) {
  critic_loss_body<true>(q, q_next, sub, n_sub, rewards, masks, logp_next, lagrange, backup_entropy, gamma, grad_scale, target_q, dq,
                         info, E, B, w, delta);
}

// ---------------------------------------------------------------------------------------------
// Actor loss: L = -mean_b(qbar_b - alpha * logp_b), qbar = mean_e Q_e(s, a).
// Backward w.r.t. the policy head outputs, given da = dL/da from the critic input-gradient
// (critic seeded with dQ[e,b] = -1/(E*B)):
//   du_i = da_i (1 - a_i^2) + (alpha/B) * 2 a_i ;  dmu_i = du_i ;
//   dlogstd_i = [du_i * std_i * eps_i - alpha/B] * 1[std unclipped]          (exp, uniform: d std/d x = std)
//   dx_i = [du_i * eps_i - alpha/(B std_i)] * sigmoid(x_i) * 1[std unclipped]  (softplus)
// info[0..2] = {actor_loss, temperature(alpha), entropy}
// ---------------------------------------------------------------------------------------------
template <int kStd>
__global__ void __launch_bounds__(1024) actor_loss_kernel(const float* __restrict__ q, const float* __restrict__ logp,
                                                          const float* __restrict__ lagrange, const float* __restrict__ da, int ld_da,
                                                          const float* __restrict__ act, int ld_act, const float* __restrict__ std,
                                                          const float* __restrict__ log_std, int ld_ls, const float* __restrict__ eps,
                                                          float std_min, float std_max, float grad_scale,
                                                          float* __restrict__ dmu, float* __restrict__ dlogstd,
                                                          float* __restrict__ info, int E, int B, int A) {
  pdl_prologue();
  __shared__ float red[64];
  const float alpha = softplusf(lagrange[0]);
  float sobj = 0.f, slp = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float qb = 0.f;
    for (int e = 0; e < E; ++e) qb += q[(size_t)e * B + b];
    qb /= (float)E;
    sobj += qb - alpha * logp[b];
    slp += logp[b];
    for (int i = 0; i < A; ++i) {
      const float a = act[(size_t)b * ld_act + i];
      const float du = da[(size_t)b * ld_da + i] * (1.f - a * a) + grad_scale * (alpha / (float)B) * 2.f * a;
      dmu[b * A + i] = du;
      const float x = log_std[b * ld_ls + i];
      const float raw = raw_std<kStd>(x);
      const bool inside = raw >= std_min && raw <= std_max;
      if constexpr (kStd == SERL_STD_SOFTPLUS) {
        const float sig = 1.f / (1.f + expf(-x));
        dlogstd[b * A + i] = inside ? (du * eps[b * A + i] - grad_scale * alpha / ((float)B * std[b * A + i])) * sig : 0.f;
      } else {
        dlogstd[b * A + i] = inside ? (du * std[b * A + i] * eps[b * A + i] - grad_scale * alpha / (float)B) : 0.f;
      }
    }
  }
  block_sum2(sobj, slp, red);
  if (threadIdx.x == 0) { info[0] = grad_scale * -sobj / (float)B; info[1] = grad_scale * alpha; info[2] = grad_scale * -slp / (float)B; }
}

// dQ seed for the actor pass: every entry -grad_scale/(E*B)
__global__ void fill_kernel(float* x, float v, int n) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = v;
}

// Temperature loss: L = softplus(lambda) * (entropy - target), entropy = -mean logp'.  dL/dlambda = sigmoid(lambda) * (...)
__global__ void __launch_bounds__(1024) temperature_loss_kernel(const float* __restrict__ logp, const float* __restrict__ lagrange,
                                                                float target_entropy, float grad_scale, float* __restrict__ dlagrange,
                                                                float* __restrict__ info, int B) {
  pdl_prologue();
  __shared__ float red[64];
  float s = 0.f, dummy = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) s += logp[b];
  block_sum2(s, dummy, red);
  if (threadIdx.x == 0) {
    const float ent = -s / (float)B, lam = lagrange[0];
    info[0] = grad_scale * softplusf(lam) * (ent - target_entropy);
    dlagrange[0] = grad_scale * (1.f / (1.f + expf(-lam))) * (ent - target_entropy);
  }
}

// ---------------------------------------------------------------------------------------------
// Fused optimizer step over the flat trainable buffer.
// Every `update` call ticks all three txs (common.py:142-147).  A trainable leaf whose gradient under a tx is
// identically zero keeps zero moments and a zero update there, so only the txs that ever see a non-zero gradient
// need state: one per leaf, except the proprio-encoder leaves [aux_lo, aux_hi), which the critic loss AND the actor
// loss both differentiate (encoding.py:48-70: stop_gradient covers the image embeddings only) - they carry a second
// (actor-tx) moment pair in the aux tail.  For group gid: g = live ? grad : 0.
//   m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; p += -lr_t * (m / (1-b1^t)) / (sqrt(v / (1-b2^t)) + eps)
// then, if polyak: target = p_new * tau + target * (1 - tau)   (common.py:131-133, over the whole tree).
// counts[3] (device, int32) are incremented by the tail thread; lr_t follows optimizers.py:23-29.
// ---------------------------------------------------------------------------------------------
struct AdamArgs {
  float* p; float* target; float* m; float* v; const float* grad;
  int n;
  int seg_end[3];            // flat layout: [0,seg_end[0]) group 0, gap, [seg_end[0]+gap,seg_end[1]) group 1, ...
  int live[3];
  int32_t* counts;           // per group
  float lr[3]; int warmup[3];
  float b1, b2, eps, tau;
  int polyak;
  float* lr_out;             // (3) learning rates actually used (info["*_lr"])
  int gap, aux_lo, aux_hi, aux_off;   // info gap after group 0; leaves with a second (actor-tx) Adam state at [i + aux_off]
  // serl_adam_polyak_opts only (kOpts): per-tx global-norm clip thresholds (<= 0: off), cosine decay steps (<= 0: off)
  float clip[3]; int decay[3];
  const float* norms;
};

// learning rate of tx gid at optax count cnt (inject_hyperparams evaluates the schedule before the count increments)
template <bool kOpts>
__device__ inline float sched_lr(const AdamArgs& a, int gid, int cnt) {
  if (kOpts && a.decay[gid] > 0 && cnt >= a.warmup[gid]) {
    // warmup_cosine_decay_schedule, decay branch: lr * 0.5 (1 + cos(pi * min(c - w, D - w) / (D - w)))
    const int span = a.decay[gid] - a.warmup[gid];
    const float x = (float)min(cnt - a.warmup[gid], span) / (float)span;
    return a.lr[gid] * (0.5f * (1.f + cospif(x)));
  }
  return cnt < a.warmup[gid] ? a.lr[gid] * ((float)cnt / (float)a.warmup[gid]) : a.lr[gid];
}

// clip_by_global_norm ahead of the Adam moments: g unchanged if norm < max_norm, else (g / norm) * max_norm
template <bool kOpts>
__device__ inline float clip_grad(const AdamArgs& a, int gid, float g) {
  if (kOpts && a.clip[gid] > 0.f) {
    const float nrm = a.norms[gid];
    if (!(nrm < a.clip[gid])) g = (g / nrm) * a.clip[gid];
  }
  return g;
}

// one optax adam transform on one element: returns the update -lr * mhat / (sqrt(vhat) + eps)
template <bool kOpts>
__device__ inline float adam_update(const AdamArgs& a, int gid, float g, float* mp, float* vp) {
  const int cnt = a.counts[gid];
  const float t = (float)(cnt + 1);
  const float lr = sched_lr<kOpts>(a, gid, cnt);
  g = clip_grad<kOpts>(a, gid, g);
  const float m = a.b1 * *mp + (1.f - a.b1) * g;
  const float v = a.b2 * *vp + (1.f - a.b2) * g * g;
  *mp = m; *vp = v;
  const float mhat = m / (1.f - powf(a.b1, t));
  const float vhat = v / (1.f - powf(a.b2, t));
  return (mhat / (sqrtf(vhat) + a.eps)) * (-lr);             // optax: scale_by_adam then scale(-lr)
}

template <bool kOpts>
__device__ inline void adam_polyak_body(const AdamArgs& a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  if (i >= a.seg_end[0] && i < a.seg_end[0] + a.gap) return;   // info scalars, not parameters
  const int gid = i < a.seg_end[0] ? 0 : (i < a.seg_end[1] ? 1 : 2);
  float u = adam_update<kOpts>(a, gid, a.live[gid] ? a.grad[i] : 0.f, a.m + i, a.v + i);
  if (i >= a.aux_lo && i < a.aux_hi) {                         // second transform (actor tx); updates summed in tx order actor, critic
    const int j = i + a.aux_off;
    u = adam_update<kOpts>(a, 1, a.live[1] ? a.grad[j] : 0.f, a.m + j, a.v + j) + u;
  }
  const float pn = a.p[i] + u;
  a.p[i] = pn;
  if (a.polyak) a.target[i] = pn * a.tau + a.target[i] * (1.f - a.tau);
}

__global__ void adam_polyak_kernel(const AdamArgs a) {
  pdl_prologue();
  adam_polyak_body<false>(a);
}

__global__ void adam_polyak_opts_kernel(const AdamArgs a) {
  pdl_prologue();
  adam_polyak_body<true>(a);
}

// ---------------------------------------------------------------------------------------------
// Global gradient norm per tx (optax.global_norm over the gradient tree the tx receives, common.py:136-168).
// Pass 1: SERL_GRAD_NORM_CTAS CTAs stride over the buffer in float4s (every segment boundary is 16-byte aligned,
// params.py) and write fixed-order float64 partials.  Pass 2: one CTA sums them in a fixed order.  No atomics, so
// every data-parallel rank computes the same bits from the same all-reduced buffer.
// ---------------------------------------------------------------------------------------------
constexpr int kNormThreads = 256;

struct NormArgs {
  const float* grad;
  int n;                               // slots read: the parameter slots, or up to the end of the twin slots
  int s0, g0, s1, s2, x_lo, x_hi;      // [0,s0) tx 0 | gap | [g0,s1) tx 1 | [s1,s2) tx 2 | [x_lo,x_hi) tx 1 (twin slots)
  int want[3];                         // live and clipping
  double* partials;                    // [3][SERL_GRAD_NORM_CTAS]
  float* norms;
};

__device__ inline int norm_tx(const NormArgs& a, int i) {
  const int t = i < a.s0 ? 0 : i < a.g0 ? -1 : i < a.s1 ? 1 : i < a.s2 ? 2 : (i >= a.x_lo && i < a.x_hi) ? 1 : -1;
  return (t >= 0 && a.want[t]) ? t : -1;
}

// fixed-order block sum of three doubles; result valid in thread 0
__device__ inline void block_sum3_f64(double (&s)[3], double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < 3; ++k)
    for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_down_sync(0xffffffffu, s[k], o);
  if (lane == 0) for (int k = 0; k < 3; ++k) red[3 * warp + k] = s[k];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < 3; ++k) {
      double t = 0.0;
      for (int w = 0; w < nw; ++w) t += red[3 * w + k];
      s[k] = t;
    }
  }
}

__global__ void __launch_bounds__(kNormThreads) grad_sumsq_kernel(const NormArgs a) {
  pdl_prologue();
  __shared__ double red[3 * kNormThreads / 32];
  double s[3] = {0.0, 0.0, 0.0};
  const int n4 = a.n >> 2;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += gridDim.x * blockDim.x) {
    const int t = norm_tx(a, 4 * q);
    if (t < 0) continue;
    const float4 g = reinterpret_cast<const float4*>(a.grad)[q];
    const double v = (double)g.x * g.x + (double)g.y * g.y + (double)g.z * g.z + (double)g.w * g.w;
    s[0] += t == 0 ? v : 0.0; s[1] += t == 1 ? v : 0.0; s[2] += t == 2 ? v : 0.0;
  }
  if (blockIdx.x == 0) {                                 // scalar tail (n is a multiple of 4 for the agents' layouts)
    for (int i = 4 * n4 + threadIdx.x; i < a.n; i += blockDim.x) {
      const int t = norm_tx(a, i);
      if (t >= 0) s[t] += (double)a.grad[i] * a.grad[i];
    }
  }
  block_sum3_f64(s, red);
  if (threadIdx.x == 0)
    for (int k = 0; k < 3; ++k) a.partials[k * SERL_GRAD_NORM_CTAS + blockIdx.x] = s[k];
}

__global__ void __launch_bounds__(SERL_GRAD_NORM_CTAS) grad_norm_finish_kernel(const NormArgs a) {
  pdl_prologue();
  __shared__ double red[3 * SERL_GRAD_NORM_CTAS / 32];
  double s[3];
  for (int k = 0; k < 3; ++k) s[k] = a.partials[k * SERL_GRAD_NORM_CTAS + threadIdx.x];
  block_sum3_f64(s, red);
  if (threadIdx.x == 0)
    for (int k = 0; k < 3; ++k) a.norms[k] = a.want[k] ? (float)sqrt(s[k]) : 0.f;
}

// ---------------------------------------------------------------------------------------------
// Behaviour cloning (agents/continuous/bc.py:36-76): Dense -> tanh layers of the launcher's BC policy (MLP without LayerNorm,
// utils/launcher.py:26-47) and the loss  -mean_b log N(a_b; mu_b, diag(std_b^2)),  std = clip(exp(log_std), std_min, std_max).
// ---------------------------------------------------------------------------------------------
__global__ void tanh_fwd_kernel(const float* __restrict__ z, float* __restrict__ out, int n) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = tanhf(z[i]);
}
__global__ void tanh_bwd_kernel(const float* __restrict__ dt, const float* __restrict__ t, float* __restrict__ dz, int n) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const float tv = t[i]; dz[i] = dt[i] * (1.f - tv * tv); }
}
// info[0] = actor_loss, info[1] = mse (both * grad_scale: see critic_loss_kernel); one CTA, fixed-order reductions.
// Generalised over the std head (x = the head's (B, A) output; "uniform": the (A,) log_stds leaf broadcast over the rows, whose
// gradient is the caller's column sum of dx) and over the tanh squash (bc.py:46-69 with Policy's TanhMultivariateNormalDiag):
//   u = squash ? atanh(a) : a,  -logp = sum_j [0.5 ((u - mu)/std)^2 + log std + 0.5 log 2pi] (+ sum_j 2 (log 2 - u - softplus(-2u)))
//   mse = sum_j (mode - a)^2,  mode = squash ? tanh(mu) : mu.
// The log-det term holds no parameter, so dmu and dstd have the same form in u with and without the squash.  Clip ties: a std
// exactly on std_min / std_max passes no gradient (strictly inside only), as the <exp, no squash> instantiation (serl_bc_loss)
// always did; DESIGN.md section 5.  "fixed" (Policy's fixed_std): x is the constant (A,) std broadcast over the rows, and dx is not
// written.
template <int kStd, bool kSquash>
__global__ void __launch_bounds__(1024) bc_loss_kernel(const float* __restrict__ mu, const float* __restrict__ x, const float* __restrict__ act,
                                                       float std_min, float std_max, float grad_scale, float* __restrict__ dmu,
                                                       float* __restrict__ dx, float* __restrict__ info, int B, int A) {
  pdl_prologue();
  __shared__ float red[64];
  float sl = 0.f, sm = 0.f;
  const float inv = grad_scale / (float)B;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float lp = 0.f, se = 0.f;
    for (int j = 0; j < A; ++j) {
      const float m = mu[b * A + j], xs = x[(kStd == SERL_STD_UNIFORM || kStd == SERL_STD_FIXED) ? j : b * A + j], a = act[b * A + j];
      const float raw = raw_std<kStd>(xs);
      const float sd = fminf(fmaxf(raw, std_min), std_max);
      const float u = kSquash ? atanhf(a) : a;
      const float d = u - m, z = d / sd;
      lp += -0.5f * z * z - logf(sd) - 0.918938533204672742f;
      if constexpr (kSquash) {
        lp -= 2.f * (0.693147180559945309f - u - softplusf(-2.f * u));
        const float e = a - tanhf(m);
        se += e * e;
      } else {
        se += d * d;
      }
      dmu[b * A + j] = -(d / (sd * sd)) * inv;                                   // d(-logp)/dmu
      if constexpr (kStd == SERL_STD_FIXED) continue;                             // a constant std: no parameter, no gradient
      const float dsd = -(d * d / (sd * sd * sd) - 1.f / sd) * inv;               // d(-logp)/dstd
      if constexpr (kStd == SERL_STD_SOFTPLUS)                                    // clip passes the gradient strictly inside only
        dx[b * A + j] = (raw > std_min && raw < std_max) ? dsd * (1.f / (1.f + expf(-xs))) : 0.f;
      else
        dx[b * A + j] = (raw > std_min && raw < std_max) ? dsd * raw : 0.f;
    }
    sl -= lp; sm += se;
  }
  block_sum2(sl, sm, red);
  if (threadIdx.x == 0) { info[0] = sl * inv; info[1] = sm * inv; }
}

template <bool kOpts>
__global__ void adam_tick_kernel(const AdamArgs a) {
  pdl_prologue();
  const int gid = threadIdx.x;
  if (gid < 3) {
    const int cnt = a.counts[gid];
    if (a.lr_out) a.lr_out[gid] = sched_lr<kOpts>(a, gid, cnt);
    a.counts[gid] = cnt + 1;
  }
}

}  // namespace serl

using namespace serl;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int serl_rng_schedule(uint32_t* rng_state, uint32_t* keys, int do_aug, int do_update, void* stream) {
  launch_k(rng_schedule_kernel, 1, 32, 0, ST(stream), rng_state, keys, do_aug, do_update);
  return check_launch("rng_schedule_kernel");
}

extern "C" int serl_mlp_dropout_keys(const uint32_t* rng_state, uint32_t* keys, int do_aug, void* stream) {
  launch_k(mlp_dropout_keys_kernel, 1, 32, 0, ST(stream), rng_state, keys, do_aug);
  return check_launch("mlp_dropout_keys_kernel");
}

extern "C" int serl_bc_key_chain(uint32_t* rng_state, uint32_t* key, void* stream) {
  launch_k(bc_key_chain_kernel, 1, 32, 0, ST(stream), rng_state, key);
  return check_launch("bc_key_chain_kernel");
}

extern "C" int serl_host_bc_key_chain(uint32_t* rng, uint32_t* key) {
  bc_key_chain(rng, key);
  return SERL_OK;
}

extern "C" int serl_host_mlp_dropout_keys(const uint32_t* rng, uint32_t* keys, int do_aug) {
  mlp_dropout_keys(u32x2{rng[0], rng[1]}, do_aug, keys);
  return SERL_OK;
}

extern "C" int serl_host_rng_schedule(uint32_t* rng, uint32_t* keys, int do_aug, int do_update) {
  // host mirror of rng_schedule_kernel (same __host__ __device__ primitives) for CPU tests
  u32x2 r{rng[0], rng[1]};
  auto put = [&](int slot, u32x2 k) { keys[2 * slot] = k.x; keys[2 * slot + 1] = k.y; };
  if (do_aug) { put(SERL_KEY_CROP_OBS, jax_split_at(r, 3, 1)); put(SERL_KEY_CROP_NEXT, jax_split_at(r, 3, 2)); r = jax_split_at(r, 3, 0); }
  if (do_update) {
    const u32x2 k_actor = jax_split_at(r, 4, 1), k_critic = jax_split_at(r, 4, 2), k_temp = jax_split_at(r, 4, 3);
    const u32x2 c1 = jax_split_at(k_critic, 2, 0);
    put(SERL_KEY_CRITIC_NEXT, jax_split_at(k_critic, 2, 1));
    put(SERL_KEY_CRITIC_SUBSAMPLE, jax_split_at(c1, 2, 1));
    put(SERL_KEY_ACTOR_DROPOUT, jax_split_at(k_actor, 4, 1));
    put(SERL_KEY_ACTOR_SAMPLE, jax_split_at(k_actor, 4, 2));
    put(SERL_KEY_TEMP_NEXT, jax_split_at(k_temp, 2, 1));
    r = jax_split_at(r, 2, 0);
  }
  rng[0] = r.x; rng[1] = r.y;
  return SERL_OK;
}

extern "C" int serl_normal_fill(const uint32_t* key, float* out, int n, void* stream) {
  launch_k(normal_fill_kernel, ceil_div(n, 128), 128, 0, ST(stream), key, out, n);
  return check_launch("normal_fill_kernel");
}

extern "C" int serl_dropout_mask_fill(const uint32_t* key, uint32_t fold, float keep, uint8_t* mask, int n, void* stream) {
  launch_k(dropout_mask_kernel, ceil_div(n, 256), 256, 0, ST(stream), key, fold, keep, mask, n);
  return check_launch("dropout_mask_kernel");
}

extern "C" int serl_subsample_idx(const uint32_t* key, int ensemble, int32_t* out, int n, void* stream) {
  if (n < 1 || n > 32 || ensemble < 1 || ensemble > 65535) { set_last_error("serl_subsample_idx: need 1 <= n <= 32, 1 <= ensemble < 65536"); return SERL_ERR_INVALID; }
  launch_k(subsample_idx_kernel, 1, 32, 0, ST(stream), key, ensemble, out, n);
  return check_launch("subsample_idx_kernel");
}

extern "C" int serl_tanh_gaussian_fwd(const float* mu, const float* log_std, const float* eps, float std_min, float std_max,
                                      float* act, int ld_act, float* logp, float* u_out, float* std_out, int B, int A,
                                      int deterministic, void* stream) {
  if (!deterministic && !eps) { set_last_error("serl_tanh_gaussian_fwd: eps required unless deterministic"); return SERL_ERR_INVALID; }
  launch_k(tanh_gaussian_fwd_kernel<SERL_STD_EXP>, ceil_div(B, 128), 128, 0, ST(stream), mu, log_std, A, eps, std_min, std_max, act, ld_act,
           logp, u_out, std_out, B, A, deterministic);
  return check_launch("tanh_gaussian_fwd_kernel");
}

extern "C" int serl_tanh_gaussian_fwd_std(const float* mu, const float* x, int ld_x, int std_param, const float* eps, float std_min,
                                          float std_max, float* act, int ld_act, float* logp, float* u_out, float* std_out, int B, int A,
                                          int deterministic, void* stream) {
  if (!deterministic && !eps) { set_last_error("serl_tanh_gaussian_fwd_std: eps required unless deterministic"); return SERL_ERR_INVALID; }
  auto k = std_param == SERL_STD_EXP ? tanh_gaussian_fwd_kernel<SERL_STD_EXP> : std_param == SERL_STD_SOFTPLUS ? tanh_gaussian_fwd_kernel<SERL_STD_SOFTPLUS>
         : std_param == SERL_STD_UNIFORM ? tanh_gaussian_fwd_kernel<SERL_STD_UNIFORM>
         : std_param == SERL_STD_FIXED ? tanh_gaussian_fwd_kernel<SERL_STD_FIXED> : nullptr;
  const bool broadcast = std_param == SERL_STD_UNIFORM || std_param == SERL_STD_FIXED;
  if (!k || ld_x < 0 || broadcast != (ld_x == 0)) {
    set_last_error("serl_tanh_gaussian_fwd_std: unknown std_param %d or row stride %d (0 exactly for uniform / fixed)", std_param, ld_x);
    return SERL_ERR_INVALID;
  }
  launch_k(k, ceil_div(B, 128), 128, 0, ST(stream), mu, x, ld_x, eps, std_min, std_max, act, ld_act, logp, u_out, std_out, B, A, deterministic);
  return check_launch("tanh_gaussian_fwd_kernel");
}

extern "C" int serl_critic_loss(const float* q, const float* q_next, const int32_t* sub, int n_sub, const float* rewards,
                                const float* masks, const float* logp_next, const float* lagrange, int backup_entropy,
                                float gamma, float grad_scale, float* target_q, float* dq, float* info, int E, int B, void* stream) {
  launch_k(critic_loss_kernel, 1, 1024, 0, ST(stream), q, q_next, sub, n_sub, rewards, masks, logp_next, lagrange, backup_entropy, gamma,
                                                 grad_scale, target_q, dq, info, E, B);
  return check_launch("critic_loss_kernel");
}

extern "C" int serl_critic_loss_weighted(const float* q, const float* q_next, const int32_t* sub, int n_sub, const float* rewards,
                                         const float* masks, const float* logp_next, const float* lagrange, int backup_entropy,
                                         float gamma, float grad_scale, const float* w, float* target_q, float* dq, float* delta,
                                         float* info, int E, int B, void* stream) {
  if (!w || !delta) { set_last_error("serl_critic_loss_weighted: weights and delta are required"); return SERL_ERR_INVALID; }
  launch_k(critic_loss_weighted_kernel, 1, 1024, 0, ST(stream), q, q_next, sub, n_sub, rewards, masks, logp_next, lagrange, backup_entropy,
           gamma, grad_scale, target_q, dq, info, E, B, w, delta);
  return check_launch("critic_loss_weighted_kernel");
}

extern "C" int serl_fill_f32(float* x, float v, int n, void* stream) {
  launch_k(fill_kernel, ceil_div(n, 256), 256, 0, ST(stream), x, v, n);
  return check_launch("fill_kernel");
}

extern "C" int serl_actor_loss(const float* q, const float* logp, const float* lagrange, const float* da, int ld_da,
                               const float* act, int ld_act, const float* std, const float* log_std, const float* eps,
                               float std_min, float std_max, float grad_scale, float* dmu, float* dlogstd, float* info,
                               int E, int B, int A, void* stream) {
  launch_k(actor_loss_kernel<SERL_STD_EXP>, 1, 1024, 0, ST(stream), q, logp, lagrange, da, ld_da, act, ld_act, std, log_std, A, eps, std_min,
           std_max, grad_scale, dmu, dlogstd, info, E, B, A);
  return check_launch("actor_loss_kernel");
}

extern "C" int serl_actor_loss_std(const float* q, const float* logp, const float* lagrange, const float* da, int ld_da,
                                   const float* act, int ld_act, const float* std, const float* x, int ld_x, int std_param, const float* eps,
                                   float std_min, float std_max, float grad_scale, float* dmu, float* dx, float* info,
                                   int E, int B, int A, void* stream) {
  auto k = std_param == SERL_STD_EXP ? actor_loss_kernel<SERL_STD_EXP> : std_param == SERL_STD_SOFTPLUS ? actor_loss_kernel<SERL_STD_SOFTPLUS>
         : std_param == SERL_STD_UNIFORM ? actor_loss_kernel<SERL_STD_UNIFORM> : nullptr;
  if (!k || ld_x < 0 || (std_param == SERL_STD_UNIFORM) != (ld_x == 0)) {
    set_last_error("serl_actor_loss_std: unknown std_param %d or row stride %d (0 exactly for uniform)", std_param, ld_x); return SERL_ERR_INVALID;
  }
  launch_k(k, 1, 1024, 0, ST(stream), q, logp, lagrange, da, ld_da, act, ld_act, std, x, ld_x, eps, std_min, std_max, grad_scale, dmu, dx,
           info, E, B, A);
  return check_launch("actor_loss_kernel");
}

extern "C" int serl_temperature_loss(const float* logp, const float* lagrange, float target_entropy, float grad_scale,
                                     float* dlagrange, float* info, int B, void* stream) {
  launch_k(temperature_loss_kernel, 1, 1024, 0, ST(stream), logp, lagrange, target_entropy, grad_scale, dlagrange, info, B);
  return check_launch("temperature_loss_kernel");
}

extern "C" int serl_tanh_fwd(const float* z, float* out, int n, void* stream) {
  launch_k(tanh_fwd_kernel, ceil_div(n, 256), 256, 0, ST(stream), z, out, n);
  return check_launch("tanh_fwd_kernel");
}
extern "C" int serl_tanh_bwd(const float* dt, const float* t, float* dz, int n, void* stream) {
  launch_k(tanh_bwd_kernel, ceil_div(n, 256), 256, 0, ST(stream), dt, t, dz, n);
  return check_launch("tanh_bwd_kernel");
}
extern "C" int serl_bc_loss(const float* mu, const float* log_std, const float* actions, float std_min, float std_max, float grad_scale,
                            float* dmu, float* dlogstd, float* info, int B, int A, void* stream) {
  if (!mu || !log_std || !actions || !dmu || !dlogstd || !info || B < 1 || A < 1) { set_last_error("serl_bc_loss: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(bc_loss_kernel<SERL_STD_EXP, false>, 1, 1024, 0, ST(stream), mu, log_std, actions, std_min, std_max, grad_scale, dmu, dlogstd,
           info, B, A);
  return check_launch("bc_loss_kernel");
}

extern "C" int serl_bc_loss_std(const float* mu, const float* x, int ld_x, int std_param, int tanh_squash, const float* actions, float std_min,
                                float std_max, float grad_scale, float* dmu, float* dx, float* info, int B, int A, void* stream) {
  using Fn = decltype(&bc_loss_kernel<SERL_STD_EXP, false>);
  Fn k = nullptr;
  switch (std_param) {
    case SERL_STD_EXP: k = tanh_squash ? bc_loss_kernel<SERL_STD_EXP, true> : bc_loss_kernel<SERL_STD_EXP, false>; break;
    case SERL_STD_SOFTPLUS: k = tanh_squash ? bc_loss_kernel<SERL_STD_SOFTPLUS, true> : bc_loss_kernel<SERL_STD_SOFTPLUS, false>; break;
    case SERL_STD_UNIFORM: k = tanh_squash ? bc_loss_kernel<SERL_STD_UNIFORM, true> : bc_loss_kernel<SERL_STD_UNIFORM, false>; break;
    case SERL_STD_FIXED: k = tanh_squash ? bc_loss_kernel<SERL_STD_FIXED, true> : bc_loss_kernel<SERL_STD_FIXED, false>; break;
    default: break;
  }
  const bool broadcast = std_param == SERL_STD_UNIFORM || std_param == SERL_STD_FIXED;
  if (!k || ld_x != (broadcast ? 0 : A) || !mu || !x || !actions || !dmu || (!dx && std_param != SERL_STD_FIXED) || !info || B < 1 || A < 1) {
    set_last_error("serl_bc_loss_std: unknown std_param %d, row stride %d (0 for uniform / fixed, A otherwise) or invalid arguments",
                   std_param, ld_x);
    return SERL_ERR_INVALID;
  }
  launch_k(k, 1, 1024, 0, ST(stream), mu, x, actions, std_min, std_max, grad_scale, dmu, dx, info, B, A);
  return check_launch("bc_loss_kernel");
}

// descriptor -> kernel arguments; 0 or SERL_ERR_INVALID (message set, prefixed with `who`)
static int adam_args(const serl_adam_desc* d, const char* who, AdamArgs& a) {
  char msg[160];
  if (!d || d->n < 1 || !d->params || !d->m || !d->v || !d->grad || !d->counts) {
    snprintf(msg, sizeof msg, "%s: invalid descriptor", who); set_last_error(msg); return SERL_ERR_INVALID;
  }
  if (d->polyak && !d->target) { snprintf(msg, sizeof msg, "%s: polyak needs target", who); set_last_error(msg); return SERL_ERR_INVALID; }
  a = AdamArgs{};
  a.p = d->params; a.target = d->target; a.m = d->m; a.v = d->v; a.grad = d->grad; a.n = d->n; a.counts = d->counts;
  for (int g = 0; g < 3; ++g) { a.seg_end[g] = d->seg_end[g]; a.live[g] = d->live[g]; a.lr[g] = d->lr[g]; a.warmup[g] = d->warmup[g]; }
  a.b1 = d->b1; a.b2 = d->b2; a.eps = d->eps; a.tau = d->tau; a.polyak = d->polyak; a.lr_out = d->lr_out;
  a.gap = d->gap; a.aux_lo = d->aux_lo; a.aux_hi = d->aux_hi; a.aux_off = d->aux_off;
  if (a.gap < 0 || a.aux_lo > a.aux_hi || (a.aux_hi > a.aux_lo && (a.aux_lo < 0 || a.aux_hi > d->seg_end[0] || a.aux_lo + a.aux_off < d->n))) {
    snprintf(msg, sizeof msg, "%s: invalid gap / aux range", who); set_last_error(msg); return SERL_ERR_INVALID;
  }
  return 0;
}

extern "C" int serl_adam_polyak(const serl_adam_desc* d, void* stream) {
  AdamArgs a;
  if (int e = adam_args(d, "serl_adam_polyak", a)) return e;
  launch_k(adam_polyak_kernel, ceil_div(d->n, 256), 256, 0, ST(stream), a);
  if (int e = check_launch("adam_polyak_kernel")) return e;
  launch_k(adam_tick_kernel<false>, 1, 32, 0, ST(stream), a);
  return check_launch("adam_tick_kernel");
}

extern "C" int serl_adam_polyak_opts(const serl_adam_desc* d, const serl_adam_opts* o, void* stream) {
  AdamArgs a;
  if (int e = adam_args(d, "serl_adam_polyak_opts", a)) return e;
  if (!o) { set_last_error("serl_adam_polyak_opts: options required"); return SERL_ERR_INVALID; }
  for (int g = 0; g < 3; ++g) {
    a.clip[g] = o->clip[g] > 0.f ? o->clip[g] : 0.f;
    a.decay[g] = o->decay_steps[g] > 0 ? o->decay_steps[g] : 0;
    if (a.decay[g] > 0 && a.decay[g] <= d->warmup[g]) { set_last_error("serl_adam_polyak_opts: decay_steps must exceed warmup"); return SERL_ERR_INVALID; }
    if (a.clip[g] > 0.f && d->live[g] && !o->norms) { set_last_error("serl_adam_polyak_opts: clipping needs norms"); return SERL_ERR_INVALID; }
    if (!d->live[g]) a.clip[g] = 0.f;                           // zero gradient: norm 0 < clip, never clipped
  }
  a.norms = o->norms;
  launch_k(adam_polyak_opts_kernel, ceil_div(d->n, 256), 256, 0, ST(stream), a);
  if (int e = check_launch("adam_polyak_opts_kernel")) return e;
  launch_k(adam_tick_kernel<true>, 1, 32, 0, ST(stream), a);
  return check_launch("adam_tick_kernel");
}

extern "C" int serl_grad_global_norms(const serl_adam_desc* d, const int32_t want[3], double* partials, float* norms, void* stream) {
  if (!d || !d->grad || d->n < 1 || !want || !partials || !norms) { set_last_error("serl_grad_global_norms: invalid arguments"); return SERL_ERR_INVALID; }
  if (d->gap < 0 || d->aux_lo > d->aux_hi || d->seg_end[0] < 0 || d->seg_end[0] + d->gap > d->seg_end[1] || d->seg_end[1] > d->seg_end[2] ||
      d->seg_end[2] > d->n || (d->aux_hi > d->aux_lo && (d->aux_lo < 0 || d->aux_lo + d->aux_off < d->n))) {
    set_last_error("serl_grad_global_norms: invalid flat layout"); return SERL_ERR_INVALID;
  }
  NormArgs a{};
  a.grad = d->grad; a.n = d->n;
  a.s0 = d->seg_end[0]; a.g0 = d->seg_end[0] + d->gap; a.s1 = d->seg_end[1]; a.s2 = d->seg_end[2];
  a.x_lo = a.x_hi = 0;
  if (d->aux_hi > d->aux_lo) {                     // the twin slots lie past the n parameter slots: read up to their end
    a.x_lo = d->aux_lo + d->aux_off; a.x_hi = d->aux_hi + d->aux_off;
    a.n = a.x_hi;
  }
  for (int g = 0; g < 3; ++g) a.want[g] = want[g] && d->live[g];
  a.partials = partials; a.norms = norms;
  launch_k(grad_sumsq_kernel, SERL_GRAD_NORM_CTAS, kNormThreads, 0, ST(stream), a);
  if (int e = check_launch("grad_sumsq_kernel")) return e;
  launch_k(grad_norm_finish_kernel, 1, SERL_GRAD_NORM_CTAS, 0, ST(stream), a);
  return check_launch("grad_norm_finish_kernel");
}

// ---- forward-only passes of the public API (agents/continuous/sac.py:33-116) ------------------------------------------------------
namespace serl {
// log-probability of given actions: the tanh_gaussian_fwd_kernel formula with u = atanh(x) instead of mu + std * eps
__global__ void tanh_normal_log_prob_kernel(const float* __restrict__ mu, const float* __restrict__ std, const float* __restrict__ x,
                                            float* __restrict__ logp, int B, int A) {
  pdl_prologue();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float lp = 0.f;
  for (int i = 0; i < A; ++i) {
    const float m = mu[b * A + i], sd = std[b * A + i];
    const float u = atanhf(x[b * A + i]);
    const float z = (u - m) / sd;
    lp += -0.5f * z * z - logf(sd) - 0.918938533204672742f;
    lp -= 2.f * (0.693147180559945309f - u - softplusf(-2.f * u));
  }
  logp[b] = lp;
}

__global__ void lagrange_penalty_kernel(const float* __restrict__ lagrange, const float* __restrict__ lhs, float rhs, float* __restrict__ out,
                                        int n) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float m = softplusf(lagrange[0]);
  out[i] = lhs ? m * (lhs[i] - rhs) : m;
}
}  // namespace serl

extern "C" int serl_tanh_normal_log_prob(const float* mu, const float* std, const float* x, float* logp, int B, int A, void* stream) {
  if (!mu || !std || !x || !logp || B < 1 || A < 1) { set_last_error("serl_tanh_normal_log_prob: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(tanh_normal_log_prob_kernel, ceil_div(B, 128), 128, 0, ST(stream), mu, std, x, logp, B, A);
  return check_launch("tanh_normal_log_prob_kernel");
}

extern "C" int serl_lagrange_penalty(const float* lagrange, const float* lhs, float rhs, float* out, int n, void* stream) {
  if (!lagrange || !out || n < 1) { set_last_error("serl_lagrange_penalty: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(lagrange_penalty_kernel, ceil_div(n, 256), 256, 0, ST(stream), lagrange, lhs, rhs, out, n);
  return check_launch("lagrange_penalty_kernel");
}
