"""Thin torch-tensor wrappers over the C-ABI ops (pointer + stream extraction only; no math here).

torch is plumbing: it owns device memory and the current stream.  Every function launches
hand-written kernels from libserl_b200.so and raises if the library or a launch fails.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib as L


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _s():
    return L.stream_ptr()


def _chk(t: torch.Tensor, dtype, name):
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    return t


# ---- trunk (fp32) ----------------------------------------------------------------------------------
def conv2d_nhwc(x, w, y, stride, pad_lo, pad_hi):
    """x (N,Hi,Wi,Ci) u8|f32, w (kh,kw,Ci,Co) f32 -> y (N,Ho,Wo,Co) f32."""
    N, Hi, Wi, Ci = x.shape
    kh, kw, ci2, Co = w.shape
    assert ci2 == Ci and x.is_contiguous() and w.is_contiguous() and y.is_contiguous()
    L.call("serl_conv2d_nhwc_f32", _p(x), int(x.dtype == torch.uint8), _p(w), _p(y), N, Hi, Wi, Ci, Co, kh, kw, stride,
           pad_lo, pad_hi, _s())
    return y


# ---- DrQ "small" encoder (3x3 / stride-2 VALID convs) --------------------------------------------------
SCONV_CTAS = 4 * 132          # wgrad split-K target: about four CTAs per SM, whatever the shape


def sconv_wgrad_splits(N, H, W, Ci, Co):
    """The split count serl_sconv_wgrad is given for a shape (a function of the shape only: the summation order is fixed)."""
    Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
    tiles = -(-(9 * Ci + 1) // 64) * -(-Co // 64)
    return max(1, min(-(-N * Ho * Wo // 256), SCONV_CTAS // tiles))


def sconv_wgrad_workspace(N, H, W, Ci, Co):
    """Floats of split-K partials serl_sconv_wgrad needs for a shape."""
    Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
    K = N * Ho * Wo
    ks = -(-(-(-K // sconv_wgrad_splits(N, H, W, Ci, Co))) // 16) * 16
    return -(-K // ks) * (9 * Ci + 1) * Co


def sconv_fwd(x, w, b, y, N, H, W, Ci, Co, x_is_u8, tc=False):
    """y (N,Ho,Wo,Co) = relu(conv3x3/2 VALID (x) + b); x u8 (scaled by 1/255) or f32 NHWC; addresses.  tc: on the tensor cores
    (3xTF32 wgmma), else on the CUDA cores."""
    L.call("serl_sconv_fwd", x, int(x_is_u8), w, b, y, N, H, W, Ci, Co, int(tc), _s())


def sconv_dgrad(dz, w, x, dx, N, H, W, Ci, Co, tc=False):
    """dx (N,H,W,Ci) = input gradient of the conv given dz (N,Ho,Wo,Co), gated by x > 0 (x: the layer input)."""
    L.call("serl_sconv_dgrad", dz, w, x, dx, N, H, W, Ci, Co, int(tc), _s())


def sconv_wgrad(x, x_is_u8, dz, dw, db, ws: torch.Tensor, N, H, W, Ci, Co, tc=False):
    """dw (3,3,Ci,Co), db (Co) of the conv from its input x and pre-activation gradient dz (fixed-order split-K in ws)."""
    L.call("serl_sconv_wgrad", x, int(x_is_u8), dz, dw, db, ws.data_ptr(), ws.numel() * 4, sconv_wgrad_splits(N, H, W, Ci, Co),
           N, H, W, Ci, Co, int(tc), _s())


def sconv_mean_fwd(y, out, N, P, C):
    L.call("serl_sconv_mean_fwd", y, out, N, P, C, _s())


def sconv_mean_bwd(dout, ld, y, dz, N, P, C):
    L.call("serl_sconv_mean_bwd", dout, ld, y, dz, N, P, C, _s())


# ---- DrQ "resnet" encoder (a trainable ResNet-10): convs at any kernel / stride / padding, GroupNorm and max-pool backward ----
# Addresses in, no shapes inferred.  tc: the tensor-core (3xTF32 wgmma) convs of the 16-bit builds, else the CUDA-core ones.
def rconv_fwd(x, w, y, N, H, W, Ci, Cw, Co, k, stride, pad_lo, pad_hi, tc):
    """y (N,Ho,Wo,Co) = conv(x (N,H,W,Ci), w (k,k,Cw,Co)); Cw < Ci: x's extra channels are zero padding."""
    L.call("serl_rconv_fwd", x, w, y, N, H, W, Ci, Cw, Co, k, k, stride, pad_lo, pad_hi, int(tc), _s())


def rconv_dgrad(dz, w, dx, N, H, W, Ci, Co, k, stride, pad_lo, pad_hi, accumulate, tc):
    """dx (N,H,W,Ci) (+)= the conv's input gradient from dz (N,Ho,Wo,Co)."""
    L.call("serl_rconv_dgrad", dz, w, dx, N, H, W, Ci, Co, k, k, stride, pad_lo, pad_hi, int(accumulate), int(tc), _s())


def rconv_wgrad_workspace(N, H, W, Ci, Co, k, stride, pad_lo, pad_hi) -> int:
    """Floats of split-K partials rconv_wgrad needs for a shape."""
    out = C.c_longlong(0)
    L.call("serl_rconv_wgrad_workspace", N, H, W, Ci, Co, k, k, stride, pad_lo, pad_hi, C.byref(out))
    return int(out.value)


def rconv_wgrad(x, dz, dw, ws: torch.Tensor, N, H, W, Ci, Cw, Co, k, stride, pad_lo, pad_hi, tc):
    """dw (k,k,Cw,Co) = the conv's weight gradient from its input x and output gradient dz (fixed-order split-K in ws)."""
    L.call("serl_rconv_wgrad", x, dz, dw, ws.data_ptr(), ws.numel() * 4, N, H, W, Ci, Cw, Co, k, k, stride, pad_lo, pad_hi, int(tc), _s())


def rconv_stem_prep(x, y, N, H, W, Ci=3):
    """y (N,H,W,4) fp32 = ImageNet-normalised x (N,H,W,3) uint8 with a zero fourth channel.  A stack of T frames on the channel
    axis (Ci = 3T > 3): y (N,H,W,stem_channels(Ci)), channel c normalised like channel c mod 3, the padding channels zero."""
    if Ci == 3:
        L.call("serl_rconv_stem_prep", x, y, N, H, W, _s())
    else:
        L.call("serl_rconv_stem_prep_stacked", x, y, N, H, W, Ci, _s())


def stem_channels(Ci: int) -> int:
    """Channels of the stem's normalised copy of a Ci-channel image: Ci rounded up to a multiple of 4 (the tensor-core convs'
    input granule)."""
    return -(-Ci // 4) * 4


def groupnorm_bwd_workspace(N, C_, groups) -> int:
    return 2 * N * C_ + 2 * N * groups


def groupnorm_bwd_nhwc(x, y, dy, scale, dx, dres, dscale, dbias, ws: torch.Tensor, N, HW, C_, groups, eps, relu):
    """Backward of groupnorm_nhwc: dx, dres (the residual's gradient, nullable), dscale / dbias from the forward's input x and
    output y (its ReLU mask) and dy; ws >= groupnorm_bwd_workspace floats."""
    assert ws.numel() >= groupnorm_bwd_workspace(N, C_, groups)
    L.call("serl_groupnorm_bwd_nhwc", x, y, dy, scale, dx, dres, dscale, dbias, ws.data_ptr(), N, HW, C_, groups, float(eps), int(relu),
           _s())


def maxpool3x3s2_bwd_nhwc(x, dy, dx, N, H, W, C_):
    """dx (N,H,W,C) of maxpool3x3s2_nhwc from its input x and dy (N,(H+1)//2,(W+1)//2,C); first-max rule."""
    L.call("serl_maxpool3x3s2_bwd_nhwc", x, dy, dx, N, H, W, C_, _s())


def sle_input_grad(ds, ld_ds, kernel, dx, R, P, C_):
    """dx (R,P,C) = the SpatialLearnedEmbeddings input gradient from ds (R, C*F) rows of stride ld_ds (F = 8)."""
    L.call("serl_vice_sle_input_grad", ds, ld_ds, kernel, dx, R, P, C_, _s())


def groupnorm_nhwc(x, y, scale, bias, residual, groups, eps, relu):
    N, H, W, Cc = x.shape
    L.call("serl_groupnorm_nhwc_f32", _p(x), _p(y), _p(scale), _p(bias), _p(residual), N, H * W, Cc, groups, float(eps),
           int(relu), _s())
    return y


def maxpool3x3s2_nhwc(x, y):
    N, H, W, Cc = x.shape
    L.call("serl_maxpool3x3s2_nhwc_f32", _p(x), _p(y), N, H, W, Cc, _s())
    return y


# ---- GEMM -------------------------------------------------------------------------------------------
class Workspace:
    """Caller-owned scratch for split-K / batch-reduce partials."""

    GEMM_IMPLS = {"f32": "serl_gemm_f32", "tf32x3": "serl_gemm_tf32x3"}

    def __init__(self, nbytes: int, device, gemm_impl: str = "f32"):
        self.buf = torch.empty(nbytes // 4, dtype=torch.float32, device=device)
        self.nbytes = self.buf.numel() * 4
        self.gemm_fn = self.GEMM_IMPLS[gemm_impl]      # CUDA-core SGEMM (1e-5 build) or tensor-core 3xTF32 (speed builds)


def gemm(ws: Workspace, A_ptr, B_ptr, C_ptr, M, N, K, *, sAm, sAk, sBk, sBn, ldc, Z=1, sAz=0, sBz=0, sCz=0,
         bias_ptr=None, sBiasZ=0, accumulate=False, reduce_z=False):
    d = L.GemmDesc()
    d.A, d.B, d.C, d.bias = A_ptr, B_ptr, C_ptr, bias_ptr
    d.workspace, d.workspace_bytes = ws.buf.data_ptr(), ws.nbytes
    d.M, d.N, d.K, d.Z = M, N, K, Z
    d.sAz, d.sAm, d.sAk, d.sBz, d.sBk, d.sBn, d.sCz, d.sBiasZ = sAz, sAm, sAk, sBz, sBk, sBn, sCz, sBiasZ
    d.ldc, d.accumulate, d.reduce_z = ldc, int(accumulate), int(reduce_z)
    L.call(ws.gemm_fn, C.byref(d), _s())


def at(t: torch.Tensor, elem_offset: int = 0) -> int:
    """Device address of element `elem_offset` of a tensor's storage view."""
    return t.data_ptr() + elem_offset * t.element_size()


def dense_fwd(ws, x, ldx, w, b, out, ldo, M, K, N, *, Z=1, x_z=0, w_z=None, b_z=None, out_z=0):
    """out[z] (M,N) = x[z] (M,K) @ w[z] (K,N) + b[z];  x/out given as (address, ld)."""
    gemm(ws, x, w, out, M, N, K, sAm=ldx, sAk=1, sBk=N, sBn=1, ldc=ldo, Z=Z, sAz=x_z, sBz=(K * N if w_z is None else w_z),
         sCz=out_z, bias_ptr=b, sBiasZ=(N if b_z is None else b_z))


def dense_bwd_weight(ws, x, ldx, dz, lddz, dw, M, K, N, *, Z=1, x_z=0, dz_z=0, dw_z=None):
    """dw[z] (K,N) = x[z]^T (K,M) @ dz[z] (M,N)."""
    gemm(ws, x, dz, dw, K, N, M, sAm=1, sAk=ldx, sBk=lddz, sBn=1, ldc=N, Z=Z, sAz=x_z, sBz=dz_z,
         sCz=(K * N if dw_z is None else dw_z))


def dense_bwd_input(ws, dz, lddz, w, dx, lddx, M, K, N, *, Z=1, dz_z=0, w_z=None, dx_z=0, reduce_z=False, accumulate=False):
    """dx[z] (M,K) = dz[z] (M,N) @ w[z]^T (N,K)   (w stored (K,N) row-major)."""
    gemm(ws, dz, w, dx, M, K, N, sAm=lddz, sAk=1, sBk=1, sBn=N, ldc=lddx, Z=Z, sAz=dz_z, sBz=(K * N if w_z is None else w_z),
         sCz=dx_z, reduce_z=reduce_z, accumulate=accumulate)


# ---- heads -------------------------------------------------------------------------------------------
def sle_fwd(feat, kernel, keep_mask, keep, out, ld_out):
    N, Pp, Cc = feat.shape[0], feat.shape[1] * feat.shape[2], feat.shape[3]
    L.call("serl_sle_fwd", _p(feat), _p(kernel), _p(keep_mask), float(keep), out, N, Pp, Cc, kernel.shape[-1], ld_out, _s())


def sle_bwd_kernel_grad(ws, feat, dout, ld_dout, dkernel):
    N, Pp, Cc = feat.shape[0], feat.shape[1] * feat.shape[2], feat.shape[3]
    L.call("serl_sle_bwd_kernel_grad", _p(feat), dout, dkernel, ws.buf.data_ptr(), ws.nbytes, N, Pp, Cc, 8, ld_dout, _s())


def ln_tanh_fwd(z, ld_z, scale, bias, rows_per_group, group_stride, out, ld_out, xhat, rstd, R, D, eps=1e-6):
    L.call("serl_layernorm_tanh_fwd", z, ld_z, scale, bias, rows_per_group, group_stride, out, ld_out, xhat, rstd, R, D,
           float(eps), _s())


def ln_tanh_bwd(dt, ld_dt, t, ld_t, xhat, rstd, scale, rows_per_group, group_stride, dz, dy, dscale, dbias, R, D):
    L.call("serl_layernorm_tanh_bwd", dt, ld_dt, t, ld_t, xhat, rstd, scale, rows_per_group, group_stride, dz, dy, dscale,
           dbias, R, D, _s())


def ln_act_fwd(z, ld_z, scale, bias, rows_per_group, group_stride, out, ld_out, xhat, rstd, R, D, act, layer_norm, eps=1e-6):
    """[LayerNorm +] activation (act: L.ACT_*); without LayerNorm scale / bias / xhat / rstd are unused."""
    L.call("serl_layernorm_act_fwd", z, ld_z, scale, bias, rows_per_group, group_stride, out, ld_out, xhat, rstd, R, D,
           float(eps), int(act), int(layer_norm), _s())


def ln_act_bwd(dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride, dz, dy, R, D, act, layer_norm):
    """dz of [LayerNorm +] activation; with LayerNorm dy is kept for ln_param_grad."""
    L.call("serl_layernorm_act_bwd", dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride, dz, dy,
           R, D, int(act), int(layer_norm), _s())


def ln_act_dropout_fwd(z, ld_z, scale, bias, rows_per_group, group_stride, mask, inv_keep, out, ld_out, xhat, rstd, R, D, act, layer_norm,
                       eps=1e-6, mask_rows=None):
    """ln_act_fwd with the layer's Dropout first (mask (R, D) uint8 tensor); without LayerNorm the dropped-out z is written back to z.
    mask_rows: row r reads mask row r % mask_rows (a critic ensemble's E*B rows share one (B, D) mask with mask_rows = B)."""
    if mask_rows is None:
        L.call("serl_ln_act_dropout_fwd", z, ld_z, scale, bias, rows_per_group, group_stride, _p(mask), float(inv_keep), out, ld_out, xhat, rstd,
               R, D, float(eps), int(act), int(layer_norm), _s())
    else:
        L.call("serl_ln_act_dropout_rows_fwd", z, ld_z, scale, bias, rows_per_group, group_stride, _p(mask), int(mask_rows), float(inv_keep),
               out, ld_out, xhat, rstd, R, D, float(eps), int(act), int(layer_norm), _s())


def ln_act_dropout_bwd(dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride, mask, inv_keep, dz, dy, R, D,
                       act, layer_norm, mask_rows=None):
    if mask_rows is None:
        L.call("serl_ln_act_dropout_bwd", dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride, _p(mask),
               float(inv_keep), dz, dy, R, D, int(act), int(layer_norm), _s())
    else:
        L.call("serl_ln_act_dropout_rows_bwd", dt, ld_dt, t, ld_t, pre, ld_pre, xhat, rstd, scale, bias, rows_per_group, group_stride,
               _p(mask), int(mask_rows), float(inv_keep), dz, dy, R, D, int(act), int(layer_norm), _s())


def ln_param_grad(dy, xhat, dscale, dbias, rows_per_group, R, D):
    L.call("serl_layernorm_param_grad", dy, xhat, dscale, dbias, rows_per_group, R, D, _s())


def colsum(x, out, groups, rows, D, ld, accumulate=False):
    L.call("serl_colsum_f32", x, out, groups, rows, D, ld, int(accumulate), _s())


def copy2d(src, ld_src, dst, ld_dst, R, D):
    L.call("serl_copy2d_f32", src, ld_src, dst, ld_dst, R, D, _s())


def fill(x, v, n):
    L.call("serl_fill_f32", x, float(v), n, _s())


# ---- rng ---------------------------------------------------------------------------------------------
def rng_schedule(rng_state, keys, do_aug, do_update, mlp_dropout=False):
    """mlp_dropout: the agent's critic or policy MLP has dropout - an update also writes the critic-MLP keys (KEY_MLP_*; keys then
    holds NUM_KEYS_MLP slots), from the rng before it advances."""
    if mlp_dropout and do_update:
        L.call("serl_mlp_dropout_keys", _p(_chk(rng_state, torch.uint32, "rng")), _p(keys), int(do_aug), _s())
    L.call("serl_rng_schedule", _p(_chk(rng_state, torch.uint32, "rng")), _p(keys), int(do_aug), int(do_update), _s())


def bc_key_chain(rng_state, key):
    """BCAgent.update's key chain on the device: key = split(split(rng)[1])[1] (the step's dropout key), rng = split(rng)[0].
    Host tensors (the host-logic dry runs of a device="cpu" agent) take the same chain compiled for the host."""
    args = _p(_chk(rng_state, torch.uint32, "rng")), _p(_chk(key, torch.uint32, "key"))
    if rng_state.device.type == "cpu":
        L.call("serl_host_bc_key_chain", *args)
    else:
        L.call("serl_bc_key_chain", *args, _s())


def key_ptr(keys: torch.Tensor, slot: int) -> int:
    return keys.data_ptr() + 8 * slot


def normal_fill(key_addr, out, n):
    L.call("serl_normal_fill", key_addr, _p(out), n, _s())


def dropout_mask_fill(key_addr, fold, keep, mask, n):
    L.call("serl_dropout_mask_fill", key_addr, fold, float(keep), _p(mask), n, _s())


def subsample_idx(key_addr, ensemble, out, n):
    L.call("serl_subsample_idx", key_addr, ensemble, _p(out), int(n), _s())


def counter_add(counter, inc=1):
    L.call("serl_counter_add", _p(counter), inc, _s())


# ---- prioritized replay (include/serl_b200.h: sum tree layout, draw, writers) --------------------------------------------
def priority_tree(nodes: torch.Tensor, max_dev: torch.Tensor, capacity: int, valid: Optional[torch.Tensor] = None) -> L.PriorityTree:
    t = L.PriorityTree()
    t.nodes, t.max_dev, t.capacity = _p(_chk(nodes, torch.float32, "nodes")), _p(_chk(max_dev, torch.float32, "max_dev")), int(capacity)
    t.valid = _p(valid)
    return t


def priority_set(tree: L.PriorityTree, slots: torch.Tensor, n: int, *, td: Optional[torch.Tensor] = None,
                 valid: Optional[torch.Tensor] = None, alpha: float = 0.0, eps: float = 0.0):
    """Leaves slots[:n] <- (|td| + eps)^alpha (td given) or valid ? m : 0; a slot named twice takes its last entry."""
    L.call("serl_replay_priority_set", C.byref(tree), _p(_chk(slots, torch.int32, "slots")),
           _p(None if td is None else _chk(td, torch.float32, "td")), _p(valid), int(n), float(alpha), float(eps), _s())


def priority_rebuild(tree: L.PriorityTree):
    L.call("serl_replay_priority_rebuild", C.byref(tree), _s())


def priority_weights(prio: torch.Tensor, n: int, beta_dev: torch.Tensor, w: torch.Tensor):
    """w[:n] = (min(prio[:n]) / prio[:n]) ^ beta, beta read from beta_dev on the device."""
    L.call("serl_replay_priority_weights", _p(_chk(prio, torch.float32, "prio")), int(n), _p(_chk(beta_dev, torch.float32, "beta")),
           _p(_chk(w, torch.float32, "w")), _s())


# ---- losses / optimizer ------------------------------------------------------------------------------
def tanh_gaussian_fwd(mu, log_std, eps, std_min, std_max, act, ld_act, logp, u, std, B, A, deterministic=False):
    L.call("serl_tanh_gaussian_fwd", _p(mu), _p(log_std), _p(eps), float(std_min), float(std_max), act, ld_act, _p(logp),
           _p(u), _p(std), B, A, int(deterministic), _s())


def tanh_gaussian_fwd_std(mu, x, ld_x, std_param, eps, std_min, std_max, act, ld_act, logp, u, std, B, A, deterministic=False):
    """tanh_gaussian_fwd for any std parameterisation (L.STD_*): x is the std head's output (row stride ld_x, 0 for "uniform")."""
    L.call("serl_tanh_gaussian_fwd_std", _p(mu), x, ld_x, int(std_param), _p(eps), float(std_min), float(std_max), act, ld_act, _p(logp),
           _p(u), _p(std), B, A, int(deterministic), _s())


def actor_loss_std(q, logp, lagrange, da, ld_da, act, ld_act, std, x, ld_x, std_param, eps, std_min, std_max, grad_scale, dmu, dx,
                   info, E, B, A):
    """actor_loss for any std parameterisation; dx (B, A) is the gradient w.r.t. the std head's output per row."""
    L.call("serl_actor_loss_std", _p(q), _p(logp), lagrange, da, ld_da, act, ld_act, _p(std), x, ld_x, int(std_param), _p(eps),
           float(std_min), float(std_max), float(grad_scale), _p(dmu), _p(dx), info, E, B, A, _s())


def critic_loss(q, q_next, sub, n_sub, rewards, masks, logp_next, lagrange, backup_entropy, gamma, grad_scale, target_q,
                dq, info, E, B, weights=None, delta=None):
    """weights (B) given: serl_critic_loss_weighted, which also writes each row's TD error to delta (B)."""
    if weights is None:
        L.call("serl_critic_loss", _p(q), _p(q_next), _p(sub), n_sub, _p(rewards), _p(masks), _p(logp_next), lagrange,
               int(backup_entropy), float(gamma), float(grad_scale), _p(target_q), _p(dq), info, E, B, _s())
    else:
        L.call("serl_critic_loss_weighted", _p(q), _p(q_next), _p(sub), n_sub, _p(rewards), _p(masks), _p(logp_next), lagrange,
               int(backup_entropy), float(gamma), float(grad_scale), _p(weights), _p(target_q), _p(dq), _p(delta), info, E, B, _s())


def actor_loss(q, logp, lagrange, da, ld_da, act, ld_act, std, log_std, eps, std_min, std_max, grad_scale, dmu, dlogstd,
               info, E, B, A):
    L.call("serl_actor_loss", _p(q), _p(logp), lagrange, da, ld_da, act, ld_act, _p(std), _p(log_std), _p(eps),
           float(std_min), float(std_max), float(grad_scale), _p(dmu), _p(dlogstd), info, E, B, A, _s())


def bc_loss_std(mu, x, ld_x, std_param, tanh_squash, actions, std_min, std_max, grad_scale, dmu, dx, info, B, A):
    """serl_bc_loss for any std head (x: address of the head's output, ld_x = A, or of the "uniform" log_stds, ld_x = 0) and the tanh
    squash; dx (B, A) per row, info address of {loss, mse}."""
    L.call("serl_bc_loss_std", _p(mu), x, ld_x, int(std_param), int(tanh_squash), _p(actions), float(std_min), float(std_max),
           float(grad_scale), _p(dmu), _p(dx), info, B, A, _s())


def temperature_loss(logp, lagrange, target_entropy, grad_scale, dlagrange, info, B):
    L.call("serl_temperature_loss", _p(logp), lagrange, float(target_entropy), float(grad_scale), dlagrange, info, B, _s())


def critic_multi_action_fwd(P, actions, w_act, w_act_z, scale, bias, z, out, E, B, N, A, H, act, layer_norm, eps=1e-6):
    """First critic layer for N candidate actions per state: out (E, B*N, H) = [LayerNorm +] act(P[e, b] + a[b, n] @ W_act[e]).
    P (E, B, H) and the (B, N, A) actions are tensors; w_act / scale / bias addresses (w_act_z: member stride in floats)."""
    L.call("serl_critic_multi_action_fwd", _p(P), _p(actions), w_act, int(w_act_z), scale, bias, _p(z), _p(out), E, B, N, A, H, float(eps),
           int(act), int(layer_norm), _s())


def tanh_normal_log_prob(mu, std, x, logp, B, A):
    """logp (B,) of given actions x (B, A) under the tanh-Gaussian with mean mu and clipped std (all (B, A) tensors)."""
    L.call("serl_tanh_normal_log_prob", _p(mu), _p(std), _p(x), _p(logp), B, A, _s())


def lagrange_penalty(lagrange, lhs, rhs, out, n):
    """out = softplus(lagrange) * (lhs - rhs), or softplus(lagrange) when lhs is None (lagrange: address)."""
    L.call("serl_lagrange_penalty", lagrange, _p(lhs), float(rhs), _p(out), n, _s())


def ln_relu_head_fwd(z, mask, keep, scale, bias, w, b, h, xhat, rstd, logit, R, D=256, eps=1e-6):
    """Reward-classifier hidden layer: [dropout] -> LayerNorm -> relu -> Dense(1).  Addresses (int) or None for the optionals."""
    L.call("serl_layernorm_relu_head_fwd", z, mask, float(keep), scale, bias, w, b, h, xhat, rstd, logit, R, D, float(eps), _s())


def ln_relu_head_bwd(dlogit, w, h, xhat, rstd, scale, mask, keep, dy, dz, R, D=256):
    L.call("serl_layernorm_relu_head_bwd", dlogit, w, h, xhat, rstd, scale, mask, float(keep), dy, dz, R, D, _s())


def bce_logits_loss(logits_train, logits_eval, labels, grad_scale, dlogit, info, B):
    L.call("serl_bce_logits_loss", logits_train, logits_eval, labels, float(grad_scale), dlogit, info, B, _s())


def dropout_bwd(dx, mask, keep, n):
    """In place: dx = mask ? dx / keep : 0."""
    L.call("serl_dropout_bwd_f32", dx, mask, float(keep), int(n), _s())


def adam_desc(params, target, m, v, grad, seg_end: Sequence[int], live: Sequence[int], counts, lr, warmup, tau, polyak,
              lr_out=None, b1=0.9, b2=0.999, eps=1e-8, n=None, gap=0, aux=(0, 0, 0)):
    """aux = (aux_lo, aux_hi, aux_off): leaves with a second (actor-tx) Adam state at flat index i + aux_off."""
    d = L.AdamDesc()
    d.params, d.target, d.m, d.v, d.grad = _p(params), _p(target), _p(m), _p(v), _p(grad)
    d.n = params.numel() if n is None else int(n)
    d.gap, d.aux_lo, d.aux_hi, d.aux_off = int(gap), int(aux[0]), int(aux[1]), int(aux[2])
    for g in range(3):
        d.seg_end[g], d.live[g], d.lr[g], d.warmup[g] = int(seg_end[g]), int(live[g]), float(lr[g]), int(warmup[g])
    d.counts = _p(counts)
    d.b1, d.b2, d.eps, d.tau, d.polyak = b1, b2, eps, float(tau), int(polyak)
    d.lr_out = _p(lr_out)
    return d


def adam_polyak(*args, **kw):
    """Fused Adam of the three txs + polyak (arguments: adam_desc)."""
    L.call("serl_adam_polyak", C.byref(adam_desc(*args, **kw)), _s())


def adam_single(store, lr: float, live: bool = True, warmup: int = 0, tau: Optional[float] = None, polyak: bool = False):
    """One Adam tx over every leaf of a params.FlatParams store (a tx that is not live still ticks its count).  With tau the
    store's target is part of the step and moves by polyak averaging when `polyak`."""
    n = store.n
    adam_polyak(store.params, None if tau is None else store.target, store.m, store.v, store.grad, [n, n, n], [int(live), 0, 0],
                store.counts, [lr] * 3, [warmup, 0, 0], tau or 0.0, polyak, lr_out=store.lr_info, n=n, gap=0, aux=(0, 0, 0))


def grad_global_norms(d, want: Sequence[int], partials: torch.Tensor, norms: torch.Tensor):
    """norms[g] = global gradient norm of tx g (live and want[g]) over the flat layout of AdamDesc d; partials: float64
    workspace of 3 * GRAD_NORM_CTAS."""
    w = (C.c_int32 * 3)(*[int(x) for x in want])
    L.call("serl_grad_global_norms", C.byref(d), w, _chk(partials, torch.float64, "partials").data_ptr(),
           _chk(norms, torch.float32, "norms").data_ptr(), _s())


def adam_polyak_opts(d, clip: Sequence[float], decay_steps: Sequence[int], norms: Optional[torch.Tensor]):
    """adam_polyak with per-tx clip_by_global_norm thresholds (0: off; norms from grad_global_norms) and cosine decay steps
    (0: linear warm-up then constant)."""
    o = L.AdamOpts()
    for g in range(3):
        o.clip[g], o.decay_steps[g] = float(clip[g]), int(decay_steps[g])
    o.norms = _p(norms)
    L.call("serl_adam_polyak_opts", C.byref(d), C.byref(o), _s())


# ---- single-pass TF32 GEMM with TMA-fed operands and fused epilogues (heads of the 16-bit builds) -------------------
def tgemm_problem(A, B, *, sAm, sAk, sBk, sBn, Z=1, sAz=0, sBz=0, C_=None, sCz=0, ldc=0, bias=None, sBiasZ=0, ln_scale=None,
                  ln_bias=None, sLnZ=0, xhat=None, rstd=None, sXhatZ=0, sRstdZ=0, head_w=None, head_b=None, sHeadWz=0, sHeadBz=0,
                  head_out=None, sHeadOutZ=0, ld_head=1, head_w2=None, head_b2=None, head_out2=None, noise=None, act=None, ld_act=0,
                  logp=None, u_out=None, std_out=None):
    """One problem of a serl_tgemm_tf32 launch; every operand is a device ADDRESS (int) or None, strides in floats."""
    p = L.TgemmProblem()
    p.A, p.B, p.sAz, p.sAm, p.sAk, p.sBz, p.sBk, p.sBn, p.Z = A, B, sAz, sAm, sAk, sBz, sBk, sBn, Z
    p.C, p.sCz, p.ldc, p.bias, p.sBiasZ = C_, sCz, ldc, bias, sBiasZ
    p.ln_scale, p.ln_bias, p.sLnZ, p.xhat, p.rstd, p.sXhatZ, p.sRstdZ = ln_scale, ln_bias, sLnZ, xhat, rstd, sXhatZ, sRstdZ
    p.head_w, p.head_b, p.sHeadWz, p.sHeadBz, p.head_out, p.sHeadOutZ, p.ld_head = head_w, head_b, sHeadWz, sHeadBz, head_out, sHeadOutZ, ld_head
    p.head_w2, p.head_b2, p.head_out2 = head_w2, head_b2, head_out2
    p.noise, p.act, p.ld_act, p.logp, p.u_out, p.std_out = noise, act, ld_act, logp, u_out, std_out
    return p


def tgemm(ws: Optional[Workspace], problems, M, N, K, *, epilogue=L.TGEMM_STORE, head_n=0, accumulate=False, reduce_z=False, splits=0,
          ln_eps=1e-6, std_min=1e-5, std_max=5.0, deterministic=False, error=None, masks=None, inv_keep=1.0):
    """C[z] = A[z] @ B[z] on the tensor cores (TF32, fp32 accumulate) for up to 6 problems of one shape; see include/serl_b200.h.
    masks: one (M, 256) uint8 Dropout keep mask per problem (LayerNorm epilogues; z' = mask ? z * inv_keep : 0), or None."""
    arr = (L.TgemmProblem * len(problems))(*problems)
    d = L.TgemmDesc()
    d.problems, d.num_problems, d.M, d.N, d.K = arr, len(problems), M, N, K
    d.epilogue, d.head_n, d.accumulate, d.reduce_z, d.splits = epilogue, head_n, int(accumulate), int(reduce_z), splits
    d.ln_eps, d.std_min, d.std_max, d.deterministic = float(ln_eps), float(std_min), float(std_max), int(deterministic)
    if ws is not None:
        d.workspace, d.workspace_bytes = ws.buf.data_ptr(), ws.nbytes
    d.error = _p(error)
    if masks is None:
        L.call("serl_tgemm_tf32", C.byref(d), _s())
    else:
        ptrs = (C.c_void_p * len(masks))(*[_p(m) for m in masks])
        L.call("serl_tgemm_tf32_masked", C.byref(d), ptrs, float(inv_keep), _s())


def tgemm_splits(K: int, want: int) -> int:
    """Largest S <= want such that S k-splits of whole 32-wide k-blocks cover K with no empty split."""
    for S in range(max(want, 1), 0, -1):
        kc = -(-(-(-K // S)) // 32) * 32
        if -(-K // kc) == S:
            return S
    return 1


def sle_fwd_multi(problems, keep, N, P, C_):
    """problems: (feat, kernel, keep_mask | None, out, ld_out) device addresses; one launch."""
    arr = (L.SleProblem * len(problems))()
    for q, (feat, kern, mask, out, ld) in zip(arr, problems):
        q.feat, q.kernel, q.keep_mask, q.out, q.ld_out = feat, kern, mask, out, ld
    L.call("serl_sle_fwd_multi", arr, len(problems), float(keep), N, P, C_, 8, _s())


def sle_bwd_multi(ws: Workspace, problems, N, P, C_):
    """problems: (feat, dout, ld_dout, dkernel) device addresses; SLE kernel gradients of all cameras in two launches."""
    arr = (L.SleBwdProblem * len(problems))()
    for q, (feat, dout, ld, dk) in zip(arr, problems):
        q.feat, q.dout, q.ld_dout, q.dkernel = feat, dout, ld, dk
    L.call("serl_sle_bwd_multi", arr, len(problems), ws.buf.data_ptr(), ws.nbytes, N, P, C_, 8, _s())


def enc_finish(problems, rows, eps=1e-6):
    """problems: dicts with partials+S or x+ld_x+w+K, and bias, ln_scale, ln_bias, out, ld_out, D, optional xhat, rstd."""
    arr = (L.EncFinishProblem * len(problems))()
    for q, p in zip(arr, problems):
        q.partials, q.S, q.x, q.ld_x, q.w, q.K = p.get("partials"), p.get("S", 0), p.get("x"), p.get("ld_x", 0), p.get("w"), p.get("K", 0)
        q.bias, q.ln_scale, q.ln_bias, q.out, q.ld_out = p["bias"], p["ln_scale"], p["ln_bias"], p["out"], p["ld_out"]
        q.xhat, q.rstd, q.D = p.get("xhat"), p.get("rstd"), p["D"]
    L.call("serl_enc_finish", arr, len(problems), rows, float(eps), _s())


def ln_tanh_bwd_multi(problems, masks=None, mask_rows=1, inv_keep=1.0):
    """problems: dicts with dt+ld_dt (or dq+head_w[+head_w_stride]), optional dt2+ld_dt2, t, ld_t, xhat, rstd, scale,
    rows_per_group, group_stride, dz, optional dy, R, D.  masks: per problem the forward's Dropout keep mask, row r reading mask
    row r % mask_rows (dz *= mask * inv_keep), or None."""
    arr = (L.LnBwdProblem * len(problems))()
    for q, p in zip(arr, problems):
        q.dt, q.ld_dt, q.dt2, q.ld_dt2 = p.get("dt"), p.get("ld_dt", 0), p.get("dt2"), p.get("ld_dt2", 0)
        q.dq, q.head_w, q.head_w_stride = p.get("dq"), p.get("head_w"), p.get("head_w_stride", 0)
        q.t, q.ld_t, q.xhat, q.rstd, q.scale = p["t"], p["ld_t"], p["xhat"], p["rstd"], p["scale"]
        q.rows_per_group, q.group_stride, q.dz, q.dy, q.R, q.D = p["rows_per_group"], p.get("group_stride", 0), p["dz"], p.get("dy"), p["R"], p["D"]
        q.dt_parts, q.dt_part_stride = p.get("dt_parts", 1), p.get("dt_part_stride", 0)
    if masks is None:
        L.call("serl_layernorm_tanh_bwd_multi", arr, len(problems), _s())
    else:
        ptrs = (C.c_void_p * len(masks))(*[_p(m) for m in masks])
        L.call("serl_layernorm_tanh_bwd_multi_masked", arr, len(problems), ptrs, int(mask_rows), float(inv_keep), _s())


def small_grads(jobs):
    """jobs: (kind, x, ld_x, y | None, ld_y, out_a, out_b | None, groups, rows, D)."""
    arr = (L.SmallGradJob * len(jobs))()
    for q, (kind, x, ld_x, y, ld_y, out_a, out_b, groups, rows, D) in zip(arr, jobs):
        q.kind, q.x, q.ld_x, q.y, q.ld_y, q.out_a, q.out_b, q.groups, q.rows, q.D = kind, x, ld_x, y, ld_y, out_a, out_b, groups, rows, D
    L.call("serl_small_grads", arr, len(jobs), _s())


# ---- image augmentations (vision/data_augmentations.py) -------------------------------------------------------------------------
# src / dst: contiguous (n, H, W, C) images on the device, keys: uint32 pairs viewed as int32 (one per image, or one split n ways
# by aug_crop's split_n).  draws: optional float32 records of each image's random decisions (the tests compare them).
def aug_crop(src, dst, keys, split_n, n, H, W, C_, padding):
    L.call("serl_aug_crop", _p(src), _p(dst), _p(keys), int(split_n), n, H, W, C_ * src.element_size(), int(padding), _s())


def aug_color(src, dst, keys, draws, n, H, W, lo, hi, enabled, shuffle, apply_prob, jitter_prob, gray_prob):
    d = L.ColorDesc((L.f32 * 4)(*lo), (L.f32 * 4)(*hi), int(enabled), int(shuffle), float(apply_prob), float(jitter_prob),
                    float(gray_prob))
    L.call("serl_aug_color", _p(src), _p(dst), _p(keys), _p(draws), n, H, W, C.byref(d), _s())


def aug_blur(src, dst, keys, draws, n, H, W, C_, radius, sigma_min, sigma_max, apply_prob):
    L.call("serl_aug_blur", _p(src), _p(dst), _p(keys), _p(draws), n, H, W, C_, int(radius), float(sigma_min), float(sigma_max),
           float(apply_prob), _s())


def aug_flip(src, dst, keys, n, H, W, C_):
    L.call("serl_aug_flip", _p(src), _p(dst), _p(keys), n, H, W, C_, _s())


def aug_solarize(src, dst, keys, n, H, W, C_, threshold, apply_prob):
    L.call("serl_aug_solarize", _p(src), _p(dst), _p(keys), n, H, W, C_, float(threshold), float(apply_prob), _s())
