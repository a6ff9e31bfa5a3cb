"""Float64 CPU restatement of VICEAgent.update_vice and vice_reward (agents/continuous/vice.py:357-560 of the reference), on the
functions of oracle/drq.py and oracle/jax_prng.py.  PARITY UNPINNED like oracle/drq.py.

Decisions restated here (DESIGN.md §4): lam = uniform(key_0) (Beta(1, 1) in distribution); permutation(key_1, N) as jax's
_shuffle; dropout keys folded per camera (SLE) and at ncams (hidden), the penalty's masks one row broadcast over the samples;
lam / y_a / y_b of the LAST camera in the loss; the penalty's norms per (camera, row), averaged over ncams * B rows.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import drq as O
from oracle import jax_prng as P

VICE = "modules_vice"
KEEP = 0.9
SLOPE = 0.01


def permutation(key, n):
    """jax.random.permutation(key, n): per round key, sub = split(key); stable sort of the rows by random_bits(sub, (n,))."""
    x = np.arange(n)
    rounds = int(np.ceil(3 * np.log(max(1, n)) / np.log(np.iinfo(np.uint32).max)))
    key = np.asarray(key, np.uint32)
    for _ in range(rounds):
        key, sub = P.split(key)
        x = x[np.argsort(P.random_bits(sub, (n,)), kind="stable")]
    return x


def keys(rng, ncams):
    """update_vice's key chain (vice.py:370-446) and apply_loss_fns' split(rng, 5) (tree order actor, critic, temperature, vice)."""
    rng = np.asarray(rng, np.uint32)
    k_aug, r = P.split(rng)
    cams = []
    for _ in range(ncams):
        _, r = P.split(r)
        k0, k1, r = P.split(r, 3)
        k_eps, r = P.split(r)
        cams.append((k0, k1, k_eps))
    k_drop, r = P.split(r)
    return dict(aug=k_aug, cams=cams, drop=k_drop, vice=P.split(rng, 5)[4], final=r)


def draws(k, N):
    k0, k1, k_eps = k
    return float(P.uniform01(k0, ())), permutation(k1, N), P.uniform01(k_eps, (N // 2,))


def labels(N):
    y = np.concatenate([np.ones(N // 2, np.float32), np.zeros(N // 2, np.float32)])
    return (y * np.float32(1 - 0.2) + np.float32(0.5 * 0.2)).astype(np.float32)


def forward(params, cams, feats, sle_masks=None, hidden_mask=None):
    """BinaryClassifier(classify_encoded=True) -> logits (R,).  feats {cam: (R, 4, 4, 512)}; masks None: train=False."""
    outs = []
    for cam in cams:
        pre = f"{VICE}/encoder/encoder_{cam}"
        k = params[f"{pre}/SpatialLearnedEmbeddings_0/kernel"]
        f = feats[cam]
        s = torch.einsum("bhwc,hwcf->bcf", f, k).reshape(f.shape[0], -1)
        if sle_masks is not None:
            s = torch.where(torch.as_tensor(np.asarray(sle_masks[cam])).bool(), s / KEEP, torch.zeros_like(s))
        z = s @ params[f"{pre}/Dense_0/kernel"] + params[f"{pre}/Dense_0/bias"]
        outs.append(torch.tanh(O.layer_norm(z, params[f"{pre}/LayerNorm_0/scale"], params[f"{pre}/LayerNorm_0/bias"])))
    x = torch.cat(outs, dim=-1)
    z = x @ params[f"{VICE}/network/Dense_0/kernel"] + params[f"{VICE}/network/Dense_0/bias"]
    if hidden_mask is not None:
        z = torch.where(torch.as_tensor(np.asarray(hidden_mask)).bool(), z / KEEP, torch.zeros_like(z))
    h = torch.nn.functional.leaky_relu(O.layer_norm(z, params[f"{VICE}/network/LayerNorm_0/scale"],
                                                    params[f"{VICE}/network/LayerNorm_0/bias"]), SLOPE)
    return (h @ params[f"{VICE}/Dense_0/kernel"] + params[f"{VICE}/Dense_0/bias"])[:, 0]


def bce(x, y):
    return x.clamp_min(0) - x * y + torch.log1p(torch.exp(-x.abs()))


def loss(params, cams, raw, k, *, last_camera_labels=True, per_camera_norms=True, per_camera_draws=True, dtype=torch.float64):
    """bce + 10 gp of update_vice from the trunk features raw {cam: (2B, 4, 4, 512)} of [goal, goal crop, obs, obs crop].
    Returns (total, info); info holds the draws, masks and both loss terms.  The two flags switch off the reference's
    last-camera labels (use camera 0's), per-(camera, row) norms (one norm per row over all cameras) and per-camera draws (every
    camera mixed with camera 0's lam / permutation / eps) for the tests that show each changes the result."""
    nc = len(cams)
    N = next(iter(raw.values())).shape[0]
    B = N // 2
    mix, gp_in, d = {}, {}, []
    for j, cam in enumerate(cams):
        lam, perm, eps = draws(k["cams"][j if per_camera_draws else 0], N)
        f = torch.as_tensor(np.asarray(raw[cam])).to(dtype)
        m = lam * f + (1 - lam) * f[perm]
        e = torch.as_tensor(eps).to(dtype).view(B, 1, 1, 1)
        mix[cam], gp_in[cam] = m, e * m[:B] + (1 - e) * m[B:]
        d.append((lam, perm, eps))
    lam, perm, _ = d[-1] if last_camera_labels else d[0]
    y = torch.as_tensor(labels(N)).to(dtype)
    sle_m = {cam: P.bernoulli(P.fold_in(k["drop"], j), KEEP, (N, 4096)) for j, cam in enumerate(cams)}
    hid_m = P.bernoulli(P.fold_in(k["drop"], nc), KEEP, (N, 256))
    logits = forward(params, cams, mix, sle_m, hid_m)
    b = lam * bce(logits, y).mean() + (1 - lam) * bce(logits, y[perm]).mean()
    gsle = {cam: np.ascontiguousarray(np.broadcast_to(P.bernoulli(P.fold_in(k["vice"], j), KEEP, (4096,)), (B, 4096))) for j, cam in enumerate(cams)}
    ghid = np.ascontiguousarray(np.broadcast_to(P.bernoulli(P.fold_in(k["vice"], nc), KEEP, (256,)), (B, 256)))
    x = {cam: v.detach().requires_grad_(True) for cam, v in gp_in.items()}
    out = forward(params, cams, x, gsle, ghid)
    g = torch.autograd.grad(out.sum(), [x[c] for c in cams], create_graph=True)     # rows are independent: per-sample gradients
    if per_camera_norms:
        gg = torch.cat([t.reshape(B, -1) for t in g], dim=0)
    else:
        gg = torch.cat([t.reshape(B, -1) for t in g], dim=1)
    norms = torch.sqrt(torch.sum(gg ** 2 + 1e-6, dim=1))
    gp = torch.mean((norms - 1) ** 2)
    total = b + 10 * gp
    return total, dict(bce=b, gp=gp, grad_norm=norms.mean(), draws=d, sle_masks=sle_m, hidden_mask=hid_m, logits=logits)


def update_vice_grads(params, cams, raw, k, dtype=torch.float64):
    """(gradients of every vice leaf, info) of one update_vice step."""
    p = {n: torch.as_tensor(np.asarray(v)).to(dtype).requires_grad_(True) for n, v in params.items()}
    total, info = loss(p, cams, raw, k, dtype=dtype)
    gs = torch.autograd.grad(total, list(p.values()))
    info["total"] = total
    return {n: g for n, g in zip(p, gs)}, info


def act(name, u):
    """The VICE activations as jax writes them: tanh, and leaky_relu = where(u >= 0, u, 0.01 u) (slope 1 at u = 0)."""
    return torch.tanh(u) if name == "tanh" else torch.where(u >= 0, u, SLOPE * u)


def ln_act(z, scale, bias, act_name, mask=None, pre_bias=None, keep=KEEP, eps=1e-6):
    """act(LN(mask(z + pre_bias)) * scale + bias) row by row, flax's fast variance max(E[x^2] - E[x]^2, 0); scale / bias (D,) or
    one row per input row; mask (R, D) bool (kept units scaled by 1 / keep)."""
    x = z if pre_bias is None else z + pre_bias
    if mask is not None:
        x = torch.where(torch.as_tensor(mask).bool(), x / keep, torch.zeros_like(x))
    mean = x.mean(-1, keepdim=True)
    var = ((x * x).mean(-1, keepdim=True) - mean * mean).clamp_min(0)
    return act(act_name, (x - mean) * torch.rsqrt(var + eps) * scale + bias)


def ln_act_jvp(z, zdot, scale, bias, act_name, mask=None, pre_bias=None, keep=KEEP):
    """(y, ydot): ln_act at z and its directional derivative along zdot (the tangent rows of serl_vice_ln_act_fwd), by
    forward-mode autograd; both stay differentiable in z, zdot, scale and bias."""
    return torch.func.jvp(lambda zz: ln_act(zz, scale, bias, act_name, mask, pre_bias, keep), (z,), (zdot,))


def vice_reward(params, cams, feats, dtype=torch.float64):
    p = {n: torch.as_tensor(np.asarray(v)).to(dtype) for n, v in params.items()}
    return torch.sigmoid(forward(p, cams, {c: torch.as_tensor(np.asarray(f)).to(dtype) for c, f in feats.items()}))
