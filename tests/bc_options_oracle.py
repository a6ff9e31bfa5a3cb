"""Float64 restatement of BCAgent.update for every accepted configuration (test infrastructure only).

Extends oracle/bc.py's launcher-only restatement to the reference constructor's options (agents/continuous/bc.py:117-229):
the MLP of networks/mlp.py:10-32 (widths, activation, LayerNorm, dropout_rate; Dense -> Dropout -> [LayerNorm] -> activation),
Policy's std heads ("exp", "softplus", "uniform" log_stds) clipped to [std_min, std_max], the tanh-squashed distribution and
pixel-only encoders.  Encoder, trunk and Adam algebra are oracle/drq.py's; activations are tests/arch_oracle.py's.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from arch_oracle import ACTIVATIONS
from oracle import drq as O
from oracle.jax_prng import bernoulli, fold_in, split

ENC = O.ENC


def mlp_masks(drop_key, ncams, B, hidden, rate):
    """Hidden layer i's keep mask: bernoulli(fold_in(key, ncams + i), 1 - rate, (B, H_i)) (DESIGN.md §4)."""
    return [bernoulli(fold_in(drop_key, ncams + i), 1.0 - rate, (B, H)) for i, H in enumerate(hidden)]


def encode(params, cams, feats, state, masks, use_proprio):
    """oracle.drq.encode with stop_gradient=True; without proprio the image embeddings alone."""
    if use_proprio:
        return O.encode(params, cams, feats, state, masks, stop_gradient=True)
    dummy = dict(params)
    dummy[f"{ENC}/Dense_0/kernel"] = torch.zeros(1, 1, dtype=params[f"{ENC}/encoder_{cams[0]}/Dense_0/kernel"].dtype)
    dummy[f"{ENC}/Dense_0/bias"] = torch.zeros(1, dtype=dummy[f"{ENC}/Dense_0/kernel"].dtype)
    dummy[f"{ENC}/LayerNorm_0/scale"] = torch.ones(1, dtype=dummy[f"{ENC}/Dense_0/kernel"].dtype)
    dummy[f"{ENC}/LayerNorm_0/bias"] = torch.zeros(1, dtype=dummy[f"{ENC}/Dense_0/kernel"].dtype)
    B = next(iter(feats.values())).shape[0]
    enc = O.encode(dummy, cams, feats, torch.zeros(B, 1, dtype=dummy[f"{ENC}/Dense_0/kernel"].dtype), masks, stop_gradient=True)
    return enc[:, :256 * len(cams)]


def policy(params, enc, arch, std, std_min, std_max, hidden_masks=None, temperature=1.0):
    """Policy.__call__ (actor_critic_nets.py:178-227) -> (mu, std * sqrt(temperature)).  hidden_masks: train=True Dropout."""
    n = "modules_actor/network"
    x = enc
    for i, _ in enumerate(arch.hidden):
        x = x @ params[f"{n}/Dense_{i}/kernel"] + params[f"{n}/Dense_{i}/bias"]
        if hidden_masks is not None and arch.dropout:
            m = torch.as_tensor(np.asarray(hidden_masks[i]))
            x = torch.where(m, x / (1.0 - arch.dropout), torch.zeros_like(x))
        if arch.layer_norm:
            x = O.layer_norm(x, params[f"{n}/LayerNorm_{i}/scale"], params[f"{n}/LayerNorm_{i}/bias"])
        x = ACTIVATIONS[arch.act](x)
    mu = x @ params["modules_actor/Dense_0/kernel"] + params["modules_actor/Dense_0/bias"]
    if std == "uniform":
        raw = torch.exp(params["modules_actor/log_stds"]).expand_as(mu)
    else:
        ls = x @ params["modules_actor/Dense_1/kernel"] + params["modules_actor/Dense_1/bias"]
        raw = F.softplus(ls) if std == "softplus" else torch.exp(ls)
    return mu, torch.clamp(raw, std_min, std_max) * math.sqrt(temperature)


def log_prob(mu, sd, a, squash):
    """MultivariateNormalDiag / TanhMultivariateNormalDiag log_prob (the latter at u = atanh a)."""
    u = torch.atanh(a) if squash else a
    z = (u - mu) / sd
    lp = (-0.5 * z * z - torch.log(sd) - 0.5 * math.log(2 * math.pi)).sum(-1)
    if squash:
        lp = lp - (2.0 * (math.log(2.0) - u - F.softplus(-2.0 * u))).sum(-1)
    return lp


def mode(mu, squash):
    return torch.tanh(mu) if squash else mu


def update(params, opt, rng, cams, feats, state, actions, opts, dropout_masks=None, hidden_masks=None, lr=3e-4, dtype=torch.float64):
    """One BCAgent.update on given trunk features.  opts = dict(arch, std, std_min, std_max, squash, use_proprio).  Masks None ->
    keyed masks.  Returns (new_params, opt, new_rng, info, grads, masks)."""
    arch = opts["arch"]
    new_rng, k = split(np.asarray(rng, np.uint32), 2)
    drop_key = split(k, 2)[1]
    B = actions.shape[0]
    if dropout_masks is None:
        dropout_masks = O._dropout_masks(drop_key, cams, B)
    if hidden_masks is None and arch.dropout:
        hidden_masks = mlp_masks(drop_key, len(cams), B, arch.hidden, arch.dropout)
    p = {kk: torch.as_tensor(np.asarray(v)).to(dtype) for kk, v in params.items()}
    train = {kk: v.clone().requires_grad_(True) for kk, v in p.items() if "pretrained_encoder" not in kk}
    full = {**p, **train}
    masks = {c: torch.as_tensor(np.asarray(m)).bool() for c, m in dropout_masks.items()}
    enc = encode(full, cams, {c: f.to(dtype) for c, f in feats.items()}, None if state is None else torch.as_tensor(np.asarray(state)).to(dtype),
                 masks, opts["use_proprio"])
    mu, sd = policy(full, enc, arch, opts["std"], opts["std_min"], opts["std_max"], hidden_masks)
    a = torch.as_tensor(np.asarray(actions)).to(dtype)
    loss = -log_prob(mu, sd, a, opts["squash"]).mean()
    mse = ((mode(mu, opts["squash"]) - a) ** 2).sum(-1).mean()
    gs = torch.autograd.grad(loss, list(train.values()), allow_unused=True)
    grads = {kk: (torch.zeros_like(v) if g is None else g) for (kk, v), g in zip(train.items(), gs)}
    upd = O.adam_tx_update(grads, opt, lr)
    new_params = dict(p)
    for kk in train:
        new_params[kk] = p[kk] + upd[kk]
    info = {"actor_loss": loss.item(), "mse": mse.item()}
    return new_params, opt, new_rng, info, grads, {"sle": dropout_masks, "mlp": hidden_masks}
