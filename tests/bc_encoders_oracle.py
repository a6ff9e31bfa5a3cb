"""Float64 restatement of BCAgent with the trainable "small" and "resnet" encoders and with a fixed std (test infrastructure only).

Composes tests/small_encoder_oracle.py / tests/resnet_encoder_oracle.py (each camera's encoder on its uint8 frames) with
tests/bc_options_oracle.py (policy MLP, std heads, log-prob, mode, MLP dropout masks) and oracle/drq.py's Adam:
  agents/continuous/bc.py:36-76              loss = -mean_b log pi(a_b | o_b), mse = mean_b sum (mode_b - a_b)^2
  networks/actor_critic_nets.py:185          the encoder runs with stop_gradient=True: every encoder leaf gets a zero gradient
  networks/actor_critic_nets.py:205-212      fixed std: std = clip(fixed_std, std_min, std_max) * sqrt(temperature), no parameter
The key chain is bc_options_oracle's: new_rng, k = split(rng); dropout key = split(k)[1]; camera j's SLE mask folds j ("resnet"
only: the small encoder has no Dropout), hidden layer i's MLP mask folds ncams + i.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import resnet_encoder_oracle
import small_encoder_oracle
from bc_options_oracle import log_prob, mlp_masks, mode
from bc_options_oracle import policy as _policy
from oracle import drq as O
from oracle.jax_prng import split

ENCODE = {"small": small_encoder_oracle.encode, "resnet": resnet_encoder_oracle.encode}


def encode(params, encoder, cams, images, state, masks):
    """The concatenated embeddings behind the policy's stop_gradient; the proprio block is there when the tree has its leaves."""
    kw = {"dropout_masks": masks} if encoder == "resnet" else {}
    return ENCODE[encoder](params, cams, images, state, stop_gradient=True, **kw)


def policy(params, enc, opts, hidden_masks=None, temperature=1.0):
    """bc_options_oracle.policy, plus the fixed std (opts["fixed_std"]): the means of the same MLP, a constant clipped std."""
    if opts["std"] != "fixed":
        return _policy(params, enc, opts["arch"], opts["std"], opts["std_min"], opts["std_max"], hidden_masks, temperature)
    A = params["modules_actor/Dense_0/bias"].shape[0]
    no_head = dict(params, **{"modules_actor/log_stds": torch.zeros(A, dtype=enc.dtype)})
    mu, _ = _policy(no_head, enc, opts["arch"], "uniform", opts["std_min"], opts["std_max"], hidden_masks)
    fixed = torch.as_tensor(np.asarray(opts["fixed_std"], np.float32)).to(enc.dtype)
    return mu, (torch.clamp(fixed, opts["std_min"], opts["std_max"]) * math.sqrt(temperature)).expand_as(mu)


def keyed_masks(rng, encoder, cams, B, arch):
    """The dropout masks one update draws from the state's rng: ({cam: (B, 4096)} or None, [(B, H_i)] or None)."""
    k = split(np.asarray(rng, np.uint32), 2)[1]
    drop_key = split(k, 2)[1]
    sle = O._dropout_masks(drop_key, cams, B) if encoder == "resnet" else None
    return sle, (mlp_masks(drop_key, len(cams), B, arch.hidden, arch.dropout) if arch.dropout else None)


def loss_fn(params, opts, cams, images, state, actions, sle_masks=None, hidden_masks=None):
    """(loss, mse) of one BC batch; sle_masks / hidden_masks None: train=False (no Dropout)."""
    masks = None if sle_masks is None else {c: torch.as_tensor(np.asarray(m)).bool() for c, m in sle_masks.items()}
    enc = encode(params, opts["encoder"], cams, images, None if state is None else torch.as_tensor(np.asarray(state)), masks)
    mu, sd = policy(params, enc, opts, hidden_masks)
    a = torch.as_tensor(np.asarray(actions)).to(enc.dtype)
    return -log_prob(mu, sd, a, opts["squash"]).mean(), ((mode(mu, opts["squash"]) - a) ** 2).sum(-1).mean()


def update(params, opt, rng, cams, images, state, actions, opts, sle_masks=None, hidden_masks=None, lr=3e-4, dtype=torch.float64):
    """One BCAgent.update on the uint8 frames `images` {cam: (B, H, W, 3)}.  opts = dict(encoder, arch, std, std_min, std_max,
    squash, use_proprio[, fixed_std]).  Masks None -> the keyed masks.  Returns (new_params, opt, new_rng, info, grads, masks)."""
    B = np.asarray(actions).shape[0]
    new_rng = split(np.asarray(rng, np.uint32), 2)[0]
    ks, kh = keyed_masks(rng, opts["encoder"], cams, B, opts["arch"])
    sle_masks = ks if sle_masks is None else sle_masks
    hidden_masks = kh if hidden_masks is None else hidden_masks
    p = {k: torch.as_tensor(np.asarray(v)).to(dtype) for k, v in params.items()}
    train = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    loss, mse = loss_fn(train, opts, cams, images, state, actions, sle_masks, hidden_masks)
    gs = torch.autograd.grad(loss, list(train.values()), allow_unused=True)
    grads = {k: (torch.zeros_like(v) if g is None else g) for (k, v), g in zip(train.items(), gs)}
    upd = O.adam_tx_update(grads, opt, lr)
    new_params = {k: p[k] + upd[k] for k in p}
    info = {"actor_loss": loss.item(), "mse": mse.item()}
    return new_params, opt, new_rng, info, grads, {"sle": sle_masks, "mlp": hidden_masks}
