"""ORACLE (test infrastructure, not product): make_optimizer's per-tx options (common/optimizers.py:6-56) on top of the
step restated in `oracle/drq.py`: a learning rate per tx, optax.warmup_cosine_decay_schedule and
optax.clip_by_global_norm ahead of each tx's Adam.

Third-party arithmetic restated from optax's published definitions: **parity unpinned**, like the rest of drq.py.

`update` runs drq.update for the losses, gradients and key chain, then redoes the optimizer tail of
common.py:136-168 with the options from the pre-step moments.  `update_critics` / `update_high_utd` run drq's entry
points with that `update` in place of drq's.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional
from unittest import mock

import torch

from . import drq

TXS = ("actor", "critic", "temperature")
_drq_update = drq.update


@dataclass
class OptimizerOptions:
    lr: Dict[str, float] = field(default_factory=dict)                 # tx -> peak learning rate (default: OracleConfig.lr)
    cosine_decay_steps: Dict[str, Optional[int]] = field(default_factory=dict)
    clip_grad_norm: Dict[str, Optional[float]] = field(default_factory=dict)


def lr_schedule(count: int, lr: float, warmup: int, decay_steps: Optional[int] = None) -> float:
    """optimizers.py:14-29.  Without decay: drq.lr_schedule (linear 0 -> lr over `warmup`, then constant).
    With decay_steps = D: optax.warmup_cosine_decay_schedule(0, lr, warmup, D, end_value=0) - the same linear warm-up,
    then cosine_decay_schedule(lr, D - warmup, alpha=0) at count - warmup: lr * 0.5 * (1 + cos(pi * min(c - w, D - w) / (D - w)))."""
    if decay_steps is None or count < warmup:
        return drq.lr_schedule(count, lr, warmup)
    span = decay_steps - warmup
    assert span > 0, "optax.cosine_decay_schedule needs decay_steps > 0"
    return lr * 0.5 * (1.0 + math.cos(math.pi * min(count - warmup, span) / span))


def global_norm(grads) -> torch.Tensor:
    """optax.global_norm: sqrt of the sum over every leaf of sum(g^2)."""
    return torch.sqrt(sum((g.to(torch.float64) ** 2).sum() for g in grads.values()))


def clip_by_global_norm(grads, max_norm: float):
    """optax.clip_by_global_norm(max_norm): every leaf unchanged if norm < max_norm, else (g / norm) * max_norm.
    Returns (clipped tree, norm)."""
    norm = global_norm(grads)
    if norm < max_norm:
        return dict(grads), norm
    return {k: (g / norm.to(g.dtype)) * max_norm for k, g in grads.items()}, norm


def update(state: drq.OracleState, cfg: drq.OracleConfig, batch: dict, rnd, nets=frozenset(TXS), dtype=torch.float64,
           new_rng=None, opts: Optional[OptimizerOptions] = None):
    """drq.update with make_optimizer's options.  info["_grad_norm"][tx] = the global norm of each clipping tx's gradient."""
    opts = opts or OptimizerOptions()
    p0, t0 = state.params, state.target_params
    opt0 = {n: {"count": o["count"], "mu": dict(o["mu"]), "nu": dict(o["nu"])} for n, o in state.opt.items()}
    info = _drq_update(state, cfg, batch, rnd, nets, dtype, new_rng)         # gradients, infos, step, rng
    state.opt = opt0
    grads = info["_grads"]
    total = {k: torch.zeros_like(v) for k, v in p0.items()}
    info["_grad_norm"] = {}
    for name in TXS:                                                        # common.py:136-168: summed in tx order
        lr = lr_schedule(state.opt[name]["count"], opts.lr.get(name, cfg.lr), cfg.warmup[name], opts.cosine_decay_steps.get(name))
        g = grads[name]
        if opts.clip_grad_norm.get(name) is not None:                      # optax.chain(clip_by_global_norm, adam)
            g, info["_grad_norm"][name] = clip_by_global_norm(g, opts.clip_grad_norm[name])
        upd = drq.adam_tx_update(g, state.opt[name], lr)
        info[f"{name}_lr"] = lr
        for k in total:
            total[k] = total[k] + upd[k]
    state.params = {k: (p0[k] + total[k]).detach() for k in p0}
    state.target_params = t0
    if "critic" in nets:                                                    # common.py:124-134
        state.target_params = {k: state.params[k] * cfg.tau + t0[k] * (1 - cfg.tau) for k in state.params}
    return info


def _with_options(entry, opts, *args, **kw):
    last = {}

    def upd(*a, **k):
        info = update(*a, **k, opts=opts)
        last["norms"] = info["_grad_norm"]
        return info

    with mock.patch.object(drq, "update", upd):
        info = entry(*args, **kw)
    info["_grad_norm"] = last["norms"]                                      # of the last update the entry point ran
    return info


def update_critics(state, cfg, batch_unpacked, opts: OptimizerOptions, dtype=torch.float64):
    return _with_options(drq.update_critics, opts, state, cfg, batch_unpacked, dtype=dtype)


def update_high_utd(state, cfg, batch_unpacked, utd_ratio: int, opts: OptimizerOptions, dtype=torch.float64, augment: bool = True):
    return _with_options(drq.update_high_utd, opts, state, cfg, batch_unpacked, utd_ratio, dtype=dtype, augment=augment)
