"""ORACLE (test infrastructure, not product): the agents' public forward passes (agents/continuous/sac.py:33-116) restated in
torch on top of `oracle/drq.py` and `tests/arch_oracle.py`, float64 by default.

Follows (relative to serl_launcher/serl_launcher):
  networks/actor_critic_nets.py:33-46    multiple_action_q_function: actions (B, N, A) -> vmap of the critic over N -> (E, B, N)
  networks/actor_critic_nets.py:230-272  TanhMultivariateNormalDiag.log_prob of given actions: distrax Transformed with a Tanh
                                         bijector, log N(atanh(x); loc, diag(scale^2)) - sum 2 (log 2 - u - softplus(-2u))
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

import arch_oracle
from oracle import drq
from oracle import jax_prng as P


def tanh_normal_log_prob(means, stds, x):
    """log-probability of given actions x under tanh(N(means, diag(stds^2))); x is not clipped (|x| = 1 gives NaN)."""
    u = torch.atanh(torch.as_tensor(x).to(means.dtype))
    z = (u - means) / stds
    base = (-0.5 * z * z - torch.log(stds) - 0.5 * math.log(2 * math.pi)).sum(-1)
    fldj = (2.0 * (math.log(2.0) - u - F.softplus(-2.0 * u))).sum(-1)
    return base - fldj


def multi_action_critic(params, enc, actions, arch, pixel_agent: bool):
    """Q (E, B, N) of N candidate actions per state: one critic pass per candidate, stacked on the last axis."""
    actions = torch.as_tensor(actions).to(enc.dtype)
    return torch.stack([arch_oracle.critic_forward(params, enc, actions[:, n], arch, pixel_agent) for n in range(actions.shape[1])], -1)


def encoder(agent, params, obs, dropout_key=None, dtype=torch.float64):
    """enc(obs) for a batch: the state itself for the state agent; trunk + image heads + proprio head for the pixel agent, with
    camera j's keep-mask bernoulli(fold_in(dropout_key, j), 0.9) when a key is given (oracle/drq.py::_dropout_masks)."""
    cfg = agent._cfg
    if not cfg.pixel:
        return torch.as_tensor(np.asarray(obs)).to(dtype).reshape(np.asarray(obs).shape[0], -1)
    feats = {}
    for cam in cfg.cams:
        img = torch.as_tensor(np.asarray(obs[cam]))
        b, t, h, w, c = img.shape
        feats[cam] = drq.trunk_forward(params, cam, img.permute(0, 2, 3, 1, 4).reshape(b, h, w, t * c), dtype)
    B = np.asarray(obs["state"]).shape[0]
    masks = None
    if dropout_key is not None:
        masks = {c: torch.as_tensor(m) for c, m in drq._dropout_masks(np.asarray(dropout_key, np.uint32), cfg.cams, B).items()}
    return drq.encode(params, cfg.cams, feats, torch.as_tensor(np.asarray(obs["state"])), masks)


def critic(agent, params, obs, actions):
    """forward_critic of a batch: (E, B) for (B, A) actions, (E, B, N) for (B, N, A)."""
    cfg = agent._cfg
    enc = encoder(agent, params, obs)
    actions = torch.as_tensor(np.asarray(actions)).to(enc.dtype)
    if actions.dim() == 3:
        return multi_action_critic(params, enc, actions, cfg.critic_arch, cfg.pixel)
    return arch_oracle.critic_forward(params, enc, actions, cfg.critic_arch, cfg.pixel)


def policy(agent, params, obs, dropout_key=None):
    """forward_policy of a batch -> (loc, clipped std)."""
    cfg = agent._cfg
    enc = encoder(agent, params, obs, dropout_key)
    return arch_oracle.policy_forward(params, enc, cfg.policy_arch, cfg.std_parameterization, cfg.std_min, cfg.std_max)


def sample_and_log_prob(means, stds, seed):
    """TanhMultivariateNormalDiag.sample_and_log_prob(seed=seed): eps = normal(seed, (B, A)) as sample_actions draws it."""
    eps = torch.as_tensor(P.normal(np.asarray(seed, np.uint32), tuple(means.shape)))
    return drq.tanh_normal_sample_logp(means, stds, eps)
