"""ORACLE (test infrastructure, not product): SAC / DrQ updates with the reference MLP's dropout_rate (dropout Q-functions), on
top of `oracle/drq.py` and `tests/arch_oracle.py`.

Follows (relative to serl_launcher/serl_launcher):
  networks/mlp.py:22-31                 Dense -> Dropout(rate) -> [LayerNorm] -> activation when train=True; kept units * 1/(1-rate)
  networks/actor_critic_nets.py:156-164 ensemblize = nn.vmap(split_rngs={"params": True}): the dropout rng is broadcast, so the E
                                        members of one critic forward share layer i's (B, H_i) mask
  agents/continuous/sac.py:134-234      which forwards run with train=True, and their keys: critic loss - policy on s' k_na, target
                                        critic c1, online critic c2 (critic_subsample_size) or c1; actor loss - policy k_p, critic
                                        critic_rng; temperature loss - policy k
Mask bits follow the repository's convention (DESIGN.md §4): hidden layer i's keep mask = bernoulli(fold_in(key, ncams + i), 1 - rate,
(B, H_i)), ncams = 0 for the state agent.

`networks(...)` runs oracle/drq.py's update / update_critics / update_high_utd with these networks: each `update` consumes the masks
`derive_mlp_masks` gives for its key, in the order the loss functions call the networks.  The masks can also be given explicitly
(`update(..., mlp_masks=...)`), so tests can hold them fixed.
"""
from __future__ import annotations

import contextlib
from unittest import mock

import numpy as np
import torch

from arch_oracle import ACTIVATIONS
from oracle import drq
from oracle import jax_prng as P


def mlp_masks(key, ncams, B, arch):
    """The (B, H_i) keep masks of one train=True forward of an MLP with key `key`; None without dropout."""
    if not arch.dropout:
        return None
    return [P.bernoulli(P.fold_in(key, ncams + i), 1.0 - arch.dropout, (B, H)) for i, H in enumerate(arch.hidden)]


def mlp(params, prefix, x, arch, ensemble: bool, masks=None):
    """arch_oracle.mlp with Dropout: masks[i] (B, H_i) broadcast over the ensemble axis."""
    act = ACTIVATIONS[arch.act]
    for i in range(len(arch.hidden)):
        w, b = params[f"{prefix}/Dense_{i}/kernel"], params[f"{prefix}/Dense_{i}/bias"]
        if ensemble:
            x = (torch.einsum("bi,eio->ebo", x, w) if x.dim() == 2 else torch.einsum("ebi,eio->ebo", x, w)) + b[:, None, :]
        else:
            x = x @ w + b
        if masks is not None:
            m = torch.as_tensor(np.asarray(masks[i]))
            x = torch.where(m, x / (1.0 - arch.dropout), torch.zeros_like(x))
        if arch.layer_norm:
            sc, bi = params[f"{prefix}/LayerNorm_{i}/scale"], params[f"{prefix}/LayerNorm_{i}/bias"]
            x = drq.layer_norm(x, sc[:, None, :], bi[:, None, :]) if ensemble else drq.layer_norm(x, sc, bi)
        x = act(x)
    return x


def critic_forward(params, enc, actions, arch, pixel_agent=True, masks=None):
    x = torch.cat([enc, actions.to(enc.dtype)], dim=-1)
    h = mlp(params, "modules_critic/network", x, arch, ensemble=True, masks=masks)
    w, b = params["modules_critic/Dense_0/kernel"], params["modules_critic/Dense_0/bias"]
    if pixel_agent:
        return (h @ w + b).squeeze(-1)
    return (torch.einsum("ebi,eio->ebo", h, w) + b[:, None, :]).squeeze(-1)


def policy_forward(params, enc, arch, std_parameterization="exp", std_min=1e-5, std_max=5.0, masks=None):
    import torch.nn.functional as F
    h = mlp(params, "modules_actor/network", enc, arch, ensemble=False, masks=masks)
    means = h @ params["modules_actor/Dense_0/kernel"] + params["modules_actor/Dense_0/bias"]
    if std_parameterization == "uniform":
        stds = torch.exp(params["modules_actor/log_stds"]).expand_as(means)
    else:
        x = h @ params["modules_actor/Dense_1/kernel"] + params["modules_actor/Dense_1/bias"]
        stds = torch.exp(x) if std_parameterization == "exp" else F.softplus(x)
    return means, torch.clamp(stds, std_min, std_max)


def update_keys(rng, nets, subsample: bool):
    """The MLP dropout keys of SACAgent.update from the rng it splits (derive_update_randomness's `rng`), per network call in the
    order the loss functions make them: [("policy" | "critic", key), ...]."""
    _, k_actor, k_critic, k_temp = P.split(rng, 4)
    calls = []
    if "critic" in nets:
        c1, k_na = P.split(k_critic)                        # sac.py:137
        c2, _ = P.split(c1)                                 # sac.py:152
        calls += [("policy", k_na), ("critic", c1), ("critic", c2 if subsample else c1)]
    if "actor" in nets:
        _, k_p, _, k_c = P.split(k_actor, 4)                # sac.py:197
        calls += [("policy", k_p), ("critic", k_c)]
    if "temperature" in nets:
        _, k = P.split(k_temp)                              # sac.py:224
        calls += [("policy", k)]
    return calls


def derive_mlp_masks(rng, nets, B, ncams, critic_arch, policy_arch, subsample: bool):
    """[(network, masks or None), ...] of one update, in call order (see update_keys)."""
    arch = {"critic": critic_arch, "policy": policy_arch}
    return [(net, mlp_masks(key, ncams, B, arch[net])) for net, key in update_keys(rng, nets, subsample)]


@contextlib.contextmanager
def networks(critic_arch, policy_arch, std_parameterization="exp", std_min=1e-5, std_max=5.0):
    """oracle/drq.py with dropout MLPs.  Every drq.update draws its masks from the rng derive_update_randomness split (or takes
    `mlp_masks=`); forward calls outside an update (sample_actions) run with train=False."""
    queue = []
    last = {}

    def cf(params, enc, actions, pixel_agent=True):
        m = None
        if queue:
            net, m = queue.pop(0)
            assert net == "critic", "the critic was called where the loss calls the policy"
        return critic_forward(params, enc, actions, critic_arch, pixel_agent, m)

    def pf(params, enc, *a, **k):
        m = None
        if queue:
            net, m = queue.pop(0)
            assert net == "policy", "the policy was called where the loss calls the critic"
        return policy_forward(params, enc, policy_arch, std_parameterization, std_min, std_max, m)

    derive, update = drq.derive_update_randomness, drq.update

    def derive_wrap(rng, B, A, cams, pixel, ensemble=10, subsample=2, nets=("critic", "actor", "temperature")):
        out = derive(rng, B, A, cams, pixel, ensemble, subsample, nets)
        last["masks"] = derive_mlp_masks(rng, nets, B, len(cams) if pixel else 0, critic_arch, policy_arch, bool(subsample))
        return out

    def update_wrap(state, cfg, batch, rnd, nets=frozenset({"actor", "critic", "temperature"}), dtype=torch.float64, new_rng=None,
                    mlp_masks=None):
        given = mlp_masks if mlp_masks is not None else last.pop("masks")
        queue[:] = list(given)
        info = update(state, cfg, batch, rnd, nets, dtype, new_rng)
        assert not queue, f"{len(queue)} mask sets left unused"
        info["_mlp_masks"] = given
        return info

    with mock.patch.object(drq, "critic_forward", cf), mock.patch.object(drq, "policy_forward", pf), \
            mock.patch.object(drq, "derive_update_randomness", derive_wrap), mock.patch.object(drq, "update", update_wrap):
        yield


def networks_of(agent):
    c = agent._cfg
    return networks(c.critic_arch, c.policy_arch, c.std_parameterization, c.std_min, c.std_max)
