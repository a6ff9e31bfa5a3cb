"""ORACLE (test infrastructure, not product): the reference's general MLP and the policy's std parameterisations, restated
in torch on top of `oracle/drq.py`, whose `mlp2` / `critic_forward` / `policy_forward` build the launcher architecture only.

Follows (relative to serl_launcher/serl_launcher):
  networks/mlp.py:10-32                 MLP: per hidden width Dense -> [LayerNorm] -> activation (activate_final=True, as the
                                        agents' constructors force it)
  networks/actor_critic_nets.py:190-210 std head: "exp" exp(Dense), "softplus" softplus(Dense), "uniform" exp(log_stds) with a
                                        free (A,) leaf; then clip(std, std_min, std_max)
Activations restated from the published flax / jax definitions (parity unpinned, like the rest of the oracle): tanh;
relu = max(x, 0) (jax's derivative at 0 is 0); swish = silu = x * sigmoid(x); leaky_relu = where(x >= 0, x, 0.01 x);
gelu(approximate=True) = x * 0.5 * (1 + tanh(sqrt(2/pi) * (x + 0.044715 x^3))).

`networks(...)` is a context manager that runs oracle/drq.py's step, update_critics, update_high_utd and sample_actions (and
oracle/optim.py's, which call them) with these networks in place of the launcher ones.
"""
from __future__ import annotations

import contextlib
import math
from unittest import mock

import torch
import torch.nn.functional as F

from oracle import drq


def _relu(x):
    return torch.where(x > 0, x, torch.zeros_like(x))


def _swish(x):
    return x * torch.sigmoid(x)


def _leaky_relu(x):
    return torch.where(x >= 0, x, 0.01 * x)


def _gelu(x):
    return x * (0.5 * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3))))


ACTIVATIONS = {"tanh": torch.tanh, "relu": _relu, "swish": _swish, "leaky_relu": _leaky_relu, "gelu": _gelu}


def mlp(params, prefix, x, arch, ensemble: bool):
    """mlp.py:22-31 for an MlpArch (hidden, act, layer_norm).  Ensemble params have a leading E axis."""
    act = ACTIVATIONS[arch.act]
    for i in range(len(arch.hidden)):
        w, b = params[f"{prefix}/Dense_{i}/kernel"], params[f"{prefix}/Dense_{i}/bias"]
        if ensemble:
            x = (torch.einsum("bi,eio->ebo", x, w) if x.dim() == 2 else torch.einsum("ebi,eio->ebo", x, w)) + b[:, None, :]
        else:
            x = x @ w + b
        if arch.layer_norm:
            sc, bi = params[f"{prefix}/LayerNorm_{i}/scale"], params[f"{prefix}/LayerNorm_{i}/bias"]
            x = drq.layer_norm(x, sc[:, None, :], bi[:, None, :]) if ensemble else drq.layer_norm(x, sc, bi)
        x = act(x)
    return x


def critic_forward(params, enc, actions, arch, pixel_agent: bool = True):
    """actor_critic_nets.py:57-73 -> (E,B), as drq.critic_forward with a general backbone."""
    x = torch.cat([enc, actions.to(enc.dtype)], dim=-1)
    h = mlp(params, "modules_critic/network", x, arch, ensemble=True)
    w, b = params["modules_critic/Dense_0/kernel"], params["modules_critic/Dense_0/bias"]
    if pixel_agent:
        return (h @ w + b).squeeze(-1)
    return (torch.einsum("ebi,eio->ebo", h, w) + b[:, None, :]).squeeze(-1)


def policy_forward(params, enc, arch, std_parameterization="exp", std_min=1e-5, std_max=5.0):
    """actor_critic_nets.py:178-210 -> (means, clipped stds)."""
    h = mlp(params, "modules_actor/network", enc, arch, ensemble=False)
    means = h @ params["modules_actor/Dense_0/kernel"] + params["modules_actor/Dense_0/bias"]
    if std_parameterization == "uniform":
        stds = torch.exp(params["modules_actor/log_stds"]).expand_as(means)
    else:
        x = h @ params["modules_actor/Dense_1/kernel"] + params["modules_actor/Dense_1/bias"]
        stds = torch.exp(x) if std_parameterization == "exp" else F.softplus(x)
    return means, torch.clamp(stds, std_min, std_max)


@contextlib.contextmanager
def networks(critic_arch, policy_arch, std_parameterization="exp", std_min=1e-5, std_max=5.0):
    """oracle/drq.py with these networks (see the module docstring)."""
    cf = lambda params, enc, actions, pixel_agent=True: critic_forward(params, enc, actions, critic_arch, pixel_agent)
    pf = lambda params, enc, *a, **k: policy_forward(params, enc, policy_arch, std_parameterization, std_min, std_max)
    with mock.patch.object(drq, "critic_forward", cf), mock.patch.object(drq, "policy_forward", pf):
        yield


def networks_of(agent):
    """networks(...) with an agent's architecture and std clip."""
    c = agent._cfg
    return networks(c.critic_arch, c.policy_arch, c.std_parameterization, c.std_min, c.std_max)
