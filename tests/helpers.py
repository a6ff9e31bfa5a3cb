"""Shared helpers for the GPU parity tests (product objects <-> oracle objects)."""
from __future__ import annotations

import contextlib
import types

import numpy as np
import torch


class Box:
    def __init__(self, shape, dtype=np.float32):
        self.shape, self.dtype = tuple(shape), np.dtype(dtype)


class DictSpace:
    def __init__(self, spaces):
        self.spaces = dict(spaces)


def pixel_spaces(cams, hw=128, T=1, S=7, A=4):
    obs = DictSpace({**{c: Box((T, hw, hw, 3), np.uint8) for c in cams}, "state": Box((T, S))})
    return obs, Box((A,))


def fake_env(cams, hw=128, T=1, S=7, A=4):
    o, a = pixel_spaces(cams, hw, T, S, A)
    return types.SimpleNamespace(observation_space=o, action_space=a)


def random_transitions(rng, n, cams, hw=128, T=1, S=7, A=4, mean_ep=12):
    """Consecutive transitions share frames like a real episode (next_obs of t == obs of t+1)."""
    out, cur = [], None
    for _ in range(n):
        if cur is None:
            cur = {c: rng.integers(0, 256, (T, hw, hw, 3), dtype=np.uint8) for c in cams}
            cur["state"] = rng.standard_normal((T, S)).astype(np.float32)
        nxt = {c: np.concatenate([cur[c][1:], rng.integers(0, 256, (1, hw, hw, 3), dtype=np.uint8)]) for c in cams}
        nxt["state"] = rng.standard_normal((T, S)).astype(np.float32)
        done = bool(rng.random() < 1.0 / mean_ep)
        out.append(dict(observations=cur, next_observations=nxt, actions=rng.uniform(-1, 1, A).astype(np.float32),
                        rewards=np.float32(rng.random()), masks=np.float32(0.0 if done else 1.0), dones=done))
        cur = None if done else nxt
    return out


def to_numpy_tree(d):
    if isinstance(d, dict):
        return {k: to_numpy_tree(v) for k, v in d.items()}
    return d.detach().cpu().numpy() if isinstance(d, torch.Tensor) else np.asarray(d)


def oracle_state_from_agent(agent, dtype=torch.float64):
    from oracle.drq import OracleState
    from serl_b200.params import flatten
    st = agent.state
    params = {k: torch.as_tensor(np.asarray(v)) for k, v in flatten(st.params).items()}
    o = OracleState.create(params, st.rng, dtype)
    o.target_params = {k: torch.as_tensor(np.asarray(v)).to(dtype) for k, v in flatten(st.target_params).items()}
    os_ = st.opt_states
    for name in ("actor", "critic", "temperature"):
        o.opt[name]["count"] = os_[name]["count"]
        o.opt[name]["mu"].update({k: torch.as_tensor(v).to(dtype) for k, v in flatten(os_[name]["mu"]).items()})
        o.opt[name]["nu"].update({k: torch.as_tensor(v).to(dtype) for k, v in flatten(os_[name]["nu"]).items()})
    return o


def oracle_cfg_from_agent(agent):
    from oracle.drq import OracleConfig
    c = agent._cfg
    return OracleConfig(cams=tuple(c.cams), discount=c.discount, tau=c.tau, target_entropy=c.target_entropy,
                        ensemble=c.ensemble, subsample=c.subsample, backup_entropy=c.backup_entropy, lr=c.lr[0],
                        warmup={"critic": c.warmup[0], "actor": c.warmup[1], "temperature": c.warmup[2]}, pixel=c.pixel)


@contextlib.contextmanager
def injected_features(pix, feats):
    """Feed the oracle an engine's own frozen-trunk features instead of its float64 trunk.

    pix[cam] (N,H,W,3) uint8 holds the crops the sampler wrote (obs rows, then next-obs rows) and feats[cam] (N,4,4,512)
    their features.  Each crop's bytes key its feature row.  While active, `oracle.drq._features` looks up every frame it
    is asked for and returns that row cast to the requested dtype.  The lookup is by content, not by call order, so it serves
    `update_critics`, `update_high_utd` and the pipelined path alike.  A frame with no match raises: the oracle's augmented
    crops must be bit-identical to the engine's.  Identical crops share the first row's features."""
    from oracle import drq as O
    tables = {}
    for cam in pix:
        p = np.ascontiguousarray(pix[cam].cpu().numpy() if isinstance(pix[cam], torch.Tensor) else pix[cam])
        rows = {}
        for i in range(p.shape[0]):
            rows.setdefault(p[i].tobytes(), i)
        tables[cam] = (rows, torch.as_tensor(feats[cam]).detach().cpu())

    def _features(state, cfg, obs, dtype):
        out = {}
        for cam in cfg.cams:
            img = np.asarray(obs[cam])                                    # (b,T,H,W,C) -> frames "B H W (T C)" as the oracle has them
            b, t, h, w, c = img.shape
            img = np.ascontiguousarray(img.transpose(0, 2, 3, 1, 4).reshape(b, h, w, t * c))
            rows, f = tables[cam]
            idx = [rows.get(img[i].tobytes()) for i in range(b)]
            missing = [i for i, j in enumerate(idx) if j is None]
            if missing:
                raise AssertionError(f"{cam}: {len(missing)} of {b} oracle frames match no engine crop (first: frame {missing[0]})")
            out[cam] = f[idx].to(dtype)
        return out

    saved = O._features
    O._features = _features
    try:
        yield
    finally:
        O._features = saved


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))
