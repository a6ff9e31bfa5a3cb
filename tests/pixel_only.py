"""Shared pieces of the pixel-only DrQ tests (use_proprio=False): an environment whose observations are camera images only, its
transitions, the agent the SERL launcher would build for it, and the float64 oracle with the encoder the reference's
EncodingWrapper builds when use_proprio=False (common/encoding.py:26-72: the per-camera image embeddings, concatenated)."""
from __future__ import annotations

import contextlib
import types
from unittest import mock

import numpy as np
import torch

from helpers import Box, DictSpace, random_transitions

LAUNCHER_POLICY = {"tanh_squash_distribution": True, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5}


def pixel_only_env(cams, hw=128, T=1, A=4):
    obs = DictSpace({c: Box((T, hw, hw, 3), np.uint8) for c in cams})
    return types.SimpleNamespace(observation_space=obs, action_space=Box((A,)))


def strip_state(tr):
    """A transition (or batch) without its "state" entries."""
    out = dict(tr)
    for k in ("observations", "next_observations"):
        out[k] = {c: v for c, v in tr[k].items() if c != "state"}
    return out


def pixel_only_transitions(rng, n, cams, hw=128, T=1, A=4, mean_ep=12):
    return [strip_state(tr) for tr in random_transitions(rng, n, cams, hw, T, 7, A, mean_ep)]


def make_agent(seed, sample_obs, sample_action, cams, use_proprio=False, precision="fp32", device=None):
    """DrQAgent.create_drq with make_drq_agent's hyper-parameters, use_proprio as given."""
    from serl_b200.agents.continuous.drq import DrQAgent
    kw = {} if device is None else {"device": device}
    return DrQAgent.create_drq(seed, sample_obs, sample_action, encoder_type="resnet-pretrained", use_proprio=use_proprio,
                               image_keys=tuple(cams), policy_kwargs=dict(LAUNCHER_POLICY), temperature_init=1e-2, discount=0.96,
                               backup_entropy=False, critic_ensemble_size=10, critic_subsample_size=2, precision=precision, **kw)


def with_empty_state(batch):
    """A host batch with zero-width "state" entries: the oracle's update reads obs["state"], which the pixel-only encoder ignores."""
    out = dict(batch)
    B = np.asarray(batch["rewards"]).shape[0]
    for k in ("observations", "next_observations"):
        out[k] = dict(batch[k])
        out[k]["state"] = np.zeros((B, 1, 0), np.float32)
    return out


@contextlib.contextmanager
def pixel_only_oracle():
    """oracle/drq.py (update, update_critics, update_high_utd, sample_actions) and tests/forward_oracle.py with the encoder
    EncodingWrapper builds for use_proprio=False (encoding.py:26-72): the concatenated camera embeddings.

    The camera embeddings are computed by oracle.drq.encode itself, so its image path (SLE contraction, dropout scaling, Dense,
    LayerNorm, tanh, stop_gradient) is the one and only restatement the tests use.  It is called with a stand-in proprio block
    whose output is identically zero (a zero state column into an all-zero Dense) and the 64 proprio columns it appends are
    dropped; the stand-in leaves are constants, so no gradient reaches or leaves them."""
    from oracle import drq
    encode = drq.encode

    def images_only(params, cams, feats, state, dropout_masks=None, stop_gradient=False):
        state = torch.as_tensor(np.asarray(state))
        assert state.numel() == 0, "the pixel-only encoder reads no state vector"
        dt = params[f"{drq.ENC}/encoder_{cams[0]}/Dense_0/kernel"].dtype
        empty = {f"{drq.ENC}/Dense_0/kernel": torch.zeros(1, 64, dtype=dt), f"{drq.ENC}/Dense_0/bias": torch.zeros(64, dtype=dt),
                 f"{drq.ENC}/LayerNorm_0/scale": torch.ones(64, dtype=dt), f"{drq.ENC}/LayerNorm_0/bias": torch.zeros(64, dtype=dt)}
        assert not any(k in params for k in empty), "a pixel-only parameter tree has no proprio leaves"
        enc = encode({**params, **empty}, cams, feats, torch.zeros(state.shape[0], 1, dtype=dt), dropout_masks, stop_gradient)
        return enc[:, :256 * len(cams)]

    with mock.patch.object(drq, "encode", images_only):
        yield
