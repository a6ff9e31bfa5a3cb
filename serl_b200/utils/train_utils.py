"""Batch plumbing helpers with the reference's names (utils/train_utils.py:16-66,69-130)."""
from __future__ import annotations

import os
import pickle as pkl

import numpy as np
import torch

from ..data.replay_buffer import BatchHandle


def concat_batches(offline_batch, online_batch, axis=1):
    """utils/train_utils.py:16-31: per-leaf concatenate (first argument's rows first).
    Lazy `BatchHandle`s are concatenated symbolically - no data moves until the agent consumes them."""
    if isinstance(offline_batch, BatchHandle) and isinstance(online_batch, BatchHandle):
        if axis != 0:
            raise ValueError("lazy replay batches concatenate along the batch axis (axis=0)")
        return offline_batch.concat(online_batch)
    if isinstance(offline_batch, BatchHandle):
        offline_batch = offline_batch.to_dict()
    if isinstance(online_batch, BatchHandle):
        online_batch = online_batch.to_dict()
    out = {}
    for k, v in offline_batch.items():
        if isinstance(v, dict):
            out[k] = concat_batches(v, online_batch[k], axis=axis)
        elif isinstance(v, torch.Tensor):
            out[k] = torch.cat((v, torch.as_tensor(online_batch[k], device=v.device)), dim=axis)
        else:
            out[k] = np.concatenate((np.asarray(v), np.asarray(online_batch[k])), axis=axis)
    return out


def _unpack(batch):
    """utils/train_utils.py:44-66: packed (B,T+1,...) pixels -> obs[:, :-1], next_obs[:, 1:]."""
    if isinstance(batch, BatchHandle):
        return batch
    obs, nobs = dict(batch["observations"]), dict(batch["next_observations"])
    for k, v in batch["observations"].items():
        if k not in batch["next_observations"]:
            obs[k], nobs[k] = v[:, :-1], v[:, 1:]
    out = dict(batch)
    out["observations"], out["next_observations"] = obs, nobs
    return out


def _resnet10_pickle(path=None):
    """The local `resnet10_params.pkl` (path, ./resnet10_params.pkl or ~/.serl/resnet10_params.pkl), loaded, or None."""
    candidates = [path, "resnet10_params.pkl", os.path.expanduser("~/.serl/resnet10_params.pkl")]
    file_path = next((p for p in candidates if p and os.path.exists(p)), None)
    if file_path is None:
        print("resnet10_params.pkl not found locally (no network): keeping synthetic ResNet-10 weights")
        return None
    with open(file_path, "rb") as f:
        return pkl.load(f)


def replace_pretrained_leaves(tree, encoder_params, image_keys, root=("modules_actor", "encoder")):
    """Writes the pickle's ResNet-10 leaves into tree[root...][f"encoder_{key}"]["pretrained_encoder"] (in place)."""
    for image_key in image_keys:
        enc = tree
        for r in root:
            enc = enc[r]
        enc = enc[f"encoder_{image_key}"]
        enc = enc.get("pretrained_encoder", enc)
        for k in list(enc):
            if k in encoder_params:
                enc[k] = {kk: np.asarray(vv) for kk, vv in encoder_params[k].items()} if isinstance(encoder_params[k], dict) \
                    else np.asarray(encoder_params[k])
                print(f"replaced {k} in pretrained_encoder")
    return tree


def load_resnet10_params(agent, image_keys=("image",), public=True, path=None):
    """utils/train_utils.py:69-130.  The reference downloads `resnet10_params.pkl` from a GitHub release;
    there is no network here, so only a local pickle is honoured (path, ./resnet10_params.pkl or
    ~/.serl/resnet10_params.pkl).  Absent file -> the agent keeps its synthetic kaiming-normal trunk.
    The reward classifier (networks/reward_classifier.py) loads the same pickle under its `encoder_def` root."""
    encoder_params = _resnet10_pickle(path)
    if encoder_params is None:
        return agent
    tree = replace_pretrained_leaves(agent.state.params, encoder_params, image_keys)
    return agent.replace(state=agent.state.replace(params=tree))
