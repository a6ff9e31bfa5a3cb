"""CPU restatement of the reference's binary reward classifier and its training step (test infrastructure only - never
imported by serl_b200/).

Follows networks/reward_classifier.py:16-89 (BinaryClassifier on EncodingWrapper(use_proprio=False, enable_stacking=True)
with one PreTrainedResNetEncoder per camera, vision/resnet_v1.py:324-376) and the train_step / augmentation of
examples/async_cable_route_drq/train_reward_classifier.py:108-157 (one optax.adam(1e-4) over the whole tree, the trunk is
stop-gradient).  Trunk, LayerNorm and Adam algebra are the functions of oracle/drq.py.  PARITY UNPINNED like oracle/drq.py
(jax / flax / optax are not installable here): the layer definitions are restated from their published forms.

Dropout keys are this repo's spec (DESIGN.md §4 (i)): camera j's SLE keep mask = bernoulli(fold_in(key, j), 0.9, (B, 4096)),
the hidden Dropout_0 keep mask = bernoulli(fold_in(key, ncams), 0.9, (B, 256)).
"""
from __future__ import annotations

import numpy as np
import torch

from . import drq as O
from . import jax_prng as P
from .replay import random_shift

ROOT = "encoder_def"
KEEP = 0.9


def features(params, cams, data, dtype):
    """Frozen-trunk features per camera from (B, 1, H, W, 3) frames ("B T H W C -> B H W (T C)", encoding.py:41-44)."""
    feats = {}
    for cam in cams:
        pre = f"{ROOT}/encoder_{cam}/pretrained_encoder/"
        trunk = {f"{O.ENC}/encoder_{cam}/pretrained_encoder/{k[len(pre):]}": v for k, v in params.items() if k.startswith(pre)}
        img = torch.as_tensor(np.asarray(data[cam]))
        b, t, h, w, c = img.shape
        feats[cam] = O.trunk_forward(trunk, cam, img.permute(0, 2, 3, 1, 4).reshape(b, h, w, t * c), dtype)
    return feats


def dropout_masks(key, cams, B):
    """(SLE keep masks {cam: (B, 4096)}, hidden keep mask (B, 256)) of one train_step key."""
    sle = {cam: P.bernoulli(P.fold_in(key, j), KEEP, (B, 4096)) for j, cam in enumerate(cams)}
    return sle, P.bernoulli(P.fold_in(key, len(cams)), KEEP, (B, 256))


def forward(params, cams, feats, sle_masks=None, hidden_mask=None, hidden_live=None, saves=None):
    """BinaryClassifier.__call__ -> logits (B, 1).  Masks None: train=False (no dropout).

    hidden_live: optional (B, 256) bool, the hidden relu's active set to use instead of `pre > 0`.  An implementation whose
    pre-activation lands on the other side of 0 within its rounding takes the other branch of relu's derivative, which moves
    a gradient leaf by about 1/B of its max; passing that implementation's own active set compares the rest of the step.
    saves: optional dict; receives the hidden LayerNorm output (the relu's input) under "hidden_pre"."""
    outs = []
    for cam in cams:
        pre = f"{ROOT}/encoder_{cam}"
        k = params[f"{pre}/SpatialLearnedEmbeddings_0/kernel"]
        f = feats[cam].to(k.dtype)
        sle = torch.einsum("bhwc,hwcf->bcf", f, k).reshape(f.shape[0], -1)           # index c*8+f
        if sle_masks is not None:
            sle = torch.where(torch.as_tensor(np.asarray(sle_masks[cam])).bool(), sle / KEEP, torch.zeros_like(sle))
        z = sle @ params[f"{pre}/Dense_0/kernel"] + params[f"{pre}/Dense_0/bias"]
        outs.append(torch.tanh(O.layer_norm(z, params[f"{pre}/LayerNorm_0/scale"], params[f"{pre}/LayerNorm_0/bias"])))
    x = torch.cat(outs, dim=-1)
    z = x @ params["Dense_0/kernel"] + params["Dense_0/bias"]
    if hidden_mask is not None:                                                     # Dropout BEFORE the LayerNorm
        z = torch.where(torch.as_tensor(np.asarray(hidden_mask)).bool(), z / KEEP, torch.zeros_like(z))
    pre = O.layer_norm(z, params["LayerNorm_0/scale"], params["LayerNorm_0/bias"])
    if saves is not None:
        saves["hidden_pre"] = pre.detach()
    if hidden_live is None:
        h = torch.relu(pre)
    else:
        h = torch.where(torch.as_tensor(np.asarray(hidden_live)).bool(), pre, torch.zeros_like(pre))
    return h @ params["Dense_1/kernel"] + params["Dense_1/bias"]


def bce(logits, labels):
    """optax.sigmoid_binary_cross_entropy, element-wise, in the overflow-free form max(x,0) - x*y + log1p(exp(-|x|))."""
    return logits.clamp_min(0) - logits * labels + torch.log1p(torch.exp(-logits.abs()))


def accuracy(logits_eval, labels):
    """mean((sigmoid(logits) >= 0.5) == labels) with sigmoid evaluated in float32 (a tiny negative logit rounds to exactly 0.5)."""
    x = np.asarray(logits_eval, np.float32)
    s = np.float32(1) / (np.float32(1) + np.exp(-x))
    return float(np.mean((s >= np.float32(0.5)).astype(np.float32) == np.asarray(labels, np.float32)))


def train_step(params, opt, cams, batch, key=None, masks=None, lr=1e-4, dtype=torch.float64, hidden_live=None):
    """One train_step.  params: flat {path: tensor} incl. the frozen trunk; opt = {"count", "mu", "nu"} over the trainable leaves;
    masks: (sle masks, hidden mask) or None -> keyed by `key`; hidden_live: the train pass's relu active set (see `forward`).
    Returns (new_params, opt, info, grads); info["_hidden_pre"] is the train pass's relu input."""
    data = batch["data"]
    labels = torch.as_tensor(np.asarray(batch["labels"])).to(dtype).reshape(-1, 1)
    B = labels.shape[0]
    p = {k: v.detach().to(dtype) for k, v in params.items()}
    train = {k: v.clone().requires_grad_(True) for k, v in p.items() if "pretrained_encoder" not in k}
    full = {**p, **train}
    feats = features(p, cams, data, dtype)
    sle_m, hid_m = masks if masks is not None else dropout_masks(np.asarray(key, np.uint32), cams, B)
    saves = {}
    logits = forward(full, cams, feats, sle_m, hid_m, hidden_live, saves)
    loss = bce(logits, labels).mean()
    gs = torch.autograd.grad(loss, list(train.values()))
    grads = {k: g for k, g in zip(train, gs)}
    with torch.no_grad():
        logits_eval = forward(p, cams, feats)
    upd = O.adam_tx_update(grads, opt, lr)
    new_params = dict(p)
    for k in train:
        new_params[k] = p[k] + upd[k]
    info = {"loss": loss.item(), "accuracy": accuracy(logits_eval.numpy(), labels.numpy()), "_logits": logits.detach(),
            "_logits_eval": logits_eval, "_hidden_pre": saves["hidden_pre"]}
    return new_params, opt, info, grads


def crop_batch(pos_next_frames, neg_obs_frames, key):
    """The script's data_augmentation_fn on concat(positive next_observations, negative observations): one
    batched_random_crop(key, padding=4, num_batch_dims=2) over the whole batch, the same offsets for every camera.
    frames: {cam: (B/2, 1, H, W, 3)} -> {cam: (B, 1, H, W, 3)}."""
    out = {}
    for cam in pos_next_frames:
        x = np.concatenate([np.asarray(pos_next_frames[cam]), np.asarray(neg_obs_frames[cam])])
        b, t = x.shape[:2]
        off = P.crop_offsets(np.asarray(key, np.uint32), b * t)                       # frame i uses split(key, B*T)[i]
        out[cam] = random_shift(x.reshape(b * t, *x.shape[2:]), off).reshape(x.shape)
    return out
