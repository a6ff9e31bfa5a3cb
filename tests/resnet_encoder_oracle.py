"""ORACLE (test infrastructure, not product): DrQ's trainable "resnet" encoder restated in torch, float64 by default, plugged
into oracle/drq.py and tests/forward_oracle.py.

Follows (relative to serl_launcher/serl_launcher):
  agents/continuous/drq.py:153-166     ResNetEncoder(stage_sizes=(1,1,1,1), ResNetBlock, pre_pooling=False,
                                       pooling_method="spatial_learned_embeddings", num_spatial_blocks=8, bottleneck_dim=256) per
                                       camera, named encoder_<cam>; the `encode=` argument EncodingWrapper passes is dropped
  vision/resnet_v1.py:217-286          x = (uint8 / 255 - mean) / std; conv_init 7x7/2 pad (3, 3) -> GroupNorm -> relu ->
                                       max_pool 3x3/2 SAME; four ResNetBlocks (:129-156); then (pre_pooling=False) the
                                       SpatialLearnedEmbeddings(8) -> Dropout(0.1) -> Dense(256) -> LayerNorm -> tanh head
  common/encoding.py:26-72             per-camera embeddings (stop_gradient for the policy), concat, proprio Dense(64) ->
                                       LayerNorm -> tanh when the tree has its leaves
Max-pool gradient: to the first maximal element of each window in row-major window order (XLA select_and_scatter with `ge`),
pinned here by argmax (torch returns the first maximal index).
"""
from __future__ import annotations

import contextlib
from unittest import mock

import numpy as np
import torch
import torch.nn.functional as F

from oracle import drq


def max_pool_first_max(x):
    """max_pool 3x3 / stride 2, XLA SAME, on NHWC x; the gradient reaches each window's first maximal element."""
    N, H, W, C = x.shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    ph, pw = max((Ho - 1) * 2 + 3 - H, 0), max((Wo - 1) * 2 + 3 - W, 0)
    xp = F.pad(x.permute(0, 3, 1, 2), (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=float("-inf"))
    win = xp.unfold(2, 3, 2).unfold(3, 3, 2).reshape(N, C, Ho, Wo, 9)
    out = win.gather(-1, win.argmax(-1, keepdim=True)).squeeze(-1)
    return out.permute(0, 2, 3, 1)


def trunk(params, cam, images, dtype=torch.float64, keep=False):
    """images (N,H,W,3) uint8 -> the last block's output (N,H/32,W/32,512), differentiable w.r.t. the leaves under
    encoder_<cam>; keep: also return {name: activation} of the stem and blocks."""
    p = f"{drq.ENC}/encoder_{cam}"
    g = lambda k: params[f"{p}/{k}"].to(dtype)
    mean, std = torch.tensor(drq.IMAGENET_MEAN, dtype=dtype), torch.tensor(drq.IMAGENET_STD, dtype=dtype)
    x = (torch.as_tensor(np.asarray(images)).to(dtype) / 255.0 - mean) / std
    acts = {}
    x = drq.conv_nhwc(x, g("conv_init/kernel"), 2, 3, 3)
    x = drq.group_norm_nhwc(x, g("norm_init/scale"), g("norm_init/bias")).relu()
    acts["stem"] = x
    x = max_pool_first_max(x)
    acts["pool"] = x
    for i, (filters, stride) in enumerate(drq.STAGES):
        b = f"ResNetBlock_{i}"
        res = x
        lo, hi = drq.same_pads(x.shape[1], 3, stride)
        y = drq.conv_nhwc(x, g(f"{b}/Conv_0/kernel"), stride, lo, hi)
        y = drq.group_norm_nhwc(y, g(f"{b}/MyGroupNorm_0/scale"), g(f"{b}/MyGroupNorm_0/bias")).relu()
        y = drq.conv_nhwc(y, g(f"{b}/Conv_1/kernel"), 1, 1, 1)
        y = drq.group_norm_nhwc(y, g(f"{b}/MyGroupNorm_1/scale"), g(f"{b}/MyGroupNorm_1/bias"))
        if res.shape != y.shape:
            res = drq.conv_nhwc(res, g(f"{b}/conv_proj/kernel"), stride, 0, 0)
            res = drq.group_norm_nhwc(res, g(f"{b}/norm_proj/scale"), g(f"{b}/norm_proj/bias"))
        x = (res + y).relu()
        acts[b] = x
    return (x, acts) if keep else x


def image_embedding(params, cam, images, dropout_mask=None, dtype=torch.float64):
    p = f"{drq.ENC}/encoder_{cam}"
    f = trunk(params, cam, images, dtype)
    k = params[f"{p}/SpatialLearnedEmbeddings_0/kernel"]
    sle = torch.einsum("bhwc,hwcf->bcf", f, k).reshape(f.shape[0], -1)       # index c*8+f
    if dropout_mask is not None:
        sle = torch.where(torch.as_tensor(dropout_mask).bool(), sle / 0.9, torch.zeros_like(sle))
    z = sle @ params[f"{p}/Dense_0/kernel"] + params[f"{p}/Dense_0/bias"]
    return torch.tanh(drq.layer_norm(z, params[f"{p}/LayerNorm_0/scale"], params[f"{p}/LayerNorm_0/bias"]))


def encode(params, cams, images, state, dropout_masks=None, stop_gradient=False):
    """oracle.drq.encode for the resnet encoder: images[cam] are the (B,H,W,3) crops (what `trunk_forward` passes through
    below).  The proprio block is there when the tree has its leaves."""
    dt = params[f"{drq.ENC}/encoder_{cams[0]}/Dense_0/kernel"].dtype
    outs = []
    for cam in cams:
        img = image_embedding(params, cam, images[cam], None if dropout_masks is None else dropout_masks[cam], dt)
        outs.append(img.detach() if stop_gradient else img)
    if f"{drq.ENC}/Dense_0/kernel" in params:
        s = torch.as_tensor(np.asarray(state)).reshape(outs[0].shape[0], -1).to(dt)
        z = s @ params[f"{drq.ENC}/Dense_0/kernel"] + params[f"{drq.ENC}/Dense_0/bias"]
        outs.append(torch.tanh(drq.layer_norm(z, params[f"{drq.ENC}/LayerNorm_0/scale"], params[f"{drq.ENC}/LayerNorm_0/bias"])))
    return torch.cat(outs, dim=-1)


@contextlib.contextmanager
def resnet_encoder_oracle():
    """oracle/drq.py and tests/forward_oracle.py with the resnet encoder: the "trunk" passes the uint8 crops through, and
    `encode` runs the trainable ResNet-10 with whichever parameter tree it is given."""
    with mock.patch.object(drq, "trunk_forward", lambda params, cam, images_u8, dtype: torch.as_tensor(images_u8)), \
            mock.patch.object(drq, "encode", encode):
        yield
