"""ORACLE (test infrastructure, not product): DrQ's "small" encoder restated in torch, float64 by default, plugged into
oracle/drq.py and tests/forward_oracle.py.

Follows (relative to serl_launcher/serl_launcher):
  agents/continuous/drq.py:137-152     SmallEncoder(features=(32, 64, 128, 256), kernel_sizes 3, strides 2, padding="VALID",
                                       pool_method="avg", bottleneck_dim=256) per camera, named encoder_<cam>
  vision/small_encoders.py:20-55       x = uint8 / 255; 4 x [nn.Conv (with bias) -> relu]; mean over the positions;
                                       Dense(256) -> LayerNorm -> tanh.  No SpatialLearnedEmbeddings, no Dropout.
  common/encoding.py:26-72             EncodingWrapper: per-camera embeddings (stop_gradient for the policy), concat, proprio
                                       Dense(64) -> LayerNorm -> tanh when use_proprio.  The `encode=` argument the reference
                                       passes to every encoder (:46) is dropped: SmallEncoder does not take it.
"""
from __future__ import annotations

import contextlib
from unittest import mock

import numpy as np
import torch

from oracle import drq

SMALL_CONVS = ((3, 32), (32, 64), (64, 128), (128, 256))


def conv_stack(params, cam, images, dtype=torch.float64, keep=False):
    """images (N,H,W,3) uint8 -> pooled (N,256); keep: also return the four post-ReLU maps."""
    p = f"{drq.ENC}/encoder_{cam}"
    x = torch.as_tensor(images).to(dtype) / 255.0
    maps = []
    for i in range(len(SMALL_CONVS)):
        x = (drq.conv_nhwc(x, params[f"{p}/Conv_{i}/kernel"], 2, 0, 0) + params[f"{p}/Conv_{i}/bias"]).relu()
        maps.append(x)
    pooled = x.mean(dim=(1, 2))
    return (pooled, maps) if keep else pooled


def image_embedding(params, cam, images, dtype=torch.float64):
    p = f"{drq.ENC}/encoder_{cam}"
    z = conv_stack(params, cam, images, dtype) @ params[f"{p}/Dense_0/kernel"] + params[f"{p}/Dense_0/bias"]
    return torch.tanh(drq.layer_norm(z, params[f"{p}/LayerNorm_0/scale"], params[f"{p}/LayerNorm_0/bias"]))


def encode(params, cams, images, state, dropout_masks=None, stop_gradient=False):
    """oracle.drq.encode for the small encoder: images[cam] are the (B,H,W,3) crops (what `trunk_forward` passes through below),
    dropout_masks do not apply.  The proprio block is there when the tree has its leaves."""
    dt = params[f"{drq.ENC}/encoder_{cams[0]}/Dense_0/kernel"].dtype
    outs = []
    for cam in cams:
        img = image_embedding(params, cam, images[cam], dt)
        outs.append(img.detach() if stop_gradient else img)
    if f"{drq.ENC}/Dense_0/kernel" in params:
        s = torch.as_tensor(np.asarray(state)).reshape(outs[0].shape[0], -1).to(dt)
        z = s @ params[f"{drq.ENC}/Dense_0/kernel"] + params[f"{drq.ENC}/Dense_0/bias"]
        outs.append(torch.tanh(drq.layer_norm(z, params[f"{drq.ENC}/LayerNorm_0/scale"], params[f"{drq.ENC}/LayerNorm_0/bias"])))
    return torch.cat(outs, dim=-1)


@contextlib.contextmanager
def small_encoder_oracle():
    """oracle/drq.py (update, update_critics, update_high_utd, sample_actions) and tests/forward_oracle.py with the small
    encoder: the "trunk" passes the uint8 crops through unchanged, and `encode` runs the conv stack with whichever parameter
    tree it is given (the differentiated leaves, the constant params or the target params)."""
    with mock.patch.object(drq, "trunk_forward", lambda params, cam, images_u8, dtype: torch.as_tensor(images_u8)), \
            mock.patch.object(drq, "encode", encode):
        yield
