"""ORACLE (test infrastructure, not product): the trainable encoders on stacks of T frames, as EncodingWrapper(enable_stacking=True)
feeds them (common/encoding.py:36-70): "B T H W C -> B H W (T C)", channel t*C + c is channel c of frame t, oldest frame first.

oracle/drq.py already crops each of the B*T frames with its own key and rearranges the stack before the encoder; the small
encoder's convs (tests/small_encoder_oracle.py) take any input width.  The ResNet's stem normalises by the ImageNet statistics
(resnet_v1.py:222-224), which broadcast over the channel axis: channel c of a stack takes those of channel c mod 3.
"""
from __future__ import annotations

import contextlib
from unittest import mock

import numpy as np

from oracle import drq
from resnet_encoder_oracle import resnet_encoder_oracle


def stack(images):
    """(B, T, H, W, C) -> (B, H, W, T*C), oldest frame first; (T, H, W, C) -> (H, W, T*C)."""
    x = np.asarray(images)
    if x.ndim == 4:
        return stack(x[None])[0]
    B, T, H, W, C = x.shape
    return np.ascontiguousarray(x.transpose(0, 2, 3, 1, 4).reshape(B, H, W, T * C))


@contextlib.contextmanager
def resnet_stack_oracle(T: int):
    """resnet_encoder_oracle on (B, H, W, 3T) stacks: the stem's mean / std tiled T times along the channel axis."""
    with mock.patch.object(drq, "IMAGENET_MEAN", list(drq.IMAGENET_MEAN) * T), \
            mock.patch.object(drq, "IMAGENET_STD", list(drq.IMAGENET_STD) * T), resnet_encoder_oracle():
        yield
