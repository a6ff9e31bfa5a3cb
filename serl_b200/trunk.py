"""The frozen ResNet-10 trunk (reference vision/resnet_v1.py:217-286) of one agent or classifier.

`FrozenTrunk` is created once per agent or classifier.  It holds the fp32 HWIO leaves per camera, reads and writes them as the
`pretrained_encoder` subtrees of a parameter tree (`dump` / `load`: what `TrainState`, checkpoints and `replace` go through), and
keeps their packed 16-bit copy for the tensor-core build and every runner it handed out.

Both builds encode 128x128 frames only: the trunk maps them to the (4, 4, 512) features every consumer allocates and the SLE
head's kernel expects.

A `TrunkRunner` is one caller's scratch for passes over up to N images: the fp32 build's activation buffers (the cameras run one
after the other), or one 16-bit plan per camera (the cameras of a step may run concurrently), and the flag the 16-bit kernels
raise on a pipeline-barrier timeout.  Callers that run concurrently (the two engines of the step pipeline, an inference engine
next to them) each take their own runner.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib as L
from . import ops, trunk_bf16
from .params import STAGES

f32 = torch.float32


class FrozenTrunk:
    def __init__(self, leaves: Dict[str, Dict[str, torch.Tensor]], precision: str, image_hw: int = 128):
        if leaves and image_hw != 128:
            raise NotImplementedError(f"FrozenTrunk: the frozen ResNet-10 trunk takes 128x128 frames (its (4, 4, 512) features), "
                                      f"got {image_hw}x{image_hw}")
        self.leaves, self.precision, self.image_hw = leaves, precision, image_hw
        self._packed: Dict[str, tuple] = {}          # cam -> (leaf versions, packed 16-bit weights)
        self._runners: List[TrunkRunner] = []

    def runner(self, N: int, device) -> "TrunkRunner":
        r = TrunkRunner(self, N, device)
        self._runners.append(r)
        return r

    def packed(self, cam: str) -> dict:
        """The 16-bit weights of `cam`, packed again when a leaf has been written since the last packing (its `_version` moved).
        Captured CUDA graphs hold the packed tensors' addresses and the stem sign mask: whoever writes the leaves drops the graphs
        that read them (and, with `drop_packed`, the packing) before the next replay."""
        w = self.leaves[cam]
        ver = tuple(t._version for t in w.values())
        if cam not in self._packed or self._packed[cam][0] != ver:
            self._packed[cam] = (ver, trunk_bf16.pack_trunk(w, trunk_bf16.FMT[self.precision][1]))
        return self._packed[cam][1]

    def drop_packed(self):
        """Frees the packed copy; the next 16-bit pass packs the leaves again."""
        self._packed.clear()

    def dump(self, prefix: Callable[[str], str], cams: Optional[Sequence[str]] = None) -> Dict[str, np.ndarray]:
        """{f"{prefix(cam)}/{leaf}": host array} of every camera (or of `cams`); prefix(cam) is the tree path of the camera's
        `pretrained_encoder`."""
        return {f"{prefix(cam)}/{k}": v.detach().cpu().numpy() for cam in (self.leaves if cams is None else cams)
                for k, v in self.leaves[cam].items()}

    def load(self, flat: Dict[str, object], prefix: Callable[[str], str]):
        """Writes the leaves `flat` holds under prefix(cam) and drops the 16-bit packing made from the old ones."""
        for cam, w in self.leaves.items():
            for k, t in w.items():
                key = f"{prefix(cam)}/{k}"
                if key in flat:
                    t.copy_(torch.as_tensor(np.asarray(flat[key], np.float32)).reshape(t.shape))
        self.drop_packed()

    def check_error(self):
        """Raises if a 16-bit trunk kernel of any runner flagged a pipeline-barrier timeout (synchronises)."""
        for r in self._runners:
            if int(r.error.item()):
                raise L.SerlError("frozen trunk: a tensor-core convolution timed out on a pipeline barrier (flagged by the kernel)")


class TrunkRunner:
    def __init__(self, owner: FrozenTrunk, N: int, device):
        self.owner, self.N, self.dev = owner, N, torch.device(device)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.plans: Dict[str, trunk_bf16._Plan] = {}
        self._f32 = None

    def plan(self, cam: str) -> trunk_bf16._Plan:
        """The 16-bit activation buffers of `cam`, allocated by its first pass."""
        if cam not in self.plans:
            self.plans[cam] = trunk_bf16._Plan(self.N, self.owner.image_hw, self.dev, self.owner.precision, self.error)
        return self.plans[cam]

    def _on_device(self, t: torch.Tensor) -> bool:
        d = self.dev
        if t.device.type != d.type:
            return False
        return d.index is None or t.device.index == d.index

    def check_pass(self, pix: torch.Tensor, feats: torch.Tensor):
        """Raises ValueError unless pix is a contiguous (n, hw, hw, 3) uint8 pass of 1 <= n <= N frames and feats contiguous fp32
        with at least n rows of (4, 4, 512), both on the runner's device: the kernels index both by n and trust those shapes."""
        hw = self.owner.image_hw
        if not (isinstance(pix, torch.Tensor) and pix.dtype == torch.uint8 and pix.dim() == 4 and tuple(pix.shape[1:]) == (hw, hw, 3)
                and pix.is_contiguous()):
            got = (tuple(pix.shape), pix.dtype, pix.is_contiguous()) if isinstance(pix, torch.Tensor) else type(pix)
            raise ValueError(f"trunk pass: pix must be a contiguous (n, {hw}, {hw}, 3) uint8 tensor, got {got}")
        n = pix.shape[0]
        if not 1 <= n <= self.N:
            raise ValueError(f"trunk pass of {n} images on a runner for 1..{self.N}")
        if not (isinstance(feats, torch.Tensor) and feats.dtype == f32 and feats.dim() == 4 and tuple(feats.shape[1:]) == (4, 4, 512)
                and feats.shape[0] >= n and feats.is_contiguous()):
            got = (tuple(feats.shape), feats.dtype, feats.is_contiguous()) if isinstance(feats, torch.Tensor) else type(feats)
            raise ValueError(f"trunk pass: feats must be contiguous float32 with at least {n} rows of (4, 4, 512), got {got}")
        if not (self._on_device(pix) and self._on_device(feats)):
            raise ValueError(f"trunk pass: pix ({pix.device}) and feats ({feats.device}) must be on the runner's device {self.dev}")

    def forward(self, cam: str, pix: torch.Tensor, feats: torch.Tensor) -> torch.Tensor:
        """pix (n, hw, hw, 3) uint8, 1 <= n <= N -> feats[:n] (n, 4, 4, 512) fp32.  Anything else is refused before any launch
        (check_pass)."""
        self.check_pass(pix, feats)
        w = self.owner.leaves[cam]
        if self.owner.precision != "fp32":
            return trunk_bf16.forward(self.plan(cam), w, self.owner.packed(cam), pix, feats)
        N, hw = pix.shape[0], pix.shape[1]
        s = hw // 2
        if self._f32 is None:
            e = lambda *sh: torch.empty(*sh, dtype=f32, device=self.dev)
            self._f32 = (e(self.N, s, s, 64), [e(self.N * (s // 2) * (s // 2) * 64) for _ in range(4)])
        a0, bufs = self._f32
        a0 = a0[:N]
        ops.conv2d_nhwc(pix, w["conv_init/kernel"], a0, 2, 3, 3)
        ops.groupnorm_nhwc(a0, a0, w["norm_init/scale"], w["norm_init/bias"], None, 4, 1e-5, True)
        s //= 2
        x = bufs[0][:N * s * s * 64].view(N, s, s, 64)
        ops.maxpool3x3s2_nhwc(a0, x)
        free = [1, 2, 3]
        cur = 0
        cin = 64
        for i, (f, stride) in enumerate(STAGES):
            b = f"ResNetBlock_{i}"
            so = s // stride
            iy, iy2, ir = free
            y = bufs[iy][:N * so * so * f].view(N, so, so, f)
            lo, hi = (1, 1) if stride == 1 else (0, 1)           # XLA SAME on even sizes
            ops.conv2d_nhwc(x, w[f"{b}/Conv_0/kernel"], y, stride, lo, hi)
            ops.groupnorm_nhwc(y, y, w[f"{b}/MyGroupNorm_0/scale"], w[f"{b}/MyGroupNorm_0/bias"], None, 4, 1e-5, True)
            last = i == len(STAGES) - 1
            y2 = feats[:N] if last else bufs[iy2][:N * so * so * f].view(N, so, so, f)
            ops.conv2d_nhwc(y, w[f"{b}/Conv_1/kernel"], y2, 1, 1, 1)
            if stride != 1 or cin != f:
                r = bufs[ir][:N * so * so * f].view(N, so, so, f)
                ops.conv2d_nhwc(x, w[f"{b}/conv_proj/kernel"], r, stride, 0, 0)
                ops.groupnorm_nhwc(r, r, w[f"{b}/norm_proj/scale"], w[f"{b}/norm_proj/bias"], None, 4, 1e-5, False)
            else:
                r = x
            ops.groupnorm_nhwc(y2, y2, w[f"{b}/MyGroupNorm_1/scale"], w[f"{b}/MyGroupNorm_1/bias"], r, 4, 1e-5, True)
            if not last:
                free = [cur, iy, ir]
                cur = iy2
                x, s, cin = y2, so, f
        return feats
