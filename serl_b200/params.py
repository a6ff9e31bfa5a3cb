"""Parameter layout of the DrQ / SAC agents: one flat fp32 buffer in HBM whose leaves are addressed by
their Flax tree paths (SURVEY.md Appendix D), grouped by the optimizer that owns them.

Mirrors what `ModuleDict.init` + `JaxRLTrainState.create` produce in the reference
(agents/continuous/drq.py:70-84, common/common.py:223-245) - the tree paths, shapes and initialiser
*distributions* (flax defaults: xavier_uniform Dense kernels in MLP/Policy/Critic heads
[common/common.py:15, networks/mlp.py:23], lecun_normal for the bottleneck Dense and the
SpatialLearnedEmbeddings kernel [vision/resnet_v1.py:86,371], kaiming_normal convs [:232], zeros bias,
ones/zeros norms, lagrange = softplus^-1(temperature_init) [networks/lagrange.py:27-35]).  The random
stream is NumPy's (flax's init key-path folding is version-coupled and not reproducible here), so
initial VALUES differ from a JAX run with the same seed; parity tests therefore feed both sides the
same parameters.

Optimizer groups (DESIGN.md "Adam groups"): 0 = critic tx (trainable encoder heads + critic),
1 = actor tx (policy MLP + heads), 2 = temperature tx (lagrange).  Leaves are 16-byte aligned.

Flat layout (floats):  [ group 0 | info gap (INFO_GAP) | group 1 | group 2 | aux ]
  * info gap: in the GRADIENT buffer it holds the loss kernels' info scalars ([0:4] critic, [4:12] actor /
    temperature), so that a data-parallel step exchanges gradients AND infos with ONE all-reduce of one
    contiguous range (critic step: [0, seg_end[0]+4); actor/temperature step: [seg_end[0]+4, n)).
  * aux: the proprio-encoder leaves (`modules_actor/encoder/{Dense_0,LayerNorm_0}`) are the only leaves that
    receive a non-zero gradient from TWO losses - the critic loss, and the actor loss, whose `stop_gradient`
    covers the image embeddings only (common/encoding.py:48-49 vs :55-70).  Both Adam transforms therefore
    keep live moments for them (common/common.py:136-168).  The aux tail of the grad / m / v buffers holds the
    ACTOR tx's gradient and moments of those leaves (same relative order); params / target have no aux part.
    A pixel-only agent (use_proprio=False) has no such leaves: the aux tail is empty and n == n_main.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

ENC = "modules_actor/encoder"
INFO_GAP = 16
PROPRIO_LEAVES = (f"{ENC}/Dense_0/kernel", f"{ENC}/Dense_0/bias", f"{ENC}/LayerNorm_0/scale", f"{ENC}/LayerNorm_0/bias")
STAGES = ((64, 1), (128, 2), (256, 2), (512, 2))
# DrQ's "small" encoder (drq.py:137-152, small_encoders.py:9-55): (Ci, Co) of its four 3x3 / stride-2 VALID convs
SMALL_CONVS = ((3, 32), (32, 64), (64, 128), (128, 256))
ENCODER_TYPES = ("resnet-pretrained", "small")


@dataclass
class Leaf:
    path: str
    shape: Tuple[int, ...]
    group: int
    offset: int = 0

    @property
    def size(self):
        return int(np.prod(self.shape)) if len(self.shape) else 1


def _trunc_normal(rng, shape, std):
    # flax variance_scaling(..., "truncated_normal"): N(0,1) truncated to [-2,2], rescaled by std/.8796
    out = rng.standard_normal(shape)
    bad = np.abs(out) > 2
    while bad.any():
        out[bad] = rng.standard_normal(int(bad.sum()))
        bad = np.abs(out) > 2
    return (out * (std / 0.87962566103423978)).astype(np.float32)


def _fans(shape):
    rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
    return shape[-2] * rf, shape[-1] * rf


def xavier_uniform(rng, shape):
    fi, fo = _fans(shape)
    lim = math.sqrt(6.0 / (fi + fo))
    return rng.uniform(-lim, lim, shape).astype(np.float32)


def lecun_normal(rng, shape):
    return _trunc_normal(rng, shape, math.sqrt(1.0 / _fans(shape)[0]))


def kaiming_normal(rng, shape):
    return _trunc_normal(rng, shape, math.sqrt(2.0 / _fans(shape)[0]))


def trunk_spec(in_channels: int = 3) -> List[Tuple[str, Tuple[int, ...]]]:
    """Leaves of `pretrained_encoder` (vision/resnet_v1.py:189-286, config resnetv1-10-frozen)."""
    spec = [("conv_init/kernel", (7, 7, in_channels, 64)), ("norm_init/scale", (64,)), ("norm_init/bias", (64,))]
    cin = 64
    for i, (f, s) in enumerate(STAGES):
        b = f"ResNetBlock_{i}"
        spec += [(f"{b}/Conv_0/kernel", (3, 3, cin, f)), (f"{b}/MyGroupNorm_0/scale", (f,)), (f"{b}/MyGroupNorm_0/bias", (f,)),
                 (f"{b}/Conv_1/kernel", (3, 3, f, f)), (f"{b}/MyGroupNorm_1/scale", (f,)), (f"{b}/MyGroupNorm_1/bias", (f,))]
        if s != 1 or cin != f:
            spec += [(f"{b}/conv_proj/kernel", (1, 1, cin, f)), (f"{b}/norm_proj/scale", (f,)), (f"{b}/norm_proj/bias", (f,))]
        cin = f
    return spec


def init_trunk(rng, in_channels: int = 3) -> Dict[str, np.ndarray]:
    out = {}
    for k, shp in trunk_spec(in_channels):
        if k.endswith("kernel"):
            out[k] = kaiming_normal(rng, shp)
        elif k.endswith("scale"):
            out[k] = np.ones(shp, np.float32)
        else:
            out[k] = np.zeros(shp, np.float32)
    return out


@dataclass(frozen=True)
class MlpArch:
    """One MLP of networks/mlp.py:10-32 as the agents build it (activate_final=True): Dense -> [Dropout] -> [LayerNorm] ->
    activation per hidden width.  act: "tanh" | "relu" | "swish" | "leaky_relu" | "gelu".  dropout: the MLP's dropout_rate (BC
    only; 0: no Dropout layer)."""
    hidden: Tuple[int, ...] = (256, 256)
    act: str = "tanh"
    layer_norm: bool = True
    dropout: float = 0.0


LAUNCHER_MLP = MlpArch()                                   # utils/launcher.py:61-66,95-104
STD_PARAMETERIZATIONS = ("exp", "softplus", "uniform")


def _mlp_leaves(prefix: str, fan_in: int, arch: MlpArch, group: int, lead: Tuple[int, ...] = ()) -> List[Leaf]:
    out, k = [], fan_in
    for i, h in enumerate(arch.hidden):
        out += [Leaf(f"{prefix}/Dense_{i}/kernel", lead + (k, h), group), Leaf(f"{prefix}/Dense_{i}/bias", lead + (h,), group)]
        if arch.layer_norm:
            out += [Leaf(f"{prefix}/LayerNorm_{i}/scale", lead + (h,), group), Leaf(f"{prefix}/LayerNorm_{i}/bias", lead + (h,), group)]
        k = h
    return out


def trainable_spec(cams: Sequence[str], state_in: int, action_dim: int, ensemble: int, pixel: bool, critic: MlpArch = LAUNCHER_MLP,
                   policy: MlpArch = LAUNCHER_MLP, std_parameterization: str = "exp", use_proprio: bool = True,
                   encoder: str = "resnet-pretrained") -> List[Leaf]:
    """Trainable leaves in flat order (group-major).  The policy's std head is `modules_actor/Dense_1` ("exp", "softplus") or the
    free `modules_actor/log_stds` vector ("uniform"), actor_critic_nets.py:190-207.  A pixel agent with use_proprio=False has
    no proprio Dense / LayerNorm (encoding.py:26-72 builds them only with use_proprio): the encoder is the image heads alone.
    encoder "small": each camera's encoder is the trainable conv stack Conv_0..3 (3,3,Ci,Co) + bias, then Dense_0 (256, 256) and
    LayerNorm_0 (no SpatialLearnedEmbeddings, no Dropout: pool_method="avg"); all in the critic group like the other heads."""
    L: List[Leaf] = []
    E, A = ensemble, action_dim
    if pixel:
        F = 256 * len(cams) + (64 if use_proprio else 0)
        for cam in cams:
            p = f"{ENC}/encoder_{cam}"
            if encoder == "small":
                for i, (ci, co) in enumerate(SMALL_CONVS):
                    L += [Leaf(f"{p}/Conv_{i}/kernel", (3, 3, ci, co), 0), Leaf(f"{p}/Conv_{i}/bias", (co,), 0)]
                L += [Leaf(f"{p}/Dense_0/kernel", (256, 256), 0)]
            else:
                L += [Leaf(f"{p}/SpatialLearnedEmbeddings_0/kernel", (4, 4, 512, 8), 0), Leaf(f"{p}/Dense_0/kernel", (4096, 256), 0)]
            L += [Leaf(f"{p}/Dense_0/bias", (256,), 0), Leaf(f"{p}/LayerNorm_0/scale", (256,), 0), Leaf(f"{p}/LayerNorm_0/bias", (256,), 0)]
        if use_proprio:
            L += [Leaf(f"{ENC}/Dense_0/kernel", (state_in, 64), 0), Leaf(f"{ENC}/Dense_0/bias", (64,), 0),
                  Leaf(f"{ENC}/LayerNorm_0/scale", (64,), 0), Leaf(f"{ENC}/LayerNorm_0/bias", (64,), 0)]
    else:
        F = state_in
    L += _mlp_leaves("modules_critic/network", F + A, critic, 0, (E,))
    H = critic.hidden[-1]                                     # the value head reads the last hidden layer
    if pixel:   # one shared value head (drq.py:201-207)
        L += [Leaf("modules_critic/Dense_0/kernel", (H, 1), 0), Leaf("modules_critic/Dense_0/bias", (1,), 0)]
    else:       # whole critic vmapped (sac.py:523-524)
        L += [Leaf("modules_critic/Dense_0/kernel", (E, H, 1), 0), Leaf("modules_critic/Dense_0/bias", (E, 1), 0)]
    L += _mlp_leaves("modules_actor/network", F, policy, 1)
    H = policy.hidden[-1]
    L += [Leaf("modules_actor/Dense_0/kernel", (H, A), 1), Leaf("modules_actor/Dense_0/bias", (A,), 1)]
    if std_parameterization == "uniform":
        L += [Leaf("modules_actor/log_stds", (A,), 1)]
    else:
        L += [Leaf("modules_actor/Dense_1/kernel", (H, A), 1), Leaf("modules_actor/Dense_1/bias", (A,), 1)]
    L += [Leaf("modules_temperature/lagrange", (), 2)]
    off, group = 0, 0
    for leaf in L:
        if leaf.group != group and group == 0:
            off += INFO_GAP                                   # info scalars live between group 0 and group 1 (gradient buffer)
        group = leaf.group
        leaf.offset = off
        off += (leaf.size + 3) // 4 * 4
    return L


def init_trainable(rng, spec: List[Leaf], temperature_init: float) -> Dict[str, np.ndarray]:
    out = {}
    for leaf in spec:
        p, shp = leaf.path, leaf.shape
        if p.endswith("lagrange"):
            v = np.array(math.log(math.exp(temperature_init) - 1.0), np.float32)
        elif p.endswith("SpatialLearnedEmbeddings_0/kernel"):
            v = lecun_normal(rng, shp)
        elif p.endswith("kernel"):
            if "/encoder_" in p:                                   # bottleneck nn.Dense / small-encoder nn.Conv default init
                v = lecun_normal(rng, shp)
            elif len(shp) == 3:                                    # vmapped: each member initialised independently
                v = np.stack([xavier_uniform(rng, shp[1:]) for _ in range(shp[0])])
            else:
                v = xavier_uniform(rng, shp)
        elif p.endswith("scale"):
            v = np.ones(shp, np.float32)
        else:
            v = np.zeros(shp, np.float32)
        out[p] = v.astype(np.float32)
    return out


class ParamStore:
    """Flat device buffers + per-leaf views (params, target, Adam moments, gradients)."""

    def __init__(self, spec: List[Leaf], device):
        self.spec = spec
        self.leaf = {l.path: l for l in spec}
        self.n_main = spec[-1].offset + (spec[-1].size + 3) // 4 * 4
        self.seg_end = [0, 0, 0]
        for l in spec:
            self.seg_end[l.group] = l.offset + (l.size + 3) // 4 * 4
        self.info_off = self.seg_end[0]                       # [info_off, info_off + INFO_GAP): info scalars in the grad buffer
        self.seg_end[1] = max(self.seg_end[1], self.seg_end[0] + INFO_GAP)
        self.seg_end[2] = self.n_main
        # leaves with two live Adam txs (critic + actor): contiguous in the spec; their actor-tx state lives in the aux tail
        two = [self.leaf[p] for p in PROPRIO_LEAVES if p in self.leaf]
        self.aux_lo = two[0].offset if two else 0
        self.aux_hi = (two[-1].offset + (two[-1].size + 3) // 4 * 4) if two else 0
        assert all(a.offset + (a.size + 3) // 4 * 4 == b.offset for a, b in zip(two, two[1:])), "proprio leaves must be contiguous"
        self.aux_off = self.n_main - self.aux_lo             # aux index of flat index i in [aux_lo, aux_hi) = i + aux_off
        self.n = self.n_main + (self.aux_hi - self.aux_lo)
        z = lambda: torch.zeros(self.n, dtype=torch.float32, device=device)
        self.params, self.target, self.m, self.v, self.grad = z(), z(), z(), z(), z()
        self.counts = torch.zeros(3, dtype=torch.int32, device=device)
        self.version = 0                                      # bumped by every out-of-band parameter write (TrainState.replace)

    def two_tx(self, path: str) -> bool:
        return self.aux_lo <= self.leaf[path].offset < self.aux_hi

    def aux_view(self, buf: torch.Tensor, path: str) -> torch.Tensor:
        """Actor-tx twin (gradient / moments) of a proprio-encoder leaf."""
        l = self.leaf[path]
        assert self.two_tx(path)
        return buf[l.offset + self.aux_off:l.offset + self.aux_off + l.size].view(l.shape)

    def aux_addr(self, buf: torch.Tensor, path: str) -> int:
        assert self.two_tx(path)
        return buf.data_ptr() + 4 * (self.leaf[path].offset + self.aux_off)

    def view(self, buf: torch.Tensor, path: str) -> torch.Tensor:
        l = self.leaf[path]
        return buf[l.offset:l.offset + l.size].view(l.shape)

    def addr(self, buf: torch.Tensor, path: str) -> int:
        return buf.data_ptr() + 4 * self.leaf[path].offset

    def load(self, buf: torch.Tensor, values: Dict[str, np.ndarray], aux_values: Dict[str, np.ndarray] = None):
        host = torch.zeros(self.n, dtype=torch.float32)
        for l in self.spec:
            host[l.offset:l.offset + l.size] = torch.as_tensor(np.asarray(values[l.path], np.float32)).reshape(-1)
            if aux_values is not None and self.two_tx(l.path):
                o = l.offset + self.aux_off
                host[o:o + l.size] = torch.as_tensor(np.asarray(aux_values[l.path], np.float32)).reshape(-1)
        buf.copy_(host)
        self.version += 1

    def dump_aux(self, buf: torch.Tensor) -> Dict[str, np.ndarray]:
        host = buf.detach().cpu().numpy()
        return {l.path: host[l.offset + self.aux_off:l.offset + self.aux_off + l.size].reshape(l.shape).copy()
                for l in self.spec if self.two_tx(l.path)}

    def dump(self, buf: torch.Tensor) -> Dict[str, np.ndarray]:
        host = buf.detach().cpu().numpy()
        return {l.path: host[l.offset:l.offset + l.size].reshape(l.shape).copy() for l in self.spec}


def nest(flat: Dict[str, object]) -> dict:
    """{"a/b/c": v} -> {"a": {"b": {"c": v}}} (the Flax tree the JAX actor consumes)."""
    out: dict = {}
    for k, v in flat.items():
        d = out
        parts = k.split("/")
        for p in parts[:-1]:
            d = d.setdefault(p, {})
        d[parts[-1]] = v
    return out


def flatten(tree: dict, prefix: str = "") -> Dict[str, object]:
    out = {}
    for k, v in tree.items():
        p = f"{prefix}/{k}" if prefix else k
        if isinstance(v, dict):
            out.update(flatten(v, p))
        else:
            out[p] = v
    return out
