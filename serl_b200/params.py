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
TRUNK_PATH = ENC + "/encoder_{}/pretrained_encoder"        # TRUNK_PATH.format(cam): the agents' frozen trunk in the parameter tree
INFO_GAP = 16
PROPRIO_LEAVES = (f"{ENC}/Dense_0/kernel", f"{ENC}/Dense_0/bias", f"{ENC}/LayerNorm_0/scale", f"{ENC}/LayerNorm_0/bias")
STAGES = ((64, 1), (128, 2), (256, 2), (512, 2))
# DrQ's "small" encoder (drq.py:137-152, small_encoders.py:9-55): (Ci, Co) of its four 3x3 / stride-2 VALID convs
SMALL_CONVS = ((3, 32), (32, 64), (64, 128), (128, 256))
ENCODER_TYPES = ("resnet-pretrained", "small", "resnet")


@dataclass
class Leaf:
    path: str
    shape: Tuple[int, ...]
    group: int
    offset: int = 0

    @property
    def size(self):
        return int(np.prod(self.shape)) if len(self.shape) else 1

    @property
    def end(self):
        """Offset behind the leaf, rounded up to 16 bytes: where the next leaf starts."""
        return self.offset + (self.size + 3) // 4 * 4


def assign_offsets(leaves: List["Leaf"], start: int = 0) -> int:
    """Lays the leaves out one after the other from `start` (floats), each 16-byte aligned; returns the offset behind the last."""
    for leaf in leaves:
        leaf.offset = start
        start = leaf.end
    return start


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
    activation per hidden width.  act: "tanh" | "relu" | "swish" | "leaky_relu" | "gelu".  dropout: the MLP's dropout_rate (BC,
    SAC and DrQ; 0: no Dropout layer)."""
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


def image_head_leaves(prefix: str, width: int = 256, group: int = 0) -> List[Leaf]:
    """One camera's head on the frozen trunk's features: SpatialLearnedEmbeddings, Dense(4096 -> width), LayerNorm."""
    return [Leaf(f"{prefix}/SpatialLearnedEmbeddings_0/kernel", (4, 4, 512, 8), group), Leaf(f"{prefix}/Dense_0/kernel", (4096, width), group),
            Leaf(f"{prefix}/Dense_0/bias", (width,), group), Leaf(f"{prefix}/LayerNorm_0/scale", (width,), group),
            Leaf(f"{prefix}/LayerNorm_0/bias", (width,), group)]


def camera_encoder_leaves(prefix: str, encoder: str, group: int = 0, in_channels: int = 3) -> List[Leaf]:
    """One camera's trainable encoder leaves under `prefix` (encoder_<cam>): "resnet-pretrained" the image head on the frozen
    trunk's features; "small" the conv stack Conv_0..3 (3,3,Ci,Co) + bias, then Dense_0 (256, 256) and LayerNorm_0 (no
    SpatialLearnedEmbeddings, no Dropout: pool_method="avg"); "resnet" the `trunk_spec` leaves directly under encoder_<cam> (no
    pretrained_encoder level), followed by the image head.  in_channels: the channels of the image the first conv (Conv_0,
    conv_init) reads, 3T for a stack of T RGB frames (EncodingWrapper's enable_stacking)."""
    if encoder == "small":
        out = []
        for i, (ci, co) in enumerate(SMALL_CONVS):
            ci = in_channels if i == 0 else ci
            out += [Leaf(f"{prefix}/Conv_{i}/kernel", (3, 3, ci, co), group), Leaf(f"{prefix}/Conv_{i}/bias", (co,), group)]
        return out + [Leaf(f"{prefix}/Dense_0/kernel", (256, 256), group), Leaf(f"{prefix}/Dense_0/bias", (256,), group),
                      Leaf(f"{prefix}/LayerNorm_0/scale", (256,), group), Leaf(f"{prefix}/LayerNorm_0/bias", (256,), group)]
    trunk = [Leaf(f"{prefix}/{k}", shp, group) for k, shp in trunk_spec(in_channels)] if encoder == "resnet" else []
    return trunk + image_head_leaves(prefix, group=group)


def proprio_leaves(state_in: int, group: int = 0) -> List[Leaf]:
    shapes = ((state_in, 64), (64,), (64,), (64,))
    return [Leaf(p, shp, group) for p, shp in zip(PROPRIO_LEAVES, shapes)]


def policy_leaves(F: int, action_dim: int, arch: MlpArch, std_parameterization: str, group: int) -> List[Leaf]:
    """The policy MLP on F features, the means head `modules_actor/Dense_0` and the std head: `modules_actor/Dense_1` ("exp",
    "softplus"), the free `modules_actor/log_stds` vector ("uniform") or none ("fixed": a constant std), actor_critic_nets.py:190-212."""
    H, A = arch.hidden[-1], action_dim
    L = _mlp_leaves("modules_actor/network", F, arch, group)
    L += [Leaf("modules_actor/Dense_0/kernel", (H, A), group), Leaf("modules_actor/Dense_0/bias", (A,), group)]
    if std_parameterization == "fixed":
        return L
    if std_parameterization == "uniform":
        return L + [Leaf("modules_actor/log_stds", (A,), group)]
    return L + [Leaf("modules_actor/Dense_1/kernel", (H, A), group), Leaf("modules_actor/Dense_1/bias", (A,), group)]


def trainable_spec(cams: Sequence[str], state_in: int, action_dim: int, ensemble: int, pixel: bool, critic: MlpArch = LAUNCHER_MLP,
                   policy: MlpArch = LAUNCHER_MLP, std_parameterization: str = "exp", use_proprio: bool = True,
                   encoder: str = "resnet-pretrained", in_channels: int = 3) -> List[Leaf]:
    """Trainable leaves in flat order (group-major).  A pixel agent with use_proprio=False has no proprio Dense / LayerNorm
    (encoding.py:26-72 builds them only with use_proprio): the encoder is the image heads alone.
    encoder "small": each camera's encoder is the trainable conv stack Conv_0..3 (3,3,Ci,Co) + bias, then Dense_0 (256, 256) and
    LayerNorm_0 (no SpatialLearnedEmbeddings, no Dropout: pool_method="avg"); all in the critic group like the other heads.
    encoder "resnet": each camera's encoder is a trainable ResNet-10, the `trunk_spec` leaves directly under encoder_<cam> (no
    pretrained_encoder level), followed by the SpatialLearnedEmbeddings / Dense / LayerNorm head; all in the critic group.
    in_channels: channels of the trainable encoders' input image (3T for a stack of T frames)."""
    L: List[Leaf] = []
    E, A = ensemble, action_dim
    if pixel:
        F = 256 * len(cams) + (64 if use_proprio else 0)
        for cam in cams:
            L += camera_encoder_leaves(f"{ENC}/encoder_{cam}", encoder, in_channels=in_channels)
        if use_proprio:
            L += proprio_leaves(state_in)
    else:
        F = state_in
    L += _mlp_leaves("modules_critic/network", F + A, critic, 0, (E,))
    H = critic.hidden[-1]                                     # the value head reads the last hidden layer
    if pixel:   # one shared value head (drq.py:201-207)
        L += [Leaf("modules_critic/Dense_0/kernel", (H, 1), 0), Leaf("modules_critic/Dense_0/bias", (1,), 0)]
    else:       # whole critic vmapped (sac.py:523-524)
        L += [Leaf("modules_critic/Dense_0/kernel", (E, H, 1), 0), Leaf("modules_critic/Dense_0/bias", (E, 1), 0)]
    n0 = len(L)
    L += policy_leaves(F, A, policy, std_parameterization, 1)
    L += [Leaf("modules_temperature/lagrange", (), 2)]
    assign_offsets(L[n0:], assign_offsets(L[:n0]) + INFO_GAP)    # info scalars live between group 0 and group 1 (gradient buffer)
    return L


def init_leaves(rng, spec: List[Leaf], xavier=lambda path: False, lagrange: float = 0.0, kaiming=lambda path: False) -> Dict[str, np.ndarray]:
    """Initial values drawn leaf by leaf in spec order (flax defaults): kernels lecun_normal, or xavier_uniform where xavier(path)
    says so (each member of a vmapped (E, K, H) kernel drawn independently), or kaiming_normal where kaiming(path) says so,
    scales 1, `lagrange` its given value, the rest 0."""
    out = {}
    for leaf in spec:
        p, shp = leaf.path, leaf.shape
        if p.endswith("lagrange"):
            v = np.array(lagrange, np.float32)
        elif p.endswith("kernel"):
            if kaiming(p):
                v = kaiming_normal(rng, shp)
            elif not xavier(p):
                v = lecun_normal(rng, shp)
            elif len(shp) == 3:
                v = np.stack([xavier_uniform(rng, shp[1:]) for _ in range(shp[0])])
            else:
                v = xavier_uniform(rng, shp)
        elif p.endswith("scale"):
            v = np.ones(shp, np.float32)
        else:
            v = np.zeros(shp, np.float32)
        out[p] = v.astype(np.float32)
    return out


def xavier_outside_encoders(path: str) -> bool:
    """SAC / DrQ / BC: Dense kernels of the MLPs and output heads are xavier_uniform; a camera encoder's SpatialLearnedEmbeddings,
    bottleneck nn.Dense and small-encoder nn.Conv keep flax's default lecun_normal."""
    return "/encoder_" not in path


def kaiming_in_resnet_encoder(path: str) -> bool:
    """The trainable ResNet-10's conv kernels (conv_init, ResNetBlock_*/Conv_* and conv_proj directly under encoder_<cam>) are
    kaiming_normal (resnet_v1.py:232: variance_scaling(2.0, "fan_in", "truncated_normal"))."""
    if "/encoder_" not in path or "/pretrained_encoder/" in path:
        return False
    return "/conv_init/" in path or "/ResNetBlock_" in path


def init_trainable(rng, spec: List[Leaf], temperature_init: float) -> Dict[str, np.ndarray]:
    return init_leaves(rng, spec, xavier_outside_encoders, math.log(math.exp(temperature_init) - 1.0), kaiming_in_resnet_encoder)


class FlatParams:
    """One flat fp32 device buffer per role (params, optional target, Adam moments m / v, gradient) over the leaves of a spec, with
    per-leaf addresses and views, and the {path: array} export / import of a buffer.  `tail` floats follow the leaves in every
    buffer; `info` more floats follow in the gradient buffer only (`grad_info` = gradient + infos: one all-reduce for both)."""

    def __init__(self, spec: List[Leaf], device, target: bool = True, tail: int = 0, info: int = 0):
        self.spec = spec
        self.leaf = {l.path: l for l in spec}
        self.n = spec[-1].end + tail
        z = lambda n: torch.zeros(n, dtype=torch.float32, device=device)
        self.params, self.m, self.v = z(self.n), z(self.n), z(self.n)
        self.target = z(self.n) if target else None
        self.grad_info = z(self.n + info)
        self.grad, self.info = self.grad_info[:self.n], self.grad_info[self.n:]
        self.counts = torch.zeros(3, dtype=torch.int32, device=device)
        self.lr_info = z(4)                                   # the learning rates the last single-tx Adam step applied

    def view(self, buf: torch.Tensor, path: str) -> torch.Tensor:
        l = self.leaf[path]
        return buf[l.offset:l.offset + l.size].view(l.shape)

    def addr(self, buf: torch.Tensor, path: str) -> int:
        return buf.data_ptr() + 4 * self.leaf[path].offset

    def P(self, path: str) -> int:
        return self.addr(self.params, path)

    def G(self, path: str) -> int:
        return self.addr(self.grad, path)

    def load(self, buf: torch.Tensor, values: Dict[str, np.ndarray]):
        """Writes the leaves `values` names; the others keep what the buffer holds."""
        host = buf.detach().cpu()
        for l in self.spec:
            if l.path in values:
                host[l.offset:l.offset + l.size] = torch.as_tensor(np.asarray(values[l.path], np.float32)).reshape(-1)
        buf.copy_(host)

    def dump(self, buf: torch.Tensor) -> Dict[str, np.ndarray]:
        host = buf.detach().cpu().numpy()
        return {l.path: host[l.offset:l.offset + l.size].reshape(l.shape).copy() for l in self.spec}


class ParamStore(FlatParams):
    """The three-tx store of the SAC / DrQ agents: optimizer groups, the info gap and the aux tail (module docstring)."""

    def __init__(self, spec: List[Leaf], device):
        # leaves with two live Adam txs (critic + actor): contiguous in the spec; their actor-tx state lives in the aux tail
        two = [l for l in spec if l.path in PROPRIO_LEAVES]
        self.aux_lo, self.aux_hi = (two[0].offset, two[-1].end) if two else (0, 0)
        assert all(a.end == b.offset for a, b in zip(two, two[1:])), "proprio leaves must be contiguous"
        super().__init__(spec, device, tail=self.aux_hi - self.aux_lo)
        self.n_main = spec[-1].end
        self.seg_end = [0, 0, 0]
        for l in spec:
            self.seg_end[l.group] = l.end
        self.info_off = self.seg_end[0]                       # [info_off, info_off + INFO_GAP): info scalars in the grad buffer
        self.seg_end[1] = max(self.seg_end[1], self.seg_end[0] + INFO_GAP)
        self.seg_end[2] = self.n_main
        self.aux_off = self.n_main - self.aux_lo             # aux index of flat index i in [aux_lo, aux_hi) = i + aux_off
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

    def load(self, buf: torch.Tensor, values: Dict[str, np.ndarray], aux_values: Dict[str, np.ndarray] = None):
        """Writes EVERY leaf (and, with aux_values, the actor-tx twins); the rest of the buffer is zeroed."""
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
