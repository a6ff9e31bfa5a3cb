"""Device-side execution plan of one DrQ/SAC `update` call: which hand-written kernels run, in what
order, on which HBM buffers.  Pure orchestration - every arithmetic op is a C-ABI call (ops.py).

Data flow (pixel agent, one camera shown; B = batch, N = 2B images):

  sampler kernel ─ u8 crops (obs rows [0,B), next rows [B,2B)) ─ trunk (frozen ResNet-10, ONCE per step,
  shared by policy / critic / target critic; the reference recomputes it per network, SURVEY.md §3.1)
  ─ feats (N,4,4,512) ─ trainable heads (SLE, Dropout, Dense, LN, tanh; + proprio) ─ enc (B,F)
  ─ policy MLP / critic ensemble ─ losses ─ analytic backward ─ flat gradient ─ fused Adam+polyak.

Reference semantics: agents/continuous/sac.py:134-299, agents/continuous/drq.py:255-328,
common/common.py:124-221 (see oracle/drq.py for the restatement this is tested against).
"""
from __future__ import annotations

import os

from dataclasses import dataclass, replace
from typing import Dict, Optional, Sequence

import torch

from . import _lib as L
from . import ops
from .params import ENC, INFO_GAP, LAUNCHER_MLP, SMALL_CONVS, STAGES, MlpArch, ParamStore
from .trunk import FrozenTrunk

f32 = torch.float32
MAX_OBS_HORIZON = 8              # frames per stacked observation: the sampler's one-CTA-per-row kernel stages up to 8 frames' bands


@dataclass
class AgentConfig:
    cams: Sequence[str]
    state_in: int                # T * S (pixel agent) or S (state agent)
    action_dim: int
    pixel: bool = True
    ensemble: int = 10
    subsample: Optional[int] = 2
    discount: float = 0.96
    tau: float = 0.005
    target_entropy: float = -2.0
    backup_entropy: bool = False
    lr: Sequence[float] = (3e-4, 3e-4, 3e-4)            # critic, actor, temperature tx
    warmup: Sequence[int] = (0, 0, 0)
    decay: Sequence[Optional[int]] = (None, None, None)  # cosine_decay_steps per tx (None: linear warm-up, then constant)
    clip: Sequence[Optional[float]] = (None, None, None) # clip_grad_norm per tx (None: no clipping)
    std_min: float = 1e-5
    std_max: float = 5.0
    image_hw: int = 128
    precision: str = "fp32"      # trunk arithmetic: "fp32" (1e-5 parity build) | "bf16" / "fp16" (tensor-core builds)
    critic_arch: MlpArch = LAUNCHER_MLP
    policy_arch: MlpArch = LAUNCHER_MLP
    std_parameterization: str = "exp"   # "exp" | "softplus" | "uniform" (actor_critic_nets.py:190-207)
    use_proprio: bool = True     # pixel agent: proprio Dense(64) -> LayerNorm -> tanh after the image embeddings (encoding.py:55-70)
    encoder: str = "resnet-pretrained"   # pixel agent: "resnet-pretrained" (frozen trunk + SLE heads) | "small" (trainable convs)
    #                                      | "resnet" (trainable ResNet-10 + SLE heads)
    obs_horizon: int = 1         # pixel agent: frames T per observation, stacked on the channel axis (trainable encoders only)

    @property
    def in_channels(self) -> int:
        """Channels of the encoder's input image: T RGB frames stacked oldest first, "B T H W C -> B H W (T C)" (encoding.py:36-70)."""
        return 3 * self.obs_horizon

    @property
    def enc_dim(self):
        return 256 * len(self.cams) + (64 if self.use_proprio else 0) if self.pixel else self.state_in

    @property
    def proprio(self) -> bool:
        """The pixel agent's encoder has the proprio block."""
        return self.pixel and self.use_proprio

    @property
    def small(self) -> bool:
        """The pixel agent's image encoders are DrQ's trainable "small" conv stacks (no frozen trunk)."""
        return self.pixel and self.encoder == "small"

    @property
    def resnet(self) -> bool:
        """The pixel agent's image encoders are trainable ResNet-10s with the SLE heads (no frozen trunk)."""
        return self.pixel and self.encoder == "resnet"

    @property
    def trainable_encoder(self) -> bool:
        """The pixel encoder's convs are trained ("small", "resnet"): no frozen trunk, the convs run inside Engine.encode on the
        parameters of the moment, the cross-step pipeline prefetches crops only and the fused heads do not engage."""
        return self.small or self.resnet

    @property
    def mlp_dropout(self) -> bool:
        """The critic or the policy MLP has Dropout (dropout_rate > 0): the training passes draw (B, H_i) keep masks per layer."""
        return self.critic_arch.dropout > 0 or self.policy_arch.dropout > 0

    @property
    def launcher_arch(self) -> bool:
        """The architecture every SERL launcher builds: the one the fused tgemm heads implement."""
        return self.critic_arch == LAUNCHER_MLP and self.policy_arch == LAUNCHER_MLP and self.std_parameterization == "exp"

    @property
    def fused_heads_arch(self) -> bool:
        """The launcher's widths, activation, LayerNorm and std head at any dropout rate: the networks the fused tgemm heads
        implement (their LayerNorm epilogues take the MLP's Dropout masks)."""
        return (replace(self.critic_arch, dropout=0.0) == LAUNCHER_MLP and replace(self.policy_arch, dropout=0.0) == LAUNCHER_MLP
                and self.std_parameterization == "exp")


ACT_IDS = {"tanh": L.ACT_TANH, "relu": L.ACT_RELU, "swish": L.ACT_SWISH, "leaky_relu": L.ACT_LEAKY_RELU, "gelu": L.ACT_GELU}
STD_IDS = {"exp": L.STD_EXP, "softplus": L.STD_SOFTPLUS, "uniform": L.STD_UNIFORM, "fixed": L.STD_FIXED}


class _MlpActs:
    """Activations of an MLP over R rows (R = E*B for the ensemble): per layer the output h, and the LayerNorm statistics
    (xhat, rstd) or, without LayerNorm, the pre-activation z the backward reads.  With LayerNorm z is one scratch for all layers."""

    def __init__(self, R, dev, arch: MlpArch = LAUNCHER_MLP):
        e = lambda *s: torch.empty(*s, dtype=f32, device=dev)
        self.arch = arch
        self.h = [e(R, H) for H in arch.hidden]
        if arch.layer_norm:
            self.z = e(R, max(arch.hidden))
            self.zs = [self.z] * len(arch.hidden)
            self.xhat, self.rstd = [e(R, H) for H in arch.hidden], [e(R) for _ in arch.hidden]
        else:
            self.zs = [e(R, H) for H in arch.hidden]
            self.xhat = self.rstd = [None] * len(arch.hidden)

    # the launcher architecture's two layers under the names the fused heads (heads_fused.py) use
    h1 = property(lambda s: s.h[0])
    h2 = property(lambda s: s.h[1])
    xhat1 = property(lambda s: s.xhat[0])
    xhat2 = property(lambda s: s.xhat[1])
    rstd1 = property(lambda s: s.rstd[0])
    rstd2 = property(lambda s: s.rstd[1])


def mlp_act_fwd(P, arch: MlpArch, buf, prefix, i, z, out, xhat, rstd, rows_per_group, group_stride, R, D, mask=None, mask_rows=None):
    """Layer i's normalisation + activation of z (R, D) into out; P(buf, path) is a leaf's device address.  The launcher layer
    (LayerNorm + tanh) keeps its own entry.  mask: the layer's (R, D) Dropout keep mask (training with arch.dropout > 0), applied
    to z first (in place without LayerNorm); with mask_rows, a (mask_rows, D) mask that row r reads at r % mask_rows."""
    sc = P(buf, f"{prefix}/LayerNorm_{i}/scale") if arch.layer_norm else None
    bi = P(buf, f"{prefix}/LayerNorm_{i}/bias") if arch.layer_norm else None
    xh, rs = (xhat.data_ptr() if xhat is not None else None), (rstd.data_ptr() if rstd is not None else None)
    if mask is not None:
        ops.ln_act_dropout_fwd(z.data_ptr(), D, sc, bi, rows_per_group, group_stride, mask, 1.0 / (1.0 - arch.dropout), out.data_ptr(), D,
                               xh, rs, R, D, ACT_IDS[arch.act], arch.layer_norm, mask_rows=mask_rows)
    elif arch.layer_norm and arch.act == "tanh":
        ops.ln_tanh_fwd(z.data_ptr(), D, sc, bi, rows_per_group, group_stride, out.data_ptr(), D, xh, rs, R, D)
    else:
        ops.ln_act_fwd(z.data_ptr(), D, sc, bi, rows_per_group, group_stride, out.data_ptr(), D, xh, rs, R, D, ACT_IDS[arch.act],
                       arch.layer_norm)


def mlp_act_bwd(P, params, arch: MlpArch, prefix, i, acts: "_MlpActs", dt, dz, dy, rows_per_group, group_stride, R, D, dparams=None,
                mask=None, mask_rows=None):
    """dz of layer i from dt = d(layer output); dy kept for the LayerNorm parameter gradients.  dparams: (dscale, dbias)
    addresses to write them right away (current stream), or None (the caller launches ln_param_grad where it wants).  mask: the
    forward's Dropout keep mask, through which dz leaves."""
    sc = P(params, f"{prefix}/LayerNorm_{i}/scale") if arch.layer_norm else None
    xh = acts.xhat[i].data_ptr() if arch.layer_norm else None
    rs = acts.rstd[i].data_ptr() if arch.layer_norm else None
    dyp = dy.data_ptr() if dy is not None else None
    ds, db = dparams if dparams is not None else (None, None)
    bi = P(params, f"{prefix}/LayerNorm_{i}/bias") if arch.layer_norm else None
    if mask is not None:
        ops.ln_act_dropout_bwd(dt.data_ptr(), D, acts.h[i].data_ptr(), D, acts.zs[i].data_ptr(), D, xh, rs, sc, bi, rows_per_group,
                               group_stride, mask, 1.0 / (1.0 - arch.dropout), dz.data_ptr(), dyp, R, D, ACT_IDS[arch.act], arch.layer_norm,
                               mask_rows=mask_rows)
    elif arch.layer_norm and arch.act == "tanh":
        ops.ln_tanh_bwd(dt.data_ptr(), D, acts.h[i].data_ptr(), D, xh, rs, sc, rows_per_group, group_stride, dz.data_ptr(), dyp, ds, db, R, D)
        return
    else:
        ops.ln_act_bwd(dt.data_ptr(), D, acts.h[i].data_ptr(), D, acts.zs[i].data_ptr(), D, xh, rs, sc, bi, rows_per_group, group_stride,
                       dz.data_ptr(), dyp, R, D, ACT_IDS[arch.act], arch.layer_norm)
    if arch.layer_norm and dparams is not None:
        ops.ln_param_grad(dyp, xh, ds, db, rows_per_group, R, D)


POLICY = "modules_actor/network"


def policy_hidden_fwd(P, ws, arch: MlpArch, buf, X, F, acts: "_MlpActs", B, save: bool, masks=None):
    """The policy MLP's hidden layers on X (B, F) with the parameters in buf: Dense -> [Dropout: masks[i]] -> [LayerNorm] ->
    activation per layer (networks/mlp.py:22-31).  Returns (address, width) of the last layer's output."""
    x, ldx = X.data_ptr(), F
    for i, H in enumerate(arch.hidden):
        z = acts.zs[i]
        ops.dense_fwd(ws, x, ldx, P(buf, f"{POLICY}/Dense_{i}/kernel"), P(buf, f"{POLICY}/Dense_{i}/bias"), z.data_ptr(), H, B, ldx, H)
        mlp_act_fwd(P, arch, buf, POLICY, i, z, acts.h[i], acts.xhat[i] if save else None, acts.rstd[i] if save else None, B, 0, B, H,
                    mask=masks[i] if masks is not None else None)
        x, ldx = acts.h[i].data_ptr(), H
    return x, ldx


def policy_heads_fwd(P, ws, std_parameterization: str, buf, x, H, mu, ls, B, A):
    """means = h Dense_0 and, unless the std is the free log_stds vector ("uniform") or a constant ("fixed"), ls = h Dense_1."""
    ops.dense_fwd(ws, x, H, P(buf, "modules_actor/Dense_0/kernel"), P(buf, "modules_actor/Dense_0/bias"), mu.data_ptr(), A, B, H, A)
    if std_parameterization not in ("uniform", "fixed"):
        ops.dense_fwd(ws, x, H, P(buf, "modules_actor/Dense_1/kernel"), P(buf, "modules_actor/Dense_1/bias"), ls.data_ptr(), A, B, H, A)


def policy_heads_bwd(P, ws, std_parameterization: str, params, grad, h, H, dmu, dls, dh, B, A):
    """Gradients of the output heads from dmu / dls (B, A) and of their input h (address, width H): dh = dmu W0^T (+ dls W1^T).
    A "fixed" std has no head: dls is not read."""
    dmu, dls = dmu.data_ptr(), dls.data_ptr()
    ops.dense_bwd_weight(ws, h, H, dmu, A, P(grad, "modules_actor/Dense_0/kernel"), B, H, A)
    ops.colsum(dmu, P(grad, "modules_actor/Dense_0/bias"), 1, B, A, A)
    if std_parameterization in ("uniform", "fixed"):
        if std_parameterization == "uniform":              # log_stds is broadcast over the rows: its gradient is the column sum
            ops.colsum(dls, P(grad, "modules_actor/log_stds"), 1, B, A, A)
        ops.dense_bwd_input(ws, dmu, A, P(params, "modules_actor/Dense_0/kernel"), dh.data_ptr(), H, B, H, A)
    else:
        ops.dense_bwd_weight(ws, h, H, dls, A, P(grad, "modules_actor/Dense_1/kernel"), B, H, A)
        ops.colsum(dls, P(grad, "modules_actor/Dense_1/bias"), 1, B, A, A)
        ops.dense_bwd_input(ws, dmu, A, P(params, "modules_actor/Dense_0/kernel"), dh.data_ptr(), H, B, H, A)
        ops.dense_bwd_input(ws, dls, A, P(params, "modules_actor/Dense_1/kernel"), dh.data_ptr(), H, B, H, A, accumulate=True)


def policy_hidden_bwd(P, ws, arch: MlpArch, params, grad, X, F, acts: "_MlpActs", dh, dz, dy, B, masks=None):
    """Gradients of the hidden layers from dh = d(last layer's output); dh, dz, dy are scratch the layers share.  Returns dz, which
    holds the (B, hidden[0]) gradient of layer 0's Dense output."""
    for i in reversed(range(len(arch.hidden))):
        H = arch.hidden[i]
        dparams = (P(grad, f"{POLICY}/LayerNorm_{i}/scale"), P(grad, f"{POLICY}/LayerNorm_{i}/bias")) if arch.layer_norm else None
        mlp_act_bwd(P, params, arch, POLICY, i, acts, dh, dz, dy if arch.layer_norm else None, B, 0, B, H, dparams=dparams,
                    mask=masks[i] if masks is not None else None)
        x, K = (acts.h[i - 1].data_ptr(), arch.hidden[i - 1]) if i > 0 else (X.data_ptr(), F)
        ops.dense_bwd_weight(ws, x, K, dz.data_ptr(), H, P(grad, f"{POLICY}/Dense_{i}/kernel"), B, K, H)
        ops.colsum(dz.data_ptr(), P(grad, f"{POLICY}/Dense_{i}/bias"), 1, B, H, H)
        if i > 0:
            ops.dense_bwd_input(ws, dz.data_ptr(), H, P(params, f"{POLICY}/Dense_{i}/kernel"), dh.data_ptr(), K, B, K, H)
    return dz


def small_sizes(hw: int):
    """Spatial sizes of the small encoder's input and its four conv outputs (128 -> 63, 31, 15, 7)."""
    out = [hw]
    for _ in SMALL_CONVS:
        out.append((out[-1] - 3) // 2 + 1)
    return out


class _SmallActs:
    """Outputs of one small-encoder pass over up to n images: the four post-ReLU conv maps (NHWC) and the pooled (n, 256)."""

    def __init__(self, n, hw, device):
        e = lambda *s: torch.empty(*s, dtype=f32, device=device)
        S = small_sizes(hw)
        self.y = [e(n, S[i + 1], S[i + 1], co) for i, (_, co) in enumerate(SMALL_CONVS)]
        self.pooled = e(n, SMALL_CONVS[-1][1])


def resnet_convs(hw: int, in_channels: int = 3):
    """The trainable ResNet-10's convs on an hw x hw image of in_channels channels, in forward order: (leaf, k, stride, pad_lo,
    pad_hi, H_in, Ci, Co).  XLA SAME paddings: 7x7/2 (3, 3), 3x3/1 (1, 1), 3x3/2 (0, 1) and 1x1/2 (0, 0) on even sizes."""
    out = [("conv_init", 7, 2, 3, 3, hw, in_channels, 64)]
    s, cin = hw // 4, 64
    for i, (f, stride) in enumerate(STAGES):
        b = f"ResNetBlock_{i}"
        out.append((f"{b}/Conv_0", 3, stride, 1 if stride == 1 else 0, 1, s, cin, f))
        out.append((f"{b}/Conv_1", 3, 1, 1, 1, s // stride, f, f))
        if stride != 1 or cin != f:
            out.append((f"{b}/conv_proj", 1, stride, 0, 0, s, cin, f))
        s, cin = s // stride, f
    return out


class _ResActs:
    """Activations of one trainable-ResNet-10 pass over up to n images, every one the backward reads: the stem's normalised
    4-channel input (x4; ops.stem_channels(in_channels) channels for a frame stack), pre-norm conv outputs (z*), post-norm outputs
    (stem a, block h0 / rp / out) and the max-pool output."""

    def __init__(self, n, hw, device, in_channels: int = 3):
        e = lambda *s: torch.empty(*s, dtype=f32, device=device)
        s = hw // 2
        self.x4, self.z_stem, self.a_stem, self.pool = e(n, hw, hw, ops.stem_channels(in_channels)), e(n, s, s, 64), e(n, s, s, 64), e(n, s // 2, s // 2, 64)
        self.blocks = []
        s, cin = s // 2, 64
        for f, stride in STAGES:
            so = s // stride
            d = {k: e(n, so, so, f) for k in ("z0", "h0", "z1", "out")}
            if stride != 1 or cin != f:
                d["zp"], d["rp"] = e(n, so, so, f), e(n, so, so, f)
            self.blocks.append(d)
            s, cin = so, f

    @property
    def feats(self):
        return self.blocks[-1]["out"]


def small_encoder_forward(store, precision: str, buf, cam: str, pix: torch.Tensor, acts: _SmallActs):
    """pix (n, hw, hw, 3T) uint8 -> the small encoder's conv maps and pooled (n, 256) in acts, with camera cam's conv leaves of buf
    (a buffer of store: params or target).  small_encoders.py:28-44: x = pix / 255, 4 x [conv 3x3/2 VALID + bias, ReLU], mean over
    positions; Conv_0 reads the 3T channels of a stack of T frames.  The fp32 build runs the convs on the CUDA cores, the 16-bit
    builds on the tensor cores (3xTF32)."""
    n, S, p = pix.shape[0], small_sizes(pix.shape[1]), f"{ENC}/encoder_{cam}"
    x, u8 = pix.data_ptr(), True
    for i, (ci, co) in enumerate(SMALL_CONVS):
        ci = pix.shape[-1] if i == 0 else ci
        ops.sconv_fwd(x, store.addr(buf, f"{p}/Conv_{i}/kernel"), store.addr(buf, f"{p}/Conv_{i}/bias"), acts.y[i].data_ptr(), n, S[i], S[i],
                      ci, co, u8, tc=precision != "fp32")
        x, u8 = acts.y[i].data_ptr(), False
    ops.sconv_mean_fwd(x, acts.pooled.data_ptr(), n, S[-1] * S[-1], SMALL_CONVS[-1][1])


def resnet_encoder_forward(store, precision: str, buf, cam: str, pix: torch.Tensor, acts: _ResActs):
    """pix (n, hw, hw, 3T) uint8 -> every activation of camera cam's trainable ResNet-10 in acts, with the leaves of buf (a buffer of
    store: params or target): resnet_v1.py:217-286 with pre_pooling=False.  The fp32 build runs the frozen trunk's CUDA-core forward
    kernels; the 16-bit builds run the convs on the tensor cores (3xTF32) from the stem's normalised copy, zero-padded to a multiple
    of 4 channels."""
    n, hw, p, ci0 = pix.shape[0], pix.shape[1], f"{ENC}/encoder_{cam}", pix.shape[-1]
    tc = precision != "fp32"
    V = lambda leaf: store.view(buf, f"{p}/{leaf}")
    P = lambda leaf: store.addr(buf, f"{p}/{leaf}")
    convs = {c[0]: c for c in resnet_convs(hw, ci0)}

    def conv(x, leaf, y, Ci_x):
        _, k, st, lo, hi, H, ci, co = convs[leaf]
        if tc:
            ops.rconv_fwd(x.data_ptr(), P(f"{leaf}/kernel"), y.data_ptr(), n, H, H, Ci_x, ci, co, k, st, lo, hi, True)
        else:
            ops.conv2d_nhwc(x, V(f"{leaf}/kernel"), y, st, lo, hi)

    x4, z, a, pool = acts.x4[:n], acts.z_stem[:n], acts.a_stem[:n], acts.pool[:n]
    ops.rconv_stem_prep(pix.data_ptr(), x4.data_ptr(), n, hw, hw, ci0)  # the stem's wgrad input (and its tensor-core fwd input)
    conv(x4 if tc else pix, "conv_init", z, x4.shape[-1] if tc else ci0)
    ops.groupnorm_nhwc(z, a, V("norm_init/scale"), V("norm_init/bias"), None, 4, 1e-5, True)
    ops.maxpool3x3s2_nhwc(a, pool)
    x = pool
    for i, d in enumerate(acts.blocks):
        b = f"ResNetBlock_{i}"
        z0, h0, z1, out = d["z0"][:n], d["h0"][:n], d["z1"][:n], d["out"][:n]
        conv(x, f"{b}/Conv_0", z0, x.shape[-1])
        ops.groupnorm_nhwc(z0, h0, V(f"{b}/MyGroupNorm_0/scale"), V(f"{b}/MyGroupNorm_0/bias"), None, 4, 1e-5, True)
        conv(h0, f"{b}/Conv_1", z1, h0.shape[-1])
        r = x
        if "zp" in d:
            zp, r = d["zp"][:n], d["rp"][:n]
            conv(x, f"{b}/conv_proj", zp, x.shape[-1])
            ops.groupnorm_nhwc(zp, r, V(f"{b}/norm_proj/scale"), V(f"{b}/norm_proj/bias"), None, 4, 1e-5, False)
        ops.groupnorm_nhwc(z1, out, V(f"{b}/MyGroupNorm_1/scale"), V(f"{b}/MyGroupNorm_1/bias"), r, 4, 1e-5, True)
        x = out


class _EncScratch:
    """Scratch of one encoder-heads pass; each concurrently running branch of the step owns one."""

    def __init__(self, cfg, B, device, ws):
        e = lambda *s: torch.empty(*s, dtype=f32, device=device)
        self.ws = ws
        if cfg.pixel:
            if cfg.small:
                self.small = _SmallActs(B, cfg.image_hw, device)
            else:
                self.sle = {c: e(B, 4096) for c in cfg.cams}
            if cfg.resnet:
                self.res = _ResActs(B, cfg.image_hw, device, cfg.in_channels)
            self.enc_z, self.enc_zp = e(B, 256), e(B, 64)


class Engine:
    def __init__(self, cfg: AgentConfig, store: ParamStore, trunk: FrozenTrunk, batch: int, device):
        self.cfg, self.store, self.B, self.dev = cfg, store, batch, device
        B, E, A, F = batch, cfg.ensemble, cfg.action_dim, cfg.enc_dim
        self.F, self.FA = F, F + A
        e = lambda *s: torch.empty(*s, dtype=f32, device=device)
        # heads GEMMs: CUDA-core SGEMM in the 1e-5 build, tensor-core 3xTF32 (fp32-class accuracy) next to the 16-bit trunk
        gemm_impl = os.environ.get("SERL_HEADS_GEMM") or ("f32" if cfg.precision == "fp32" else "tf32x3")
        ws_bytes = max(48 << 20, 2 * 4 * E * B * self.FA)
        self.ws = ops.Workspace(ws_bytes, device, gemm_impl)
        # Branch-level concurrency: the heads are ~100 short, latency-bound launches, and several chains of them are
        # independent (online critic / target encoder / policy in the forward pass; weight gradients vs the dX chain in
        # the backward pass).  They run on two side streams; under CUDA-graph capture the fork / join events become graph
        # edges.  Every branch owns its scratch (split-K workspace included).
        dev = torch.device(device)
        self.side = [L.new_side_stream(dev) for _ in range(2)]
        # frozen trunk: every camera's pass on its own stream (camera 0 stays on the main stream).  At batch 256 the persistent
        # conv kernels fill the GPU and the passes serialise; at the small per-rank batches of data-parallel runs (32 rows per
        # rank on 8 GPUs) a trunk kernel covers a fraction of the SMs and the cameras overlap.
        self.cam_stream = {c: (L.new_side_stream(dev) if j > 0 else None) for j, c in enumerate(cfg.cams)}
        self.ws_side = [ops.Workspace(ws_bytes, device, gemm_impl) for _ in range(2)]
        # batch tensors
        self.state_o, self.state_n = e(B, cfg.state_in), e(B, cfg.state_in)
        self.actions, self.rewards, self.masks = e(B, A), e(B), e(B)
        self.dones = torch.empty(B, dtype=torch.uint8, device=device)
        self.idx = torch.empty(B, dtype=torch.int32, device=device)
        self.status = torch.zeros(1, dtype=torch.int32, device=device)
        # prioritized replay: each row's drawn priority, importance weight (1 on rows of uniform rings) and TD error, and the
        # (ring, first row, rows) of the batch's prioritized parts, whose slots get their rows' TD errors back after the loss
        self.prio, self.weights, self.delta = e(B), e(B), e(B)
        self.prio_parts: list = []
        self.state_sinks: Dict[int, tuple] = {}     # pixel-only agent: per ring state width, the (obs, next) rows nobody reads
        if cfg.pixel:
            hw, N, T = cfg.image_hw, 2 * B, cfg.obs_horizon
            self.N = N
            self.pix = {c: torch.empty(N, hw, hw, cfg.in_channels, dtype=torch.uint8, device=device) for c in cfg.cams}
            self.off = torch.empty(2, B * T, 2, dtype=torch.int32, device=device)   # applied crop offsets (obs, next), one per frame
            if cfg.small:
                # the critic-loss backward's inputs per camera (obs rows), and one set of conv-map gradients (the backward runs
                # the cameras one after the other on the main stream)
                self.small_saved = {c: _SmallActs(B, hw, device) for c in cfg.cams}
                self.small_dz = _SmallActs(B, hw, device).y
                S = small_sizes(hw)
                self.small_ws = e(max(ops.sconv_wgrad_workspace(B, S[i], S[i], cfg.in_channels if i == 0 else ci, co)
                                      for i, (ci, co) in enumerate(SMALL_CONVS)))
                self.d_pool = e(B, 256)
            elif cfg.resnet:
                # the critic-loss backward's inputs per camera (obs rows) and one set of gradient scratch (cameras run one after the
                # other on the main stream): two stem-sized maps, seven of the largest block's size, the split-K / GroupNorm partials
                self.res_saved = {c: _ResActs(B, hw, device, cfg.in_channels) for c in cfg.cams}
                s = hw // 2
                self.res_g_stem = [e(B * s * s * 64) for _ in range(2)]
                self.res_g = [e(B * (s // 2) * (s // 2) * 64) for _ in range(7)]
                self.res_ws = e(max(ops.rconv_wgrad_workspace(B, H, H, ops.stem_channels(ci), co, k, st, lo, hi)
                                    for _, k, st, lo, hi, H, ci, co in resnet_convs(hw, cfg.in_channels)))
                self.res_gn_ws = e(ops.groupnorm_bwd_workspace(B, 512, 4))
                self.d_feats = e(B, 4, 4, 512)
                self.sle_saved = {c: e(B, 4096) for c in cfg.cams}
            else:
                self.feats = {c: e(N, 4, 4, 512) for c in cfg.cams}
                self.trunk = trunk.runner(N, device)
                self.sle_saved = {c: e(B, 4096) for c in cfg.cams}
            self.enc_xhat = {c: e(B, 256) for c in cfg.cams}
            self.enc_rstd = {c: e(B) for c in cfg.cams}
            self.enc_xhat_p, self.enc_rstd_p = e(B, 64), e(B)
            self.masks_u8 = {c: torch.empty(B, 4096, dtype=torch.uint8, device=device) for c in cfg.cams}
            self.d_enc_z = {c: e(B, 256) for c in cfg.cams}          # per camera: the side stream reads it while the next one is written
            self.d_enc_y, self.d_sle = {c: e(B, 256) for c in cfg.cams}, e(B, 4096)
            self.d_enc_zp, self.d_enc_yp = e(B, 64), e(B, 64)
            # actor pass: the proprio Dense/LayerNorm stays differentiable under the policy's stop_gradient (encoding.py:48-70)
            self.enc_xhat_pa, self.enc_rstd_pa = e(B, 64), e(B)
            self.dXp_p, self.d_enc_zpa, self.d_enc_ypa = e(B, 64), e(B, 64), e(B, 64)
        self.sc_main = _EncScratch(cfg, B, device, self.ws)
        self.sc_side = [_EncScratch(cfg, B, device, w) for w in self.ws_side]
        # critic / policy activations
        self.Xc, self.Xt, self.Xp = e(B, self.FA), e(B, self.FA), e(B, F)
        ca, pa = cfg.critic_arch, cfg.policy_arch
        self.c_main, self.c_tgt = _MlpActs(E * B, device, ca), _MlpActs(E * B, device, ca)
        self.q, self.q_next, self.dq, self.target_q = e(E, B), e(E, B), e(E, B), e(B)
        self.p_acts = _MlpActs(B, device, pa)
        # MLP Dropout keep masks, (B, H_i) per hidden layer (the ensemble's members share them): the online critic of the critic
        # loss (then of the actor loss), the target critic, and the policy pass of the moment (its backward reads the actor pass's)
        self.c_mask, self.c_mask_tgt, self.p_mask = self.mlp_masks(ca), self.mlp_masks(ca), self.mlp_masks(pa)
        self.mu, self.ls, self.u, self.std, self.eps = e(B, A), e(B, A), e(B, A), e(B, A), e(B, A)
        self.logp = e(B)
        self.act_scratch = e(B, A)
        self.sub = torch.zeros(max(cfg.subsample or 1, 1), dtype=torch.int32, device=device)
        # gradient scratch.  Critic: one dz / dy per layer - the side stream still reads a layer's while the next one is written
        # (the launcher architecture's layer 1 / layer 0 pairs are dz, dy / dz0, dy0)
        Hc, Hp = max(ca.hidden), max(pa.hidden)
        self.dh = e(E * B, Hc)
        self.c_dz, self.c_dy = [e(E * B, H) for H in ca.hidden], [e(E * B, H) if ca.layer_norm else None for H in ca.hidden]
        self.dz, self.dy, self.dz0, self.dy0 = self.c_dz[-1], self.c_dy[-1], self.c_dz[0], self.c_dy[0]
        self.dX = e(B, self.FA)
        self.dmu, self.dls = e(B, A), e(B, A)
        self.pdh, self.pdz, self.pdy = e(B, Hp), e(B, Hp), e(B, Hp)
        # info scalars live INSIDE the flat gradient buffer (params.py: info gap), next to the segments they travel with in
        # the data-parallel all-reduce: [0:3] critic | [4:7] actor, [8] temperature.  Learning rates are separate.
        self.info = store.grad[store.info_off:store.info_off + INFO_GAP]
        self.info.zero_()
        self.info_hist = torch.zeros(INFO_GAP, dtype=f32, device=device)
        self.lr_info = torch.zeros(4, dtype=f32, device=device)
        # per-tx global gradient norms (clip_grad_norm) and their float64 per-CTA partials
        self.grad_norms = torch.zeros(3, dtype=f32, device=device)
        self.norm_partials = torch.zeros(3 * L.GRAD_NORM_CTAS, dtype=torch.float64, device=device)
        # 16-bit builds, pixel agent: the critic step runs on the fused head kernels (heads_fused.py: TF32 GEMMs with TMA-fed
        # operands and LayerNorm / head epilogues, batched problems); SERL_FUSED_HEADS=0 keeps the per-op chain below.  The fused
        # epilogues implement the launcher architecture (with or without MLP Dropout) only: every other architecture runs the per-op chain.
        from . import heads_fused
        self.fused = heads_fused.FusedCritic(self) if (cfg.fused_heads_arch and not cfg.trainable_encoder and heads_fused.enabled(cfg)
                                                       and (dev.type == "cuda" or os.environ.get("SERL_FUSED_HEADS") == "force")) else None

    # ------------------------------------------------------------------------------------------
    def P(self, buf, path):
        return self.store.addr(buf, path)

    def mlp_masks(self, arch: MlpArch):
        """(B, H_i) uint8 keep masks for an MLP with Dropout; None without."""
        if not arch.dropout:
            return None
        return [torch.empty(self.B, H, dtype=torch.uint8, device=self.dev) for H in arch.hidden]

    def fill_mlp_masks(self, masks, arch: MlpArch, key_addr, given=None):
        """Hidden layer i's keep mask bernoulli(fold_in(key, ncams + i), 1 - rate, (B, H_i)) (DESIGN.md §4; ncams = 0 for the state
        agent), or the given (B, H_i) masks (tests' explicit randomness)."""
        ncams = len(self.cfg.cams) if self.cfg.pixel else 0
        for i, m in enumerate(masks):
            if given is None:
                ops.dropout_mask_fill(key_addr, ncams + i, 1.0 - arch.dropout, m, m.numel())
            else:
                m.copy_(torch.as_tensor(given[i]).to(self.dev, torch.uint8))

    def state_sink(self, n: int):
        """Scratch (B, n) x 2 for the state rows the sampler gathers from a ring that stores n state values per sample when the
        agent has no proprio input (use_proprio=False).  Allocated on the first eager step with such a ring, before any capture."""
        if n not in self.state_sinks:
            self.state_sinks[n] = tuple(torch.empty(self.B, n, dtype=f32, device=self.dev) for _ in range(2))
        return self.state_sinks[n]

    # ---- frozen trunk (vision/resnet_v1.py:217-286) -------------------------------------------
    def trunk_forward(self, cam: str, pix: torch.Tensor, feats: torch.Tensor):
        """pix (n, hw, hw, 3) uint8 -> feats[:n] on this engine's trunk runner."""
        return self.trunk.forward(cam, pix, feats)

    # ---- trainable encoder heads (common/encoding.py:26-72, vision/resnet_v1.py:340-374) -------
    def encode(self, buf, feats_rows: slice, state: torch.Tensor, out: torch.Tensor, ld_out: int,
               masks: Optional[Dict[str, torch.Tensor]], save: bool, sc: Optional[_EncScratch] = None, save_proprio_actor: bool = False):
        """save: keep what the critic-loss backward needs (every head).  save_proprio_actor: keep the proprio LayerNorm
        statistics for the ACTOR-loss backward (the only encoder branch the policy's stop_gradient leaves differentiable)."""
        sc = sc or self.sc_main
        cfg, B, ws = self.cfg, self.B, sc.ws
        if not cfg.pixel:
            ops.copy2d(state.data_ptr(), cfg.state_in, out.data_ptr(), ld_out, B, cfg.state_in)
            return
        for j, cam in enumerate(cfg.cams):
            p = f"{ENC}/encoder_{cam}"
            if cfg.small:            # no Dropout in the small encoder (pool_method="avg"): masks do not apply
                acts = self.small_saved[cam] if save else sc.small
                self.small_forward(buf, cam, self.pix[cam][feats_rows], acts)
                x, K = acts.pooled.data_ptr(), 256
            else:
                if cfg.resnet:
                    acts = self.res_saved[cam] if save else sc.res
                    pix = self.pix[cam][feats_rows]
                    self.resnet_forward(buf, cam, pix, acts)
                    feats = acts.feats[:pix.shape[0]]
                else:
                    feats = self.feats[cam][feats_rows]
                sle = self.sle_saved[cam] if save else sc.sle[cam]
                ops.sle_fwd(feats, self.store.view(buf, f"{p}/SpatialLearnedEmbeddings_0/kernel"),
                            None if masks is None else masks[cam], 0.9, sle.data_ptr(), 4096)
                x, K = sle.data_ptr(), 4096
            ops.dense_fwd(ws, x, K, self.P(buf, f"{p}/Dense_0/kernel"), self.P(buf, f"{p}/Dense_0/bias"),
                          sc.enc_z.data_ptr(), 256, B, K, 256)
            ops.ln_tanh_fwd(sc.enc_z.data_ptr(), 256, self.P(buf, f"{p}/LayerNorm_0/scale"), self.P(buf, f"{p}/LayerNorm_0/bias"),
                            B, 0, ops.at(out, 256 * j), ld_out, self.enc_xhat[cam].data_ptr() if save else None,
                            self.enc_rstd[cam].data_ptr() if save else None, B, 256)
        if not cfg.use_proprio:           # pixel-only encoder: the image embeddings are all of enc
            return
        ops.dense_fwd(ws, state.data_ptr(), cfg.state_in, self.P(buf, f"{ENC}/Dense_0/kernel"), self.P(buf, f"{ENC}/Dense_0/bias"),
                      sc.enc_zp.data_ptr(), 64, B, cfg.state_in, 64)
        xh, rs = (self.enc_xhat_p, self.enc_rstd_p) if save else ((self.enc_xhat_pa, self.enc_rstd_pa) if save_proprio_actor else (None, None))
        ops.ln_tanh_fwd(sc.enc_zp.data_ptr(), 64, self.P(buf, f"{ENC}/LayerNorm_0/scale"), self.P(buf, f"{ENC}/LayerNorm_0/bias"),
                        B, 0, ops.at(out, 256 * len(cfg.cams)), ld_out, None if xh is None else xh.data_ptr(),
                        None if rs is None else rs.data_ptr(), B, 64)

    def small_forward(self, buf, cam: str, pix: torch.Tensor, acts: _SmallActs):
        small_encoder_forward(self.store, self.cfg.precision, buf, cam, pix, acts)

    def resnet_forward(self, buf, cam: str, pix: torch.Tensor, acts: _ResActs):
        resnet_encoder_forward(self.store, self.cfg.precision, buf, cam, pix, acts)

    def resnet_backward(self, cam: str, d_feats: torch.Tensor):
        """Gradients of camera cam's trunk leaves (into store.grad) from d(block 3 output) (B, 4, 4, 512), through the saved obs-row
        activations: per block GN_1 (ReLU mask, residual split) -> [norm_proj -> conv_proj] -> conv_1 -> GN_0 -> conv_0, the
        block input's gradient summed over the residual / projection and conv_0 paths; then the max-pool, the stem GroupNorm and
        the stem conv's weight gradient (the image needs no input gradient)."""
        B, hw, p = self.B, self.cfg.image_hw, f"{ENC}/encoder_{cam}"
        G, Pm, acts, tc = self.store.grad, self.store.params, self.res_saved[cam], self.cfg.precision != "fp32"
        convs = {c[0]: c for c in resnet_convs(hw, self.cfg.in_channels)}
        GA = lambda leaf: self.P(G, f"{p}/{leaf}")
        PA = lambda leaf: self.P(Pm, f"{p}/{leaf}")

        def gbuf(i, like):
            return self.res_g[i][:like.numel()].view(like.shape)

        def gn_bwd(x, y, dy, norm, dx, dres, relu):
            N, H, W, C = x.shape
            ops.groupnorm_bwd_nhwc(x.data_ptr(), y.data_ptr(), dy.data_ptr(), PA(f"{norm}/scale"), dx.data_ptr(),
                                   None if dres is None else dres.data_ptr(), GA(f"{norm}/scale"), GA(f"{norm}/bias"), self.res_gn_ws,
                                   N, H * W, C, 4, 1e-5, relu)

        def wgrad(x, leaf, dz, Ci_x):
            _, k, st, lo, hi, H, ci, co = convs[leaf]
            ops.rconv_wgrad(x.data_ptr(), dz.data_ptr(), GA(f"{leaf}/kernel"), self.res_ws, B, H, H, Ci_x, ci, co, k, st, lo, hi, tc)

        def dgrad(dz, leaf, dx, accumulate):
            _, k, st, lo, hi, H, ci, co = convs[leaf]
            ops.rconv_dgrad(dz.data_ptr(), PA(f"{leaf}/kernel"), dx.data_ptr(), B, H, H, ci, co, k, st, lo, hi, accumulate, tc)

        dy = d_feats
        cur = 0                                               # res_g index holding dy (the last block's dy is d_feats)
        for i in reversed(range(len(acts.blocks))):
            b, d = f"ResNetBlock_{i}", acts.blocks[i]
            x = acts.pool if i == 0 else acts.blocks[i - 1]["out"]
            free = [j for j in range(7) if j != cur or i == len(acts.blocks) - 1]
            dz1, dh0, dz0, dx = gbuf(free[0], d["z1"]), gbuf(free[1], d["z1"]), gbuf(free[2], d["z1"]), gbuf(free[3], x)
            if "zp" in d:
                dr, dzp = gbuf(free[4], d["rp"]), gbuf(free[5], d["zp"])
                gn_bwd(d["z1"], d["out"], dy, f"{b}/MyGroupNorm_1", dz1, dr, True)
                gn_bwd(d["zp"], d["rp"], dr, f"{b}/norm_proj", dzp, None, False)
                wgrad(x, f"{b}/conv_proj", dzp, x.shape[-1])
                dgrad(dzp, f"{b}/conv_proj", dx, False)
            else:
                gn_bwd(d["z1"], d["out"], dy, f"{b}/MyGroupNorm_1", dz1, dx, True)
            wgrad(d["h0"], f"{b}/Conv_1", dz1, d["h0"].shape[-1])
            dgrad(dz1, f"{b}/Conv_1", dh0, False)
            gn_bwd(d["z0"], d["h0"], dh0, f"{b}/MyGroupNorm_0", dz0, None, True)
            wgrad(x, f"{b}/Conv_0", dz0, x.shape[-1])
            dgrad(dz0, f"{b}/Conv_0", dx, True)
            dy, cur = dx, free[3]
        da = self.res_g_stem[0][:acts.a_stem.numel()].view(acts.a_stem.shape)
        dz = self.res_g_stem[1][:acts.z_stem.numel()].view(acts.z_stem.shape)
        N, H, W, C = acts.a_stem.shape
        ops.maxpool3x3s2_bwd_nhwc(acts.a_stem.data_ptr(), dy.data_ptr(), da.data_ptr(), N, H, W, C)
        gn_bwd(acts.z_stem, acts.a_stem, da, "norm_init", dz, None, True)
        wgrad(acts.x4, "conv_init", dz, acts.x4.shape[-1])

    def small_backward(self, cam: str, pix: torch.Tensor, d_pool: torch.Tensor):
        """Gradients of camera cam's conv leaves (into store.grad) from d(pooled) (B, 256), through the saved obs-row maps."""
        B, S, p, G, Pm = self.B, small_sizes(self.cfg.image_hw), f"{ENC}/encoder_{cam}", self.store.grad, self.store.params
        tc = self.cfg.precision != "fp32"            # 16-bit builds: the tensor-core (3xTF32 wgmma) kernels
        acts, dz = self.small_saved[cam], self.small_dz
        ops.sconv_mean_bwd(d_pool.data_ptr(), 256, acts.y[-1].data_ptr(), dz[-1].data_ptr(), B, S[-1] * S[-1], SMALL_CONVS[-1][1])
        for i in reversed(range(len(SMALL_CONVS))):
            ci, co = SMALL_CONVS[i] if i > 0 else (pix.shape[-1], SMALL_CONVS[0][1])
            x = acts.y[i - 1].data_ptr() if i > 0 else pix.data_ptr()
            ops.sconv_wgrad(x, i == 0, dz[i].data_ptr(), self.P(G, f"{p}/Conv_{i}/kernel"), self.P(G, f"{p}/Conv_{i}/bias"), self.small_ws,
                            B, S[i], S[i], ci, co, tc=tc)
            if i > 0:                                        # layer 0's input is the image: no input gradient
                ops.sconv_dgrad(dz[i].data_ptr(), self.P(Pm, f"{p}/Conv_{i}/kernel"), x, dz[i - 1].data_ptr(), B, S[i], S[i], ci, co, tc=tc)

    def encode_backward(self, dX: torch.Tensor, X: torch.Tensor, feats_rows: slice, state: torch.Tensor):
        """Gradients of the trainable heads given d(enc) = dX[:, :F]; the frozen trunk is stop-gradient, the small encoder's convs
        are not.  Weight / bias gradients of the Dense / LayerNorm heads run on side stream 0, the d_enc_z -> d_sle -> SLE-kernel
        chain (small encoder: d_enc_z -> d_pool -> conv backward) stays on the main stream."""
        cfg, B, ws, st = self.cfg, self.B, self.ws, self.store
        G = st.grad
        ld = self.FA
        side, wss = self.side[0], self.ws_side[0]
        for j, cam in enumerate(cfg.cams):
            p = f"{ENC}/encoder_{cam}"
            dez = self.d_enc_z[cam]
            dey = self.d_enc_y[cam]
            ops.ln_tanh_bwd(ops.at(dX, 256 * j), ld, ops.at(X, 256 * j), ld, self.enc_xhat[cam].data_ptr(), self.enc_rstd[cam].data_ptr(),
                            self.P(st.params, f"{p}/LayerNorm_0/scale"), B, 0, dez.data_ptr(), dey.data_ptr(), None, None, B, 256)
            x, K = (self.small_saved[cam].pooled, 256) if cfg.small else (self.sle_saved[cam], 4096)
            side.fork()
            with side:
                ops.ln_param_grad(dey.data_ptr(), self.enc_xhat[cam].data_ptr(), self.P(G, f"{p}/LayerNorm_0/scale"),
                                  self.P(G, f"{p}/LayerNorm_0/bias"), B, B, 256)
                ops.dense_bwd_weight(wss, x.data_ptr(), K, dez.data_ptr(), 256, self.P(G, f"{p}/Dense_0/kernel"), B, K, 256)
                ops.colsum(dez.data_ptr(), self.P(G, f"{p}/Dense_0/bias"), 1, B, 256, 256)
            dx = self.d_pool if cfg.small else self.d_sle
            ops.dense_bwd_input(ws, dez.data_ptr(), 256, self.P(st.params, f"{p}/Dense_0/kernel"), dx.data_ptr(), K, B, K, 256)
            if cfg.small:
                self.small_backward(cam, self.pix[cam][feats_rows], dx)
            else:
                feats = self.res_saved[cam].feats if cfg.resnet else self.feats[cam][feats_rows]
                ops.sle_bwd_kernel_grad(ws, feats, self.d_sle.data_ptr(), 4096, self.P(G, f"{p}/SpatialLearnedEmbeddings_0/kernel"))
                if cfg.resnet:
                    ops.sle_input_grad(self.d_sle.data_ptr(), 4096, self.P(st.params, f"{p}/SpatialLearnedEmbeddings_0/kernel"),
                                       self.d_feats.data_ptr(), B, 16, 512)
                    self.resnet_backward(cam, self.d_feats)
        if not cfg.use_proprio:
            return
        off = 256 * len(cfg.cams)
        ops.ln_tanh_bwd(ops.at(dX, off), ld, ops.at(X, off), ld, self.enc_xhat_p.data_ptr(), self.enc_rstd_p.data_ptr(),
                        self.P(st.params, f"{ENC}/LayerNorm_0/scale"), B, 0, self.d_enc_zp.data_ptr(), self.d_enc_yp.data_ptr(),
                        None, None, B, 64)
        side.fork()
        with side:
            ops.ln_param_grad(self.d_enc_yp.data_ptr(), self.enc_xhat_p.data_ptr(), self.P(G, f"{ENC}/LayerNorm_0/scale"),
                              self.P(G, f"{ENC}/LayerNorm_0/bias"), B, B, 64)
            ops.dense_bwd_weight(wss, state.data_ptr(), cfg.state_in, self.d_enc_zp.data_ptr(), 64, self.P(G, f"{ENC}/Dense_0/kernel"),
                                 B, cfg.state_in, 64)
            ops.colsum(self.d_enc_zp.data_ptr(), self.P(G, f"{ENC}/Dense_0/bias"), 1, B, 64, 64)

    # ---- MLP layers: [LayerNorm +] activation, forward and backward ----------------------------------------------------------
    def _act_fwd(self, arch: MlpArch, buf, prefix, i, z, out, xhat, rstd, rows_per_group, group_stride, R, D, mask=None):
        mlp_act_fwd(self.P, arch, buf, prefix, i, z, out, xhat, rstd, rows_per_group, group_stride, R, D, mask=mask,
                    mask_rows=None if mask is None else self.B)

    def _act_bwd(self, arch: MlpArch, prefix, i, acts: "_MlpActs", dt, dz, dy, rows_per_group, group_stride, R, D, dparams=None, mask=None):
        mlp_act_bwd(self.P, self.store.params, arch, prefix, i, acts, dt, dz, dy, rows_per_group, group_stride, R, D, dparams=dparams,
                    mask=mask, mask_rows=None if mask is None else self.B)

    # ---- critic ensemble (networks/actor_critic_nets.py:57-73, networks/mlp.py:22-31) ----------
    def critic_forward(self, buf, X: torch.Tensor, acts: _MlpActs, q: torch.Tensor, save: bool, ws: Optional[ops.Workspace] = None,
                       masks=None):
        """masks: the (B, H_i) Dropout keep masks of a train=True pass, shared by the E members (nn.vmap broadcasts the dropout
        rng, actor_critic_nets.py:156-164)."""
        cfg, B, E, ws = self.cfg, self.B, self.cfg.ensemble, ws or self.ws
        c, arch = "modules_critic/network", self.cfg.critic_arch
        x, ldx, x_z = X.data_ptr(), self.FA, 0                   # layer 0's input is broadcast over the ensemble
        for i, H in enumerate(arch.hidden):
            z = acts.zs[i]
            ops.dense_fwd(ws, x, ldx, self.P(buf, f"{c}/Dense_{i}/kernel"), self.P(buf, f"{c}/Dense_{i}/bias"), z.data_ptr(), H,
                          B, ldx, H, Z=E, x_z=x_z, out_z=B * H)
            self._act_fwd(arch, buf, c, i, z, acts.h[i], acts.xhat[i] if save else None, acts.rstd[i] if save else None, B, H, E * B, H,
                          mask=masks[i] if masks is not None else None)
            x, ldx, x_z = acts.h[i].data_ptr(), H, B * H
        H = arch.hidden[-1]
        wk, wb = self.P(buf, "modules_critic/Dense_0/kernel"), self.P(buf, "modules_critic/Dense_0/bias")
        if cfg.pixel:     # one shared value head over all E*B rows
            ops.dense_fwd(ws, x, H, wk, wb, q.data_ptr(), 1, E * B, H, 1)
        else:             # per-member head
            ops.dense_fwd(ws, x, H, wk, wb, q.data_ptr(), 1, B, H, 1, Z=E, x_z=B * H, w_z=H, b_z=1, out_z=B)

    def critic_backward(self, X: torch.Tensor, acts: _MlpActs, dq: torch.Tensor, param_grads: bool, need_dx: bool, masks=None):
        """The dq -> dh -> dz -> ... -> dX chain runs on the main stream; each layer's weight / bias gradient only needs that
        layer's (input, dz) pair, so it is forked to side stream 0 as soon as dz exists (joined by the caller).  masks: the
        forward's Dropout keep masks."""
        cfg, B, E, ws, st = self.cfg, self.B, self.cfg.ensemble, self.ws, self.store
        G, Pm = st.grad, st.params
        c, arch = "modules_critic/network", self.cfg.critic_arch
        FA, R, n = self.FA, E * B, len(arch.hidden)
        side, wss = self.side[0], self.ws_side[0]
        H = arch.hidden[-1]
        hl, dh = acts.h[-1].data_ptr(), self.dh
        wk = self.P(Pm, "modules_critic/Dense_0/kernel")
        if param_grads:
            side.fork()
            with side:
                if cfg.pixel:
                    ops.dense_bwd_weight(wss, hl, H, dq.data_ptr(), 1, self.P(G, "modules_critic/Dense_0/kernel"), R, H, 1)
                    ops.colsum(dq.data_ptr(), self.P(G, "modules_critic/Dense_0/bias"), 1, R, 1, 1)
                else:
                    ops.dense_bwd_weight(wss, hl, H, dq.data_ptr(), 1, self.P(G, "modules_critic/Dense_0/kernel"), B, H, 1,
                                         Z=E, x_z=B * H, dz_z=B, dw_z=H)
                    ops.colsum(dq.data_ptr(), self.P(G, "modules_critic/Dense_0/bias"), E, B, 1, 1)
        if cfg.pixel:
            ops.dense_bwd_input(ws, dq.data_ptr(), 1, wk, dh.data_ptr(), H, R, H, 1)
        else:
            ops.dense_bwd_input(ws, dq.data_ptr(), 1, wk, dh.data_ptr(), H, B, H, 1, Z=E, dz_z=B, w_z=H, dx_z=B * H)
        for i in reversed(range(n)):
            H = arch.hidden[i]
            dz, dy = self.c_dz[i], self.c_dy[i]
            self._act_bwd(arch, c, i, acts, dh, dz, dy, B, H, R, H, mask=masks[i] if masks is not None else None)
            x, K, x_z = (acts.h[i - 1].data_ptr(), arch.hidden[i - 1], B * arch.hidden[i - 1]) if i > 0 else (X.data_ptr(), FA, 0)
            if param_grads:
                side.fork()
                with side:
                    if arch.layer_norm:
                        ops.ln_param_grad(dy.data_ptr(), acts.xhat[i].data_ptr(), self.P(G, f"{c}/LayerNorm_{i}/scale"),
                                          self.P(G, f"{c}/LayerNorm_{i}/bias"), B, R, H)
                    ops.dense_bwd_weight(wss, x, K, dz.data_ptr(), H, self.P(G, f"{c}/Dense_{i}/kernel"), B, K, H, Z=E, x_z=x_z, dz_z=B * H)
                    ops.colsum(dz.data_ptr(), self.P(G, f"{c}/Dense_{i}/bias"), E, B, H, H)
            if i > 0:
                ops.dense_bwd_input(ws, dz.data_ptr(), H, self.P(Pm, f"{c}/Dense_{i}/kernel"), dh.data_ptr(), K, B, K, H, Z=E, dz_z=B * H,
                                    dx_z=B * K)
        if need_dx:       # input is broadcast over the ensemble: dX = sum_e dZ1_e W1_e^T
            H0 = arch.hidden[0]
            ops.dense_bwd_input(ws, self.c_dz[0].data_ptr(), H0, self.P(Pm, f"{c}/Dense_0/kernel"), self.dX.data_ptr(), FA, B, FA, H0, Z=E,
                                dz_z=B * H0, reduce_z=True)

    # ---- policy (networks/actor_critic_nets.py:178-227) ------------------------------------------
    def std_input(self, buf):
        """(address, row stride) of the std head's output the tanh-Gaussian reads: Dense_1's (B, A) rows, or the (A,) log_stds
        leaf broadcast to every row ("uniform")."""
        if self.cfg.std_parameterization == "uniform":
            return self.P(buf, "modules_actor/log_stds"), 0
        return self.ls.data_ptr(), self.cfg.action_dim

    def policy_forward(self, buf, Xp: torch.Tensor, save: bool, masks=None):
        cfg = self.cfg
        x, H = policy_hidden_fwd(self.P, self.ws, cfg.policy_arch, buf, Xp, self.F, self.p_acts, self.B, save, masks=masks)
        policy_heads_fwd(self.P, self.ws, cfg.std_parameterization, buf, x, H, self.mu, self.ls, self.B, cfg.action_dim)

    def tanh_gaussian(self, buf, act_out, ld_act, logp, u, std, deterministic=False):
        """std head -> clipped std -> tanh-Gaussian sample / log-prob; the "exp" head keeps the launcher's entry point."""
        cfg, B, A = self.cfg, self.B, self.cfg.action_dim
        if cfg.std_parameterization == "exp":
            ops.tanh_gaussian_fwd(self.mu, self.ls, self.eps, cfg.std_min, cfg.std_max, act_out, ld_act, logp, u, std, B, A,
                                  deterministic=deterministic)
        else:
            x, ld = self.std_input(buf)
            ops.tanh_gaussian_fwd_std(self.mu, x, ld, STD_IDS[cfg.std_parameterization], self.eps, cfg.std_min, cfg.std_max, act_out,
                                      ld_act, logp, u, std, B, A, deterministic=deterministic)

    def policy_backward(self, Xp: torch.Tensor):
        cfg, B, ws, a, st = self.cfg, self.B, self.ws, self.p_acts, self.store
        G, Pm = st.grad, st.params
        n, arch, F = POLICY, cfg.policy_arch, self.F
        policy_heads_bwd(self.P, ws, cfg.std_parameterization, Pm, G, a.h[-1].data_ptr(), arch.hidden[-1], self.dmu, self.dls, self.pdh,
                         B, cfg.action_dim)
        dz = policy_hidden_bwd(self.P, ws, arch, Pm, G, Xp, F, a, self.pdh, self.pdz, self.pdy, B, masks=self.p_mask)
        if self.cfg.proprio:              # (pixel-only: the actor loss reaches no encoder leaf)
            # Policy.__call__ -> encoder(..., stop_gradient=True) (actor_critic_nets.py:185) stops the gradient at the per-camera
            # image embeddings only (encoding.py:48-49); the proprio Dense -> LayerNorm -> tanh (:55-70) is differentiated by
            # jax.grad(policy_loss_fn) w.r.t. the full tree (sac.py:198-200).  Its gradient goes to the ACTOR-tx twin (aux tail)
            # of those leaves: d enc[:, off:] = dz0 @ W0[off:, :]^T, then back through LayerNorm / tanh / Dense.
            off, S, H0 = 256 * len(self.cfg.cams), self.cfg.state_in, arch.hidden[0]
            ops.dense_bwd_input(ws, dz.data_ptr(), H0, self.P(Pm, f"{n}/Dense_0/kernel") + 4 * off * H0, self.dXp_p.data_ptr(), 64, B, 64, H0)
            ops.ln_tanh_bwd(self.dXp_p.data_ptr(), 64, ops.at(Xp, off), F, self.enc_xhat_pa.data_ptr(), self.enc_rstd_pa.data_ptr(),
                            self.P(Pm, f"{ENC}/LayerNorm_0/scale"), B, 0, self.d_enc_zpa.data_ptr(), self.d_enc_ypa.data_ptr(),
                            st.aux_addr(G, f"{ENC}/LayerNorm_0/scale"), st.aux_addr(G, f"{ENC}/LayerNorm_0/bias"), B, 64)
            ops.dense_bwd_weight(ws, self.pol_state.data_ptr(), S, self.d_enc_zpa.data_ptr(), 64, st.aux_addr(G, f"{ENC}/Dense_0/kernel"), B, S, 64)
            ops.colsum(self.d_enc_zpa.data_ptr(), st.aux_addr(G, f"{ENC}/Dense_0/bias"), 1, B, 64, 64)

    # ---- the three losses --------------------------------------------------------------------------
    def _policy_pass(self, feats_rows, state, key_slot_eps, key_slot_drop, keys, act_out, ld_act, save, explicit=None):
        """enc(train=True -> dropout) -> policy -> tanh-Gaussian sample.  Writes actions to act_out."""
        cfg, B, A, st = self.cfg, self.B, self.cfg.action_dim, self.store
        if explicit is None:
            ops.normal_fill(ops.key_ptr(keys, key_slot_eps), self.eps, B * A)
            if cfg.pixel and not cfg.small:
                for j, cam in enumerate(cfg.cams):
                    ops.dropout_mask_fill(ops.key_ptr(keys, key_slot_drop), j, 0.9, self.masks_u8[cam], B * 4096)
        else:
            self.eps.copy_(explicit["eps"])
            for cam in (cfg.cams if cfg.pixel and not cfg.small else ()):
                self.masks_u8[cam].copy_(explicit["dropout"][cam])
        if self.p_mask is not None:                              # the policy MLP's masks, from the pass's dropout key
            self.fill_mlp_masks(self.p_mask, cfg.policy_arch, ops.key_ptr(keys, key_slot_drop), _given(explicit, "mlp_policy"))
        self.encode(st.params, feats_rows, state, self.Xp, self.F, self.masks_u8 if cfg.pixel and not cfg.small else None, save=False,
                    save_proprio_actor=save and cfg.pixel)
        self.pol_state = state                                   # proprio input of the pass policy_backward differentiates
        self.policy_forward(st.params, self.Xp, save, masks=self.p_mask)
        self.tanh_gaussian(st.params, act_out, ld_act, self.logp, self.u, self.std)

    def critic_loss_and_grads(self, keys, grad_scale=1.0, explicit=None):
        """sac.py:134-191 + its gradient w.r.t. group-0 parameters (written to store.grad)."""
        if self.fused is not None:
            return self.fused.critic_loss_and_grads(keys, grad_scale=grad_scale, explicit=explicit)
        cfg, B, E, st = self.cfg, self.B, self.cfg.ensemble, self.store
        obs_rows, next_rows = slice(0, B), slice(B, 2 * B)
        # three independent forward branches:
        #   side 0: Q(s, a) with params, saved for backward      side 1: target-encoder heads on s'
        #   main:   a', logp' ~ pi(s') (params, train=True), then Q'(s', a') with target params once side 1 has delivered enc(s')
        # critic-MLP dropout (sac.py:141-176): the target critic draws its masks from c1, the online critic from c2 with
        # critic_subsample_size and from c1 without it (the same bits as the target's then)
        ca, ex = cfg.critic_arch, None if explicit is None else explicit["critic"]
        s0, s1 = self.side
        s0.fork()
        s1.fork()
        with s0:
            self.encode(st.params, obs_rows, self.state_o, self.Xc, self.FA, None, save=True, sc=self.sc_side[0])
            ops.copy2d(self.actions.data_ptr(), cfg.action_dim, ops.at(self.Xc, self.F), self.FA, B, cfg.action_dim)
            if self.c_mask is not None:
                slot = L.KEY_MLP_CRITIC_SUBSAMPLED if cfg.subsample is not None else L.KEY_MLP_CRITIC_TARGET
                self.fill_mlp_masks(self.c_mask, ca, ops.key_ptr(keys, slot), _given(ex, "mlp_critic"))
            self.critic_forward(st.params, self.Xc, self.c_main, self.q, save=True, ws=self.ws_side[0], masks=self.c_mask)
        with s1:
            self.encode(st.target, next_rows, self.state_n, self.Xt, self.FA, None, save=False, sc=self.sc_side[1])
        self._policy_pass(next_rows, self.state_n, L.KEY_CRITIC_NEXT, L.KEY_CRITIC_NEXT, keys, ops.at(self.Xt, self.F), self.FA, save=False,
                          explicit=None if explicit is None else explicit["critic"])
        n_sub = 0
        if cfg.subsample is not None:
            if explicit is None:
                ops.subsample_idx(ops.key_ptr(keys, L.KEY_CRITIC_SUBSAMPLE), E, self.sub, cfg.subsample)
            else:
                self.sub.copy_(explicit["critic"]["subsample"])
            n_sub = cfg.subsample
        if self.c_mask_tgt is not None:
            self.fill_mlp_masks(self.c_mask_tgt, ca, ops.key_ptr(keys, L.KEY_MLP_CRITIC_TARGET), _given(ex, "mlp_critic_target"))
        s1.join()
        self.critic_forward(st.target, self.Xt, self.c_tgt, self.q_next, save=False, masks=self.c_mask_tgt)
        s0.join()
        ops.critic_loss(self.q, self.q_next, self.sub, n_sub, self.rewards, self.masks, self.logp, self.P(st.params, "modules_temperature/lagrange"),
                        cfg.backup_entropy, cfg.discount, grad_scale, self.target_q, self.dq, self.info.data_ptr(), E, B,
                        weights=self.weights if self.prio_parts else None, delta=self.delta)
        self.critic_backward(self.Xc, self.c_main, self.dq, param_grads=True, need_dx=cfg.pixel, masks=self.c_mask)
        if cfg.pixel:
            self.encode_backward(self.dX, self.Xc, obs_rows, self.state_o)
        s0.join()                                               # weight / bias gradients

    def actor_temp_loss_and_grads(self, keys, grad_scale=1.0, explicit=None, do_actor=True, do_temperature=True):
        """sac.py:193-234 + gradients w.r.t. group-1 / group-2 parameters (and the actor-tx twin of the proprio encoder)."""
        if self.fused is not None and os.environ.get("SERL_FUSED_ACTOR", "1") != "0":
            return self.fused.actor_temp_loss_and_grads(keys, grad_scale=grad_scale, explicit=explicit, do_actor=do_actor, do_temperature=do_temperature)
        cfg, B, E, A, st = self.cfg, self.B, self.cfg.ensemble, self.cfg.action_dim, self.store
        obs_rows, next_rows = slice(0, B), slice(B, 2 * B)
        lam = self.P(st.params, "modules_temperature/lagrange")
        if do_actor:
            self._actor_loss_and_grads(keys, grad_scale, explicit, obs_rows, lam)
        if do_temperature:
            # temperature: entropy of pi(.|s') with a fresh dropout mask / sample
            self._policy_pass(next_rows, self.state_n, L.KEY_TEMP_NEXT, L.KEY_TEMP_NEXT, keys, self.act_scratch.data_ptr(), A, save=False,
                              explicit=None if explicit is None else explicit["temperature"])
            ops.temperature_loss(self.logp, lam, cfg.target_entropy, grad_scale, self.P(st.grad, "modules_temperature/lagrange"), ops.at(self.info, 8), B)

    def _actor_loss_and_grads(self, keys, grad_scale, explicit, obs_rows, lam):
        cfg, B, E, A, st = self.cfg, self.B, self.cfg.ensemble, self.cfg.action_dim, self.store
        # actor: a, logp ~ pi_theta(s); q = mean_e Q_e(s, a) with constant critic params
        self._policy_pass(obs_rows, self.state_o, L.KEY_ACTOR_SAMPLE, L.KEY_ACTOR_DROPOUT, keys, ops.at(self.Xc, self.F), self.FA, save=True,
                          explicit=None if explicit is None else explicit["actor"])
        self.encode(st.params, obs_rows, self.state_o, self.Xc, self.FA, None, save=False)
        if self.c_mask is not None:                              # the critic on (s, pi(s)) drops out under the loss's critic_rng
            self.fill_mlp_masks(self.c_mask, cfg.critic_arch, ops.key_ptr(keys, L.KEY_MLP_ACTOR_CRITIC),
                                _given(None if explicit is None else explicit["actor"], "mlp_critic"))
        self.critic_forward(st.params, self.Xc, self.c_main, self.q, save=True, masks=self.c_mask)
        ops.fill(self.dq.data_ptr(), -grad_scale / (E * B), E * B)
        self.critic_backward(self.Xc, self.c_main, self.dq, param_grads=False, need_dx=True, masks=self.c_mask)
        if cfg.std_parameterization == "exp":
            ops.actor_loss(self.q, self.logp, lam, ops.at(self.dX, self.F), self.FA, ops.at(self.Xc, self.F), self.FA, self.std, self.ls, self.eps,
                           cfg.std_min, cfg.std_max, grad_scale, self.dmu, self.dls, ops.at(self.info, 4), E, B, A)
        else:
            x, ld = self.std_input(st.params)
            ops.actor_loss_std(self.q, self.logp, lam, ops.at(self.dX, self.F), self.FA, ops.at(self.Xc, self.F), self.FA, self.std, x, ld,
                               STD_IDS[cfg.std_parameterization], self.eps, cfg.std_min, cfg.std_max, grad_scale, self.dmu, self.dls,
                               ops.at(self.info, 4), E, B, A)
        self.policy_backward(self.Xp)

    def optimizer_step(self, live, polyak: bool):
        """The three txs of common.py:136-168 in one fused pass.  With clip_grad_norm on a live tx, the global norms of the
        gradients each tx receives are computed first (on the device, from the all-reduced buffer under data parallelism)."""
        cfg, st = self.cfg, self.store
        args = (st.params, st.target, st.m, st.v, st.grad, st.seg_end, live, st.counts, cfg.lr, cfg.warmup, cfg.tau, polyak)
        kw = dict(lr_out=self.lr_info, n=st.n_main, gap=INFO_GAP, aux=(st.aux_lo, st.aux_hi, st.aux_off))
        clip = [c or 0.0 for c in cfg.clip]
        decay = [s or 0 for s in cfg.decay]
        if not any(clip) and not any(decay):
            ops.adam_polyak(*args, **kw)
            return
        d = ops.adam_desc(*args, **kw)
        want = [int(bool(c) and bool(g)) for c, g in zip(clip, live)]
        if any(want):
            ops.grad_global_norms(d, want, self.norm_partials, self.grad_norms)
        ops.adam_polyak_opts(d, clip, decay, self.grad_norms)


def _given(explicit, name):
    """Explicit MLP masks of one loss (explicit_randomness[loss][name], a list of (B, H_i) keep masks), or None: key-derived."""
    return None if explicit is None else explicit.get(name)


class InferenceEngine(Engine):
    """Forward-only buffers of one batch size for `sample_actions` and the public forward passes (`forward_critic`,
    `forward_policy`, ...).  It shares the parameters and the frozen trunk with the training engines but none of their buffers,
    so an inference call never touches a step's batch, crops, features or the pipeline's prefetched next step.  No backward
    scratch, no info / optimizer buffers, no fused-heads state: the forward passes run on the per-op kernels (same kernels and
    workspace size as the training engines' forward passes, so `sample_actions` gives the same bits on either)."""

    def __init__(self, cfg: AgentConfig, store: ParamStore, trunk: FrozenTrunk, batch: int, device):
        self.cfg, self.store, self.B, self.dev = cfg, store, batch, device
        B, E, A, F = batch, cfg.ensemble, cfg.action_dim, cfg.enc_dim
        self.F, self.FA = F, F + A
        e = lambda *s: torch.empty(*s, dtype=f32, device=device)
        gemm_impl = os.environ.get("SERL_HEADS_GEMM") or ("f32" if cfg.precision == "fp32" else "tf32x3")
        self.ws = ops.Workspace(max(48 << 20, 2 * 4 * E * B * self.FA), device, gemm_impl)
        self.state_o = e(B, cfg.state_in)
        if cfg.pixel:
            hw = cfg.image_hw
            self.pix = {c: torch.empty(B, hw, hw, cfg.in_channels, dtype=torch.uint8, device=device) for c in cfg.cams}
            if not cfg.trainable_encoder:
                self.feats = {c: e(B, 4, 4, 512) for c in cfg.cams}
                self.trunk = trunk.runner(B, device)
            self.masks_u8 = {c: torch.empty(B, 4096, dtype=torch.uint8, device=device) for c in cfg.cams}
        self.sc_main = _EncScratch(cfg, B, device, self.ws)
        self.Xc, self.Xp = e(B, self.FA), e(B, F)
        self.c_main = _MlpActs(E * B, device, cfg.critic_arch)
        self.q = e(E, B)
        self.p_acts = _MlpActs(B, device, cfg.policy_arch)
        self.mu, self.ls, self.eps, self.std = e(B, A), e(B, A), e(B, A), e(B, A)
        self.act_scratch = e(B, A)
        self.multi = {}                 # N -> (P, first-layer scratch, activations over E*B*N rows, q)
        self.fused = None
        self._mlp_mask_bufs = {}

    def mlp_masks(self, arch: MlpArch):
        """The keep-mask buffers of a train=True forward (forward_critic / forward_policy), one set per architecture."""
        if arch not in self._mlp_mask_bufs:
            self._mlp_mask_bufs[arch] = Engine.mlp_masks(self, arch)
        return self._mlp_mask_bufs[arch]

    def critic_forward_multi(self, buf, X: torch.Tensor, actions: torch.Tensor, N: int) -> torch.Tensor:
        """Q (E, B*N) of N candidate actions per state (actions (B, N, A) contiguous); X[:, :F] holds enc(obs).  Layer 0 is split
        as W0 = [W_enc; W_act]: P = enc @ W_enc + b0 once per (member, state) on the GEMM, then serl_critic_multi_action_fwd adds
        a @ W_act per candidate with the layer's LayerNorm + activation; the other layers and the value head run on E*B*N rows."""
        cfg, B, E, A, F, FA = self.cfg, self.B, self.cfg.ensemble, self.cfg.action_dim, self.F, self.FA
        c, arch = "modules_critic/network", cfg.critic_arch
        if N not in self.multi:
            e = lambda *s: torch.empty(*s, dtype=f32, device=self.dev)
            self.multi[N] = (e(E, B, arch.hidden[0]), _MlpActs(E * B * N, self.dev, arch), e(E, B * N))
        P, acts, q = self.multi[N]
        M, H0 = B * N, arch.hidden[0]
        w0 = self.P(buf, f"{c}/Dense_0/kernel")
        ops.dense_fwd(self.ws, X.data_ptr(), FA, w0, self.P(buf, f"{c}/Dense_0/bias"), P.data_ptr(), H0, B, F, H0, Z=E, x_z=0,
                      w_z=FA * H0, out_z=B * H0)
        ln = arch.layer_norm
        ops.critic_multi_action_fwd(P, actions, w0 + 4 * F * H0, FA * H0, self.P(buf, f"{c}/LayerNorm_0/scale") if ln else None,
                                    self.P(buf, f"{c}/LayerNorm_0/bias") if ln else None, acts.zs[0], acts.h[0], E, B, N, A, H0,
                                    ACT_IDS[arch.act], ln)
        x, ldx = acts.h[0].data_ptr(), H0
        for i in range(1, len(arch.hidden)):
            H = arch.hidden[i]
            z = acts.zs[i]
            ops.dense_fwd(self.ws, x, ldx, self.P(buf, f"{c}/Dense_{i}/kernel"), self.P(buf, f"{c}/Dense_{i}/bias"), z.data_ptr(), H,
                          M, ldx, H, Z=E, x_z=M * ldx, out_z=M * H)
            self._act_fwd(arch, buf, c, i, z, acts.h[i], None, None, M, H, E * M, H)
            x, ldx = acts.h[i].data_ptr(), H
        H = arch.hidden[-1]
        wk, wb = self.P(buf, "modules_critic/Dense_0/kernel"), self.P(buf, "modules_critic/Dense_0/bias")
        if cfg.pixel:     # one shared value head over all E*B*N rows
            ops.dense_fwd(self.ws, x, H, wk, wb, q.data_ptr(), 1, E * M, H, 1)
        else:             # per-member head
            ops.dense_fwd(self.ws, x, H, wk, wb, q.data_ptr(), 1, M, H, 1, Z=E, x_z=M * H, w_z=H, b_z=1, out_z=M)
        return q
