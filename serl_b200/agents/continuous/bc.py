"""BCAgent on the hand-written sm_90a kernels of the learner (SURVEY.md §8 row f4: reuse of the encoder by behaviour cloning).

Mirrors the reference's `BCAgent` (agents/continuous/bc.py:21-226).  `make_bc_agent` (utils/launcher.py:26-47) builds
`resnet-pretrained` encoders (frozen ResNet-10 trunk + SpatialLearnedEmbeddings / Dense / LayerNorm / tanh head per camera,
Dropout(0.1) when training), proprio Dense(64) -> LayerNorm -> tanh, policy MLP [256, 256] with tanh and NO LayerNorm,
exp-parameterised std clipped to [1e-5, 5], no tanh squash; one Adam(3e-4).  `BCAgent.create` also takes the reference's other
options: any MLP of networks/mlp.py (widths, activation, LayerNorm, dropout_rate), the "exp" / "softplus" / "uniform" std heads
and the constant "fixed" std, the tanh-squashed distribution, pixel-only encoders (use_proprio=False) and the trainable encoder
types "small" (the default, as in the reference) and "resnet" (bc.py:124-163).

    loss = -mean_b log pi(a_b | o_b),  info = {actor_loss, mse = mean_b sum (mode_b - a_b)^2}                 (bc.py:46-69)

Gradient semantics: `Policy.__call__` calls the encoder with `stop_gradient=True` (networks/actor_critic_nets.py:185), which
stops the gradient at each camera's image embedding (common/encoding.py:48-49): the image heads receive a ZERO gradient (Adam
leaves them at their initial values - a property of the reference), the proprio Dense / LayerNorm, the MLP and the output heads
are trained.  With "small" / "resnet" that holds for the whole image path: convs, norms, pooling head, Dense and LayerNorm keep
their initial values and zero Adam moments, and no encoder backward runs.  Key chain (common/common.py:198-200 with one loss), on the device (`ops.bc_key_chain`): new_rng, k = split(rng);
dropout key = split(k)[1]; camera j's SLE mask folds j, hidden layer i's MLP mask folds ncams + i (DESIGN.md §4).

Same kernels as the DrQ / SAC step: trunk (fp32 or tensor-core build), DrQ's trainable encoder forwards
(`engine.small_encoder_forward` / `engine.resnet_encoder_forward`), `sle_fwd`, GEMMs, the engine's policy-MLP loops, LayerNorm +
tanh, fused Adam.  The parameters live in one `params.FlatParams` store (`agent._store`; its `target` is the
never-updated `target_params`), and the frozen trunk's subtree of `state.params` is read and written by `FrozenTrunk` (which holds
no leaves for the trainable encoder types: their convs are leaves of the store).
"""
from __future__ import annotations

import ctypes as C
from collections.abc import Mapping
from typing import Dict, Iterable, Optional

import numpy as np
import torch

from ... import _lib as L
from ... import ops
from ...data.replay_buffer import BatchHandle, refuse_nstep, refuse_prioritized
from ...engine import (MAX_OBS_HORIZON, STD_IDS, AgentConfig, _MlpActs, _ResActs, _SmallActs, policy_heads_bwd, policy_heads_fwd, policy_hidden_bwd,
                       policy_hidden_fwd, resnet_encoder_forward, small_encoder_forward, small_sizes)
from ...params import (ENC, ENCODER_TYPES, STD_PARAMETERIZATIONS, TRUNK_PATH, FlatParams, MlpArch, assign_offsets, camera_encoder_leaves, flatten,
                       init_leaves, init_trunk, kaiming_in_resnet_encoder, nest, policy_leaves, proprio_leaves, xavier_outside_encoders)
from ...step_graphs import StepGraphs
from ...trunk import FrozenTrunk
from .sac import _host_split, resolve_mlp

f32 = torch.float32


BC_LAUNCHER_MLP = MlpArch((256, 256), "tanh", False)         # utils/launcher.py:26-47
_BC_LAUNCHER_NET_KWARGS = {"activations": "tanh", "use_layer_norm": False, "hidden_dims": [256, 256]}
_POLICY_KEYS = {"std_parameterization", "std_min", "std_max", "tanh_squash_distribution", "fixed_std"}


def bc_options(network_kwargs: Optional[dict], policy_kwargs: Optional[dict]):
    """BCAgent.create's `network_kwargs` / `policy_kwargs` -> (MlpArch, std_parameterization, std_min, std_max, tanh_squash).
    Omitted network_kwargs build the launcher's MLP; a dict that differs from it must state `activations` and `use_layer_norm`
    (sac.resolve_mlp).  Policy's defaults: "exp" std in [1e-5, 10], no squash (actor_critic_nets.py:167-177).  A fixed std is
    std_parameterization="fixed" together with a 1-D `fixed_std` (`resolve_fixed_std` reads it); either one alone is refused, as Policy
    refuses it (actor_critic_nets.py:190-210)."""
    arch = resolve_mlp("network_kwargs", network_kwargs, BC_LAUNCHER_MLP, _BC_LAUNCHER_NET_KWARGS, allow_dropout=True)
    pk = dict(policy_kwargs or {})
    unknown = set(pk) - _POLICY_KEYS
    if unknown:
        raise TypeError(f"policy_kwargs: unexpected keys {sorted(unknown)} (Policy takes {sorted(_POLICY_KEYS)})")
    std = pk.get("std_parameterization", "exp")
    if (std == "fixed") != (pk.get("fixed_std") is not None):
        raise NotImplementedError(f"policy_kwargs={pk}: a fixed std takes both std_parameterization='fixed' and fixed_std")
    if std == "fixed":
        resolve_fixed_std(pk)
    elif std not in STD_PARAMETERIZATIONS:
        raise NotImplementedError(f"policy_kwargs={pk}: std_parameterization={std!r} is not supported (implemented: "
                                  f"{STD_PARAMETERIZATIONS + ('fixed',)})")
    return arch, std, float(pk.get("std_min", 1e-5)), float(pk.get("std_max", 10.0)), bool(pk.get("tanh_squash_distribution", False))


def resolve_fixed_std(policy_kwargs) -> np.ndarray:
    """policy_kwargs["fixed_std"] as a 1-D float32 vector of finite values (one per action dimension)."""
    v = np.asarray(policy_kwargs["fixed_std"], dtype=np.float64)
    if v.ndim != 1 or v.size < 1 or not np.isfinite(v).all():
        raise ValueError(f"policy_kwargs: fixed_std must be a 1-D vector of finite values, one per action dimension (got {v!r})")
    return v.astype(np.float32)


def bc_spec(cams, state_in: int, action_dim: int, arch: MlpArch = BC_LAUNCHER_MLP, std_parameterization: str = "exp",
            use_proprio: bool = True, encoder: str = "resnet-pretrained", in_channels: int = 3):
    """Trainable leaves in the Flax layout: per-camera encoders (params.camera_encoder_leaves: the image heads of
    "resnet-pretrained", the conv stack + Dense / LayerNorm of "small", the ResNet-10 + image head of "resnet"), the proprio
    Dense / LayerNorm (use_proprio), the policy MLP (`modules_actor/network/Dense_i` [+ `LayerNorm_i`]), the means head
    `modules_actor/Dense_0` and the std head `modules_actor/Dense_1` ("exp", "softplus"), the free `modules_actor/log_stds` vector
    ("uniform") or none ("fixed").  in_channels: the trainable encoders' input channels (3T for stacks of T frames)."""
    leaves = [l for cam in cams for l in camera_encoder_leaves(f"{ENC}/encoder_{cam}", encoder, in_channels=in_channels)]
    if use_proprio:
        leaves += proprio_leaves(state_in)
    leaves += policy_leaves(256 * len(cams) + (64 if use_proprio else 0), action_dim, arch, std_parameterization, 0)
    return leaves, assign_offsets(leaves)


class _BCState:
    """`agent.state` of the BC agent: the JaxRLTrainState fields of one optax.adam (step, params in the Flax tree layout incl. the
    frozen trunk, target_params, opt_states {count, mu, nu}, rng), read from and written to the agent's device buffers.
    `state_dict()` is what checkpoints store: nested dicts of NumPy arrays and ints."""

    def __init__(self, agent):
        self._a = agent
        self.step = 0

    def _tree(self, buf):
        a = self._a
        return nest({**a._store.dump(buf), **a._frozen_trunk.dump(TRUNK_PATH.format)})

    @property
    def params(self):
        return self._tree(self._a._store.params)

    @property
    def target_params(self):           # JaxRLTrainState.create(target_params=params): never updated by BC (no target_update call)
        return self._tree(self._a._store.target)

    @property
    def rng(self):
        return self._a._rng.cpu().numpy().copy()

    @property
    def opt_states(self):
        st = self._a._store
        return {"count": int(st.counts[0].item()), "mu": nest(st.dump(st.m)), "nu": nest(st.dump(st.v))}

    def state_dict(self) -> dict:
        return {"step": int(self.step), "params": self.params, "target_params": self.target_params, "opt_states": self.opt_states,
                "rng": self.rng}

    def load_state_dict(self, d) -> "_BCState":
        return self.replace(**{k: d[k] for k in ("step", "params", "target_params", "opt_states", "rng")})

    def replace(self, **kw):
        """state.replace(params=tree, target_params=tree, opt_states={count, mu, nu}, rng=key, step=n), any subset: params writes
        the trainable leaves and the frozen trunk from a Flax-layout tree.  Any write drops the agent's captured step graphs."""
        a = self._a
        st = a._store
        unknown = set(kw) - {"params", "target_params", "opt_states", "rng", "step"}
        if unknown:
            raise TypeError(f"replace: unknown fields {sorted(unknown)}")
        if "params" in kw:
            flat = flatten(kw["params"])
            st.load(st.params, flat)
            a._frozen_trunk.load(flat, TRUNK_PATH.format)
        if "target_params" in kw:
            st.load(st.target, flatten(kw["target_params"]))
        if "opt_states" in kw:
            o = kw["opt_states"]
            st.load(st.m, flatten(o["mu"]))
            st.load(st.v, flatten(o["nu"]))
            st.counts.fill_(int(o["count"]))                      # adam_single ticks all three counts every step
        if "rng" in kw:
            key = np.ascontiguousarray(np.asarray(kw["rng"]), dtype=np.uint32).reshape(2)
            a._rng.copy_(torch.from_numpy(key.view(np.int32)).view(torch.uint32))
        if "step" in kw:
            self.step = int(kw["step"])
        if set(kw) - {"step"}:
            a.invalidate_graphs()
        return self


class BCAgent:
    def __init__(self, cfg: AgentConfig, spec, trunk, device):
        self._cfg, self._trunk, self.device = cfg, trunk, torch.device(device)
        self._frozen_trunk = FrozenTrunk(trunk, cfg.precision, cfg.image_hw)
        self._store = FlatParams(spec, device)
        # the store's layout, parameter and gradient buffers (the same tensors) under the names the GPU parity tests read
        self._spec, self._n, self._params, self._grad = spec, self._store.n, self._store.params, self._store.grad
        self._rng = torch.zeros(2, dtype=torch.uint32, device=device)
        self._key = torch.zeros(2, dtype=torch.uint32, device=device)
        self._info = torch.zeros(4, dtype=f32, device=device)
        self.learning_rate, self.std_min, self.std_max = 3e-4, 1e-5, 5.0
        self.arch, self.std_parameterization, self.tanh_squash = BC_LAUNCHER_MLP, "exp", False
        self.fixed_std = None                   # "fixed": the constant (A,) std on the device
        self.config = dict(image_keys=tuple(cfg.cams))
        self.state = _BCState(self)
        # tests: {cam: (B, 4096) keep mask (not for "small"), "mlp": [(B, H_i) keep mask per layer]} instead of the keyed masks
        self.explicit_dropout = None
        self.use_cuda_graphs = True             # replay the step on a replay-ring batch as one CUDA graph from its 2nd identical call on
        self._graphs = StepGraphs()
        self._bufs: Dict[int, dict] = {}

    # ---- construction (bc.py:113-226, utils/launcher.py:26-47) ---------------------------------------------
    @classmethod
    def create(cls, seed: int, observations, actions, *, encoder_type: str = "small", image_keys: Iterable[str] = ("image",),
               use_proprio: bool = False, network_kwargs: Optional[dict] = None, policy_kwargs: Optional[dict] = None,
               learning_rate: float = 3e-4, precision: str = "fp32", device=None):
        """BCAgent.create (bc.py:113-226).  encoder_type "small" and "resnet" build the reference's networks with the `encode=`
        argument EncodingWrapper passes dropped (neither encoder takes it, so the reference's own branches fail at their first
        forward; DrQ's encoders do the same, drq.py): "small" is SmallEncoder((32, 64, 128, 256), 3x3 / stride 2 VALID, mean pool,
        Dense(256) -> LayerNorm -> tanh) on frames of at least 31x31 (the fourth conv's input must keep 3x3 positions); "resnet" is a
        resnetv1-10 with the SpatialLearnedEmbeddings(8) -> Dropout(0.1) -> Dense(256) -> LayerNorm -> tanh head on 128x128 frames,
        from kaiming-normal initial weights.  Both sit behind the policy's stop_gradient and keep their initial values.

        With observations of ChunkingWrapper(obs_horizon=T), images (T, H, W, C), "small" and "resnet" take stacks of T <= 8 frames on
        the channel axis, "B T H W C -> B H W (T C)" (EncodingWrapper's enable_stacking): their first conv reads 3T channels."""
        if encoder_type not in ENCODER_TYPES:
            raise NotImplementedError(f"encoder_type={encoder_type!r}: supported are {ENCODER_TYPES}")
        arch, std, std_min, std_max, squash = bc_options(network_kwargs, policy_kwargs)
        cams = tuple(image_keys)
        img = np.asarray(observations[cams[0]])
        hw = int(img.shape[-2])
        # "resnet-pretrained" keeps one frame per observation: a stack is refused where the batch is read
        T = int(img.shape[-4]) if img.ndim >= 4 and encoder_type != "resnet-pretrained" else 1
        if not 1 <= T <= MAX_OBS_HORIZON:
            raise NotImplementedError(f"obs_horizon={T}: stacks of 1 to {MAX_OBS_HORIZON} frames are supported")
        if encoder_type == "resnet" and hw != 128:
            # the SLE head's (4, 4, 512, 8) kernel expects the trunk's 4x4 output of a 128x128 frame
            raise NotImplementedError(f"encoder_type='resnet' takes 128x128 frames (got {hw}x{hw})")
        if encoder_type == "small" and small_sizes(hw)[-2] < 3:
            raise NotImplementedError(f"encoder_type='small' takes frames of at least 31x31 (got {hw}x{hw})")
        L.load()
        device = torch.device(device if device is not None else "cuda")
        L.require_cuda(device)
        S = 0
        if use_proprio:
            if "state" not in observations:
                raise ValueError("BCAgent.create(use_proprio=True): the observations have no 'state' entry for the proprio encoder")
            S = int(np.prod(np.asarray(observations["state"]).shape))
        A = int(np.asarray(actions).shape[-1])
        fixed = None
        if std == "fixed":
            fixed = resolve_fixed_std(policy_kwargs)
            if fixed.shape != (A,):
                raise ValueError(f"policy_kwargs: fixed_std has {fixed.size} values for {A} action dimensions")
        cfg = AgentConfig(cams=cams, state_in=S, action_dim=A, pixel=True, image_hw=hw, precision=precision, policy_arch=arch,
                          std_parameterization=std, use_proprio=bool(use_proprio), encoder=encoder_type, obs_horizon=T)
        spec, _ = bc_spec(cams, S, A, arch, std, bool(use_proprio), encoder_type, in_channels=cfg.in_channels)
        rng = np.random.default_rng(seed)
        trunk = {}
        if encoder_type == "resnet-pretrained":
            trunk = {cam: {k: torch.as_tensor(v).to(device).contiguous() for k, v in init_trunk(rng).items()} for cam in cams}
        agent = cls(cfg, spec, trunk, device)
        agent.learning_rate = float(learning_rate)
        agent.std_min, agent.std_max = std_min, std_max
        agent.arch, agent.std_parameterization, agent.tanh_squash = arch, std, squash
        if fixed is not None:
            agent.fixed_std = torch.from_numpy(fixed).to(device)
        st = agent._store
        st.load(st.params, init_leaves(rng, spec, xavier_outside_encoders, kaiming=kaiming_in_resnet_encoder))
        st.target.copy_(st.params)
        # rng, init_rng = split(PRNGKey(seed)); rng, create_rng = split(rng)   (bc.py:196-206)
        key = np.array([(seed >> 32) & 0xFFFFFFFF, seed & 0xFFFFFFFF], dtype=np.uint32)
        create = _host_split(_host_split(key, 2)[0], 2)[1]
        agent._rng.copy_(torch.from_numpy(create.view(np.int32)).view(torch.uint32))
        if encoder_type != "resnet-pretrained":
            return agent
        from ...utils.train_utils import load_resnet10_params
        return load_resnet10_params(agent, cams)

    # ---- helpers --------------------------------------------------------------------------------------------
    @property
    def _launcher_mlp(self) -> bool:
        """The launcher's MLP keeps its own kernel sequence (serl_tanh_fwd / _bwd); every other MLP runs the engine's layer loop."""
        return self.arch == BC_LAUNCHER_MLP

    def _b(self, B):
        if B not in self._bufs:
            cfg, dev, arch = self._cfg, self.device, self.arch
            e = lambda *s: torch.empty(*s, dtype=f32, device=dev)
            F, A, Hm = cfg.enc_dim, cfg.action_dim, max(arch.hidden)
            gemm_impl = "f32" if cfg.precision == "fp32" else "tf32x3"
            self._bufs[B] = dict(
                ws=ops.Workspace(48 << 20, dev, gemm_impl),
                pix={c: torch.empty(B, cfg.image_hw, cfg.image_hw, cfg.in_channels, dtype=torch.uint8, device=dev) for c in cfg.cams},
                masks={c: torch.empty(B, 4096, dtype=torch.uint8, device=dev) for c in cfg.cams} if not cfg.small else {},
                sle=e(B, 4096), enc_z=e(B, 256), enc_zp=e(B, 64), xhat_p=e(B, 64), rstd_p=e(B), state=e(B, cfg.state_in), act=e(B, A),
                X=e(B, F), mu=e(B, A), ls=e(B, A), dmu=e(B, A), dls=e(B, A), dXp=e(B, 64), dzp=e(B, 64), dyp=e(B, 64), std=e(B, A))
            # the image encoders' activations: the cameras run one after the other and nothing reads them back (no encoder backward)
            if cfg.small:
                self._bufs[B]["small"] = _SmallActs(B, cfg.image_hw, dev)
            elif cfg.resnet:
                self._bufs[B]["res"] = _ResActs(B, cfg.image_hw, dev, cfg.in_channels)
            else:
                self._bufs[B].update(trunk=self._frozen_trunk.runner(B, dev), feats={c: e(B, 4, 4, 512) for c in cfg.cams})
            if self._launcher_mlp:
                self._bufs[B].update(z1=e(B, 256), h1=e(B, 256), z2=e(B, 256), h2=e(B, 256), dh=e(B, 256), dz2=e(B, 256), dz1=e(B, 256))
            else:
                self._bufs[B].update(acts=_MlpActs(B, dev, arch), dh=e(B, Hm), dz=e(B, Hm), dy=e(B, Hm) if arch.layer_norm else None,
                                     mlp_masks=[torch.empty(B, H, dtype=torch.uint8, device=dev) for H in arch.hidden] if arch.dropout else None)
        return self._bufs[B]

    def _ingest(self, b, observations, actions=None):
        """Reference-layout observations (dict of host / device arrays, (B, T[+1], H, W, 3) pixels, (B, T, S) state) -> device buffers.
        A pixel-only agent ignores a "state" entry."""
        cfg = self._cfg
        for cam in cfg.cams:
            px = observations[cam]
            px = px if isinstance(px, torch.Tensor) else torch.as_tensor(np.asarray(px))
            T = cfg.obs_horizon
            if px.dim() == 5 and T == 1:
                if px.shape[1] > 2:
                    raise NotImplementedError("BCAgent: obs_horizon 1 (one frame per observation), like every SERL example")
                px = px[:, 0]
            elif px.dim() == 5:                      # (B, T[+1], H, W, C) -> (B, H, W, T*C), oldest frame first
                if px.shape[1] not in (T, T + 1):
                    raise ValueError(f"BCAgent: {cam!r} frames of shape {tuple(px.shape)}; the agent takes stacks of {T} frames")
                px = px[:, :T].permute(0, 2, 3, 1, 4).reshape(px.shape[0], px.shape[2], px.shape[3], px.shape[4] * T)
            b["pix"][cam].copy_(px.to(self.device, torch.uint8))
        if cfg.use_proprio:
            if "state" not in observations:
                raise ValueError("BCAgent (use_proprio=True): the observations have no 'state' entry")
            st = observations["state"]
            st = st if isinstance(st, torch.Tensor) else torch.as_tensor(np.asarray(st))
            b["state"].copy_(st.to(self.device, f32).reshape(b["state"].shape))
        if actions is not None:
            ac = actions if isinstance(actions, torch.Tensor) else torch.as_tensor(np.asarray(actions))
            b["act"].copy_(ac.to(self.device, f32))

    def _on_device(self, batch) -> bool:
        """A replay-ring batch whose rows the sampler can write straight into the step's buffers: one frame per observation,
        the agent's cameras, frame size, state and action widths, drawn by the ring's own index draw."""
        if not isinstance(batch, BatchHandle) or self.explicit_dropout is not None or self.device.type != "cuda":
            return False
        cfg = self._cfg
        for p in batch.parts:
            r = p["ring"]
            if (p.get("indx") is not None or r.shards is not None or r.cams != cfg.cams or r.T != cfg.obs_horizon or r.A != cfg.action_dim
                    or r.frame_shape != (cfg.image_hw, cfg.image_hw, 3) or (cfg.use_proprio and r.T * r.S != cfg.state_in)):
                return False
        return True

    def _sample(self, b, batch: BatchHandle, B: int, graph_mode: bool):
        """The sampler's draw of `batch` into the step's buffers: frames (identity crop, a stack's frames on the channel axis) ->
        pix, state -> state (a pixel-only agent's go to scratch), actions -> act; next frames, next state, rewards, masks, dones and
        indices to scratch."""
        cfg, dev, T = self._cfg, self.device, self._cfg.obs_horizon
        if "smp" not in b:
            e = lambda *s, dt=f32: torch.empty(*s, dtype=dt, device=dev)
            b["smp"] = dict(next_pix={c: e(B, cfg.image_hw, cfg.image_hw, cfg.in_channels, dt=torch.uint8) for c in cfg.cams}, rew=e(B),
                            mask=e(B), done=e(B, dt=torch.uint8), idx=e(B, dt=torch.int32),
                            status=torch.zeros(1, dtype=torch.int32, device=dev),
                            ident=torch.full((B * T, 2), 4, dtype=torch.int32, device=dev), sinks={})
        s = b["smp"]
        out = L.BatchOut()
        for j, cam in enumerate(cfg.cams):
            out.obs_pix[j], out.next_pix[j] = b["pix"][cam].data_ptr(), s["next_pix"][cam].data_ptr()
        out.actions, out.rewards, out.masks, out.dones = b["act"].data_ptr(), s["rew"].data_ptr(), s["mask"].data_ptr(), s["done"].data_ptr()
        out.idx, out.status = s["idx"].data_ptr(), s["status"].data_ptr()
        out.stacked = 1
        row = 0
        for part in batch.parts:
            ring = part["ring"]
            n = max(ring.T * ring.S, 1)
            if n not in s["sinks"]:
                s["sinks"][n] = (torch.empty(B, n, dtype=f32, device=dev), torch.empty(B, n, dtype=f32, device=dev))
            sink_o, sink_n = s["sinks"][n]
            out.obs_state = (b["state"] if cfg.use_proprio else sink_o).data_ptr()
            out.next_state = sink_n.data_ptr()
            ring.launch_sample(part, out, crop_total=B * T, out_row_offset=row, explicit_off=(s["ident"], s["ident"]),
                               step_dev=ring.step_dev if graph_mode else None, record_event=not graph_mode)
            if graph_mode:
                ops.counter_add(ring.step_dev, 1)
            row += part["batch"]

    def check_status(self):
        """Raises if a replay draw that loaded a step's batch on the device found no valid slot (synchronises)."""
        for b in self._bufs.values():
            if "smp" in b and int(b["smp"]["status"].item()):
                raise L.SerlError("replay draw failed: no valid slot within the redraw budget")

    def invalidate_graphs(self):
        """Drops every captured step graph and the packed 16-bit trunk weights they read: called when the state was written from
        outside the step (`state.replace`, a checkpoint restore)."""
        self._graphs.clear()
        self._frozen_trunk.drop_packed()

    def _std_input(self, b):
        """(address, row stride) of the std head's output: Dense_1's (B, A) rows, the "uniform" (A,) log_stds leaf or the "fixed"
        (A,) std."""
        if self.std_parameterization == "uniform":
            return self._store.addr(self._store.params, "modules_actor/log_stds"), 0
        if self.std_parameterization == "fixed":
            return self.fixed_std.data_ptr(), 0
        return b["ls"].data_ptr(), self._cfg.action_dim

    def _forward(self, b, B, train: bool, save: bool):
        """encoder (common/encoding.py:26-72; dropout when train) -> MLP (networks/mlp.py:22-31; Dense -> [Dropout when train] ->
        [LayerNorm] -> activation per layer) -> means, std head."""
        cfg, P, Pm, ws = self._cfg, self._store.addr, self._store.params, b["ws"]
        if not cfg.trainable_encoder:
            for cam in cfg.cams:
                b["trunk"].forward(cam, b["pix"][cam], b["feats"][cam])
        F = cfg.enc_dim
        for j, cam in enumerate(cfg.cams):
            p = f"{ENC}/encoder_{cam}"
            if cfg.small:               # conv stack -> mean pool (no SpatialLearnedEmbeddings, no Dropout)
                small_encoder_forward(self._store, cfg.precision, Pm, cam, b["pix"][cam], b["small"])
                x, K = b["small"].pooled.data_ptr(), 256
            else:
                if cfg.resnet:
                    resnet_encoder_forward(self._store, cfg.precision, Pm, cam, b["pix"][cam], b["res"])
                feats = b["res"].feats if cfg.resnet else b["feats"][cam]
                ops.sle_fwd(feats, self._store.view(Pm, f"{p}/SpatialLearnedEmbeddings_0/kernel"), b["masks"][cam] if train else None, 0.9,
                            b["sle"].data_ptr(), 4096)
                x, K = b["sle"].data_ptr(), 4096
            ops.dense_fwd(ws, x, K, P(Pm, f"{p}/Dense_0/kernel"), P(Pm, f"{p}/Dense_0/bias"), b["enc_z"].data_ptr(), 256, B, K, 256)
            ops.ln_tanh_fwd(b["enc_z"].data_ptr(), 256, P(Pm, f"{p}/LayerNorm_0/scale"), P(Pm, f"{p}/LayerNorm_0/bias"), B, 0,
                            ops.at(b["X"], 256 * j), F, None, None, B, 256)
        if cfg.use_proprio:
            ops.dense_fwd(ws, b["state"].data_ptr(), cfg.state_in, P(Pm, f"{ENC}/Dense_0/kernel"), P(Pm, f"{ENC}/Dense_0/bias"), b["enc_zp"].data_ptr(), 64, B, cfg.state_in, 64)
            ops.ln_tanh_fwd(b["enc_zp"].data_ptr(), 64, P(Pm, f"{ENC}/LayerNorm_0/scale"), P(Pm, f"{ENC}/LayerNorm_0/bias"), B, 0,
                            ops.at(b["X"], 256 * len(cfg.cams)), F, b["xhat_p"].data_ptr() if save else None, b["rstd_p"].data_ptr() if save else None, B, 64)
        n, A = "modules_actor/network", cfg.action_dim
        if self._launcher_mlp:
            ops.dense_fwd(ws, b["X"].data_ptr(), F, P(Pm, f"{n}/Dense_0/kernel"), P(Pm, f"{n}/Dense_0/bias"), b["z1"].data_ptr(), 256, B, F, 256)
            L.call("serl_tanh_fwd", b["z1"].data_ptr(), b["h1"].data_ptr(), B * 256, L.stream_ptr())
            ops.dense_fwd(ws, b["h1"].data_ptr(), 256, P(Pm, f"{n}/Dense_1/kernel"), P(Pm, f"{n}/Dense_1/bias"), b["z2"].data_ptr(), 256, B, 256, 256)
            L.call("serl_tanh_fwd", b["z2"].data_ptr(), b["h2"].data_ptr(), B * 256, L.stream_ptr())
            x, H = b["h2"].data_ptr(), 256
        else:
            x, H = policy_hidden_fwd(P, ws, self.arch, Pm, b["X"], F, b["acts"], B, save, masks=b["mlp_masks"] if train else None)
        policy_heads_fwd(P, ws, self.std_parameterization, Pm, x, H, b["mu"], b["ls"], B, A)

    def _mlp_backward(self, b, B):
        """Gradients of the output heads and the MLP from dmu / dls; returns the (B, H0) dz of the MLP's first layer."""
        st, ws, A, F = self._store, b["ws"], self._cfg.action_dim, self._cfg.enc_dim
        P, Pm, G = st.addr, st.params, st.grad
        n, std = "modules_actor/network", self.std_parameterization
        if self._launcher_mlp:
            policy_heads_bwd(P, ws, std, Pm, G, b["h2"].data_ptr(), 256, b["dmu"], b["dls"], b["dh"], B, A)
            L.call("serl_tanh_bwd", b["dh"].data_ptr(), b["h2"].data_ptr(), b["dz2"].data_ptr(), B * 256, L.stream_ptr())
            ops.dense_bwd_weight(ws, b["h1"].data_ptr(), 256, b["dz2"].data_ptr(), 256, P(G, f"{n}/Dense_1/kernel"), B, 256, 256)
            ops.colsum(b["dz2"].data_ptr(), P(G, f"{n}/Dense_1/bias"), 1, B, 256, 256)
            ops.dense_bwd_input(ws, b["dz2"].data_ptr(), 256, P(Pm, f"{n}/Dense_1/kernel"), b["dh"].data_ptr(), 256, B, 256, 256)
            L.call("serl_tanh_bwd", b["dh"].data_ptr(), b["h1"].data_ptr(), b["dz1"].data_ptr(), B * 256, L.stream_ptr())
            ops.dense_bwd_weight(ws, b["X"].data_ptr(), F, b["dz1"].data_ptr(), 256, P(G, f"{n}/Dense_0/kernel"), B, F, 256)
            ops.colsum(b["dz1"].data_ptr(), P(G, f"{n}/Dense_0/bias"), 1, B, 256, 256)
            return b["dz1"]
        arch, acts = self.arch, b["acts"]
        policy_heads_bwd(P, ws, std, Pm, G, acts.h[-1].data_ptr(), arch.hidden[-1], b["dmu"], b["dls"], b["dh"], B, A)
        return policy_hidden_bwd(P, ws, arch, Pm, G, b["X"], F, acts, b["dh"], b["dz"], b["dy"], B, masks=b["mlp_masks"])

    # ---- update (bc.py:36-76) -------------------------------------------------------------------------------
    def update(self, batch, pmap_axis: Optional[str] = None):
        """One BC step.  A replay-ring batch (`_on_device`) is drawn by the sampler straight into the step's buffers and, with
        `use_cuda_graphs`, replayed as one CUDA graph per (batch size, rings); the step then never waits for the host.  Dict
        batches, `explicit_dropout` and other handles go through `_ingest`.  Infos are 0-d device tensors."""
        refuse_nstep(batch, "BCAgent.update", "behaviour cloning reads no rewards")
        refuse_prioritized(batch, "BCAgent.update")
        dist = None
        if pmap_axis is not None:
            import torch.distributed as dist_
            if dist_.is_available() and dist_.is_initialized() and dist_.get_world_size() > 1:
                dist = dist_
        if self._on_device(batch):
            B = batch.batch_size
            key = (B, tuple((id(p["ring"]), p["batch"]) for p in batch.parts)) if self.use_cuda_graphs and dist is None else None
            self._graphs.run(key, [(p["ring"], p["step"], 1) for p in batch.parts],
                             lambda graph_mode: self._step(batch, B, dist, graph_mode), self.state)
        else:
            if isinstance(batch, BatchHandle):
                batch = batch.to_dict()
            B = int(batch["actions"].shape[0])
            self._ingest(self._b(B), batch["observations"], batch["actions"])
            self._step(None, B, dist, False)
        snap = self._info.clone()
        return self, {"actor_loss": snap[0], "mse": snap[1]}

    def _step(self, handle: Optional[BatchHandle], B: int, dist, graph_mode: bool):
        """Enqueues one step on the buffers of batch size B: the sampler's draw of `handle` (None: the batch is already ingested),
        the key chain and dropout masks, forward, loss, backward, the data-parallel all-reduces (`dist`, eager only) and Adam."""
        b, cfg, st = self._b(B), self._cfg, self._store
        P, Pm, G = st.addr, st.params, st.grad
        ws, A, F = b["ws"], cfg.action_dim, cfg.enc_dim
        if handle is not None:
            self._sample(b, handle, B, graph_mode)
        # key chain: new_rng, k = split(rng) (common.py:198-200, one loss); rng, key = split(k) (bc.py:48); dropout key = key.
        # One key for the whole forward pass: camera j's SLE mask folds j, hidden layer i's MLP mask folds ncams + i (DESIGN.md §4).
        ops.bc_key_chain(self._rng, self._key)
        mlp_masks = b.get("mlp_masks")
        if self.explicit_dropout is not None:
            for cam in b["masks"]:
                b["masks"][cam].copy_(torch.as_tensor(np.asarray(self.explicit_dropout[cam])).to(self.device, torch.uint8))
            for m, e in zip(mlp_masks or (), self.explicit_dropout.get("mlp", ())):
                m.copy_(torch.as_tensor(np.asarray(e)).to(self.device, torch.uint8))
        else:
            for j, cam in enumerate(cfg.cams):
                if cam in b["masks"]:                                # the small encoder has no Dropout
                    ops.dropout_mask_fill(self._key.data_ptr(), j, 0.9, b["masks"][cam], B * 4096)
            for i, m in enumerate(mlp_masks or ()):
                ops.dropout_mask_fill(self._key.data_ptr(), len(cfg.cams) + i, 1.0 - self.arch.dropout, m, m.numel())
        self._forward(b, B, train=True, save=True)
        world = dist.get_world_size() if dist is not None else 1
        if self.std_parameterization == "exp" and not self.tanh_squash:
            L.call("serl_bc_loss", b["mu"].data_ptr(), b["ls"].data_ptr(), b["act"].data_ptr(), self.std_min, self.std_max, 1.0 / world,
                   b["dmu"].data_ptr(), b["dls"].data_ptr(), self._info.data_ptr(), B, A, L.stream_ptr())
        else:
            x, ld = self._std_input(b)
            ops.bc_loss_std(b["mu"], x, ld, STD_IDS[self.std_parameterization], self.tanh_squash, b["act"], self.std_min, self.std_max,
                            1.0 / world, b["dmu"], b["dls"], self._info.data_ptr(), B, A)
        # ---- backward: heads -> MLP -> proprio encoder (the image embeddings are behind stop_gradient) ----
        G.zero_()
        dz0 = self._mlp_backward(b, B)
        if cfg.use_proprio:
            n, H0 = "modules_actor/network", self.arch.hidden[0]
            off = 256 * len(cfg.cams)
            ops.dense_bwd_input(ws, dz0.data_ptr(), H0, P(Pm, f"{n}/Dense_0/kernel") + 4 * off * H0, b["dXp"].data_ptr(), 64, B, 64, H0)
            ops.ln_tanh_bwd(b["dXp"].data_ptr(), 64, ops.at(b["X"], off), F, b["xhat_p"].data_ptr(), b["rstd_p"].data_ptr(), P(Pm, f"{ENC}/LayerNorm_0/scale"), B, 0,
                            b["dzp"].data_ptr(), b["dyp"].data_ptr(), P(G, f"{ENC}/LayerNorm_0/scale"), P(G, f"{ENC}/LayerNorm_0/bias"), B, 64)
            ops.dense_bwd_weight(ws, b["state"].data_ptr(), cfg.state_in, b["dzp"].data_ptr(), 64, P(G, f"{ENC}/Dense_0/kernel"), B, cfg.state_in, 64)
            ops.colsum(b["dzp"].data_ptr(), P(G, f"{ENC}/Dense_0/bias"), 1, B, 64, 64)
        if dist is not None:                                        # jax.lax.pmean(grads_and_aux) (common.py:213-214)
            dist.all_reduce(G, op=dist.ReduceOp.SUM)
            dist.all_reduce(self._info, op=dist.ReduceOp.SUM)
        ops.adam_single(st, self.learning_rate)
        self.state.step += 1

    # ---- inference (bc.py:78-111) ---------------------------------------------------------------------------
    def _dist_params(self, observations):
        """train=False forward -> (mu, std, single): the base Gaussian's means and clipped std of every row."""
        px = observations[self._cfg.cams[0]]
        single = (px.dim() if isinstance(px, torch.Tensor) else np.asarray(px).ndim) == 4       # one (T, H, W, 3) observation
        obs = {k: (np.asarray(v)[None] if single else v) for k, v in observations.items()} if single else observations
        px = obs[self._cfg.cams[0]]
        B = int(px.shape[0])
        b = self._b(B)
        self._ingest(b, obs)
        self._forward(b, B, train=False, save=False)
        mu = b["mu"].clone()
        if self.std_parameterization == "exp":
            std = torch.clamp(torch.exp(b["ls"]), self.std_min, self.std_max)          # thin glue on outputs, not on the hot path
        else:
            x, ld = self._std_input(b)
            ops.tanh_gaussian_fwd_std(b["mu"], x, ld, STD_IDS[self.std_parameterization], None, self.std_min, self.std_max, b["dmu"].data_ptr(),
                                      self._cfg.action_dim, None, None, b["std"], B, self._cfg.action_dim, deterministic=True)
            std = b["std"].clone()
        return mu, std, single

    def sample_actions(self, observations, *, seed=None, temperature: float = 1.0, argmax: bool = False):
        """dist.mode() (argmax) or dist.sample(seed) of the policy with std * sqrt(temperature); tanh of both when squashed."""
        mu, std, single = self._dist_params(observations)
        if argmax:
            out = mu
        else:
            B, A = mu.shape
            key = np.asarray(seed, dtype=np.uint32).reshape(2)
            self._key.copy_(torch.from_numpy(key.view(np.int32)).view(torch.uint32))
            eps = torch.empty(B, A, dtype=f32, device=self.device)
            ops.normal_fill(self._key.data_ptr(), eps, B * A)
            out = mu + std * (temperature ** 0.5) * eps
        if self.tanh_squash:
            out = torch.tanh(out)
        out = out.detach().cpu().numpy()
        return out[0] if single else out

    def get_debug_metrics(self, batch, **kwargs):
        if isinstance(batch, BatchHandle):
            batch = batch.to_dict()
        mu, std, _ = self._dist_params(batch["observations"])
        a = (batch["actions"] if isinstance(batch["actions"], torch.Tensor) else torch.as_tensor(np.asarray(batch["actions"]))).to(self.device, f32)
        if self.tanh_squash:
            mode = torch.tanh(mu)
            logp = torch.empty(mu.shape[0], dtype=f32, device=self.device)
            ops.tanh_normal_log_prob(mu, std, a.contiguous(), logp, mu.shape[0], mu.shape[1])
        else:
            mode = mu
            z = (a - mu) / std
            logp = (-0.5 * z * z - torch.log(std) - 0.918938533204672742).sum(-1)
        return {"mse": ((mode - a) ** 2).sum(-1), "log_probs": logp, "pi_actions": mode}

    def replace(self, **kw):
        """replace(state=s) installs a checkpointed state: a `_BCState` (what `restore_checkpoint(dir, agent.state)` returns, or
        another BC agent's state) or its `state_dict()` (what `restore_checkpoint(dir, None)` returns)."""
        if "state" in kw:
            s = kw.pop("state")
            if s is not self.state:                   # restore_checkpoint(dir, agent.state) has already loaded it into this agent
                if isinstance(s, _BCState):
                    s = s.state_dict()
                elif not isinstance(s, Mapping):
                    raise TypeError(f"replace(state=...): expected a BC state or its state_dict(), got {type(s).__name__}")
                self.state.load_state_dict(s)
        if kw:
            raise TypeError(f"replace: unknown fields {sorted(kw)}")
        return self


def _register_flax_serialization():
    try:
        from flax import serialization
    except Exception:                                   # noqa: BLE001
        return False
    try:
        serialization.register_serialization_state(_BCState, lambda s: s.state_dict(), lambda s, d: s.load_state_dict(d))
    except ValueError:
        pass
    return True


_register_flax_serialization()
