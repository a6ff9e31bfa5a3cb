"""BCAgent on the hand-written sm_100a kernels of the learner (SURVEY.md §8 row f4: reuse of the encoder by behaviour cloning).

Mirrors the reference's `BCAgent` (agents/continuous/bc.py:21-226) in the configuration `make_bc_agent` builds
(utils/launcher.py:26-47): `resnet-pretrained` encoders (frozen ResNet-10 trunk + SpatialLearnedEmbeddings / Dense / LayerNorm /
tanh head per camera, Dropout(0.1) when training), proprio Dense(64) -> LayerNorm -> tanh, policy MLP [256, 256] with tanh and
NO LayerNorm, exp-parameterised std clipped to [1e-5, 5], no tanh squash; one Adam(3e-4).

    loss = -mean_b log N(a_b; mu_b, diag(std_b^2)),  info = {actor_loss, mse}                       (bc.py:47-70)

Gradient semantics: `Policy.__call__` calls the encoder with `stop_gradient=True` (networks/actor_critic_nets.py:185), which
stops the gradient at each camera's image embedding (common/encoding.py:48-49): the image heads receive a ZERO gradient (Adam
leaves them at their initial values - a property of the reference), the proprio Dense / LayerNorm, the MLP and the two output
heads are trained.  Key chain (common/common.py:198-200 with one loss): new_rng, k = split(rng); dropout key = split(k)[1].

Same kernels as the DrQ / SAC step: trunk (fp32 or tcgen05 build), `sle_fwd`, GEMMs, LayerNorm + tanh, fused Adam.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, Optional

import numpy as np
import torch

from ... import _lib as L
from ... import ops
from ...data.replay_buffer import BatchHandle
from ...engine import AgentConfig
from ...params import ENC, Leaf, init_trunk, lecun_normal, nest, xavier_uniform
from ...trunk import FrozenTrunk
from .sac import _host_split

f32 = torch.float32


def bc_spec(cams, state_in: int, action_dim: int):
    leaves, H, A = [], 256, action_dim
    for cam in cams:
        p = f"{ENC}/encoder_{cam}"
        leaves += [Leaf(f"{p}/SpatialLearnedEmbeddings_0/kernel", (4, 4, 512, 8), 0), Leaf(f"{p}/Dense_0/kernel", (4096, 256), 0),
                   Leaf(f"{p}/Dense_0/bias", (256,), 0), Leaf(f"{p}/LayerNorm_0/scale", (256,), 0), Leaf(f"{p}/LayerNorm_0/bias", (256,), 0)]
    leaves += [Leaf(f"{ENC}/Dense_0/kernel", (state_in, 64), 0), Leaf(f"{ENC}/Dense_0/bias", (64,), 0),
               Leaf(f"{ENC}/LayerNorm_0/scale", (64,), 0), Leaf(f"{ENC}/LayerNorm_0/bias", (64,), 0)]
    F = 256 * len(cams) + 64
    a = "modules_actor/network"
    leaves += [Leaf(f"{a}/Dense_0/kernel", (F, H), 0), Leaf(f"{a}/Dense_0/bias", (H,), 0), Leaf(f"{a}/Dense_1/kernel", (H, H), 0),
               Leaf(f"{a}/Dense_1/bias", (H,), 0), Leaf("modules_actor/Dense_0/kernel", (H, A), 0), Leaf("modules_actor/Dense_0/bias", (A,), 0),
               Leaf("modules_actor/Dense_1/kernel", (H, A), 0), Leaf("modules_actor/Dense_1/bias", (A,), 0)]
    off = 0
    for l in leaves:
        l.offset = off
        off += (l.size + 3) // 4 * 4
    return leaves, off


class _BCState:
    """`agent.state` of the BC agent: params in the Flax tree layout (incl. the frozen trunk), rng, step (JaxRLTrainState fields)."""

    def __init__(self, agent):
        self._a = agent
        self.step = 0

    def _tree(self, buf):
        a = self._a
        host = buf.detach().cpu().numpy()
        flat = {l.path: host[l.offset:l.offset + l.size].reshape(l.shape).copy() for l in a._spec}
        for cam, leaves in a._trunk.items():
            for k, v in leaves.items():
                flat[f"{ENC}/encoder_{cam}/pretrained_encoder/{k}"] = v.detach().cpu().numpy()
        return nest(flat)

    @property
    def params(self):
        return self._tree(self._a._params)

    @property
    def target_params(self):           # JaxRLTrainState.create(target_params=params): never updated by BC (no target_update call)
        return self._tree(self._a._params0)

    @property
    def rng(self):
        return self._a._rng.cpu().numpy().copy()

    @property
    def opt_states(self):
        a = self._a
        return {"count": int(a._counts[0].item()), "mu": self._tree_plain(a._m), "nu": self._tree_plain(a._v)}

    def replace(self, **kw):
        """state.replace(params=tree[, rng=key, step=n]): writes the trainable leaves and the frozen trunk from a Flax-layout tree."""
        from ...params import flatten
        a = self._a
        if "params" in kw:
            flat = flatten(kw.pop("params"))
            host = a._params.detach().cpu()
            for l in a._spec:
                if l.path in flat:
                    host[l.offset:l.offset + l.size] = torch.as_tensor(np.asarray(flat[l.path], np.float32)).reshape(-1)
            a._params.copy_(host)
            for cam, leaves in a._trunk.items():
                for k in leaves:
                    key = f"{ENC}/encoder_{cam}/pretrained_encoder/{k}"
                    if key in flat:
                        leaves[k].copy_(torch.as_tensor(np.asarray(flat[key], np.float32)).to(leaves[k].device))
            a._frozen_trunk.drop_packed()
        if "rng" in kw:
            a._rng.copy_(torch.from_numpy(np.asarray(kw.pop("rng"), np.uint32).view(np.int32)).view(torch.uint32))
        if "step" in kw:
            self.step = int(kw.pop("step"))
        if kw:
            raise TypeError(f"replace: unknown fields {sorted(kw)}")
        return self

    def _tree_plain(self, buf):
        host = buf.detach().cpu().numpy()
        return nest({l.path: host[l.offset:l.offset + l.size].reshape(l.shape).copy() for l in self._a._spec})


class BCAgent:
    def __init__(self, cfg: AgentConfig, spec, n, trunk, device, seed):
        self._cfg, self._spec, self._n, self._trunk, self.device = cfg, spec, n, trunk, torch.device(device)
        self._frozen_trunk = FrozenTrunk(trunk, cfg.precision, cfg.image_hw)
        self._leaf = {l.path: l for l in spec}
        z = lambda: torch.zeros(n, dtype=f32, device=device)
        self._params, self._params0, self._m, self._v, self._grad = z(), z(), z(), z(), z()
        self._counts = torch.zeros(3, dtype=torch.int32, device=device)
        self._rng = torch.zeros(2, dtype=torch.uint32, device=device)
        self._key = torch.zeros(2, dtype=torch.uint32, device=device)
        self._info = torch.zeros(4, dtype=f32, device=device)
        self._lr_info = torch.zeros(4, dtype=f32, device=device)
        self.learning_rate, self.std_min, self.std_max = 3e-4, 1e-5, 5.0
        self.config = dict(image_keys=tuple(cfg.cams))
        self.state = _BCState(self)
        self.explicit_dropout = None            # tests: {cam: (B, 4096) keep mask} instead of the keyed masks
        self._bufs: Dict[int, dict] = {}

    # ---- construction (bc.py:113-226, utils/launcher.py:26-47) ---------------------------------------------
    @classmethod
    def create(cls, seed: int, observations, actions, *, encoder_type: str = "small", image_keys: Iterable[str] = ("image",),
               use_proprio: bool = False, network_kwargs: Optional[dict] = None, policy_kwargs: Optional[dict] = None,
               learning_rate: float = 3e-4, precision: str = "fp32", device=None):
        if encoder_type != "resnet-pretrained":
            raise NotImplementedError("BCAgent: only encoder_type='resnet-pretrained' is implemented (the encoder the DrQ launchers share)")
        nk, pk = network_kwargs or {}, policy_kwargs or {}
        act = nk.get("activations", "tanh")
        if (getattr(act, "__name__", act) != "tanh" or nk.get("use_layer_norm", False) or list(nk.get("hidden_dims", [256, 256])) != [256, 256]
                or pk.get("tanh_squash_distribution", False) or pk.get("std_parameterization", "exp") != "exp" or not use_proprio):
            raise NotImplementedError("BCAgent: the launcher's configuration only (make_bc_agent: tanh MLP [256, 256] without LayerNorm, "
                                      "exp std, no tanh squash, use_proprio=True)")
        L.load()
        device = torch.device(device if device is not None else "cuda")
        L.require_cuda(device)
        cams = tuple(image_keys)
        state = np.asarray(observations["state"])
        S, A = int(np.prod(state.shape)), int(np.asarray(actions).shape[-1])
        hw = int(np.asarray(observations[cams[0]]).shape[-2])
        cfg = AgentConfig(cams=cams, state_in=S, action_dim=A, pixel=True, image_hw=hw, precision=precision)
        spec, n = bc_spec(cams, S, A)
        rng = np.random.default_rng(seed)
        trunk = {cam: {k: torch.as_tensor(v).to(device).contiguous() for k, v in init_trunk(rng).items()} for cam in cams}
        agent = cls(cfg, spec, n, trunk, device, seed)
        agent.learning_rate = float(learning_rate)
        agent.std_min, agent.std_max = float(pk.get("std_min", 1e-5)), float(pk.get("std_max", 10.0))
        host = torch.zeros(n, dtype=f32)
        for l in spec:
            if l.path.endswith("kernel"):
                v = lecun_normal(rng, l.shape) if "/encoder_" in l.path else xavier_uniform(rng, l.shape)
            elif l.path.endswith("scale"):
                v = np.ones(l.shape, np.float32)
            else:
                v = np.zeros(l.shape, np.float32)
            host[l.offset:l.offset + l.size] = torch.as_tensor(v).reshape(-1)
        agent._params.copy_(host)
        agent._params0.copy_(host)
        # rng, init_rng = split(PRNGKey(seed)); rng, create_rng = split(rng)   (bc.py:196-206)
        key = np.array([(seed >> 32) & 0xFFFFFFFF, seed & 0xFFFFFFFF], dtype=np.uint32)
        create = _host_split(_host_split(key, 2)[0], 2)[1]
        agent._rng.copy_(torch.from_numpy(create.view(np.int32)).view(torch.uint32))
        from ...utils.train_utils import load_resnet10_params
        return load_resnet10_params(agent, cams)

    # ---- helpers --------------------------------------------------------------------------------------------
    def _P(self, buf, path):
        return buf.data_ptr() + 4 * self._leaf[path].offset

    def _b(self, B):
        if B not in self._bufs:
            cfg, dev = self._cfg, self.device
            e = lambda *s: torch.empty(*s, dtype=f32, device=dev)
            F = cfg.enc_dim
            gemm_impl = "f32" if cfg.precision == "fp32" else "tf32x3"
            self._bufs[B] = dict(
                trunk=self._frozen_trunk.runner(B, dev), ws=ops.Workspace(48 << 20, dev, gemm_impl),
                pix={c: torch.empty(B, cfg.image_hw, cfg.image_hw, 3, dtype=torch.uint8, device=dev) for c in cfg.cams},
                feats={c: e(B, 4, 4, 512) for c in cfg.cams}, masks={c: torch.empty(B, 4096, dtype=torch.uint8, device=dev) for c in cfg.cams},
                sle=e(B, 4096), enc_z=e(B, 256), enc_zp=e(B, 64), xhat_p=e(B, 64), rstd_p=e(B), state=e(B, cfg.state_in), act=e(B, cfg.action_dim),
                X=e(B, F), z1=e(B, 256), h1=e(B, 256), z2=e(B, 256), h2=e(B, 256), mu=e(B, cfg.action_dim), ls=e(B, cfg.action_dim),
                dmu=e(B, cfg.action_dim), dls=e(B, cfg.action_dim), dh=e(B, 256), dz2=e(B, 256), dz1=e(B, 256), dXp=e(B, 64), dzp=e(B, 64), dyp=e(B, 64))
        return self._bufs[B]

    def _ingest(self, b, observations, actions=None):
        """Reference-layout observations (dict of host / device arrays, (B, T[+1], H, W, 3) pixels, (B, T, S) state) -> device buffers."""
        cfg = self._cfg
        for cam in cfg.cams:
            px = observations[cam]
            px = px if isinstance(px, torch.Tensor) else torch.as_tensor(np.asarray(px))
            if px.dim() == 5:
                if px.shape[1] > 2:
                    raise NotImplementedError("BCAgent: obs_horizon 1 (one frame per observation), like every SERL example")
                px = px[:, 0]
            b["pix"][cam].copy_(px.to(self.device, torch.uint8))
        st = observations["state"]
        st = st if isinstance(st, torch.Tensor) else torch.as_tensor(np.asarray(st))
        b["state"].copy_(st.to(self.device, f32).reshape(b["state"].shape))
        if actions is not None:
            ac = actions if isinstance(actions, torch.Tensor) else torch.as_tensor(np.asarray(actions))
            b["act"].copy_(ac.to(self.device, f32))

    def _forward(self, b, B, train: bool, save: bool):
        """encoder (common/encoding.py:26-72; dropout when train) -> MLP (Dense + tanh, twice) -> means, log-stds."""
        cfg, P, Pm, ws = self._cfg, self._P, self._params, b["ws"]
        for cam in cfg.cams:
            b["trunk"].forward(cam, b["pix"][cam], b["feats"][cam])
        F = cfg.enc_dim
        for j, cam in enumerate(cfg.cams):
            p = f"{ENC}/encoder_{cam}"
            l = self._leaf[f"{p}/SpatialLearnedEmbeddings_0/kernel"]
            ops.sle_fwd(b["feats"][cam], Pm[l.offset:l.offset + l.size].view(l.shape), b["masks"][cam] if train else None, 0.9, b["sle"].data_ptr(), 4096)
            ops.dense_fwd(ws, b["sle"].data_ptr(), 4096, P(Pm, f"{p}/Dense_0/kernel"), P(Pm, f"{p}/Dense_0/bias"), b["enc_z"].data_ptr(), 256, B, 4096, 256)
            ops.ln_tanh_fwd(b["enc_z"].data_ptr(), 256, P(Pm, f"{p}/LayerNorm_0/scale"), P(Pm, f"{p}/LayerNorm_0/bias"), B, 0,
                            ops.at(b["X"], 256 * j), F, None, None, B, 256)
        ops.dense_fwd(ws, b["state"].data_ptr(), cfg.state_in, P(Pm, f"{ENC}/Dense_0/kernel"), P(Pm, f"{ENC}/Dense_0/bias"), b["enc_zp"].data_ptr(), 64, B, cfg.state_in, 64)
        ops.ln_tanh_fwd(b["enc_zp"].data_ptr(), 64, P(Pm, f"{ENC}/LayerNorm_0/scale"), P(Pm, f"{ENC}/LayerNorm_0/bias"), B, 0,
                        ops.at(b["X"], 256 * len(cfg.cams)), F, b["xhat_p"].data_ptr() if save else None, b["rstd_p"].data_ptr() if save else None, B, 64)
        n, A = "modules_actor/network", cfg.action_dim
        ops.dense_fwd(ws, b["X"].data_ptr(), F, P(Pm, f"{n}/Dense_0/kernel"), P(Pm, f"{n}/Dense_0/bias"), b["z1"].data_ptr(), 256, B, F, 256)
        L.call("serl_tanh_fwd", b["z1"].data_ptr(), b["h1"].data_ptr(), B * 256, L.stream_ptr())
        ops.dense_fwd(ws, b["h1"].data_ptr(), 256, P(Pm, f"{n}/Dense_1/kernel"), P(Pm, f"{n}/Dense_1/bias"), b["z2"].data_ptr(), 256, B, 256, 256)
        L.call("serl_tanh_fwd", b["z2"].data_ptr(), b["h2"].data_ptr(), B * 256, L.stream_ptr())
        ops.dense_fwd(ws, b["h2"].data_ptr(), 256, P(Pm, "modules_actor/Dense_0/kernel"), P(Pm, "modules_actor/Dense_0/bias"), b["mu"].data_ptr(), A, B, 256, A)
        ops.dense_fwd(ws, b["h2"].data_ptr(), 256, P(Pm, "modules_actor/Dense_1/kernel"), P(Pm, "modules_actor/Dense_1/bias"), b["ls"].data_ptr(), A, B, 256, A)

    # ---- update (bc.py:36-76) -------------------------------------------------------------------------------
    def update(self, batch, pmap_axis: Optional[str] = None):
        if isinstance(batch, BatchHandle):
            batch = batch.to_dict()
        actions = batch["actions"]
        B = int(actions.shape[0])
        b, cfg, P, Pm, G = self._b(B), self._cfg, self._P, self._params, self._grad
        ws, A, F = b["ws"], cfg.action_dim, cfg.enc_dim
        self._ingest(b, batch["observations"], actions)
        # key chain: new_rng, k = split(rng) (common.py:198-200, one loss); rng, key = split(k) (bc.py:48); dropout key = key
        r = self.state.rng
        new_rng, k = _host_split(r, 2)
        drop = _host_split(k, 2)[1]
        self._rng.copy_(torch.from_numpy(new_rng.view(np.int32)).view(torch.uint32))
        if self.explicit_dropout is not None:
            for cam in cfg.cams:
                b["masks"][cam].copy_(torch.as_tensor(np.asarray(self.explicit_dropout[cam])).to(self.device, torch.uint8))
        else:
            self._key.copy_(torch.from_numpy(drop.view(np.int32)).view(torch.uint32))
            for j, cam in enumerate(cfg.cams):
                ops.dropout_mask_fill(self._key.data_ptr(), j, 0.9, b["masks"][cam], B * 4096)
        self._forward(b, B, train=True, save=True)
        world = 1
        dist = None
        if pmap_axis is not None:
            import torch.distributed as dist_
            if dist_.is_available() and dist_.is_initialized() and dist_.get_world_size() > 1:
                dist, world = dist_, dist_.get_world_size()
        L.call("serl_bc_loss", b["mu"].data_ptr(), b["ls"].data_ptr(), b["act"].data_ptr(), self.std_min, self.std_max, 1.0 / world,
               b["dmu"].data_ptr(), b["dls"].data_ptr(), self._info.data_ptr(), B, A, L.stream_ptr())
        # ---- backward: heads -> MLP -> proprio encoder (the image embeddings are behind stop_gradient) ----
        self._grad.zero_()
        n = "modules_actor/network"
        ops.dense_bwd_weight(ws, b["h2"].data_ptr(), 256, b["dmu"].data_ptr(), A, P(G, "modules_actor/Dense_0/kernel"), B, 256, A)
        ops.colsum(b["dmu"].data_ptr(), P(G, "modules_actor/Dense_0/bias"), 1, B, A, A)
        ops.dense_bwd_weight(ws, b["h2"].data_ptr(), 256, b["dls"].data_ptr(), A, P(G, "modules_actor/Dense_1/kernel"), B, 256, A)
        ops.colsum(b["dls"].data_ptr(), P(G, "modules_actor/Dense_1/bias"), 1, B, A, A)
        ops.dense_bwd_input(ws, b["dmu"].data_ptr(), A, P(Pm, "modules_actor/Dense_0/kernel"), b["dh"].data_ptr(), 256, B, 256, A)
        ops.dense_bwd_input(ws, b["dls"].data_ptr(), A, P(Pm, "modules_actor/Dense_1/kernel"), b["dh"].data_ptr(), 256, B, 256, A, accumulate=True)
        L.call("serl_tanh_bwd", b["dh"].data_ptr(), b["h2"].data_ptr(), b["dz2"].data_ptr(), B * 256, L.stream_ptr())
        ops.dense_bwd_weight(ws, b["h1"].data_ptr(), 256, b["dz2"].data_ptr(), 256, P(G, f"{n}/Dense_1/kernel"), B, 256, 256)
        ops.colsum(b["dz2"].data_ptr(), P(G, f"{n}/Dense_1/bias"), 1, B, 256, 256)
        ops.dense_bwd_input(ws, b["dz2"].data_ptr(), 256, P(Pm, f"{n}/Dense_1/kernel"), b["dh"].data_ptr(), 256, B, 256, 256)
        L.call("serl_tanh_bwd", b["dh"].data_ptr(), b["h1"].data_ptr(), b["dz1"].data_ptr(), B * 256, L.stream_ptr())
        ops.dense_bwd_weight(ws, b["X"].data_ptr(), F, b["dz1"].data_ptr(), 256, P(G, f"{n}/Dense_0/kernel"), B, F, 256)
        ops.colsum(b["dz1"].data_ptr(), P(G, f"{n}/Dense_0/bias"), 1, B, 256, 256)
        off = 256 * len(cfg.cams)
        ops.dense_bwd_input(ws, b["dz1"].data_ptr(), 256, P(Pm, f"{n}/Dense_0/kernel") + 4 * off * 256, b["dXp"].data_ptr(), 64, B, 64, 256)
        ops.ln_tanh_bwd(b["dXp"].data_ptr(), 64, ops.at(b["X"], off), F, b["xhat_p"].data_ptr(), b["rstd_p"].data_ptr(), P(Pm, f"{ENC}/LayerNorm_0/scale"), B, 0,
                        b["dzp"].data_ptr(), b["dyp"].data_ptr(), P(G, f"{ENC}/LayerNorm_0/scale"), P(G, f"{ENC}/LayerNorm_0/bias"), B, 64)
        ops.dense_bwd_weight(ws, b["state"].data_ptr(), cfg.state_in, b["dzp"].data_ptr(), 64, P(G, f"{ENC}/Dense_0/kernel"), B, cfg.state_in, 64)
        ops.colsum(b["dzp"].data_ptr(), P(G, f"{ENC}/Dense_0/bias"), 1, B, 64, 64)
        if dist is not None:                                        # jax.lax.pmean(grads_and_aux) (common.py:213-214)
            dist.all_reduce(self._grad, op=dist.ReduceOp.SUM)
            dist.all_reduce(self._info, op=dist.ReduceOp.SUM)
        n_ = self._n
        ops.adam_polyak(self._params, None, self._m, self._v, self._grad, [n_, n_, n_], [1, 0, 0], self._counts, [self.learning_rate] * 3, [0, 0, 0], 0.0, False,
                        lr_out=self._lr_info, n=n_, gap=0, aux=(0, 0, 0))
        self.state.step += 1
        snap = self._info.clone()
        return self, {"actor_loss": snap[0], "mse": snap[1]}

    # ---- inference (bc.py:78-111) ---------------------------------------------------------------------------
    def _dist_params(self, observations):
        single = np.asarray(observations["state"]).ndim == 2
        obs = {k: (np.asarray(v)[None] if single else v) for k, v in observations.items()} if single else observations
        B = int(np.asarray(obs["state"]).shape[0]) if not isinstance(obs["state"], torch.Tensor) else int(obs["state"].shape[0])
        b = self._b(B)
        self._ingest(b, obs)
        self._forward(b, B, train=False, save=False)
        mu = b["mu"].clone()
        std = torch.clamp(torch.exp(b["ls"]), self.std_min, self.std_max)          # thin glue on outputs, not on the hot path
        return mu, std, single

    def sample_actions(self, observations, *, seed=None, temperature: float = 1.0, argmax: bool = False):
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
        out = out.detach().cpu().numpy()
        return out[0] if single else out

    def get_debug_metrics(self, batch, **kwargs):
        if isinstance(batch, BatchHandle):
            batch = batch.to_dict()
        mu, std, _ = self._dist_params(batch["observations"])
        a = (batch["actions"] if isinstance(batch["actions"], torch.Tensor) else torch.as_tensor(np.asarray(batch["actions"]))).to(self.device, f32)
        z = (a - mu) / std
        logp = (-0.5 * z * z - torch.log(std) - 0.918938533204672742).sum(-1)
        return {"mse": ((mu - a) ** 2).sum(-1), "log_probs": logp, "pi_actions": mu}

    def replace(self, **kw):
        if "state" in kw:
            kw.pop("state")
        if kw:
            raise TypeError(f"replace: unknown fields {sorted(kw)}")
        return self
