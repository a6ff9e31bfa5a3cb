"""VICEAgent: DrQ with a success reward learned by a classifier on the frozen ResNet-10 trunk (agents/continuous/vice.py).

    per camera k:  e_k  = tanh(LN(Dense_4096->512(Dropout_0.1(SLE(trunk(image_k))))))     (the agent's own frozen trunk)
    h     = leaky_relu(LN(Dropout_0.1(Dense_{512 ncams}->256(concat_k e_k))))              (MLP([256], activate_final))
    logit = Dense_256->1(h)

`update_vice(batch)` trains it on `batch["next_observations"]`, whose second half holds goal images: mixup of the trunk
features (lam = uniform(key_0), one permutation of the 2B rows), smoothed labels, BCE plus 10 x the gradient penalty
mean((|d logit / d x| - 1)^2) on interpolates of the mixed features.  The penalty's parameter gradient is the reverse-mode
gradient of a forward-mode directional derivative, on the kernels of csrc/vice.cu (see there).  `update_critics` and
`update_high_utd` replace the batch rewards by (sigmoid(logit(next_obs crop)) >= 0.5) from the trunk features the critic step
already computed; `update` does not.  Four Adam txs tick on every update: the SAC step ticks the vice tx with a zero gradient,
`update_vice` ticks the other three.

Randomness (DESIGN.md §4): the key chain of vice.py:370-446 restated step by step (`update_vice_keys`), dropout keys folded as
for the reward classifier: camera j's SLE mask = bernoulli(fold_in(k, j), 0.9), the hidden mask = fold_in(k, ncams); the
penalty's masks are ONE row broadcast over the samples (jax.vmap does not batch the key).

Supported: encoder_type="resnet-pretrained" and the launcher's vice_network_kwargs.  The VICE heads run on the fp32 CUDA-core
GEMMs in every build.  Their parameters live in a `params.FlatParams` store of their own (`agent._vice`, 4 info floats behind its
gradient); the trunk copies of the "modules_vice" subtree are written by `FrozenTrunk.dump`.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from ... import _lib as L
from ... import ops
from ...common.common import TrainState
from ...data.replay_buffer import BatchHandle, DeviceRing, refuse_nstep, refuse_prioritized
from ...params import FlatParams, Leaf, MlpArch, _mlp_leaves, assign_offsets, flatten, image_head_leaves, init_leaves, nest
from .drq import DrQAgent
from .sac import _dist, _host_split, _leaf, register_pytree

f32 = torch.float32
VICE = "modules_vice"
KEEP = 0.9
HIDDEN = 256
BOTTLENECK = 512
GP_WEIGHT = 10.0
LAUNCHER_VICE_NETWORK = {"hidden_dims": [256], "activations": "leaky_relu", "use_layer_norm": True, "dropout_rate": 0.1}


def vice_spec(cams):
    """Trainable leaves of the VICE classifier in the Flax layout (16-byte aligned, one flat buffer)."""
    leaves = [l for cam in cams for l in image_head_leaves(f"{VICE}/encoder/encoder_{cam}", BOTTLENECK)]
    leaves += _mlp_leaves(f"{VICE}/network", BOTTLENECK * len(cams), MlpArch((HIDDEN,), "leaky_relu", True), 0)
    leaves += [Leaf(f"{VICE}/Dense_0/kernel", (HIDDEN, 1), 0), Leaf(f"{VICE}/Dense_0/bias", (1,), 0)]
    return leaves, assign_offsets(leaves)


def trunk_clone_paths(cams):
    """Where the reference's tree holds the VICE module's trunk copies (inferred layout, [3P - verify]): the one shared by
    `update_vice` and one per camera encoder for `vice_reward`.  Both hold the agent's trunk here."""
    return [f"{VICE}/pretrained_encoder"] + [f"{VICE}/encoder/encoder_{cam}/pretrained_encoder" for cam in cams]


def init_vice(rng, spec):
    """xavier_uniform for the MLP's Dense (networks/mlp.py:23), flax's lecun_normal for the encoder heads and the logit Dense."""
    return init_leaves(rng, spec, lambda path: "/network/" in path)


def permutation_rounds(n: int) -> int:
    """Sort rounds of jax's _shuffle for n elements: ceil(3 ln(n) / ln(2^32 - 1))."""
    return int(np.ceil(3 * np.log(max(1, n)) / np.log(np.iinfo(np.uint32).max)))


def update_vice_keys(rng, ncams: int):
    """The key chain of update_vice (vice.py:370-446) and apply_loss_fns' five-way split (common.py:175-203)."""
    rng = np.asarray(rng, np.uint32)
    split = lambda k, n=2: _host_split(k, n)
    k_aug, r = split(rng)
    cams = []
    for _ in range(ncams):
        _k_enc, r = split(r)
        k0, k1, r = split(r, 3)
        k_eps, r = split(r)
        cams.append((k0, k1, k_eps))
    k_drop, r = split(r)
    loss = split(rng, 5)                       # [new rng, actor, critic, temperature, vice] (tree order of the loss dict)
    return dict(aug=k_aug, cams=cams, drop=k_drop, vice=loss[4], final=r)


def check_vice_network_kwargs(nk):
    if nk is None:
        return
    nk = dict(nk)
    nk.pop("activate_final", None)
    act = nk.get("activations", "leaky_relu")
    act = getattr(act, "__name__", act)
    got = {"hidden_dims": [int(h) for h in nk.get("hidden_dims", [256])], "activations": act,
           "use_layer_norm": bool(nk.get("use_layer_norm", True)), "dropout_rate": nk.get("dropout_rate", 0.1)}
    if set(nk) - set(LAUNCHER_VICE_NETWORK) or got != LAUNCHER_VICE_NETWORK:
        raise NotImplementedError(f"vice_network_kwargs={nk}: only the launcher's VICE network {LAUNCHER_VICE_NETWORK} is implemented")


class ViceTrainState(TrainState):
    """TrainState with the "modules_vice" subtree (params, target params) and the fourth Adam state "vice"."""

    def __init__(self, base: TrainState, vice: FlatParams):
        super().__init__(base._store, base._trunk, base._rng, base.step)
        self._vice = vice

    def _with_vice(self, tree, buf):
        flat = flatten(tree)
        flat.update(self._vice.dump(buf))
        cams = tuple(self._trunk.leaves)
        shared, *own = trunk_clone_paths(cams)
        flat.update(self._trunk.dump(lambda cam: shared, cams[:1]))
        flat.update(self._trunk.dump(dict(zip(cams, own)).__getitem__))
        return nest(flat)

    @property
    def params(self):
        return self._with_vice(super().params, self._vice.params)

    @property
    def target_params(self):
        return self._with_vice(super().target_params, self._vice.target)

    @property
    def opt_states(self):
        out = super().opt_states
        vs = self._vice
        vice_mu, vice_nu = nest(vs.dump(vs.m)), nest(vs.dump(vs.v))
        zero = lambda t: {k: (zero(v) if isinstance(v, dict) else np.zeros_like(v)) for k, v in t.items()}
        for name in out:                                      # the SAC txs never see a non-zero vice gradient
            out[name]["mu"][VICE] = zero(vice_mu[VICE])
            out[name]["nu"][VICE] = zero(vice_nu[VICE])
        mu, nu = zero(out["critic"]["mu"]), zero(out["critic"]["nu"])   # the same tree as the other three txs' states
        mu[VICE], nu[VICE] = vice_mu[VICE], vice_nu[VICE]
        out["vice"] = {"count": int(vs.counts[0].item()), "mu": mu, "nu": nu}
        return out

    def replace(self, **kw):
        vs = self._vice
        for key, buf in (("params", vs.params), ("target_params", vs.target)):
            if key in kw:
                vs.load(buf, flatten(kw[key]))
        if "opt_states" in kw:
            o = kw["opt_states"]
            vs.load(vs.m, flatten(o["vice"]["mu"]))
            vs.load(vs.v, flatten(o["vice"]["nu"]))
            vs.counts[0] = int(o["vice"]["count"])
            kw = dict(kw, opt_states={k: v for k, v in o.items() if k != "vice"})
        return super().replace(**kw)


_VICE_NSTEP = "the VICE reward is relabelled per transition from its one-step next observation"


class VICEAgent(DrQAgent):
    # ---- construction ---------------------------------------------------------------------------------------------
    @classmethod
    def create_vice(cls, seed: int, observations, actions, *, encoder_type: str = "small", vice_network_kwargs=None,
                    vice_optimizer_kwargs=None, image_keys=("image",), **kwargs):
        """VICEAgent.create_vice (vice.py:114-330): the DrQ agent of create_drq plus the VICE classifier.  vice_optimizer_kwargs takes
        learning_rate (default 3e-4) and warmup_steps."""
        if encoder_type != "resnet-pretrained":
            raise NotImplementedError(f"VICEAgent: encoder_type={encoder_type!r}: only 'resnet-pretrained' is implemented (the VICE "
                                      "classifier reads the frozen trunk's features)")
        check_vice_network_kwargs(vice_network_kwargs)
        for name in ("critic_network_kwargs", "policy_network_kwargs"):
            rate = (kwargs.get(name) or {}).get("dropout_rate")
            if rate not in (None, 0, 0.0):
                raise NotImplementedError(f"VICEAgent: {name} dropout_rate={rate!r} is not supported (the relabelling and VICE steps "
                                          "run the agent's networks without MLP dropout)")
        ok = dict(vice_optimizer_kwargs or {})
        for k in ("cosine_decay_steps", "clip_grad_norm", "weight_decay", "return_lr_schedule"):
            if ok.get(k) not in (None, False):
                raise NotImplementedError(f"vice_optimizer_kwargs: {k} is not supported for the vice tx")
            ok.pop(k, None)
        unknown = set(ok) - {"learning_rate", "warmup_steps"}
        if unknown:
            raise TypeError(f"vice_optimizer_kwargs: unexpected keys {sorted(unknown)}")
        agent = cls.create_drq(seed, observations, actions, encoder_type=encoder_type, image_keys=image_keys, **kwargs)
        vp = FlatParams(vice_spec(agent._cfg.cams)[0], agent.device, info=4)      # one all-reduce: gradient and infos
        vp.load(vp.params, init_vice(np.random.default_rng([int(seed), 0x51CE]), vp.spec))
        vp.target.copy_(vp.params)
        agent._vice = vp
        agent._vice_lr = float(ok.get("learning_rate", 3e-4))
        agent._vice_warmup = int(ok.get("warmup_steps", 0))
        agent._vice_bufs = {}
        agent._relabel_bufs, agent._infer_vice_bufs = {}, {}
        agent._vice_keys = torch.zeros(64, dtype=torch.uint32, device=agent.device)
        agent._vice_ws = ops.Workspace(64 << 20, agent.device, "f32")
        agent.state = ViceTrainState(agent.state, vp)
        agent.config["vice_image_keys"] = agent._cfg.cams
        return agent

    # ---- the four txs ---------------------------------------------------------------------------------------------
    def _vice_adam(self, live: bool, polyak: bool):
        ops.adam_single(self._vice, self._vice_lr, live, self._vice_warmup, self._cfg.tau, polyak)

    def _update_on_engine(self, eng, nets, pmap_axis=None, schedule_keys=True, want_info=True):
        nets = frozenset(nets) - {"vice"}
        out = super()._update_on_engine(eng, nets, pmap_axis, schedule_keys, want_info)
        self._vice_adam(False, "critic" in nets)            # the vice tx ticks with a zero gradient; polyak maps over the tree
        return out

    def update(self, batch, *, pmap_axis: Optional[str] = None, networks_to_update=frozenset({"actor", "critic", "temperature"})):
        return super().update(batch, pmap_axis=pmap_axis, networks_to_update=frozenset(networks_to_update) - {"vice"})

    # ---- VICE heads -------------------------------------------------------------------------------------------------
    def _heads_fwd(self, s, feats, sle, z1, xhat1, rstd1, X, z2, xhat2, rstd2, h, logit, smask, hmask, R0, R, tangent=False):
        """Rows [R0, R) of the stacked buffers: primal (bias, dropout) or tangent (no bias, the partner's masks, pair_off = R - R0)."""
        vp, cams, ws = self._vice, self._cfg.cams, self._vice_ws
        nc, M = len(cams), R - R0
        F = BOTTLENECK * nc
        for j, cam in enumerate(cams):
            p = f"{VICE}/encoder/encoder_{cam}"
            ops.sle_fwd_multi([(ops.at(feats[j], R0 * 8192), vp.P(f"{p}/SpatialLearnedEmbeddings_0/kernel"),
                                None if smask is None else ops.at(smask[j], R0 * 4096), ops.at(sle[j], R0 * 4096), 4096)], KEEP, M, 16, 512)
            ops.gemm(ws, ops.at(sle[j], R0 * 4096), vp.P(f"{p}/Dense_0/kernel"), ops.at(z1[j], R0 * BOTTLENECK), M, BOTTLENECK, 4096,
                     sAm=4096, sAk=1, sBk=BOTTLENECK, sBn=1, ldc=BOTTLENECK, bias_ptr=None if tangent else vp.P(f"{p}/Dense_0/bias"))
            L.call("serl_vice_ln_act_fwd", z1[j].data_ptr(), BOTTLENECK, None, None, 0, KEEP, vp.P(f"{p}/LayerNorm_0/scale"),
                   vp.P(f"{p}/LayerNorm_0/bias"), ops.at(X, BOTTLENECK * j), F, xhat1[j].data_ptr(), rstd1[j].data_ptr(), None, None, None,
                   R0, R, M if tangent else 0, int(tangent), BOTTLENECK, L.ACT_TANH, 1e-6, L.stream_ptr())
        n = f"{VICE}/network"
        ops.gemm(ws, ops.at(X, R0 * F), vp.P(f"{n}/Dense_0/kernel"), ops.at(z2, R0 * HIDDEN), M, HIDDEN, F, sAm=F, sAk=1, sBk=HIDDEN, sBn=1,
                 ldc=HIDDEN, bias_ptr=None if tangent else vp.P(f"{n}/Dense_0/bias"))
        L.call("serl_vice_ln_act_fwd", z2.data_ptr(), HIDDEN, None, None if hmask is None else hmask.data_ptr(), HIDDEN, KEEP,
               vp.P(f"{n}/LayerNorm_0/scale"), vp.P(f"{n}/LayerNorm_0/bias"), None if h is None else h.data_ptr(), HIDDEN,
               xhat2.data_ptr(), rstd2.data_ptr(), None if tangent else vp.P(f"{VICE}/Dense_0/kernel"),
               None if tangent else vp.P(f"{VICE}/Dense_0/bias"), None if tangent else logit.data_ptr(), R0, R, M if tangent else 0,
               int(tangent), HIDDEN, L.ACT_LEAKY_RELU, 1e-6, L.stream_ptr())

    def _relabel_scratch(self, B, inference=False):
        """Forward scratch of the VICE heads per batch size: the training steps' relabelling, or (inference=True) vice_reward's own,
        so an inference call never touches a step's buffers (a pipelined update_critics uses them on its heads stream)."""
        bufs = self._infer_vice_bufs if inference else self._relabel_bufs
        if B not in bufs:
            nc, dev = len(self._cfg.cams), self.device
            e = lambda *s: torch.empty(*s, dtype=f32, device=dev)
            bufs[B] = dict(sle=[e(B, 4096) for _ in range(nc)], z1=[e(B, BOTTLENECK) for _ in range(nc)],
                                         xhat1=[e(B, BOTTLENECK) for _ in range(nc)], rstd1=[e(B) for _ in range(nc)],
                                         X=e(B, BOTTLENECK * nc), z2=e(B, HIDDEN), xhat2=e(B, HIDDEN), rstd2=e(B), logit=e(B), mean=e(1))
        return bufs[B]

    def _relabel(self, eng):
        """rewards <- (sigmoid(vice(next_obs crop)) >= 0.5) on the next-obs trunk features of the step (rows [B, 2B)), train=False."""
        B = eng.B
        s = self._relabel_scratch(B)
        feats = [eng.feats[cam].view(-1)[B * 8192:] for cam in self._cfg.cams]
        self._heads_fwd(s, feats, s["sle"], s["z1"], s["xhat1"], s["rstd1"], s["X"], s["z2"], s["xhat2"], s["rstd2"], None, s["logit"],
                        None, None, 0, B)
        L.call("serl_vice_reward", s["logit"].data_ptr(), eng.rewards.data_ptr(), s["mean"].data_ptr(), B, 1, L.stream_ptr())

    def update_critics(self, batch, *, pmap_axis: Optional[str] = None):
        refuse_nstep(batch, "VICEAgent.update_critics", _VICE_NSTEP)
        refuse_prioritized(batch, "VICEAgent.update_critics")
        return super().update_critics(batch, pmap_axis=pmap_axis)

    def update_high_utd(self, batch, *, utd_ratio: int, pmap_axis: Optional[str] = None):
        """vice.py:562-610 with the typo fixed: the SAC update is applied (the reference returns the agent it was called on)."""
        refuse_nstep(batch, "VICEAgent.update_high_utd", _VICE_NSTEP)
        refuse_prioritized(batch, "VICEAgent.update_high_utd")
        agent, info = super().update_high_utd(batch, utd_ratio=utd_ratio, pmap_axis=pmap_axis)
        B = batch.batch_size if isinstance(batch, BatchHandle) else int(np.asarray(_leaf(batch, "rewards")).shape[0])
        info["vice_rewards"] = self._relabel_scratch(B)["mean"].clone()[0]
        return agent, info

    def vice_reward(self, observation):
        """sigmoid(logit) of the VICE classifier, train=False: (B,) for a batch of observations, () for one."""
        cams = self._cfg.cams
        img0 = observation[cams[0]]
        img0 = img0 if isinstance(img0, torch.Tensor) else torch.as_tensor(np.asarray(img0))
        single = img0.ndim < 5
        eng, B, _ = self._infer_inputs(observation)
        s = self._relabel_scratch(B, inference=True)
        self._heads_fwd(s, [eng.feats[c].view(-1) for c in cams], s["sle"], s["z1"], s["xhat1"], s["rstd1"], s["X"], s["z2"], s["xhat2"],
                        s["rstd2"], None, s["logit"], None, None, 0, B)
        out = torch.empty(B, dtype=f32, device=self.device)
        L.call("serl_vice_reward", s["logit"].data_ptr(), out.data_ptr(), None, B, 0, L.stream_ptr())
        return out[0] if single else out

    # ---- update_vice ------------------------------------------------------------------------------------------------
    def _vice_scratch(self, B):
        if B not in self._vice_bufs:
            cams, dev = self._cfg.cams, self.device
            nc, N, T = len(cams), 2 * B, 4 * B
            e = lambda *s: torch.empty(*s, dtype=f32, device=dev)
            u8 = lambda *s: torch.empty(*s, dtype=torch.uint8, device=dev)
            self._vice_bufs[B] = dict(
                trunk=self._frozen_trunk.runner(N, dev), pix={c: u8(N, 128, 128, 3) for c in cams}, raw=e(nc, N, 8192),
                fs=e(nc, T, 8192), smask=u8(nc, T, 4096), hmask=u8(T, HIDDEN), sle=[e(T, 4096) for _ in cams],
                z1=[e(T, BOTTLENECK) for _ in cams], xhat1=[e(3 * B, BOTTLENECK) for _ in cams], rstd1=[e(3 * B) for _ in cams],
                X=e(T, BOTTLENECK * nc), z2=e(T, HIDDEN), xhat2=e(3 * B, HIDDEN), rstd2=e(3 * B), h=e(T, HIDDEN), logit=e(3 * B),
                dlogit=e(3 * B), dz2=e(T, HIDDEN), dX=e(T, BOTTLENECK * nc), dz1=e(T, BOTTLENECK), dsle=e(T, 4096), g=e(nc, B, 8192),
                dsc=e(3 * B, BOTTLENECK), dbi=e(3 * B, BOTTLENECK), dw=e(3 * B, HIDDEN), norms=e(nc * B), lam=e(nc),
                perm=torch.empty(nc, N, dtype=torch.int32, device=dev), eps=e(nc, B),
                scratch=dict(pix={c: u8(B, 128, 128, 3) for c in cams}, r=e(B), dones=u8(B), idx=torch.empty(B, dtype=torch.int32, device=dev),
                             status=torch.zeros(1, dtype=torch.int32, device=dev)),
                ident=torch.full((B, 2), 4, dtype=torch.int32, device=dev))
        return self._vice_bufs[B]

    def _vice_pixels(self, b, batch, B):
        """all_pixels of vice.py:392-404 per camera: [goal, goal crop, obs, obs crop] (B/2 rows each) from the next observations;
        crops with split(k_aug, B)[row], the same offsets for every camera."""
        if not isinstance(batch, BatchHandle):
            batch = self._handle_from_dict(batch)
        H = B // 2
        hw = self._cfg.image_hw
        fb = hw * hw * 3
        sc = b["scratch"]
        parts, row = [], 0
        S = max(p["ring"].T * p["ring"].S for p in batch.parts)
        A = max(p["ring"].A for p in batch.parts)
        if sc.get("state") is None or sc["state"].numel() < B * max(S, 1) or sc["actions"].numel() < B * max(A, 1):
            sc["state"] = torch.empty(B * max(S, 1), dtype=f32, device=self.device)      # the sampler's (B, S) / (B, A) rows nobody reads
            sc["actions"] = torch.empty(B * max(A, 1), dtype=f32, device=self.device)
        for part in batch.parts:                              # a dict batch is one part of explicit slots: split it at B/2
            n = part["batch"]
            if row < H < row + n and part.get("indx") is not None:
                c = H - row
                parts += [dict(part, batch=c, indx=part["indx"][:c]), dict(part, batch=n - c, indx=part["indx"][c:])]
            else:
                parts.append(part)
            row += n
        row = 0
        for part in parts:
            ring, n = part["ring"], part["batch"]
            if row < H < row + n:
                raise NotImplementedError("update_vice: a batch part straddles the replay / goal halves; concatenate two halves of B/2")
            goal = row >= H
            for crop in (False, True):
                dest = (0 if not crop else H) if goal else (B if not crop else B + H)
                base = (row - H) if goal else row
                out = L.BatchOut()
                for j, c in enumerate(self._cfg.cams):
                    out.obs_pix[j] = sc["pix"][c].data_ptr() - row * fb
                    out.next_pix[j] = b["pix"][c].data_ptr() + (dest + base - row) * fb
                # every output row r of this launch lands at row r of a (B, width) scratch: the sampler writes row out_row_offset + i
                so = sc["state"].data_ptr() - row * 4 * ring.T * ring.S
                out.obs_state, out.next_state, out.actions = so, so, sc["actions"].data_ptr() - row * 4 * ring.A
                out.rewards = out.masks = sc["r"].data_ptr() - row * 4
                out.dones, out.idx, out.status = sc["dones"].data_ptr() - row, sc["idx"].data_ptr() - row * 4, sc["status"].data_ptr()
                kp = ops.key_ptr(self._vice_keys, 3 * len(self._cfg.cams))
                expl = None if crop else (b["ident"], b["ident"])
                ring.launch_sample(part, out, crop_total=B, out_row_offset=row, key_obs=kp, key_next=kp, explicit_off=expl)
            row += n

    def update_vice(self, batch, *, pmap_axis: Optional[str] = None):
        """vice.py:357-517: one step of the VICE classifier on batch["next_observations"] (second half: goal images)."""
        refuse_nstep(batch, "VICEAgent.update_vice", "the classifier is trained on the one-step next observations")
        refuse_prioritized(batch, "VICEAgent.update_vice")
        B = batch.batch_size if isinstance(batch, BatchHandle) else int(np.asarray(_leaf(batch, "rewards")).shape[0])
        if B % 2 or not 2 <= 2 * B <= 2048:
            raise ValueError(f"update_vice: batch size {B} must be even and at most 1024")
        cams, vp = self._cfg.cams, self._vice
        nc, N, T, F = len(cams), 2 * B, 4 * B, BOTTLENECK * len(cams)
        self._pipe = None
        b = self._vice_scratch(B)
        ks = update_vice_keys(self.state.rng, nc)
        host_keys = np.concatenate([np.concatenate(c) for c in ks["cams"]] + [ks["aug"], ks["drop"], ks["vice"]]).astype(np.uint32)
        self._vice_keys[:host_keys.size].copy_(torch.from_numpy(host_keys.view(np.int32)).view(torch.uint32))
        kp = lambda i: ops.key_ptr(self._vice_keys, i)
        dp = (pmap_axis is not None or self.data_parallel) and _dist() is not None
        gscale = 1.0 / _dist().get_world_size() if dp else 1.0
        # ---- pixels, frozen trunk, draws, mixup and interpolates ----
        self._vice_pixels(b, batch, B)
        for j, cam in enumerate(cams):
            b["trunk"].forward(cam, b["pix"][cam], b["raw"][j].view(N, 4, 4, 512))
        L.call("serl_vice_draws", self._vice_keys.data_ptr(), nc, N, permutation_rounds(N), b["lam"].data_ptr(), b["perm"].data_ptr(),
               b["eps"].data_ptr(), L.stream_ptr())
        L.call("serl_vice_mix", b["raw"].data_ptr(), N * 8192, b["lam"].data_ptr(), b["perm"].data_ptr(), b["eps"].data_ptr(),
               b["fs"].data_ptr(), T * 8192, nc, N, 8192, L.stream_ptr())
        for j in range(nc + 1):                                # keyed masks for the mixup rows, one broadcast row for the penalty
            out, n = (b["smask"][j], 4096) if j < nc else (b["hmask"], HIDDEN)
            L.call("serl_vice_mask_fill", kp(3 * nc + 1), j, KEEP, out.data_ptr(), N, n, 0, L.stream_ptr())
            L.call("serl_vice_mask_fill", kp(3 * nc + 2), j, KEEP, ops.at(out, N * n), N, n, 1, L.stream_ptr())
        fs = [b["fs"][j] for j in range(nc)]
        heads = (b["sle"], b["z1"], b["xhat1"], b["rstd1"], b["X"], b["z2"], b["xhat2"], b["rstd2"], b["h"], b["logit"], b["smask"], b["hmask"])
        self._heads_fwd(b, fs, *heads, 0, 3 * B)
        # ---- BCE of the mixup rows ----
        L.call("serl_vice_bce", b["logit"].data_ptr(), ops.at(b["lam"], nc - 1), ops.at(b["perm"], (nc - 1) * N), gscale,
               b["dlogit"].data_ptr(), vp.info.data_ptr(), N, L.stream_ptr())
        ops.fill(ops.at(b["dlogit"], N), 0.0, B)
        # ---- penalty: input gradient of the interpolate rows (dlogit = 1), norms, v = d gp / d g ----
        ws, st = self._vice_ws, L.stream_ptr()
        n_ = f"{VICE}/network"
        self._ln_bwd(b, L.ACT_LEAKY_RELU, None, 0, None, 1.0, 0.0, b["xhat2"], b["rstd2"], None, b["hmask"], b["h"], b["dz2"],
                     n_, None, N, 3 * B, 0, HIDDEN, head=True)
        ops.dense_bwd_input(ws, ops.at(b["dz2"], N * HIDDEN), HIDDEN, vp.P(f"{n_}/Dense_0/kernel"), ops.at(b["dX"], N * F), F, B, F, HIDDEN)
        for j, cam in enumerate(cams):
            p = f"{VICE}/encoder/encoder_{cam}"
            self._ln_bwd(b, L.ACT_TANH, ops.at(b["dX"], BOTTLENECK * j), F, None, 0.0, 0.0, b["xhat1"][j], b["rstd1"][j], None, None,
                         None, b["dz1"], p, None, N, 3 * B, 0, BOTTLENECK)
            ops.dense_bwd_input(ws, ops.at(b["dz1"], N * BOTTLENECK), BOTTLENECK, vp.P(f"{p}/Dense_0/kernel"), ops.at(b["dsle"], N * 4096),
                                4096, B, 4096, BOTTLENECK)
            ops.dropout_bwd(ops.at(b["dsle"], N * 4096), ops.at(b["smask"][j], N * 4096), KEEP, B * 4096)
            L.call("serl_vice_sle_input_grad", ops.at(b["dsle"], N * 4096), 4096, vp.P(f"{p}/SpatialLearnedEmbeddings_0/kernel"),
                   b["g"][j].data_ptr(), B, 16, 512, st)
        L.call("serl_vice_gp_rows", b["g"].data_ptr(), B * 8192, ops.at(b["fs"], 3 * B * 8192), T * 8192,
               GP_WEIGHT * 2.0 / (nc * B) * gscale, b["norms"].data_ptr(), nc, B, 8192, st)
        L.call("serl_vice_gp_finish", b["norms"].data_ptr(), nc * B, GP_WEIGHT, gscale, vp.info.data_ptr(), st)
        # ---- tangent forward of the penalty rows, then ONE reverse pass over all 4B rows ----
        self._heads_fwd(b, fs, *heads, 3 * B, T, tangent=True)
        self._ln_bwd(b, L.ACT_LEAKY_RELU, None, 0, b["dlogit"], 0.0, 1.0, b["xhat2"], b["rstd2"], b["z2"], b["hmask"], b["h"], b["dz2"],
                     n_, vp, 0, 3 * B, B, HIDDEN, head=True)
        ops.dense_bwd_weight(ws, b["X"].data_ptr(), F, b["dz2"].data_ptr(), HIDDEN, vp.G(f"{n_}/Dense_0/kernel"), T, F, HIDDEN)
        ops.colsum(b["dz2"].data_ptr(), vp.G(f"{n_}/Dense_0/bias"), 1, 3 * B, HIDDEN, HIDDEN)
        ops.colsum(b["dw"].data_ptr(), vp.G(f"{VICE}/Dense_0/kernel"), 1, 3 * B, HIDDEN, HIDDEN)
        ops.colsum(b["dlogit"].data_ptr(), vp.G(f"{VICE}/Dense_0/bias"), 1, 3 * B, 1, 1)
        ops.dense_bwd_input(ws, b["dz2"].data_ptr(), HIDDEN, vp.P(f"{n_}/Dense_0/kernel"), b["dX"].data_ptr(), F, T, F, HIDDEN)
        for j, cam in enumerate(cams):
            p = f"{VICE}/encoder/encoder_{cam}"
            self._ln_bwd(b, L.ACT_TANH, ops.at(b["dX"], BOTTLENECK * j), F, None, 0.0, 0.0, b["xhat1"][j], b["rstd1"][j], b["z1"][j], None,
                         None, b["dz1"], p, vp, 0, 3 * B, B, BOTTLENECK)
            ops.dense_bwd_weight(ws, b["sle"][j].data_ptr(), 4096, b["dz1"].data_ptr(), BOTTLENECK, vp.G(f"{p}/Dense_0/kernel"), T, 4096, BOTTLENECK)
            ops.colsum(b["dz1"].data_ptr(), vp.G(f"{p}/Dense_0/bias"), 1, 3 * B, BOTTLENECK, BOTTLENECK)
            ops.dense_bwd_input(ws, b["dz1"].data_ptr(), BOTTLENECK, vp.P(f"{p}/Dense_0/kernel"), b["dsle"].data_ptr(), 4096, T, 4096, BOTTLENECK)
            ops.dropout_bwd(b["dsle"].data_ptr(), b["smask"][j].data_ptr(), KEEP, T * 4096)
            ops.sle_bwd_multi(ws, [(fs[j].data_ptr(), b["dsle"].data_ptr(), 4096, vp.G(f"{p}/SpatialLearnedEmbeddings_0/kernel"))], T, 16, 512)
        # ---- one all-reduce (gradient + infos), the four txs, the key chain ----
        if dp:
            _dist().all_reduce(vp.grad_info, op=_dist().ReduceOp.SUM)
        self._vice_adam(True, False)
        # actor / critic / temperature txs tick with zero gradients: any engine's optimizer step (they share the flat buffers)
        eng = next(iter(self._engines.values()), None) or self._engine(B)
        eng.optimizer_step([0, 0, 0], polyak=False)
        self.state.step += 1
        # the key chain moves on the device only: a rng write through TrainState.replace would mark the parameters as written
        # from outside and drop every captured step graph (the step pipeline's stale prefetch is already dropped above)
        self.state._rng.copy_(torch.from_numpy(np.ascontiguousarray(ks["final"], np.uint32).view(np.int32)).view(torch.uint32))
        snap = vp.info.clone()
        return self, {"actor": {}, "critic": {}, "temperature": {}, "vice": {"bce_loss": snap[0], "grad_norm": snap[1]}}

    def _ln_bwd(self, b, act, dy, ld_dy, dlogit, dlogit_const, tan_seed, xhat, rstd, z, mask, y, dz, prefix, vp, R0, R, R_pair, D, head=False):
        """serl_vice_ln_act_bwd; with vp the scale / bias (and head kernel) gradients of `prefix` are column sums of the row terms."""
        v = self._vice
        L.call("serl_vice_ln_act_bwd", dy, ld_dy, None if dlogit is None else dlogit.data_ptr(), float(dlogit_const),
               v.P(f"{VICE}/Dense_0/kernel") if head else None, float(tan_seed), xhat.data_ptr(), rstd.data_ptr(),
               None if z is None else z.data_ptr(), D, None if mask is None else mask.data_ptr(), D, KEEP, v.P(f"{prefix}/LayerNorm_0/scale"),
               v.P(f"{prefix}/LayerNorm_0/bias"), None if y is None else y.data_ptr(), D, dz.data_ptr(), D,
               b["dsc"].data_ptr() if vp else None, b["dbi"].data_ptr() if vp else None, b["dw"].data_ptr() if (vp and head) else None,
               R0, R, R_pair, D, act, L.stream_ptr())
        if vp is not None:
            ops.colsum(b["dsc"].data_ptr(), v.G(f"{prefix}/LayerNorm_0/scale"), 1, R, D, D)
            ops.colsum(b["dbi"].data_ptr(), v.G(f"{prefix}/LayerNorm_0/bias"), 1, R, D, D)


register_pytree(VICEAgent)
