"""SACAgent on hand-written sm_90a kernels.

Mirrors the public surface of the reference's `SACAgent` (agents/continuous/sac.py:21-596):
`create_states` / `create_pixels`-style construction, `update(batch, pmap_axis, networks_to_update)`,
`update_high_utd(batch, utd_ratio)`, `sample_actions(observations, seed, argmax)`, the forward methods (`forward_critic`,
`forward_target_critic`, `forward_policy`, `forward_temperature`, `temperature_lagrange_penalty`; sac.py:33-116), `state`,
`config`, `replace(state=...)`.  Calls return `(agent, info)` like the reference (the agent is updated in place:
its parameters live in HBM).  `info` leaves are 0-d device tensors; `float(x)` synchronises.

Semantics reproduced (SURVEY.md Appendix A): ensemble subsample with replacement + min for the TD
target, mean over the ensemble in the actor loss, shared value head for the pixel agent, same key for
dropout and action sampling in `_compute_next_actions`, ALL three Adam txs tick on every `update`
(zero-gradient momentum drift), polyak over the whole tree after critic updates, JAX key chain.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, FrozenSet, Optional, Sequence

import numpy as np
import torch

from ... import _lib as L
from ... import ops
from ...common.common import TrainState
from ...data.replay_buffer import BatchHandle, is_prioritized
from ...engine import STD_IDS, AgentConfig, Engine, InferenceEngine
from ...params import (LAUNCHER_MLP, STD_PARAMETERIZATIONS, MlpArch, ParamStore, init_trainable, init_trunk, trainable_spec,
                       trunk_spec)
from ...step_graphs import StepGraphs
from ...trunk import FrozenTrunk

ALL_NETS = frozenset({"actor", "critic", "temperature"})


def _dist():
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            return dist
    except Exception:                                   # noqa: BLE001
        pass
    return None


class SACAgent:
    def __init__(self, cfg: AgentConfig, store: ParamStore, trunk: Optional[FrozenTrunk], state: TrainState, config: dict, device):
        self._cfg, self._store, self.state, self.config, self.device = cfg, store, state, config, device
        # the frozen ResNet-10 of a "resnet-pretrained" pixel agent; the small encoder's convs are trainable leaves of the store
        self._frozen_trunk = trunk
        self._trunk = trunk.leaves if trunk is not None else {}
        self._engines: Dict[int, Engine] = {}
        # sample_actions and the forward_* methods run on engines of their own: a training engine's buffers may hold the batch,
        # crops and features of a step that is still to come (the cross-step pipeline's prefetch)
        self._infer_engines: Dict[int, InferenceEngine] = {}
        # an agent with MLP dropout also keeps the critic-MLP keys (ops.rng_schedule(mlp_dropout=True)) past the NUM_KEYS slots
        self._keys = torch.zeros(2 * (L.NUM_KEYS_MLP if cfg.mlp_dropout else L.NUM_KEYS), dtype=torch.uint32, device=device)
        self._seed_key = torch.zeros(2, dtype=torch.uint32, device=device)
        self._fwd_key = torch.zeros(2, dtype=torch.uint32, device=device)
        self.data_parallel = False          # set True to all-reduce(mean) gradients + infos (reference: pmap_axis)
        self.explicit_randomness = None     # tests: dict with eps / dropout / subsample (and crop offsets)
        self.use_cuda_graphs = True         # replay the whole step as one CUDA graph from its 2nd identical call on
        self.section_events = None          # bench: list collecting (name, start event, end event) of eagerly launched steps
        # Cross-step pipeline (DrQ pixel agent, opt-in): the frozen encoder of step i+1 does not depend on the parameters step i
        # updates, so `update_critics` can run sampler + trunk of the NEXT sequential batch next to the heads / Adam of the current
        # one (drq.py::_update_critics_pipelined).  The next batch is then drawn one call early - like the reference iterator's
        # `queue_size=2` prefetch (data/replay_buffer.py:77-90) - and a call that does not continue the sequence falls back.
        self.pipeline_critic_steps = False
        self._pipe = None
        self._eng_pair: Dict[int, list] = {}
        self._keys_pair = [self._keys, torch.zeros_like(self._keys)]
        self._rng_look = torch.zeros(2, dtype=torch.uint32, device=device)
        self._pipe_stream = None
        self._last_engine = None
        self._graphs = StepGraphs()
        self._graphs_version = store.version   # captured graphs bake parameter-derived state (packed trunk weights, stem sign mask)

    # ---- construction (sac.py:322-400,486-542) ------------------------------------------------------
    @classmethod
    def _build(cls, seed: int, cfg: AgentConfig, temperature_init: float, device, in_channels: int = 3, config_extra=None):
        L.load()
        device = torch.device(device if device is not None else "cuda")
        L.require_cuda(device)
        rng = np.random.default_rng(seed)
        spec = trainable_spec(cfg.cams, cfg.state_in, cfg.action_dim, cfg.ensemble, cfg.pixel, cfg.critic_arch, cfg.policy_arch,
                              cfg.std_parameterization, cfg.use_proprio, cfg.encoder, in_channels=cfg.in_channels)
        store = ParamStore(spec, device)
        values = init_trainable(rng, spec, temperature_init)
        store.load(store.params, values)
        store.target.copy_(store.params)                               # target_params=params (sac.py:369)
        trunk = {}
        if cfg.pixel and not cfg.trainable_encoder:
            for cam in cfg.cams:
                w = init_trunk(rng, in_channels)
                trunk[cam] = {k: torch.as_tensor(v).to(device).contiguous() for k, v in w.items()}
        # rng, init_rng = split(PRNGKey(seed)); rng, create_rng = split(rng)  (sac.py:360,368): state.rng = create_rng
        key = np.array([(seed >> 32) & 0xFFFFFFFF, seed & 0xFFFFFFFF], dtype=np.uint32)
        key = _host_split(key, 2)[0]
        create = _host_split(key, 2)[1]
        rng_dev = torch.zeros(2, dtype=torch.uint32, device=device)
        trunk = None if cfg.trainable_encoder else FrozenTrunk(trunk, cfg.precision, cfg.image_hw)
        state = TrainState(store, trunk, rng_dev)
        state.replace(rng=create)
        config = dict(critic_ensemble_size=cfg.ensemble, critic_subsample_size=cfg.subsample, discount=cfg.discount,
                      soft_target_update_rate=cfg.tau, target_entropy=cfg.target_entropy, backup_entropy=cfg.backup_entropy)
        config.update(config_extra or {})
        return cls(cfg, store, trunk, state, config, device)

    @classmethod
    def create_states(cls, seed: int, observations, actions, *, discount=0.95, critic_ensemble_size=2,
                      critic_subsample_size=None, temperature_init=1.0, backup_entropy=False, soft_target_update_rate=0.005,
                      target_entropy=None, policy_kwargs=None, actor_warmup=None, critic_warmup=None, learning_rate=None,
                      actor_optimizer_kwargs=None, critic_optimizer_kwargs=None, temperature_optimizer_kwargs=None,
                      device=None, **kwargs):
        """State-observation agent (sac.py:486-542).  Optimizer defaults follow SACAgent.create (:333-343): lr 3e-4 and a
        2000-step linear warm-up for actor and critic.  `*_optimizer_kwargs` take make_optimizer's learning_rate,
        warmup_steps, cosine_decay_steps and clip_grad_norm (see `optimizer_settings`); `critic_network_kwargs`,
        `policy_network_kwargs` and policy_kwargs["std_parameterization"] choose the networks (see `architecture_settings`)."""
        arch = architecture_settings(policy_kwargs, kwargs, pixel=False, allow_dropout=True)
        opt = optimizer_settings({"critic": critic_optimizer_kwargs, "actor": actor_optimizer_kwargs, "temperature": temperature_optimizer_kwargs},
                                 learning_rate, {"critic": critic_warmup, "actor": actor_warmup},
                                 {"critic": 2000, "actor": 2000, "temperature": 0})
        pk = policy_kwargs or {}
        S = int(np.asarray(observations).shape[-1])
        A = int(np.asarray(actions).shape[-1])
        cfg = AgentConfig(cams=(), state_in=S, action_dim=A, pixel=False, ensemble=critic_ensemble_size,
                          subsample=critic_subsample_size, discount=discount, tau=soft_target_update_rate,
                          target_entropy=(-A / 2 if target_entropy is None else target_entropy), backup_entropy=backup_entropy,
                          **opt, **arch, std_min=pk.get("std_min", 1e-5), std_max=pk.get("std_max", 10.0))
        return cls._build(seed, cfg, temperature_init, device)

    def replace(self, **kw):
        if "state" in kw:
            self.state = kw.pop("state")
            self.invalidate_graphs()
        if kw:
            raise TypeError(f"replace: unknown fields {sorted(kw)}")
        return self

    def invalidate_graphs(self):
        """Drops every captured CUDA graph (and the packed 16-bit trunk weights derived from the fp32 ones): called when
        parameters were written from outside the step (`state.replace(params=...)`, checkpoint restore)."""
        self._graphs.clear()
        self._pipe = None
        self._graphs_version = self._store.version
        if self._frozen_trunk is not None:
            self._frozen_trunk.drop_packed()

    # ---- engines ---------------------------------------------------------------------------------
    def _engine(self, B: int) -> Engine:
        if B not in self._engines:
            self._engines[B] = Engine(self._cfg, self._store, self._frozen_trunk, B, self.device)
        return self._engines[B]

    def _infer_engine(self, B: int) -> InferenceEngine:
        if B not in self._infer_engines:
            self._infer_engines[B] = InferenceEngine(self._cfg, self._store, self._frozen_trunk, B, self.device)
        return self._infer_engines[B]

    @property
    def kernel_launches(self) -> int:
        """Kernels of libserl_b200 executed so far in this process: the library's own launch counter, minus launches that
        were only recorded during graph capture, plus the recorded count for every replay."""
        return L.launch_count() + self._graphs.launch_adj

    # ---- CUDA graphs: the ~150 launches of a step are captured once and replayed -------------------------
    def _check_nstep(self, batch):
        """An n-step handle (sample_args n_step > 1) must be drawn with this agent's discount: the critic target
        R + discount * masks * min Q(s') is then the n-step target, because the sampler folds discount^(m-1) into masks."""
        if not isinstance(batch, BatchHandle):
            return
        if is_prioritized(batch) and self.data_parallel and _dist() is not None:
            raise NotImplementedError("prioritized replay under data parallelism: each rank's written priorities would have to "
                                      "reach every replica")
        n_step, discount = batch.n_step
        if n_step == 1:
            return
        if discount != float(self.config["discount"]):
            raise ValueError(f"batch drawn with n_step={n_step}, discount={discount}; the agent's discount is {self.config['discount']}")
        if self.config["backup_entropy"]:
            raise NotImplementedError("backup_entropy=True with n_step > 1: the entropy backup subtracts alpha * log pi(a'|s') "
                                      "undiscounted at the one-step next observation; an n-step version would be a new definition")

    def _graph_key(self, tag, batch):
        """Batches that can be replayed: lazy handles whose index draw reads the ring's device-resident counters.  The n-step
        setting is part of the key (a captured sampler launch bakes it in)."""
        self._check_nstep(batch)
        if not self.use_cuda_graphs or self.explicit_randomness is not None or not isinstance(batch, BatchHandle):
            return None
        if torch.device(self.device).type != "cuda":            # host-logic dry runs (tests) have nothing to capture
            return None
        if any(p.get("indx") is not None for p in batch.parts):
            return None
        return (tag, batch.batch_size, tuple((id(p["ring"]), p["batch"]) for p in batch.parts), batch.n_step)

    def _run_step(self, key, batch, body):
        """body(graph_mode) enqueues one step on `batch`, through the step-graph cache (StepGraphs.run)."""
        if self._graphs_version != self._store.version:          # TrainState.replace(params=...) since the last capture
            self.invalidate_graphs()
        self._pipe = None                                        # any step outside the pipelined path consumes the key chain: prefetch is stale
        self._keys = self._keys_pair[0]
        draws = [(p["ring"], p["step"], 1) for p in batch.parts] if key is not None else []
        self._graphs.run(key, draws, body, self.state)

    # ---- batch ingestion -------------------------------------------------------------------------------
    def _load_batch(self, eng: Engine, batch, *, augment: bool, keys, graph_mode: bool = False) -> None:
        """Fills the engine's batch buffers.  Pixel agents: obs crops to pix rows [0,B), next crops to [B,2B), the T frames of a
        stack on the channel axis (the sampler's stacked layout), one crop per frame.  Parts drawn with n_step > 1 are gathered by
        the n-step sampler (ring.launch_sample)."""
        cfg, B = self._cfg, eng.B
        if not isinstance(batch, BatchHandle):
            batch = self._handle_from_dict(batch)
        self._check_nstep(batch)
        if batch.batch_size != B:
            raise ValueError(f"batch size {batch.batch_size} != engine batch {B}")
        out = L.BatchOut()
        T = cfg.obs_horizon if cfg.pixel else 1
        if cfg.pixel:
            hw = cfg.image_hw
            for j, cam in enumerate(cfg.cams):
                out.obs_pix[j] = eng.pix[cam].data_ptr()
                out.next_pix[j] = eng.pix[cam].data_ptr() + B * hw * hw * cfg.in_channels
            out.off_obs, out.off_next = eng.off[0].data_ptr(), eng.off[1].data_ptr()
            out.stacked = 1
        out.obs_state, out.next_state, out.actions = eng.state_o.data_ptr(), eng.state_n.data_ptr(), eng.actions.data_ptr()
        out.rewards, out.masks, out.dones = eng.rewards.data_ptr(), eng.masks.data_ptr(), eng.dones.data_ptr()
        out.idx, out.status = eng.idx.data_ptr(), eng.status.data_ptr()
        expl = None
        if self.explicit_randomness is not None and "crop" in self.explicit_randomness:
            expl = tuple(torch.as_tensor(np.asarray(o), dtype=torch.int32, device=self.device).contiguous()
                         for o in self.explicit_randomness["crop"])
        elif not augment or not cfg.pixel:
            ident = torch.full((B * T, 2), 4, dtype=torch.int32, device=self.device)
            expl = (ident, ident)
        row = 0
        # prioritized parts: each row's priority, then the part's importance weights; rows of uniform parts weigh 1
        eng.prio_parts = [(p["ring"], r, p["batch"]) for p, r in zip(batch.parts, np.cumsum([0] + [q["batch"] for q in batch.parts]))
                          if p["ring"].prioritized]
        for ring, r, n in eng.prio_parts:
            if n > L.PRIO_SET_MAX:
                raise ValueError(f"a prioritized part of {n} rows: at most {L.PRIO_SET_MAX} rows write their priorities back in one step")
        if eng.prio_parts and len(eng.prio_parts) < len(batch.parts):
            ops.fill(eng.weights.data_ptr(), 1.0, B)
        # RLPD (concat_batches of an online and a demo handle): the parts gather disjoint output rows from different rings, so the
        # second part's launch runs on side stream 0 next to the first (each launch alone is one partial wave of CTAs: latency-bound)
        side = eng.side[0] if (graph_mode and len(batch.parts) == 2 and batch.parts[0]["ring"] is not batch.parts[1]["ring"]) else None
        for pi, part in enumerate(batch.parts):
            ring = part["ring"]
            if cfg.pixel and ring.T != T:
                if T == 1:
                    raise NotImplementedError("the trunk kernels take one frame per observation (obs_horizon=1), like every SERL example")
                raise ValueError(f"the agent takes stacks of {T} frames (obs_horizon={T}), the replay buffer stores {ring.T}")
            on_side = side is not None and pi == 1
            out.obs_state, out.next_state = self._state_outputs(eng, ring)
            if on_side:
                side.fork()
                side.__enter__()
            try:
                ring.launch_sample(part, out, crop_total=B * T, out_row_offset=row, key_obs=ops.key_ptr(keys, L.KEY_CROP_OBS),
                                   key_next=ops.key_ptr(keys, L.KEY_CROP_NEXT), explicit_off=expl,
                                   step_dev=ring.step_dev if graph_mode else None, record_event=not graph_mode,
                                   prio_out=eng.prio if ring.prioritized else None)
                if ring.prioritized:                                       # weights normalised over this part's rows
                    n = part["batch"]
                    ops.priority_weights(eng.prio[row:row + n], n, ring.beta_dev, eng.weights[row:row + n])
                if graph_mode:
                    ops.counter_add(ring.step_dev, 1)
            finally:
                if on_side:
                    side.__exit__(None, None, None)
            row += part["batch"]
        if side is not None:
            side.join()

    def _state_outputs(self, eng: Engine, ring):
        """Where the sampler writes a part's (obs, next obs) state rows.  A pixel-only agent has no state input: the rows of a
        ring that stores a state vector go to per-engine scratch nobody reads (a ring without one writes nothing)."""
        cfg = self._cfg
        n = ring.T * ring.S
        if cfg.proprio and n != cfg.state_in:
            raise ValueError(f"the agent's proprio encoder takes {cfg.state_in} state inputs, the replay buffer stores {n} per sample")
        if cfg.use_proprio or not cfg.pixel or n == 0:             # proprio and state agents read the rows
            return eng.state_o.data_ptr(), eng.state_n.data_ptr()
        sink_o, sink_n = eng.state_sink(n)
        return sink_o.data_ptr(), sink_n.data_ptr()

    def _handle_from_dict(self, batch: dict) -> BatchHandle:
        """Host / device dict in the reference layout -> a temporary HBM ring + explicit indices."""
        from ...data.replay_buffer import DeviceRing
        cfg = self._cfg
        dev = self.device
        t = lambda x, dt=torch.float32: torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x).to(dev, dt)
        B = int(t(batch["rewards"]).shape[0])
        if cfg.pixel:
            # row b's T + 1 frames (its obs stack, then the next observation's newest frame) fill slots b(T+1) .. b(T+1)+T; slot
            # b(T+1)+T is the row's drawn slot, whose window is the obs stack and, shifted by one, the next-obs stack
            obs, nobs = batch["observations"], batch["next_observations"]
            T = cfg.obs_horizon
            ring = DeviceRing(B * (T + 1), cfg.cams, (cfg.image_hw, cfg.image_hw, 3), T, cfg.state_in // T, cfg.action_dim, device=dev,
                              seed=0)
            for cam in cfg.cams:
                pix = t(obs[cam], torch.uint8)
                if cam in nobs:
                    npix = t(nobs[cam], torch.uint8)
                    if T > 1 and not torch.equal(npix[:, :-1], pix[:, 1:]):
                        raise ValueError(f"dict batches: next_observations[{cam!r}] must be observations[{cam!r}] shifted by one frame "
                                         "(ChunkingWrapper stacks)")
                    pix = torch.cat([pix, npix[:, -1:]], dim=1)
                if pix.shape[1] != T + 1:
                    if T == 1:
                        raise NotImplementedError("dict batches: obs_horizon must be 1")
                    raise ValueError(f"dict batches: {cam!r} frames of shape {tuple(pix.shape)}; expected (B, {T}, H, W, C) "
                                     f"observations and next_observations, or packed (B, {T + 1}, H, W, C)")
                ring.frames[cam].copy_(pix.reshape(B * (T + 1), *pix.shape[2:]))
            sl = slice(T, None, T + 1)
            if cfg.state_in:                                      # (a pixel-only agent ignores a "state" entry)
                ring.state[sl] = t(obs["state"]).reshape(B, -1)
                ring.next_state[sl] = t(nobs["state"]).reshape(B, -1)
            idx = torch.arange(B, device=dev, dtype=torch.int32) * (T + 1) + T
        else:
            ring = DeviceRing(B, (), (1, 1, 1), 1, cfg.state_in, cfg.action_dim, device=dev, seed=0)
            sl = slice(None)
            ring.state[sl] = t(batch["observations"]).reshape(B, -1)
            ring.next_state[sl] = t(batch["next_observations"]).reshape(B, -1)
            idx = torch.arange(B, device=dev, dtype=torch.int32)
        ring.actions[sl] = t(batch["actions"]).reshape(B, -1)
        ring.rewards[sl] = t(batch["rewards"])
        ring.masks[sl] = t(batch["masks"])
        ring.dones[sl] = t(batch["dones"], torch.uint8) if "dones" in batch else 0
        ring.valid.fill_(1)
        ring._size = ring._capacity
        ring.size_dev.fill_(ring._size)
        return BatchHandle([dict(ring=ring, seed=0, step=0, batch=B, indx=idx)], True)

    # ---- update (sac.py:243-299) ------------------------------------------------------------------------
    def _section(self, name):
        """Context manager timing one section of an EAGER step with CUDA events (bench.py's per-section timeline); no-op otherwise."""
        import contextlib
        if self.section_events is None or torch.cuda.is_current_stream_capturing():
            return contextlib.nullcontext()

        @contextlib.contextmanager
        def cm():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            try:
                yield
            finally:
                b.record()
                self.section_events.append((name, a, b))
        return cm()

    def _features(self, eng: Engine):
        """The frozen trunk's features of the step's crops.  A trainable encoder has no frozen part: its convs run inside
        Engine.encode, on the parameters of the moment (after the previous minibatch's Adam in update_high_utd, and never
        ahead of the current step in the cross-step pipeline, which then prefetches only the sampler's crops)."""
        if not self._cfg.pixel or self._cfg.trainable_encoder:
            return
        cams = self._cfg.cams
        # cameras 1.. first, each on its own stream (fork / join = graph edges), then camera 0 on the current stream.  The fp32
        # build shares its activation scratch between cameras and stays serial.
        side = [c for c in cams if eng.cam_stream.get(c) is not None and self._cfg.precision != "fp32"]
        for cam in side:
            cs = eng.cam_stream[cam]
            cs.fork()
            with cs:
                eng.trunk_forward(cam, eng.pix[cam], eng.feats[cam])
        for cam in cams:
            if cam not in side:
                eng.trunk_forward(cam, eng.pix[cam], eng.feats[cam])
        for cam in side:
            eng.cam_stream[cam].join()

    def _relabel(self, eng: Engine):
        """Hook between the frozen trunk and the losses of update_critics / update_high_utd: VICEAgent rewrites the batch rewards."""

    def _dp(self, pmap_axis) -> bool:
        """ONE predicate for both halves of the data-parallel exchange (1/world pre-scaling in the loss kernels and the SUM
        all-reduce): the reference's `pmap_axis is not None`, or the `data_parallel` switch, in a multi-rank job."""
        return (pmap_axis is not None or self.data_parallel) and _dist() is not None

    def _allreduce(self, lo: int, hi: int):
        """jax.lax.pmean(grads_and_aux) (common.py:213-214) as ONE collective: the loss kernels scale gradients AND info
        scalars by 1/world, and the infos sit inside the flat gradient buffer next to the segment they belong to
        (params.py), so a single SUM all-reduce of [lo, hi) yields the mean of both."""
        _dist().all_reduce(self._store.grad[lo:hi], op=_dist().ReduceOp.SUM)

    def _update_on_engine(self, eng: Engine, nets: FrozenSet[str], pmap_axis=None, schedule_keys: bool = True, want_info: bool = True):
        assert nets.issubset(ALL_NETS), f"Invalid gradient steps: {nets}"
        if schedule_keys:
            ops.rng_schedule(self.state._rng, self._keys, False, True, mlp_dropout=self._cfg.mlp_dropout)
        expl = self.explicit_randomness
        st = self._store
        dp = self._dp(pmap_axis)
        gscale = 1.0 / _dist().get_world_size() if dp else 1.0
        at = "actor" in nets or "temperature" in nets
        with self._section("heads"):
            if "critic" in nets:
                eng.critic_loss_and_grads(self._keys, grad_scale=gscale, explicit=expl)
                for ring, r, n in eng.prio_parts:                          # TD errors -> the priorities of the slots drawn
                    ops.priority_set(ring.priority_tree(), eng.idx[r:], n, td=eng.delta[r:], alpha=ring.priority_alpha,
                                     eps=ring.priority_eps)
            if at:
                # any subset is legal (sac.py:270-277): a network that is not updated contributes a zero gradient, its tx still ticks
                eng.actor_temp_loss_and_grads(self._keys, grad_scale=gscale, explicit=expl, do_actor="actor" in nets,
                                              do_temperature="temperature" in nets)
        if dp and nets:
            # [group 0 | critic infos] and/or [actor, temperature infos | groups 1, 2 | aux]: one contiguous range either way
            with self._section("allreduce"):
                self._allreduce(0 if "critic" in nets else st.info_off + 4, st.n if at else st.info_off + 4)
        with self._section("adam_polyak"):
            eng.optimizer_step([int("critic" in nets), int("actor" in nets), int("temperature" in nets)], polyak="critic" in nets)
        self.state.step += 1
        return self._info(eng, nets) if want_info else None

    def _info(self, eng: Engine, nets) -> dict:
        snap = torch.cat([eng.info[:12], eng.lr_info])
        info = {"critic": {}, "actor": {}, "temperature": {}}
        if "critic" in nets:
            info["critic"] = {"critic_loss": snap[0], "predicted_qs": snap[1], "target_qs": snap[2]}
        if "actor" in nets:
            info["actor"] = {"actor_loss": snap[4], "temperature": snap[5], "entropy": snap[6]}
        if "temperature" in nets:
            info["temperature"] = {"temperature_loss": snap[8]}
        info["critic_lr"], info["actor_lr"], info["temperature_lr"] = snap[12], snap[13], snap[14]   # sac.py:292-297
        return info

    def update(self, batch, *, pmap_axis: Optional[str] = None, networks_to_update: FrozenSet[str] = ALL_NETS):
        """One gradient step on all (or a subset of) the networks (sac.py:243-299)."""
        nets = frozenset(networks_to_update)
        B = batch.batch_size if isinstance(batch, BatchHandle) else int(np.asarray(_leaf(batch, "rewards")).shape[0])
        eng = self._engine(B)

        def body(graph_mode):
            ops.rng_schedule(self.state._rng, self._keys, False, True, mlp_dropout=self._cfg.mlp_dropout)
            self._load_batch(eng, batch, augment=False, keys=self._keys, graph_mode=graph_mode)
            self._features(eng)
            self._update_on_engine(eng, nets, pmap_axis, schedule_keys=False, want_info=False)

        self._run_step(self._graph_key(("update", tuple(sorted(nets)), pmap_axis), batch), batch, body)
        return self, self._info(eng, nets)

    def _check(self, eng: Engine):
        pass   # draw failures are surfaced lazily by check_status() to avoid a sync per step

    def check_status(self):
        for eng in list(self._engines.values()) + [pair[1] for pair in self._eng_pair.values()]:
            if int(eng.status.item()):
                raise L.SerlError("replay draw failed: no valid slot within the redraw budget")
            if getattr(eng, "fused", None) is not None:
                eng.fused.check_error()
        if self._frozen_trunk is not None:
            self._frozen_trunk.check_error()

    def update_high_utd(self, batch, *, utd_ratio: int, pmap_axis: Optional[str] = None, _augment: bool = False):
        """sac.py:544-596: utd_ratio critic updates on consecutive minibatches, then one actor+temperature update
        on the full batch."""
        self._pipe, self._keys = None, self._keys_pair[0]          # consumes the key chain: a prefetched next batch is stale
        B = batch.batch_size if isinstance(batch, BatchHandle) else int(np.asarray(_leaf(batch, "rewards")).shape[0])
        assert B % utd_ratio == 0, f"Batch size {B} must be divisible by UTD ratio {utd_ratio}"
        full = self._engine(B)
        mb = B // utd_ratio
        if utd_ratio == 1:                                         # the DrQ learner's case: one graph for the whole call
            def body(graph_mode):
                if _augment:
                    ops.rng_schedule(self.state._rng, self._keys, True, False)      # drq.py:279
                self._load_batch(full, batch, augment=_augment, keys=self._keys, graph_mode=graph_mode)
                self._features(full)
                self._relabel(full)
                self._update_on_engine(full, frozenset({"critic"}), pmap_axis, want_info=False)
                full.info_hist.copy_(full.info)                                      # critic infos of the scan step
                self._update_on_engine(full, frozenset({"actor", "temperature"}), pmap_axis, want_info=False)

            self._run_step(self._graph_key(("high_utd", _augment, pmap_axis), batch), batch, body)
            at = self._info(full, frozenset({"actor", "temperature"}))
            snap = full.info_hist.clone()
            info = {"critic": {"critic_loss": snap[0], "predicted_qs": snap[1], "target_qs": snap[2]},
                    "actor": at["actor"], "temperature": at["temperature"]}
            for k in ("critic_lr", "actor_lr", "temperature_lr"):
                info[k] = at[k]
            return self, info
        if _augment:
            ops.rng_schedule(self.state._rng, self._keys, True, False)          # drq.py:279
        self._load_batch(full, batch, augment=_augment, keys=self._keys)
        self._features(full)
        self._relabel(full)
        crit_infos = []
        for i in range(utd_ratio):
            eng = self._minibatch_engine(full, i, mb)
            crit_infos.append(self._update_on_engine(eng, frozenset({"critic"}), pmap_axis))
        at = self._update_on_engine(full, frozenset({"actor", "temperature"}), pmap_axis)
        crit = {k: torch.stack([c["critic"][k] for c in crit_infos]).mean() for k in crit_infos[0]["critic"]}
        info = {"critic": crit, "actor": at["actor"], "temperature": at["temperature"]}
        for k in ("critic_lr", "actor_lr", "temperature_lr"):
            info[k] = at[k]
        return self, info

    def _minibatch_engine(self, full: Engine, i: int, mb: int) -> Engine:
        eng = self._engine(mb)
        lo, hi, B = i * mb, (i + 1) * mb, full.B
        for name in ("state_o", "state_n", "actions", "rewards", "masks", "idx", "weights"):
            getattr(eng, name).copy_(getattr(full, name)[lo:hi])
        # the minibatch's rows of each prioritized part (weights stay those of the draw over the whole part)
        eng.prio_parts = [(ring, max(r, lo) - lo, min(r + n, hi) - max(r, lo)) for ring, r, n in full.prio_parts if max(r, lo) < min(r + n, hi)]
        if self._cfg.pixel:
            src = "pix" if self._cfg.trainable_encoder else "feats"    # a trainable encoder runs its convs on the crops themselves
            for cam in self._cfg.cams:
                getattr(eng, src)[cam][:mb].copy_(getattr(full, src)[cam][lo:hi])
                getattr(eng, src)[cam][mb:].copy_(getattr(full, src)[cam][B + lo:B + hi])
        return eng

    # ---- sample_actions (sac.py:301-320) ---------------------------------------------------------------
    def _infer_inputs(self, observations):
        """One observation or a batch (the layouts sample_actions takes) -> (inference engine, B, unbatched) with the state rows
        loaded and, for the pixel agent, the frozen trunk's features computed (the small encoder runs in Engine.encode)."""
        cfg, dev = self._cfg, self.device
        if cfg.pixel:
            if cfg.use_proprio:
                st = _as_tensor(observations["state"])
                unbatched = st.ndim == 2                                    # (T,S)
                B = 1 if unbatched else st.shape[0]
            else:                                                           # images: (T,H,W,C) one observation, (B,T,H,W,C) a batch
                img0 = _as_tensor(observations[cfg.cams[0]])
                unbatched = img0.ndim < 5
                B = 1 if unbatched else img0.shape[0]
                st = torch.zeros(B, 0)
            eng = self._infer_engine(B)
            T, hw = cfg.obs_horizon, cfg.image_hw
            for cam in cfg.cams:                                            # (B, T, H, W, C) -> (B, H, W, T*C)
                img = _as_tensor(observations[cam]).to(dev)
                eng.pix[cam].copy_(img.reshape(B, T, hw, hw, 3).permute(0, 2, 3, 1, 4).reshape(B, hw, hw, 3 * T))
                if not cfg.trainable_encoder:
                    eng.trunk_forward(cam, eng.pix[cam], eng.feats[cam])
        else:
            st = _as_tensor(observations)
            unbatched = st.ndim == 1
            B = 1 if unbatched else st.shape[0]
            eng = self._infer_engine(B)
        if cfg.state_in:
            eng.state_o.copy_(st.to(torch.float32).reshape(B, -1))
        return eng, B, unbatched

    def sample_actions(self, observations, *, seed=None, argmax: bool = False, return_device: bool = False, **kwargs):
        cfg = self._cfg
        if argmax:
            assert seed is None, "Cannot specify seed when sampling deterministically"
        eng, B, unbatched = self._infer_inputs(observations)
        eng.encode(self._store.params, slice(0, B), eng.state_o, eng.Xp, eng.F, None, save=False)   # train=False: no dropout
        eng.policy_forward(self._store.params, eng.Xp, save=False)
        A = cfg.action_dim
        if not argmax:
            _load_key(self._seed_key, seed)
            ops.normal_fill(self._seed_key.data_ptr(), eng.eps, B * A)
        eng.tanh_gaussian(self._store.params, eng.act_scratch.data_ptr(), A, None, None, None, deterministic=argmax)
        out = eng.act_scratch.clone()
        out = out[0] if unbatched else out
        return out if return_device else out.cpu().numpy()

    # ---- forward passes of the public API (sac.py:33-116) ------------------------------------------------------------------
    # Forward only, on the inference engines: they read the parameters and change nothing else (state.rng, state.step, the
    # captured step graphs and a pipelined step's prefetched batch stay as they are).  Results are device tensors.
    def forward_critic(self, observations, actions, rng, *, grad_params=None, train: bool = True):
        """Q-values of the critic ensemble: (E, B) for actions (B, A), (E, B, N) for N candidate actions per state (B, N, A)
        (multiple_action_q_function, actor_critic_nets.py:33-46); (E,) / (E, N) for one observation.  The critic calls its encoder
        with train=False.  With the critic MLP's dropout_rate, train=True applies hidden layer i's keep mask
        bernoulli(fold_in(rng, ncams + i), 1 - rate, (B, H_i)), shared by the ensemble members (DESIGN.md §4); without it `train`
        only decides whether `rng` is required, as in the reference."""
        _refuse_grad_params(grad_params, "forward_critic")
        if train:
            assert rng is not None, "Must specify rng when training"
        return self._critic_values(self._store.params, observations, actions, rng if train else None)

    def forward_target_critic(self, observations, actions, rng):
        """forward_critic with target_params (encoder heads and critic); the frozen trunk is shared."""
        assert rng is not None, "Must specify rng when training"          # sac.py:48-50 forwards with the default train=True
        return self._critic_values(self._store.target, observations, actions, rng)

    def _mlp_masks(self, eng, arch, B, rng):
        """The (B, H_i) keep masks of a train=True forward with key rng (DESIGN.md §4), in the inference engine's buffers."""
        _load_key(self._fwd_key, rng)
        ncams = len(self._cfg.cams) if self._cfg.pixel else 0
        masks = eng.mlp_masks(arch)
        for i, m in enumerate(masks):
            ops.dropout_mask_fill(self._fwd_key.data_ptr(), ncams + i, 1.0 - arch.dropout, m, B * arch.hidden[i])
        return masks

    def _critic_values(self, buf, observations, actions, rng=None):
        cfg = self._cfg
        E, A = cfg.ensemble, cfg.action_dim
        drop = rng is not None and cfg.critic_arch.dropout > 0
        eng, B, unbatched = self._infer_inputs(observations)
        a = _as_tensor(actions).to(self.device, torch.float32)
        if a.ndim not in ((1, 2) if unbatched else (2, 3)) or a.shape[-1] != A or (not unbatched and a.shape[0] != B):
            obs = "one observation" if unbatched else f"a batch of {B}"
            want = f"(A,) or (N, A)" if unbatched else f"({B}, A) or ({B}, N, A)"
            raise ValueError(f"actions of shape {tuple(a.shape)} for {obs}: expected {want} with A = {A}")
        multi = a.ndim == (2 if unbatched else 3)
        if multi and drop:
            raise NotImplementedError("forward_critic(train=True) of N candidate actions per state with the critic's dropout_rate: "
                                      "the multi-action kernel applies no dropout mask (train=False evaluates them)")
        a = (a.reshape(B, -1, A) if multi else a.reshape(B, A)).contiguous()
        eng.encode(buf, slice(0, B), eng.state_o, eng.Xc, eng.FA, None, save=False)
        if not multi:
            ops.copy2d(a.data_ptr(), A, ops.at(eng.Xc, eng.F), eng.FA, B, A)
            eng.critic_forward(buf, eng.Xc, eng.c_main, eng.q, save=False,
                               masks=self._mlp_masks(eng, cfg.critic_arch, B, rng) if drop else None)
            q = eng.q.clone()
        else:
            N = a.shape[1]
            q = eng.critic_forward_multi(buf, eng.Xc, a, N).clone().view(E, B, N)
        return q[:, 0] if unbatched else q

    def forward_policy(self, observations, rng=None, *, grad_params=None, train: bool = True) -> "TanhMultivariateNormalDiag":
        """The policy's action distribution.  train=True applies the image heads' Dropout(0.1) with the masks the update's policy
        passes draw from a key: camera j keeps bernoulli(fold_in(rng, j), 0.9) (DESIGN.md §4), and with the policy MLP's
        dropout_rate hidden layer i keeps bernoulli(fold_in(rng, ncams + i), 1 - rate, (B, H_i)); train=False applies none."""
        _refuse_grad_params(grad_params, "forward_policy")
        if train:
            assert rng is not None, "Must specify rng when training"
        cfg = self._cfg
        eng, B, unbatched = self._infer_inputs(observations)
        masks = None
        if train and cfg.pixel and not cfg.small:            # (the small encoder has no Dropout)
            _load_key(self._fwd_key, rng)
            for j, cam in enumerate(cfg.cams):
                ops.dropout_mask_fill(self._fwd_key.data_ptr(), j, 0.9, eng.masks_u8[cam], B * 4096)
            masks = eng.masks_u8
        eng.encode(self._store.params, slice(0, B), eng.state_o, eng.Xp, eng.F, masks, save=False)
        pa = cfg.policy_arch
        eng.policy_forward(self._store.params, eng.Xp, save=False,
                           masks=self._mlp_masks(eng, pa, B, rng) if train and pa.dropout > 0 else None)
        return TanhMultivariateNormalDiag(self, eng, unbatched)

    def forward_temperature(self, *, grad_params=None) -> torch.Tensor:
        """The temperature softplus(lagrange) (GeqLagrangeMultiplier, lagrange.py:9-78), a 0-d device tensor."""
        _refuse_grad_params(grad_params, "forward_temperature")
        out = torch.empty((), dtype=torch.float32, device=self.device)
        ops.lagrange_penalty(self._store.addr(self._store.params, "modules_temperature/lagrange"), None, 0.0, out, 1)
        return out

    def temperature_lagrange_penalty(self, entropy, *, grad_params=None) -> torch.Tensor:
        """softplus(lagrange) * (entropy - target_entropy), elementwise over `entropy`."""
        _refuse_grad_params(grad_params, "temperature_lagrange_penalty")
        ent = _as_tensor(entropy).to(self.device, torch.float32).contiguous()
        out = torch.empty_like(ent)
        ops.lagrange_penalty(self._store.addr(self._store.params, "modules_temperature/lagrange"), ent, self.config["target_entropy"], out,
                             ent.numel())
        return out


class TanhMultivariateNormalDiag:
    """`forward_policy`'s result: tanh(N(loc, diag(scale_diag^2))) (actor_critic_nets.py:230-272), evaluated on the library's
    kernels.  It owns copies of the policy heads' outputs, so later calls on the agent do not change it.  Shapes are (B, A) and
    (B,) for a batch, (A,) and () for one observation.

    - `mode()` = tanh(loc): the bits of `sample_actions(argmax=True)`.
    - `stddev()` = tanh(scale_diag): the reference applies the tanh bijector to the base distribution's stddev
      (`bijector.forward(distribution.stddev())`, actor_critic_nets.py:271-272); kept as it is, although it is not the standard
      deviation of the squashed distribution.
    - `sample(seed)` = tanh(loc + scale_diag * normal(seed)): the key use and bits of `sample_actions(seed=seed)`.
    - `sample_and_log_prob(seed)`: that sample and the log-probability the update uses.
    - `log_prob(x)`: u = atanh(x), the diagonal-Gaussian log-density of u minus sum 2 (log 2 - u - softplus(-2u)).  x is not
      clipped: |x| = 1 gives u = inf and a NaN log-probability, as in the reference."""

    def __init__(self, agent: SACAgent, eng: InferenceEngine, unbatched: bool):
        cfg = agent._cfg
        self._cfg, self._dev, self._unbatched = cfg, agent.device, unbatched
        B, A = eng.B, cfg.action_dim
        self._B, self._A = B, A
        self._mu = eng.mu.clone()
        if cfg.std_parameterization == "uniform":      # the (A,) log_stds leaf, read with row stride 0
            self._x, self._ld = agent._store.view(agent._store.params, "modules_actor/log_stds").clone(), 0
        else:
            self._x, self._ld = eng.ls.clone(), A
        self._mode, self._std = self._empty(B, A), self._empty(B, A)
        self._tanh_gaussian(self._mode, None, None, self._std, deterministic=True)
        self._key = torch.zeros(2, dtype=torch.uint32, device=self._dev)

    def _empty(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self._dev)

    def _out(self, t):
        return t[0] if self._unbatched else t

    def _tanh_gaussian(self, act, eps, logp, std, deterministic=False):
        cfg, B, A = self._cfg, self._B, self._A
        if cfg.std_parameterization == "exp":
            ops.tanh_gaussian_fwd(self._mu, self._x, eps, cfg.std_min, cfg.std_max, act.data_ptr(), A, logp, None, std, B, A,
                                  deterministic=deterministic)
        else:
            ops.tanh_gaussian_fwd_std(self._mu, self._x.data_ptr(), self._ld, STD_IDS[cfg.std_parameterization], eps, cfg.std_min,
                                      cfg.std_max, act.data_ptr(), A, logp, None, std, B, A, deterministic=deterministic)

    @property
    def loc(self) -> torch.Tensor:
        return self._out(self._mu)

    @property
    def scale_diag(self) -> torch.Tensor:
        """The clipped std."""
        return self._out(self._std)

    def mode(self) -> torch.Tensor:
        return self._out(self._mode)

    def stddev(self) -> torch.Tensor:
        out = self._empty(self._B, self._A)
        L.call("serl_tanh_fwd", self._std.data_ptr(), out.data_ptr(), self._B * self._A, L.stream_ptr())
        return self._out(out)

    def _sample(self, seed, logp):
        _load_key(self._key, seed)
        eps, act = self._empty(self._B, self._A), self._empty(self._B, self._A)
        ops.normal_fill(self._key.data_ptr(), eps, self._B * self._A)
        self._tanh_gaussian(act, eps, logp, None)
        return act

    def sample(self, *, seed) -> torch.Tensor:
        return self._out(self._sample(seed, None))

    def sample_and_log_prob(self, *, seed):
        logp = self._empty(self._B)
        act = self._sample(seed, logp)
        return self._out(act), self._out(logp)

    def log_prob(self, value) -> torch.Tensor:
        x = _as_tensor(value).to(self._dev, torch.float32)
        want = (self._A,) if self._unbatched else (self._B, self._A)
        if tuple(x.shape) != want:
            raise ValueError(f"log_prob: actions of shape {tuple(x.shape)}, expected {want}")
        x = x.reshape(self._B, self._A).contiguous()
        logp = self._empty(self._B)
        ops.tanh_normal_log_prob(self._mu, self._std, x, logp, self._B, self._A)
        return self._out(logp)


def _refuse_grad_params(grad_params, name):
    if grad_params is not None:
        raise NotImplementedError(f"{name}(grad_params=...): these forward passes have no autodiff; gradients come from the update methods")


def _as_tensor(x) -> torch.Tensor:
    """A torch tensor (any device) as it is; anything else through NumPy."""
    return x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))


def _load_key(dst: torch.Tensor, key) -> None:
    """A JAX PRNG key (2 uint32 words) into the device buffer dst."""
    k = np.ascontiguousarray(np.asarray(key.cpu() if isinstance(key, torch.Tensor) else key), dtype=np.uint32).reshape(2)
    dst.copy_(torch.from_numpy(k.view(np.int32)).view(torch.uint32))


_LAUNCHER_NET_KWARGS = {"activations": "tanh", "use_layer_norm": True, "hidden_dims": [256, 256]}     # utils/launcher.py:61-66,95-104
_ACTIVATIONS = {"tanh": "tanh", "relu": "relu", "swish": "swish", "silu": "swish", "leaky_relu": "leaky_relu", "gelu": "gelu"}
_NETWORK_KEYS = {"hidden_dims", "activations", "use_layer_norm", "activate_final", "dropout_rate"}


def _mlp_arch(name: str, nk: Optional[dict], allow_dropout: bool = False) -> MlpArch:
    """One `*_network_kwargs` dict (networks/mlp.py:10-32 fields) -> MlpArch.

    Omitted, or every given key equal to the launcher's value: the launcher architecture, as every SERL launcher builds it.  A
    dict with any other value must state `activations` and `use_layer_norm`: the reference's MLP would fill them with flax
    defaults (swish, no LayerNorm) that differ from the launcher's, and neither is guessed here.  allow_dropout: the caller trains
    the MLP's Dropout (SACAgent / DrQAgent); otherwise a non-zero dropout_rate raises NotImplementedError."""
    return resolve_mlp(name, nk, LAUNCHER_MLP, _LAUNCHER_NET_KWARGS, allow_dropout=allow_dropout)


def resolve_mlp(name: str, nk: Optional[dict], launcher: MlpArch, launcher_kwargs: dict, allow_dropout: bool) -> MlpArch:
    """`_mlp_arch` against a given launcher architecture.  allow_dropout: accept `dropout_rate` (None, 0 or in (0, 1)) into
    MlpArch.dropout; otherwise a non-zero rate raises NotImplementedError."""
    if nk is None:
        return launcher
    nk = dict(nk)
    unknown = set(nk) - _NETWORK_KEYS
    if unknown:
        raise TypeError(f"{name}: unexpected keys {sorted(unknown)} (MLP takes {sorted(_NETWORK_KEYS)})")
    rate = nk.pop("dropout_rate", None)
    if not allow_dropout and rate not in (None, 0, 0.0):
        raise NotImplementedError(f"{name}: dropout_rate={rate!r} is not supported here (SACAgent and DrQAgent train MLP dropout)")
    rate = 0.0 if rate is None else float(rate)
    if not (rate == 0.0 or 0.0 < rate < 1.0):
        raise ValueError(f"{name}: dropout_rate={rate!r}: need None, 0 or a rate in (0, 1)")
    nk.pop("activate_final", None)                     # the agents' constructors force activate_final=True (sac.py:511-512, drq.py:135-136)
    act = nk.get("activations", launcher.act)
    act = getattr(act, "__name__", act)                # flax / jax function or its name, as MLP accepts both
    if not isinstance(act, str) or act not in _ACTIVATIONS:
        raise NotImplementedError(f"{name}: activations={act!r} is not supported (implemented: {sorted(_ACTIVATIONS)})")
    hidden = tuple(int(h) for h in nk.get("hidden_dims", list(launcher.hidden)))
    ln = bool(nk.get("use_layer_norm", launcher.layer_norm))
    if (hidden, _ACTIVATIONS[act], ln, rate) == (launcher.hidden, launcher.act, launcher.layer_norm, launcher.dropout):
        return launcher
    missing = [k for k in ("activations", "use_layer_norm") if k not in nk]
    if missing:
        raise ValueError(f"{name}={nk}: a non-launcher architecture must give {missing} explicitly - the reference's MLP would use "
                         "the flax defaults activations=nn.swish, use_layer_norm=False (networks/mlp.py:12-14), this project's "
                         f"launcher architecture is {launcher_kwargs}")
    if not hidden or any(h % 64 or not 64 <= h <= 1024 for h in hidden):
        raise ValueError(f"{name}: hidden_dims={list(hidden)}: need a non-empty list of widths, each a multiple of 64 in [64, 1024]")
    return MlpArch(hidden, _ACTIVATIONS[act], ln, rate)


def architecture_settings(policy_kwargs, extra, pixel, allow_dropout: bool = False) -> dict:
    """AgentConfig's critic_arch / policy_arch / std_parameterization from the reference constructors' `critic_network_kwargs`,
    `policy_network_kwargs` and `policy_kwargs` (popped from `extra`).  Omitted dicts build the launcher architecture (tanh MLPs
    [256, 256] with LayerNorm, "exp" std): this differs from the reference constructors' own defaults (swish, no LayerNorm,
    "uniform" std; sac.py:486-504, drq.py:104-131).  allow_dropout: accept the MLPs' dropout_rate (see `_mlp_arch`)."""
    pk = dict(policy_kwargs or {})
    std = pk.get("std_parameterization", "exp")
    if std == "fixed" or pk.get("fixed_std") is not None:
        raise NotImplementedError(f"policy_kwargs={pk}: a fixed std is not supported")
    if std not in STD_PARAMETERIZATIONS:
        raise NotImplementedError(f"policy_kwargs={pk}: std_parameterization={std!r} is not supported (implemented: {STD_PARAMETERIZATIONS})")
    if not pk.get("tanh_squash_distribution", True):
        raise NotImplementedError(f"policy_kwargs={pk}: only the tanh-squashed Gaussian policy is implemented")
    out = dict(critic_arch=_mlp_arch("critic_network_kwargs", extra.pop("critic_network_kwargs", None), allow_dropout),
               policy_arch=_mlp_arch("policy_network_kwargs", extra.pop("policy_network_kwargs", None), allow_dropout),
               std_parameterization=std)
    if extra.pop("shared_encoder", True) is not True:
        raise NotImplementedError("shared_encoder=False is not implemented (every SERL launcher shares the encoder)")
    for k in ("image_keys", "augmentation_function"):
        if extra.get(k) not in (None, {}):
            raise NotImplementedError(f"{k}={extra[k]!r} is not supported")
        extra.pop(k, None)
    if extra:
        raise TypeError(f"unexpected keyword arguments {sorted(extra)}")
    return out


TXS = ("critic", "actor", "temperature")        # AgentConfig's per-tx order (flat-buffer groups 0, 1, 2)
_OPTIMIZER_KEYS = {"learning_rate", "warmup_steps", "cosine_decay_steps", "clip_grad_norm"}


def optimizer_settings(tx_kwargs: Dict[str, Optional[dict]], learning_rate: Optional[float], warmup: Dict[str, Optional[int]],
                       default_warmup: Dict[str, int]):
    """Per-tx (lr, warmup, cosine decay steps, clip) tuples in AgentConfig order from the reference's
    `{actor,critic,temperature}_optimizer_kwargs` (each forwarded to make_optimizer, common/optimizers.py:6-56) and this
    project's `learning_rate=` / `*_warmup=` arguments.

    A key a dict leaves out takes the argument's value (its default when the argument is not given).  An argument given
    explicitly AND a dict key that says something else is an error: neither silently wins."""
    out = {"lr": [], "warmup": [], "decay": [], "clip": []}
    for tx in TXS:
        kw = dict(tx_kwargs.get(tx) or {})
        name = f"{tx}_optimizer_kwargs"
        if kw.get("weight_decay") is not None:
            raise NotImplementedError(
                f"{name}: weight_decay is not supported.  optax.adamw in every tx decays the whole parameter tree, the frozen "
                "pretrained ResNet-10 trunk included, on every update call (also for networks outside networks_to_update); "
                "reproducing that means rewriting the resident 16-bit trunk every step (DESIGN.md section 7)")
        kw.pop("weight_decay", None)
        if kw.pop("return_lr_schedule", False):
            raise NotImplementedError(f"{name}: return_lr_schedule is not supported (make_optimizer then returns a tuple, "
                                      "which no agent's create accepts as a tx)")
        unknown = set(kw) - _OPTIMIZER_KEYS
        if unknown:
            raise TypeError(f"{name}: unexpected keys {sorted(unknown)} (make_optimizer takes {sorted(_OPTIMIZER_KEYS)})")
        for key, arg, default, argname in (("learning_rate", learning_rate, 3e-4, "learning_rate"),
                                           ("warmup_steps", warmup.get(tx), default_warmup[tx], f"{tx}_warmup")):
            if key in kw and arg is not None and kw[key] != arg:
                raise ValueError(f"{argname}={arg!r} disagrees with {name}[{key!r}]={kw[key]!r}; pass one of them")
            kw.setdefault(key, default if arg is None else arg)
        lr, w = float(kw["learning_rate"]), int(kw["warmup_steps"])
        decay, clip = kw.get("cosine_decay_steps"), kw.get("clip_grad_norm")
        if w < 0:
            raise ValueError(f"{name}: warmup_steps must be >= 0, got {w}")
        if decay is not None and int(decay) <= w:
            raise ValueError(f"{name}: cosine_decay_steps ({decay}) must exceed warmup_steps ({w}) "
                             "(optax.cosine_decay_schedule needs decay_steps - warmup_steps > 0)")
        if clip is not None and not float(clip) > 0:
            raise ValueError(f"{name}: clip_grad_norm must be > 0, got {clip}")
        out["lr"].append(lr)
        out["warmup"].append(w)
        out["decay"].append(None if decay is None else int(decay))
        out["clip"].append(None if clip is None else float(clip))
    return {k: tuple(v) for k, v in out.items()}


def register_pytree(cls):
    """The learner scripts treat the agent as a JAX pytree: `jax.device_put(jax.tree_map(jnp.array, agent), sharding)`
    (examples/async_drq_sim/async_drq_sim.py:347-349) and `jax.block_until_ready(agent)` (:296).  This agent's arrays live in
    HBM behind the C-ABI, so it registers as a LEAF-LESS pytree node (the whole object travels as static aux data): both calls
    become identity operations.  No-op when jax is not importable."""
    try:
        from jax import tree_util
    except Exception:                                   # noqa: BLE001
        return False
    try:
        tree_util.register_pytree_node(cls, lambda a: ((), a), lambda aux, _children: aux)
    except ValueError:                                  # already registered
        pass
    return True


register_pytree(SACAgent)


def _host_split(key: np.ndarray, n: int) -> np.ndarray:
    """jax.random.split on the host through the library's host mirror of the device PRNG."""
    key = np.ascontiguousarray(key, dtype=np.uint32)
    out = np.zeros((n, 2), dtype=np.uint32)
    L.call("serl_host_threefry_split", key.ctypes.data, n, out.ctypes.data)
    return out


def _leaf(batch, key):
    v = batch[key]
    return v.cpu() if isinstance(v, torch.Tensor) else v
