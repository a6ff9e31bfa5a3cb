"""DrQAgent on hand-written sm_100a kernels.

Mirrors the reference's `DrQAgent` (agents/continuous/drq.py:23-328): `create_drq`, `update_critics`,
`update_high_utd`, inheriting `update` / `sample_actions` from SACAgent.  The DrQ random shift is not a
separate pass: it is applied by the replay sampler kernel while it gathers the frames, keyed by the
same JAX key chain as `data_augmentation_fn` (drq.py:244-253,307-310; same offsets for every camera of
a sample, different keys for obs and next_obs).

Encoders: `encoder_type="resnet-pretrained"` (the frozen ResNet-10 + trainable heads every SERL example uses) and "small",
the reference's default: four trainable 3x3 / stride-2 convs, mean pooling, Dense -> LayerNorm -> tanh (drq.py:137-152,
small_encoders.py:9-55), trained through the critic loss.  The reference's own "small" branch fails at the first forward
(EncodingWrapper passes `encode=`, which SmallEncoder does not take; SURVEY.md Appendix C.1): this is that network with the
argument dropped.  "resnet" trains a ResNet-10 (resnet_v1.py:129-286, resnetv1-10 with pre_pooling=False) end to end with the
SpatialLearnedEmbeddings / Dropout / Dense / LayerNorm head of "resnet-pretrained", from kaiming-normal initial weights.
"""
from __future__ import annotations

from typing import Iterable, Optional

import numpy as np
import torch

from ... import _lib as L
from ... import ops
from ...data.replay_buffer import BatchHandle, is_prioritized
from ...engine import MAX_OBS_HORIZON, AgentConfig, small_sizes
from ...params import ENCODER_TYPES
from .sac import SACAgent, _leaf, architecture_settings, optimizer_settings, register_pytree


class DrQAgent(SACAgent):
    @classmethod
    def create_drq(cls, seed: int, observations, actions, *, encoder_type: str = "small", use_proprio: bool = True,
                   image_keys: Iterable[str] = ("image",), discount: float = 0.95, critic_ensemble_size: int = 2,
                   critic_subsample_size: Optional[int] = None, temperature_init: float = 1.0, backup_entropy: bool = False,
                   soft_target_update_rate: float = 0.005, target_entropy: Optional[float] = None, policy_kwargs=None,
                   learning_rate: Optional[float] = None, actor_optimizer_kwargs=None, critic_optimizer_kwargs=None,
                   temperature_optimizer_kwargs=None, precision: str = "fp32", device=None, **kwargs):
        """DrQAgent.create_drq.  Optimizer defaults follow DrQAgent.create (drq.py:35-43): lr 3e-4, no
        warm-up.  `*_optimizer_kwargs` take make_optimizer's learning_rate, warmup_steps, cosine_decay_steps and
        clip_grad_norm (see sac.optimizer_settings); `critic_network_kwargs`, `policy_network_kwargs` and
        policy_kwargs["std_parameterization"] choose the networks (see sac.architecture_settings).

        use_proprio defaults to True here (every SERL launcher passes it), where the reference defaults to False.  With
        use_proprio=False the encoder is the camera embeddings alone (encoding.py:26-72): no proprio Dense / LayerNorm, and a
        "state" entry in the observations and batches is ignored.

        encoder_type="small" (the default, as in the reference) trains the conv encoder through the critic loss; it has no
        pretrained weights to load.  Its convs run on the CUDA cores in the fp32 build and on the tensor cores
        (3xTF32 wgmma) in the fp16 / bf16 builds.  encoder_type="resnet" does the same with a ResNet-10 (no pretrained weights
        are loaded): drq.py:153-166 with `encode=` dropped and pre_pooling=False, the only reading under which its pooling and
        bottleneck arguments apply (DESIGN.md §3).

        Observations of ChunkingWrapper(obs_horizon=T), images (T, H, W, C) and state (T, S), train the trainable encoders on frame
        stacks (T <= 8): EncodingWrapper(enable_stacking=True) feeds the encoder "B T H W C -> B H W (T C)", so Conv_0 / conv_init
        read 3T channels, and the proprio Dense reads T*S values.  Each frame of a stack gets its own random shift.
        "resnet-pretrained" takes one frame per observation (its ImageNet weights have 3 input channels)."""
        arch = architecture_settings(policy_kwargs, kwargs, pixel=True, allow_dropout=True)
        opt = optimizer_settings({"critic": critic_optimizer_kwargs, "actor": actor_optimizer_kwargs, "temperature": temperature_optimizer_kwargs},
                                 learning_rate, {}, {"critic": 0, "actor": 0, "temperature": 0})
        if encoder_type not in ENCODER_TYPES:
            raise NotImplementedError(f"encoder_type={encoder_type!r}: supported are {ENCODER_TYPES}")
        pk = policy_kwargs or {}
        image_keys = tuple(image_keys)
        use_proprio = bool(use_proprio)
        if use_proprio:
            if "state" not in observations:
                raise ValueError(f"use_proprio=True needs a 'state' entry in the observations (got keys {sorted(observations)}); "
                                 "pass use_proprio=False for an agent that sees the camera images only")
            st = np.asarray(observations["state"])
            S = int(np.prod(st.shape[-2:])) if st.ndim >= 2 else int(st.shape[-1])
        else:
            S = 0                                                                    # a "state" entry, if any, is ignored
        img = np.asarray(observations[image_keys[0]])
        T = img.shape[-4] if img.ndim >= 4 else 1
        if T != 1 and encoder_type == "resnet-pretrained":
            raise NotImplementedError("obs_horizon must be 1 (ChunkingWrapper(obs_horizon=1) in every SERL example)")
        if not 1 <= T <= MAX_OBS_HORIZON:
            raise NotImplementedError(f"obs_horizon={T}: stacks of 1 to {MAX_OBS_HORIZON} frames are supported")
        hw = img.shape[-2]
        if encoder_type == "resnet" and (hw != 128 or img.shape[-3] != 128):
            # the SLE head's (4, 4, 512, 8) kernel and the stride-2 parity split of the trunk's input gradients assume 128x128 frames
            raise NotImplementedError(f"encoder_type='resnet' takes 128x128 frames (got {img.shape[-3]}x{hw})")
        if encoder_type == "small" and small_sizes(hw)[-2] < 3:
            raise NotImplementedError(f"encoder_type='small' takes frames of at least 31x31 (got {img.shape[-3]}x{hw})")
        A = int(np.asarray(actions).shape[-1])
        cfg = AgentConfig(cams=image_keys, state_in=S, action_dim=A, pixel=True, use_proprio=use_proprio, ensemble=critic_ensemble_size,
                          subsample=critic_subsample_size, discount=discount, tau=soft_target_update_rate,
                          target_entropy=(-A / 2 if target_entropy is None else target_entropy), backup_entropy=backup_entropy,
                          **opt, **arch, std_min=pk.get("std_min", 1e-5), std_max=pk.get("std_max", 10.0), image_hw=hw, precision=precision,
                          encoder=encoder_type, obs_horizon=T)
        agent = cls._build(seed, cfg, temperature_init, device, config_extra={"image_keys": image_keys})
        if cfg.trainable_encoder:
            return agent
        from ...utils.train_utils import load_resnet10_params
        return load_resnet10_params(agent, image_keys)                              # drq.py:237-240

    def update_critics(self, batch, *, pmap_axis: Optional[str] = None):
        """drq.py:296-328: unpack + augment + update{critic}."""
        B = batch.batch_size if isinstance(batch, BatchHandle) else int(np.asarray(_leaf(batch, "rewards")).shape[0])
        # a prioritized draw reads the priorities the previous step wrote, so it cannot be prefetched one step early: serial
        if (self.pipeline_critic_steps and self._cfg.pixel and self.section_events is None and not is_prioritized(batch)
                and self._graph_key(("update_critics", pmap_axis), batch) is not None):
            return self._update_critics_pipelined(batch, B, pmap_axis)
        eng = self._engine(B)
        nets = frozenset({"critic"})

        def body(graph_mode):
            ops.rng_schedule(self.state._rng, self._keys, True, True, mlp_dropout=self._cfg.mlp_dropout)   # split(rng,3), then split(rng,4)
            if getattr(eng, "fused", None) is not None and self.explicit_randomness is None:
                eng.fused.prefetch_rng(self._keys)
            with self._section("sample_crop"):
                self._load_batch(eng, batch, augment=True, keys=self._keys, graph_mode=graph_mode)
            with self._section("trunk"):
                self._features(eng)
            self._relabel(eng)
            self._update_on_engine(eng, nets, pmap_axis, schedule_keys=False, want_info=False)

        self._run_step(self._graph_key(("update_critics", pmap_axis), batch), batch, body)
        info = self._info(eng, nets)
        del info["actor"], info["temperature"]
        return self, info

    # ---- cross-step pipeline: heads / Adam of step i next to sampler + frozen trunk of step i+1 ---------------------------
    def _update_critics_pipelined(self, batch: BatchHandle, B: int, pmap_axis):
        """`update_critics` for a batch handle that continues a sequence of handles (same rings, step + 1): the step's own
        sampler + trunk results were produced by the PREVIOUS call on the other engine of a ping-pong pair, and this call
        produces the next step's while its heads, all-reduce and Adam run (kind "P").  A call that does not continue the
        sequence runs its own front end first (kind "W").  Same kernels, same key chain, same results as the serial path as
        long as nothing is inserted between a prefetch and its use (then the prefetched draw simply predates the insert, as
        with the reference iterator's queue)."""
        from ...engine import Engine
        nets = frozenset({"critic"})
        if self._graphs_version != self._store.version:
            self.invalidate_graphs()
        if B not in self._eng_pair:
            self._eng_pair[B] = [self._engine(B), Engine(self._cfg, self._store, self._frozen_trunk, B, self.device)]
        if self._pipe_stream is None:
            self._pipe_stream = L.new_side_stream(torch.device(self.device))
        pair, Q = self._eng_pair[B], self._pipe_stream
        sig = (B, pmap_axis, tuple((id(p["ring"]), p["batch"], p["seed"]) for p in batch.parts), batch.n_step)
        steps = tuple(p["step"] for p in batch.parts)
        pipe = self._pipe
        hit = pipe is not None and pipe["sig"] == sig and pipe["steps"] == steps
        par = pipe["par"] if hit else 0
        kind = "P" if hit else "W"
        cur, nxt = pair[par], pair[1 - par]
        Kc, Kn = self._keys_pair[par], self._keys_pair[1 - par]
        nxt_handle = BatchHandle([dict(p, step=p["step"] + 1) for p in batch.parts], batch.pack)

        def body(graph_mode):
            self._keys = Kc
            if kind == "W":                                          # this step's own front end (cold start of the pipeline)
                ops.rng_schedule(self.state._rng, Kc, True, True, mlp_dropout=self._cfg.mlp_dropout)
                self._rng_look.copy_(self.state._rng)
                if cur.fused is not None:
                    cur.fused.fill_rng_now(Kc)
                self._load_batch(cur, batch, augment=True, keys=Kc, graph_mode=graph_mode)
                self._features(cur)
            Q.fork()
            with Q:                                                  # front end of the NEXT step
                self.state._rng.copy_(self._rng_look)                # the key this step leaves behind (= what the serial path leaves)
                ops.rng_schedule(self._rng_look, Kn, True, True, mlp_dropout=self._cfg.mlp_dropout)
                if nxt.fused is not None:
                    nxt.fused.fill_rng_now(Kn)
                self._load_batch(nxt, nxt_handle, augment=True, keys=Kn, graph_mode=graph_mode)
                self._features(nxt)
            self._relabel(cur)
            self._update_on_engine(cur, nets, pmap_axis, schedule_keys=False, want_info=False)
            Q.join()

        # W draws step, then step + 1; P draws step + 1
        draws = [(p["ring"], p["step"], 2) if kind == "W" else (p["ring"], p["step"] + 1, 1) for p in batch.parts]
        self._graphs.run(("pipe", kind, par, sig) if self.use_cuda_graphs else None, draws, body, self.state)
        self._keys = Kc
        self._pipe = dict(sig=sig, steps=tuple(s + 1 for s in steps), par=1 - par)
        self._last_engine = cur                                       # the engine whose buffers hold this step
        info = self._info(cur, nets)
        del info["actor"], info["temperature"]
        return self, info

    def update_high_utd(self, batch, *, utd_ratio: int, pmap_axis: Optional[str] = None):
        """drq.py:255-294: augment once, then SACAgent.update_high_utd."""
        return super().update_high_utd(batch, utd_ratio=utd_ratio, pmap_axis=pmap_axis, _augment=True)


register_pytree(DrQAgent)
