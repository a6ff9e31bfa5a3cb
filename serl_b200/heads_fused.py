"""Critic step of the pixel agent on the fused head kernels (16-bit builds): same algebra, same buffers and the same
gradient layout as Engine.critic_loss_and_grads (engine.py; reference agents/continuous/sac.py:134-191,
networks/actor_critic_nets.py:57-73,178-227, common/encoding.py:26-72, vision/resnet_v1.py:340-374), but

  * every dense contraction is ONE serl_tgemm_tf32 launch (csrc/tgemm.cu: TF32 tensor cores, operands by TMA from the fp32
    arrays in place) with its bias + LayerNorm + tanh (+ value head / + policy heads and the tanh-Gaussian sample) in the epilogue;
  * independent problems share a launch: the three encoder passes of the step (online critic on s, target critic on s',
    policy on s' with dropout) x cameras = one SLE launch, one k-split GEMM launch, one finish launch; online and target
    critic = one launch per layer;
  * the reductions of the backward pass (bias / LayerNorm / value-head gradients) are one launch per MLP.

About 40 launches instead of ~95 for a dual-camera critic step.  Pure orchestration: every arithmetic op is a C-ABI call.
"""
from __future__ import annotations

import os

import torch

from . import _lib as L
from . import ops
from .params import ENC

f32 = torch.float32


def enabled(cfg) -> bool:
    """Fused heads serve the pixel agent of the 16-bit builds (TMA needs 16-byte row strides: enc_dim + action_dim % 4 == 0).
    The proprio Dense runs inside enc_finish, which takes at most 64 state inputs; a pixel-only encoder has none."""
    if os.environ.get("SERL_FUSED_HEADS", "1") == "0" or not cfg.pixel or cfg.precision == "fp32":
        return False
    return (cfg.enc_dim + cfg.action_dim) % 4 == 0 and cfg.action_dim <= 8 and (not cfg.use_proprio or cfg.state_in <= 64)


class FusedCritic:
    def __init__(self, eng):
        self.eng = eng
        cfg, B, dev = eng.cfg, eng.B, eng.dev
        e = lambda *s: torch.empty(*s, dtype=f32, device=dev)
        self.ncam = len(cfg.cams)
        self.sle_t = {c: e(B, 4096) for c in cfg.cams}
        self.sle_p = {c: e(B, 4096) for c in cfg.cams}
        self.d_sle = {c: e(B, 4096) for c in cfg.cams}
        nprob = 3 * self.ncam
        tiles = nprob * ((B + 127) // 128)
        self.S = ops.tgemm_splits(4096, max(1, min(132 // tiles, 32)))
        self.ws_enc = ops.Workspace(nprob * self.S * B * 256 * 4, dev)
        self.error = torch.zeros(1, dtype=torch.int32, device=dev)
        self._rng_prefetched = False

    # ------------------------------------------------------------------------------------------------------------
    def _fill_rng(self, keys):
        eng = self.eng
        cfg, B, A = eng.cfg, eng.B, eng.cfg.action_dim
        ops.normal_fill(ops.key_ptr(keys, L.KEY_CRITIC_NEXT), eng.eps, B * A)
        for j, cam in enumerate(cfg.cams):
            ops.dropout_mask_fill(ops.key_ptr(keys, L.KEY_CRITIC_NEXT), j, 0.9, eng.masks_u8[cam], B * 4096)
        if cfg.subsample is not None:                                 # the TD target's ensemble subsample (sac.py:152-158) is key-only too
            ops.subsample_idx(ops.key_ptr(keys, L.KEY_CRITIC_SUBSAMPLE), cfg.ensemble, eng.sub, cfg.subsample)
        self._fill_mlp_masks(keys, None)

    def _fill_mlp_masks(self, keys, ex):
        """The critic step's MLP Dropout masks (DESIGN.md §4): the policy pass on s' under k_na, the target critic under c1, the
        online critic under c2 with critic_subsample_size and c1 without it; ex: the tests' explicit masks of the critic loss."""
        eng = self.eng
        cfg = eng.cfg
        get = lambda name: None if ex is None else ex.get(name)
        if eng.p_mask is not None:
            eng.fill_mlp_masks(eng.p_mask, cfg.policy_arch, ops.key_ptr(keys, L.KEY_CRITIC_NEXT), get("mlp_policy"))
        if eng.c_mask is not None:
            slot = L.KEY_MLP_CRITIC_SUBSAMPLED if cfg.subsample is not None else L.KEY_MLP_CRITIC_TARGET
            eng.fill_mlp_masks(eng.c_mask, cfg.critic_arch, ops.key_ptr(keys, slot), get("mlp_critic"))
            eng.fill_mlp_masks(eng.c_mask_tgt, cfg.critic_arch, ops.key_ptr(keys, L.KEY_MLP_CRITIC_TARGET), get("mlp_critic_target"))

    def _drop(self, arch, *masks):
        """tgemm / ln_tanh_bwd_multi keyword arguments of a layer whose problems drop out with these masks (none: no Dropout)."""
        if masks[0] is None:
            return {}
        return dict(masks=list(masks), inv_keep=1.0 / (1.0 - arch.dropout))

    def prefetch_rng(self, keys):
        """The critic step's noise and dropout masks only depend on the key schedule: fill them on side stream 1 right after
        rng_schedule, next to the sampler and the trunk (joined at the top of critic_loss_and_grads)."""
        s1 = self.eng.side[1]
        s1.fork()
        with s1:
            self._fill_rng(keys)
        self._rng_prefetched = "side"

    def fill_rng_now(self, keys):
        """Same fills on the CURRENT stream, ahead of the step that consumes them (cross-step pipeline, drq.py)."""
        self._fill_rng(keys)
        self._rng_prefetched = "done"

    def critic_loss_and_grads(self, keys, grad_scale=1.0, explicit=None):
        eng = self.eng
        cfg, B, E, A, st = eng.cfg, eng.B, eng.cfg.ensemble, eng.cfg.action_dim, eng.store
        F, FA, ncam, S = eng.F, eng.FA, self.ncam, self.S
        Pm, T, G = st.params, st.target, st.grad
        P = eng.P
        obs_rows, next_rows = slice(0, B), slice(B, 2 * B)
        err = self.error
        # ---- randomness of the policy pass on s' (dropout masks + sample noise; sac.py:122-128) ----
        if self._rng_prefetched:
            if self._rng_prefetched == "side":
                eng.side[1].join()                                   # filled on side stream 1 while the sampler and the trunk ran
            self._rng_prefetched = False                             # ("done": filled in stream order by the step pipeline)
        elif explicit is None:
            self._fill_rng(keys)
        else:
            eng.eps.copy_(explicit["critic"]["eps"])
            for cam in cfg.cams:
                eng.masks_u8[cam].copy_(explicit["critic"]["dropout"][cam])
            self._fill_mlp_masks(keys, explicit["critic"])
        parch, carch = cfg.policy_arch, cfg.critic_arch
        pm, cm_, ct_ = eng.p_mask or (None, None), eng.c_mask or (None, None), eng.c_mask_tgt or (None, None)
        # ---- encoder heads: three passes x cameras in three launches ----
        passes = [(Pm, obs_rows, eng.state_o, eng.Xc, FA, None, eng.sle_saved), (T, next_rows, eng.state_n, eng.Xt, FA, None, self.sle_t),
                  (Pm, next_rows, eng.state_n, eng.Xp, F, eng.masks_u8, self.sle_p)]
        sle, gemm, fin = [], [], []
        for pi, (buf, rows, state, X, ldx, masks, sles) in enumerate(passes):
            for j, cam in enumerate(cfg.cams):
                p = f"{ENC}/encoder_{cam}"
                i = pi * ncam + j
                sle.append((eng.feats[cam][rows].data_ptr(), P(buf, f"{p}/SpatialLearnedEmbeddings_0/kernel"),
                            None if masks is None else masks[cam].data_ptr(), sles[cam].data_ptr(), 4096))
                gemm.append(ops.tgemm_problem(sles[cam].data_ptr(), P(buf, f"{p}/Dense_0/kernel"), sAm=4096, sAk=1, sBk=256, sBn=1))
                fin.append(dict(partials=self.ws_enc.buf.data_ptr() + 4 * i * S * B * 256, S=S, bias=P(buf, f"{p}/Dense_0/bias"),
                                ln_scale=P(buf, f"{p}/LayerNorm_0/scale"), ln_bias=P(buf, f"{p}/LayerNorm_0/bias"), out=ops.at(X, 256 * j),
                                ld_out=ldx, D=256, xhat=eng.enc_xhat[cam].data_ptr() if pi == 0 else None,
                                rstd=eng.enc_rstd[cam].data_ptr() if pi == 0 else None))
        for pi, (buf, rows, state, X, ldx, masks, sles) in enumerate(passes if cfg.use_proprio else ()):
            fin.append(dict(x=state.data_ptr(), ld_x=cfg.state_in, w=P(buf, f"{ENC}/Dense_0/kernel"), K=cfg.state_in,
                            bias=P(buf, f"{ENC}/Dense_0/bias"), ln_scale=P(buf, f"{ENC}/LayerNorm_0/scale"), ln_bias=P(buf, f"{ENC}/LayerNorm_0/bias"),
                            out=ops.at(X, 256 * ncam), ld_out=ldx, D=64, xhat=eng.enc_xhat_p.data_ptr() if pi == 0 else None,
                            rstd=eng.enc_rstd_p.data_ptr() if pi == 0 else None))
        ops.sle_fwd_multi(sle, 0.9, B, 16, 512)
        ops.tgemm(self.ws_enc, gemm, B, 256, 4096, epilogue=L.TGEMM_PARTIAL, splits=S, error=err)
        ops.enc_finish(fin, B)
        ops.copy2d(eng.actions.data_ptr(), A, ops.at(eng.Xc, F), FA, B, A)
        # ---- a', log pi(a'|s') (policy MLP; mean / log-std heads and the tanh-Gaussian sample in the second launch's epilogue) ----
        n, pa = "modules_actor/network", eng.p_acts
        ops.tgemm(None, [ops.tgemm_problem(eng.Xp.data_ptr(), P(Pm, f"{n}/Dense_0/kernel"), sAm=F, sAk=1, sBk=256, sBn=1, C_=pa.h1.data_ptr(), ldc=256,
                                           bias=P(Pm, f"{n}/Dense_0/bias"), ln_scale=P(Pm, f"{n}/LayerNorm_0/scale"), ln_bias=P(Pm, f"{n}/LayerNorm_0/bias"))],
                  B, 256, F, epilogue=L.TGEMM_LN_TANH, error=err, **self._drop(parch, pm[0]))
        ops.tgemm(None, [ops.tgemm_problem(pa.h1.data_ptr(), P(Pm, f"{n}/Dense_1/kernel"), sAm=256, sAk=1, sBk=256, sBn=1,
                                           bias=P(Pm, f"{n}/Dense_1/bias"), ln_scale=P(Pm, f"{n}/LayerNorm_1/scale"), ln_bias=P(Pm, f"{n}/LayerNorm_1/bias"),
                                           head_w=P(Pm, "modules_actor/Dense_0/kernel"), head_b=P(Pm, "modules_actor/Dense_0/bias"), head_out=eng.mu.data_ptr(),
                                           head_w2=P(Pm, "modules_actor/Dense_1/kernel"), head_b2=P(Pm, "modules_actor/Dense_1/bias"), head_out2=eng.ls.data_ptr(),
                                           noise=eng.eps.data_ptr(), act=ops.at(eng.Xt, F), ld_act=FA, logp=eng.logp.data_ptr(), u_out=eng.u.data_ptr(),
                                           std_out=eng.std.data_ptr())],
                  B, 256, 256, epilogue=L.TGEMM_LN_TANH_POLICY, head_n=A, std_min=cfg.std_min, std_max=cfg.std_max, error=err,
                  **self._drop(parch, pm[1]))
        # ---- Q(s, a) with params (saved for the backward pass) and Q'(s', a') with target params: one launch per layer ----
        c, cm, ct = "modules_critic/network", eng.c_main, eng.c_tgt

        def layer1(buf, X, acts, save):
            return ops.tgemm_problem(X.data_ptr(), P(buf, f"{c}/Dense_0/kernel"), sAm=FA, sAk=1, sBk=256, sBn=1, Z=E, sAz=0, sBz=FA * 256,
                                     C_=acts.h1.data_ptr(), sCz=B * 256, ldc=256, bias=P(buf, f"{c}/Dense_0/bias"), sBiasZ=256,
                                     ln_scale=P(buf, f"{c}/LayerNorm_0/scale"), ln_bias=P(buf, f"{c}/LayerNorm_0/bias"), sLnZ=256,
                                     xhat=acts.xhat1.data_ptr() if save else None, rstd=acts.rstd1.data_ptr() if save else None, sXhatZ=B * 256, sRstdZ=B)

        def layer2(buf, acts, q, save):
            return ops.tgemm_problem(acts.h1.data_ptr(), P(buf, f"{c}/Dense_1/kernel"), sAm=256, sAk=1, sBk=256, sBn=1, Z=E, sAz=B * 256, sBz=256 * 256,
                                     C_=acts.h2.data_ptr() if save else None, sCz=B * 256, ldc=256, bias=P(buf, f"{c}/Dense_1/bias"), sBiasZ=256,
                                     ln_scale=P(buf, f"{c}/LayerNorm_1/scale"), ln_bias=P(buf, f"{c}/LayerNorm_1/bias"), sLnZ=256,
                                     xhat=acts.xhat2.data_ptr() if save else None, rstd=acts.rstd2.data_ptr() if save else None, sXhatZ=B * 256, sRstdZ=B,
                                     head_w=P(buf, "modules_critic/Dense_0/kernel"), head_b=P(buf, "modules_critic/Dense_0/bias"), sHeadWz=0, sHeadBz=0,
                                     head_out=q.data_ptr(), sHeadOutZ=B, ld_head=1)

        ops.tgemm(None, [layer1(Pm, eng.Xc, cm, True), layer1(T, eng.Xt, ct, False)], B, 256, FA, epilogue=L.TGEMM_LN_TANH, error=err,
                  **self._drop(carch, cm_[0], ct_[0]))
        ops.tgemm(None, [layer2(Pm, cm, eng.q, True), layer2(T, ct, eng.q_next, False)], B, 256, 256, epilogue=L.TGEMM_LN_TANH_HEAD, head_n=1, error=err,
                  **self._drop(carch, cm_[1], ct_[1]))
        # ---- TD target, loss, dQ (sac.py:134-191) ----
        n_sub = 0
        if cfg.subsample is not None:
            if explicit is not None:                                 # (drawn with the other key-only randomness otherwise: _fill_rng)
                eng.sub.copy_(explicit["critic"]["subsample"])
            n_sub = cfg.subsample
        ops.critic_loss(eng.q, eng.q_next, eng.sub, n_sub, eng.rewards, eng.masks, eng.logp, P(Pm, "modules_temperature/lagrange"),
                        cfg.backup_entropy, cfg.discount, grad_scale, eng.target_q, eng.dq, eng.info.data_ptr(), E, B,
                        weights=eng.weights if eng.prio_parts else None, delta=eng.delta)
        self._backward()

    # ------------------------------------------------------------------------------------------------------------
    def _backward(self):
        """Gradient of the critic loss w.r.t. critic MLP, value head, image heads and proprio encoder (group 0 of the flat buffer).
        The dQ -> ... -> d(enc) -> d(SLE) chain stays on the main stream; weight gradients and reductions run on side stream 0."""
        eng = self.eng
        cfg, B, E, st = eng.cfg, eng.B, eng.cfg.ensemble, eng.store
        F, FA, ncam = eng.F, eng.FA, self.ncam
        Pm, G = st.params, st.grad
        P = eng.P
        c, cm = "modules_critic/network", eng.c_main
        R = E * B
        side, wss, err = eng.side[0], eng.ws_side[0], self.error
        dz2, dy2, dh1, dz1, dy1 = eng.dz, eng.dy, eng.dh, eng.dz0, eng.dy0
        carch, cmask = cfg.critic_arch, eng.c_mask or (None, None)
        # layer 2: dh2 = dQ (x) w_head, LayerNorm + tanh backward (dz through the forward's Dropout mask, shared by the members)
        ops.ln_tanh_bwd_multi([dict(dq=eng.dq.data_ptr(), head_w=P(Pm, "modules_critic/Dense_0/kernel"), head_w_stride=0, t=cm.h2.data_ptr(), ld_t=256,
                                    xhat=cm.xhat2.data_ptr(), rstd=cm.rstd2.data_ptr(), scale=P(Pm, f"{c}/LayerNorm_1/scale"), rows_per_group=B,
                                    group_stride=256, dz=dz2.data_ptr(), dy=dy2.data_ptr(), R=R, D=256)], mask_rows=B, **self._drop(carch, cmask[1]))
        side.fork()
        with side:            # dW2[e] = h1[e]^T dz2[e]
            ops.tgemm(wss, [ops.tgemm_problem(cm.h1.data_ptr(), dz2.data_ptr(), sAm=1, sAk=256, sBk=256, sBn=1, Z=E, sAz=B * 256, sBz=B * 256,
                                              C_=P(G, f"{c}/Dense_1/kernel"), sCz=256 * 256, ldc=256)], 256, 256, B, splits=1, error=err)
        # dh1[e] = dz2[e] @ W2[e]^T
        ops.tgemm(eng.ws, [ops.tgemm_problem(dz2.data_ptr(), P(Pm, f"{c}/Dense_1/kernel"), sAm=256, sAk=1, sBk=1, sBn=256, Z=E, sAz=B * 256, sBz=256 * 256,
                                             C_=dh1.data_ptr(), sCz=B * 256, ldc=256)], B, 256, 256, splits=1, error=err)
        ops.ln_tanh_bwd_multi([dict(dt=dh1.data_ptr(), ld_dt=256, t=cm.h1.data_ptr(), ld_t=256, xhat=cm.xhat1.data_ptr(), rstd=cm.rstd1.data_ptr(),
                                    scale=P(Pm, f"{c}/LayerNorm_0/scale"), rows_per_group=B, group_stride=256, dz=dz1.data_ptr(), dy=dy1.data_ptr(), R=R, D=256)],
                              mask_rows=B, **self._drop(carch, cmask[0]))
        side.fork()
        with side:            # dW1[e] = Xc^T dz1[e]; every bias / LayerNorm / value-head gradient of the MLP in one launch
            ops.tgemm(wss, [ops.tgemm_problem(eng.Xc.data_ptr(), dz1.data_ptr(), sAm=1, sAk=FA, sBk=256, sBn=1, Z=E, sAz=0, sBz=B * 256,
                                              C_=P(G, f"{c}/Dense_0/kernel"), sCz=FA * 256, ldc=256)], FA, 256, B, splits=1, error=err)
            ops.small_grads([
                (L.SMALL_GRAD_COLSUM, dz2.data_ptr(), 256, None, 0, P(G, f"{c}/Dense_1/bias"), None, E, B, 256),
                (L.SMALL_GRAD_COLSUM, dz1.data_ptr(), 256, None, 0, P(G, f"{c}/Dense_0/bias"), None, E, B, 256),
                (L.SMALL_GRAD_LN, dy2.data_ptr(), 256, cm.xhat2.data_ptr(), 256, P(G, f"{c}/LayerNorm_1/scale"), P(G, f"{c}/LayerNorm_1/bias"), E, B, 256),
                (L.SMALL_GRAD_LN, dy1.data_ptr(), 256, cm.xhat1.data_ptr(), 256, P(G, f"{c}/LayerNorm_0/scale"), P(G, f"{c}/LayerNorm_0/bias"), E, B, 256),
                (L.SMALL_GRAD_HEAD, cm.h2.data_ptr(), 256, eng.dq.data_ptr(), 1, P(G, "modules_critic/Dense_0/kernel"), P(G, "modules_critic/Dense_0/bias"), 1, R, 256),
            ])
        # d enc = sum_e dz1[e] @ W1[e][:F]^T  (the input is broadcast over the ensemble; only the encoder columns are needed)
        # (the E partial products stay in the workspace; the encoder heads' LayerNorm backward sums them while it reads them)
        ops.tgemm(eng.ws, [ops.tgemm_problem(dz1.data_ptr(), P(Pm, f"{c}/Dense_0/kernel"), sAm=256, sAk=1, sBk=1, sBn=256, Z=E, sAz=B * 256, sBz=FA * 256)],
                  B, F, 256, epilogue=L.TGEMM_PARTIAL, splits=1, error=err)
        dXp, parts = eng.ws.buf, dict(dt_parts=E, dt_part_stride=B * F)
        # ---- trainable encoder heads ----
        off = 256 * ncam
        lnb, wg, dsle, jobs = [], [], [], []
        for j, cam in enumerate(cfg.cams):
            p = f"{ENC}/encoder_{cam}"
            dez, dey = eng.d_enc_z[cam], eng.d_enc_y[cam]
            lnb.append(dict(dt=ops.at(dXp, 256 * j), ld_dt=F, **parts, t=ops.at(eng.Xc, 256 * j), ld_t=FA, xhat=eng.enc_xhat[cam].data_ptr(),
                            rstd=eng.enc_rstd[cam].data_ptr(), scale=P(Pm, f"{p}/LayerNorm_0/scale"), rows_per_group=B, group_stride=0,
                            dz=dez.data_ptr(), dy=dey.data_ptr(), R=B, D=256))
            wg.append(ops.tgemm_problem(eng.sle_saved[cam].data_ptr(), dez.data_ptr(), sAm=1, sAk=4096, sBk=256, sBn=1, C_=P(G, f"{p}/Dense_0/kernel"), ldc=256))
            dsle.append(ops.tgemm_problem(dez.data_ptr(), P(Pm, f"{p}/Dense_0/kernel"), sAm=256, sAk=1, sBk=1, sBn=256, C_=self.d_sle[cam].data_ptr(), ldc=4096))
            jobs.append((L.SMALL_GRAD_COLSUM, dez.data_ptr(), 256, None, 0, P(G, f"{p}/Dense_0/bias"), None, 1, B, 256))
            jobs.append((L.SMALL_GRAD_LN, dey.data_ptr(), 256, eng.enc_xhat[cam].data_ptr(), 256, P(G, f"{p}/LayerNorm_0/scale"), P(G, f"{p}/LayerNorm_0/bias"), 1, B, 256))
        if cfg.use_proprio:
            lnb.append(dict(dt=ops.at(dXp, off), ld_dt=F, **parts, t=ops.at(eng.Xc, off), ld_t=FA, xhat=eng.enc_xhat_p.data_ptr(), rstd=eng.enc_rstd_p.data_ptr(),
                            scale=P(Pm, f"{ENC}/LayerNorm_0/scale"), rows_per_group=B, group_stride=0, dz=eng.d_enc_zp.data_ptr(), dy=eng.d_enc_yp.data_ptr(), R=B, D=64))
            jobs.append((L.SMALL_GRAD_COLSUM, eng.d_enc_zp.data_ptr(), 64, None, 0, P(G, f"{ENC}/Dense_0/bias"), None, 1, B, 64))
            jobs.append((L.SMALL_GRAD_LN, eng.d_enc_yp.data_ptr(), 64, eng.enc_xhat_p.data_ptr(), 64, P(G, f"{ENC}/LayerNorm_0/scale"), P(G, f"{ENC}/LayerNorm_0/bias"), 1, B, 64))
        ops.ln_tanh_bwd_multi(lnb)
        # encoder weight gradients on side stream 1: stream 0 may be busy with the early all-reduce of the critic bucket
        side1, wss1 = eng.side[1], eng.ws_side[1]
        side1.fork()
        with side1:
            ops.tgemm(wss1, wg, 4096, 256, B, splits=1, error=err)
            ops.small_grads(jobs)
            if cfg.use_proprio:
                ops.dense_bwd_weight(wss1, eng.state_o.data_ptr(), cfg.state_in, eng.d_enc_zp.data_ptr(), 64, P(G, f"{ENC}/Dense_0/kernel"), B, cfg.state_in, 64)
        ops.tgemm(eng.ws, dsle, B, 4096, 256, splits=1, error=err)
        ops.sle_bwd_multi(eng.ws, [(eng.feats[cam][slice(0, B)].data_ptr(), self.d_sle[cam].data_ptr(), 4096,
                                    P(G, f"{ENC}/encoder_{cam}/SpatialLearnedEmbeddings_0/kernel")) for cam in cfg.cams], B, 16, 512)
        side1.join()
        side.join()

    # ------------------------------------------------------------------------------------------------------------
    def actor_temp_loss_and_grads(self, keys, grad_scale=1.0, explicit=None, do_actor=True, do_temperature=True):
        """sac.py:193-234 on the fused kernels: the forward passes of the actor loss (policy on s with dropout, saved; critic on
        (s, pi(s)) with constant parameters) and of the temperature loss (policy on s' with a fresh dropout mask / sample) share
        one SLE launch, one k-split GEMM launch and one finish launch for their encoder passes and one launch per policy layer;
        the gradient w.r.t. the ACTION columns comes back through the same TF32 GEMMs.  The loss kernels and the policy backward
        (engine.policy_backward: policy MLP, heads and the proprio encoder's actor-tx twin) are the per-op ones."""
        eng = self.eng
        cfg, B, E, A, st = eng.cfg, eng.B, eng.cfg.ensemble, eng.cfg.action_dim, eng.store
        F, FA, ncam, S = eng.F, eng.FA, self.ncam, self.S
        Pm, P, err = st.params, eng.P, self.error
        obs_rows, next_rows = slice(0, B), slice(B, 2 * B)
        lam = P(Pm, "modules_temperature/lagrange")
        if not hasattr(self, "Xp_t"):
            e = lambda *sh: torch.empty(*sh, dtype=f32, device=eng.dev)
            self.Xp_t, self.eps_t, self.logp_t, self.h1_t, self.act_t = e(B, F), e(B, A), e(B), e(B, 256), e(B, A)
            self.masks_t = {c: torch.empty(B, 4096, dtype=torch.uint8, device=eng.dev) for c in cfg.cams}
            self.sle_c2 = {c: e(B, 4096) for c in cfg.cams}
            self.p_mask_t = eng.mlp_masks(cfg.policy_arch)          # the temperature pass's policy MLP masks
        parch, carch = cfg.policy_arch, cfg.critic_arch
        # ---- randomness ----
        jobs = []
        if do_actor:
            jobs.append((eng.eps, eng.masks_u8, eng.p_mask, L.KEY_ACTOR_SAMPLE, L.KEY_ACTOR_DROPOUT, None if explicit is None else explicit["actor"]))
        if do_temperature:
            jobs.append((self.eps_t, self.masks_t, self.p_mask_t, L.KEY_TEMP_NEXT, L.KEY_TEMP_NEXT, None if explicit is None else explicit["temperature"]))
        for eps, masks, pmask, k_eps, k_drop, ex in jobs:
            if ex is None:
                ops.normal_fill(ops.key_ptr(keys, k_eps), eps, B * A)
                for j, cam in enumerate(cfg.cams):
                    ops.dropout_mask_fill(ops.key_ptr(keys, k_drop), j, 0.9, masks[cam], B * 4096)
            else:
                eps.copy_(ex["eps"])
                for cam in cfg.cams:
                    masks[cam].copy_(ex["dropout"][cam])
            if pmask is not None:                                   # the policy MLP's masks, from the pass's dropout key
                eng.fill_mlp_masks(pmask, parch, ops.key_ptr(keys, k_drop), None if ex is None else ex.get("mlp_policy"))
        # ---- encoder passes: policy(s) with dropout [actor], critic input enc(s) [actor], policy(s') with dropout [temperature] ----
        passes = []
        if do_actor:
            passes += [(obs_rows, eng.state_o, eng.Xp, F, eng.masks_u8, self.sle_p, "pa"), (obs_rows, eng.state_o, eng.Xc, FA, None, self.sle_c2, None)]
        if do_temperature:
            passes += [(next_rows, eng.state_n, self.Xp_t, F, self.masks_t, self.sle_t, None)]
        sle, gemm, fin = [], [], []
        for pi, (rows, state, X, ldx, masks, sles, save) in enumerate(passes):
            for j, cam in enumerate(cfg.cams):
                p = f"{ENC}/encoder_{cam}"
                i = pi * ncam + j
                sle.append((eng.feats[cam][rows].data_ptr(), P(Pm, f"{p}/SpatialLearnedEmbeddings_0/kernel"),
                            None if masks is None else masks[cam].data_ptr(), sles[cam].data_ptr(), 4096))
                gemm.append(ops.tgemm_problem(sles[cam].data_ptr(), P(Pm, f"{p}/Dense_0/kernel"), sAm=4096, sAk=1, sBk=256, sBn=1))
                fin.append(dict(partials=self.ws_enc.buf.data_ptr() + 4 * i * S * B * 256, S=S, bias=P(Pm, f"{p}/Dense_0/bias"),
                                ln_scale=P(Pm, f"{p}/LayerNorm_0/scale"), ln_bias=P(Pm, f"{p}/LayerNorm_0/bias"), out=ops.at(X, 256 * j), ld_out=ldx, D=256))
        for rows, state, X, ldx, masks, sles, save in (passes if cfg.use_proprio else ()):
            # the policy's stop_gradient leaves the proprio Dense / LayerNorm differentiable (encoding.py:48-70): keep its statistics
            fin.append(dict(x=state.data_ptr(), ld_x=cfg.state_in, w=P(Pm, f"{ENC}/Dense_0/kernel"), K=cfg.state_in, bias=P(Pm, f"{ENC}/Dense_0/bias"),
                            ln_scale=P(Pm, f"{ENC}/LayerNorm_0/scale"), ln_bias=P(Pm, f"{ENC}/LayerNorm_0/bias"), out=ops.at(X, 256 * ncam), ld_out=ldx, D=64,
                            xhat=eng.enc_xhat_pa.data_ptr() if save == "pa" else None, rstd=eng.enc_rstd_pa.data_ptr() if save == "pa" else None))
        ops.sle_fwd_multi(sle, 0.9, B, 16, 512)
        ops.tgemm(self.ws_enc, gemm, B, 256, 4096, epilogue=L.TGEMM_PARTIAL, splits=S, error=err)
        ops.enc_finish(fin, B)
        # ---- policy MLP(s): layer 1, then layer 2 + heads + tanh-Gaussian sample ----
        n, pa = "modules_actor/network", eng.p_acts
        l1, l2 = [], []
        if do_actor:
            l1.append(ops.tgemm_problem(eng.Xp.data_ptr(), P(Pm, f"{n}/Dense_0/kernel"), sAm=F, sAk=1, sBk=256, sBn=1, C_=pa.h1.data_ptr(), ldc=256,
                                        bias=P(Pm, f"{n}/Dense_0/bias"), ln_scale=P(Pm, f"{n}/LayerNorm_0/scale"), ln_bias=P(Pm, f"{n}/LayerNorm_0/bias"),
                                        xhat=pa.xhat1.data_ptr(), rstd=pa.rstd1.data_ptr()))
            l2.append(ops.tgemm_problem(pa.h1.data_ptr(), P(Pm, f"{n}/Dense_1/kernel"), sAm=256, sAk=1, sBk=256, sBn=1, C_=pa.h2.data_ptr(), ldc=256,
                                        bias=P(Pm, f"{n}/Dense_1/bias"), ln_scale=P(Pm, f"{n}/LayerNorm_1/scale"), ln_bias=P(Pm, f"{n}/LayerNorm_1/bias"),
                                        xhat=pa.xhat2.data_ptr(), rstd=pa.rstd2.data_ptr(),
                                        head_w=P(Pm, "modules_actor/Dense_0/kernel"), head_b=P(Pm, "modules_actor/Dense_0/bias"), head_out=eng.mu.data_ptr(),
                                        head_w2=P(Pm, "modules_actor/Dense_1/kernel"), head_b2=P(Pm, "modules_actor/Dense_1/bias"), head_out2=eng.ls.data_ptr(),
                                        noise=eng.eps.data_ptr(), act=ops.at(eng.Xc, F), ld_act=FA, logp=eng.logp.data_ptr(), u_out=eng.u.data_ptr(),
                                        std_out=eng.std.data_ptr()))
        if do_temperature:
            l1.append(ops.tgemm_problem(self.Xp_t.data_ptr(), P(Pm, f"{n}/Dense_0/kernel"), sAm=F, sAk=1, sBk=256, sBn=1, C_=self.h1_t.data_ptr(), ldc=256,
                                        bias=P(Pm, f"{n}/Dense_0/bias"), ln_scale=P(Pm, f"{n}/LayerNorm_0/scale"), ln_bias=P(Pm, f"{n}/LayerNorm_0/bias")))
            l2.append(ops.tgemm_problem(self.h1_t.data_ptr(), P(Pm, f"{n}/Dense_1/kernel"), sAm=256, sAk=1, sBk=256, sBn=1,
                                        bias=P(Pm, f"{n}/Dense_1/bias"), ln_scale=P(Pm, f"{n}/LayerNorm_1/scale"), ln_bias=P(Pm, f"{n}/LayerNorm_1/bias"),
                                        head_w=P(Pm, "modules_actor/Dense_0/kernel"), head_b=P(Pm, "modules_actor/Dense_0/bias"), head_out=self.act_t.data_ptr(),
                                        head_w2=P(Pm, "modules_actor/Dense_1/kernel"), head_b2=P(Pm, "modules_actor/Dense_1/bias"),
                                        noise=self.eps_t.data_ptr(), act=self.act_t.data_ptr(), ld_act=A, logp=self.logp_t.data_ptr()))
        pmasks = [m for m, live in ((eng.p_mask, do_actor), (self.p_mask_t, do_temperature)) if live]
        ops.tgemm(None, l1, B, 256, F, epilogue=L.TGEMM_LN_TANH, error=err, **self._drop(parch, *[m and m[0] for m in pmasks]))
        ops.tgemm(None, l2, B, 256, 256, epilogue=L.TGEMM_LN_TANH_POLICY, head_n=A, std_min=cfg.std_min, std_max=cfg.std_max, error=err,
                  **self._drop(parch, *[m and m[1] for m in pmasks]))
        if do_actor:
            # ---- q = mean_e Q_e(s, pi(s)) with constant critic parameters; dQ/da through the same GEMMs ----
            c, cm = "modules_critic/network", eng.c_main
            R = E * B
            eng.pol_state = eng.state_o
            cmask = eng.c_mask or (None, None)                     # the critic on (s, pi(s)) drops out under the loss's critic_rng
            if eng.c_mask is not None:
                eng.fill_mlp_masks(eng.c_mask, carch, ops.key_ptr(keys, L.KEY_MLP_ACTOR_CRITIC),
                                   None if explicit is None else explicit["actor"].get("mlp_critic"))
            ops.tgemm(None, [ops.tgemm_problem(eng.Xc.data_ptr(), P(Pm, f"{c}/Dense_0/kernel"), sAm=FA, sAk=1, sBk=256, sBn=1, Z=E, sAz=0, sBz=FA * 256,
                                               C_=cm.h1.data_ptr(), sCz=B * 256, ldc=256, bias=P(Pm, f"{c}/Dense_0/bias"), sBiasZ=256,
                                               ln_scale=P(Pm, f"{c}/LayerNorm_0/scale"), ln_bias=P(Pm, f"{c}/LayerNorm_0/bias"), sLnZ=256,
                                               xhat=cm.xhat1.data_ptr(), rstd=cm.rstd1.data_ptr(), sXhatZ=B * 256, sRstdZ=B)],
                      B, 256, FA, epilogue=L.TGEMM_LN_TANH, error=err, **self._drop(carch, cmask[0]))
            ops.tgemm(None, [ops.tgemm_problem(cm.h1.data_ptr(), P(Pm, f"{c}/Dense_1/kernel"), sAm=256, sAk=1, sBk=256, sBn=1, Z=E, sAz=B * 256, sBz=256 * 256,
                                               C_=cm.h2.data_ptr(), sCz=B * 256, ldc=256, bias=P(Pm, f"{c}/Dense_1/bias"), sBiasZ=256,
                                               ln_scale=P(Pm, f"{c}/LayerNorm_1/scale"), ln_bias=P(Pm, f"{c}/LayerNorm_1/bias"), sLnZ=256,
                                               xhat=cm.xhat2.data_ptr(), rstd=cm.rstd2.data_ptr(), sXhatZ=B * 256, sRstdZ=B,
                                               head_w=P(Pm, "modules_critic/Dense_0/kernel"), head_b=P(Pm, "modules_critic/Dense_0/bias"),
                                               head_out=eng.q.data_ptr(), sHeadOutZ=B, ld_head=1)],
                      B, 256, 256, epilogue=L.TGEMM_LN_TANH_HEAD, head_n=1, error=err, **self._drop(carch, cmask[1]))
            ops.fill(eng.dq.data_ptr(), -grad_scale / (E * B), E * B)
            ops.ln_tanh_bwd_multi([dict(dq=eng.dq.data_ptr(), head_w=P(Pm, "modules_critic/Dense_0/kernel"), head_w_stride=0, t=cm.h2.data_ptr(), ld_t=256,
                                        xhat=cm.xhat2.data_ptr(), rstd=cm.rstd2.data_ptr(), scale=P(Pm, f"{c}/LayerNorm_1/scale"), rows_per_group=B,
                                        group_stride=256, dz=eng.dz.data_ptr(), R=R, D=256)], mask_rows=B, **self._drop(carch, cmask[1]))
            ops.tgemm(eng.ws, [ops.tgemm_problem(eng.dz.data_ptr(), P(Pm, f"{c}/Dense_1/kernel"), sAm=256, sAk=1, sBk=1, sBn=256, Z=E, sAz=B * 256, sBz=256 * 256,
                                                 C_=eng.dh.data_ptr(), sCz=B * 256, ldc=256)], B, 256, 256, splits=1, error=err)
            ops.ln_tanh_bwd_multi([dict(dt=eng.dh.data_ptr(), ld_dt=256, t=cm.h1.data_ptr(), ld_t=256, xhat=cm.xhat1.data_ptr(), rstd=cm.rstd1.data_ptr(),
                                        scale=P(Pm, f"{c}/LayerNorm_0/scale"), rows_per_group=B, group_stride=256, dz=eng.dz0.data_ptr(), R=R, D=256)],
                                  mask_rows=B, **self._drop(carch, cmask[0]))
            # dQ/da = sum_e dz1[e] @ W1[e][F:, :]^T: the action rows of the first layer only
            ops.tgemm(eng.ws, [ops.tgemm_problem(eng.dz0.data_ptr(), P(Pm, f"{c}/Dense_0/kernel") + 4 * F * 256, sAm=256, sAk=1, sBk=1, sBn=256, Z=E,
                                                 sAz=B * 256, sBz=FA * 256, C_=ops.at(eng.dX, F), sCz=0, ldc=FA)], B, A, 256, reduce_z=True, error=err)
            ops.actor_loss(eng.q, eng.logp, lam, ops.at(eng.dX, F), FA, ops.at(eng.Xc, F), FA, eng.std, eng.ls, eng.eps, cfg.std_min, cfg.std_max, grad_scale,
                           eng.dmu, eng.dls, ops.at(eng.info, 4), E, B, A)
            eng.policy_backward(eng.Xp)
        if do_temperature:
            ops.temperature_loss(self.logp_t, lam, cfg.target_entropy, grad_scale, P(st.grad, "modules_temperature/lagrange"), ops.at(eng.info, 8), B)

    def check_error(self):
        if int(self.error.item()):
            raise L.SerlError("tgemm_tf32_kernel: pipeline barrier timeout (flagged by the kernel)")
