"""Binary reward classifier on the hand-written sm_90a kernels (training and inference).

Mirrors the reference's `networks/reward_classifier.py:16-113` (BinaryClassifier, create_classifier, load_classifier_func)
and the `train_step` / augmentation of `examples/async_cable_route_drq/train_reward_classifier.py:108-157`:

    per camera k:  e_k   = tanh(LN(Dense_4096->256(Dropout_0.1(SLE(trunk(image_k))))))     (the DrQ encoder head; frozen trunk)
    x      = concat_k e_k                                                            (use_proprio=False: "state" is ignored)
    h      = relu(LN(Dropout_0.1(Dense_F->256(x))))                                  (dropout BEFORE the LayerNorm)
    logit  = Dense_256->1(h)
    loss   = mean(sigmoid_binary_cross_entropy(logit_train, label)),  accuracy = mean((sigmoid(logit_eval) >= 0.5) == label)

with one optax.adam(1e-4) over the whole tree (the trunk is stop-gradient: its update is exactly 0, so it is not stepped).
Unlike the agents, the classifier trains the image heads THROUGH their dropout: the SLE output gradient passes the dropout
mask (serl_dropout_bwd_f32) before the SLE kernel gradient.

Dropout keys (extends DESIGN.md §4 (i)): camera j's SLE mask = bernoulli(fold_in(key, j), 0.9, (B, 4096)); the hidden
Dropout_0 mask = bernoulli(fold_in(key, ncams), 0.9, (B, 256)).

Kernels: trunk (fp32 or wgmma build), one sle_fwd_multi for the train + eval passes, the image-head Dense on the TF32 tensor
cores (16-bit builds: serl_tgemm_tf32 k-split partials) or the CUDA-core SGEMM (fp32 build), one enc_finish, one 2-problem
Dense_0 launch, the LayerNorm-relu-head forward / backward and BCE kernels (csrc/classifier.cu), the batched head backward
(ln_tanh_bwd_multi, small_grads, sle_bwd_multi) and the fused Adam.  The parameters live in one `params.FlatParams` store
(`classifier._store`); the frozen trunk's subtree of `params` is read and written by `FrozenTrunk`.
"""
from __future__ import annotations

import types
from typing import Dict, Iterable, Optional

import numpy as np
import torch

from .. import _lib as L
from .. import ops
from ..engine import AgentConfig
from ..params import FlatParams, Leaf, assign_offsets, flatten, image_head_leaves, init_leaves, init_trunk, nest
from ..trunk import FrozenTrunk

f32 = torch.float32
ROOT = "encoder_def"
KEEP = 0.9
HIDDEN = 256


def classifier_spec(cams):
    """Trainable leaves in the Flax tree layout of BinaryClassifier (16-byte aligned in one flat buffer)."""
    leaves = [l for cam in cams for l in image_head_leaves(f"{ROOT}/encoder_{cam}")]
    F = 256 * len(cams)
    leaves += [Leaf("Dense_0/kernel", (F, HIDDEN), 0), Leaf("Dense_0/bias", (HIDDEN,), 0), Leaf("LayerNorm_0/scale", (HIDDEN,), 0),
               Leaf("LayerNorm_0/bias", (HIDDEN,), 0), Leaf("Dense_1/kernel", (HIDDEN, 1), 0), Leaf("Dense_1/bias", (1,), 0)]
    return leaves, assign_offsets(leaves)


TRUNK_PATH = ROOT + "/encoder_{}/pretrained_encoder"


def _key_array(key) -> np.ndarray:
    if isinstance(key, torch.Tensor):
        key = key.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(key).astype(np.uint32).reshape(2))


def _check_frames(shape, what):
    """enable_stacking with T=1 at 128x128, like the agents' trunk kernels."""
    if len(shape) < 4 or tuple(shape[-4:]) != (1, 128, 128, 3):
        raise NotImplementedError(f"{what}: the classifier takes (..., 1, 128, 128, 3) frames (obs_horizon 1, 128x128), got {tuple(shape)}")


class RewardClassifier:
    """`TrainState` of the reference classifier: flat fp32 params + Adam moments in HBM, the frozen trunk per camera."""

    def __init__(self, cams, spec, trunk, precision, device):
        self.cams, self._trunk, self.device = tuple(cams), trunk, torch.device(device)
        self._cfg = AgentConfig(cams=self.cams, state_in=1, action_dim=1, pixel=True, image_hw=128, precision=precision)
        self._frozen_trunk = FrozenTrunk(trunk, precision, 128)
        self._store = FlatParams(spec, device, target=False)
        # the store's layout, parameter and gradient buffers (the same tensors) under the names the GPU parity tests read
        self._spec, self._n, self._params, self._grad = spec, self._store.n, self._store.params, self._store.grad
        self._info = torch.zeros(4, dtype=f32, device=device)
        self._key = torch.zeros(2, dtype=torch.uint32, device=device)
        self.learning_rate = 1e-4
        self.step = 0
        self.explicit_dropout = None            # tests: {"sle": {cam: (B, 4096) keep mask}, "hidden": (B, 256)} instead of the keyed masks
        self._bufs: Dict[int, dict] = {}
        self._tree = None                       # the tree `params` last returned (apply_fn evaluates exactly that one)

    @property
    def precision(self):
        return self._cfg.precision

    # ---- parameters in the Flax layout ---------------------------------------------------------------------
    @property
    def params(self):
        if self._tree is None:
            self._tree = nest({**self._store.dump(self._store.params), **self._frozen_trunk.dump(TRUNK_PATH.format)})
        return self._tree

    @property
    def opt_state(self):
        st = self._store
        return {"count": int(st.counts[0].item()), "mu": nest(st.dump(st.m)), "nu": nest(st.dump(st.v))}

    def replace(self, **kw):
        """classifier.replace(params=tree[, step=n]): writes the trainable leaves and the frozen trunk from a Flax-layout tree."""
        if "params" in kw:
            flat = flatten(kw.pop("params"))
            self._store.load(self._store.params, flat)
            self._frozen_trunk.load(flat, TRUNK_PATH.format)
            self._tree = None
        if "step" in kw:
            self.step = int(kw.pop("step"))
        if kw:
            raise TypeError(f"replace: unknown fields {sorted(kw)}")
        return self

    def state_dict(self) -> dict:
        return {"step": int(self.step), "params": self.params, "opt_state": self.opt_state}

    def load_state_dict(self, d: dict) -> "RewardClassifier":
        self.replace(params=d["params"], step=d["step"])
        o, st = d["opt_state"], self._store
        st.load(st.m, flatten(o["mu"]))
        st.load(st.v, flatten(o["nu"]))
        st.counts[0] = int(o["count"])
        return self

    # ---- device scratch per batch size -------------------------------------------------------------------
    def _splits(self, B, nprob):
        return ops.tgemm_splits(4096, max(1, min(132 // (nprob * ((B + 127) // 128)), 32)))

    def _b(self, B):
        if B not in self._bufs:
            cfg, dev, nc = self._cfg, self.device, len(self.cams)
            e = lambda *s: torch.empty(*s, dtype=f32, device=dev)
            u8 = lambda *s: torch.empty(*s, dtype=torch.uint8, device=dev)
            F = 256 * nc
            fp32 = cfg.precision == "fp32"
            S2, S1 = (1, 1) if fp32 else (self._splits(B, 2 * nc), self._splits(B, nc))
            self._bufs[B] = dict(
                trunk=self._frozen_trunk.runner(B, dev), ws=ops.Workspace(48 << 20, dev, "f32" if fp32 else "tf32x3"),
                ws_enc=ops.Workspace(max(2 * nc * S2, nc * S1) * B * 256 * 4, dev), S2=S2, S1=S1,
                pix={c: u8(B, 128, 128, 3) for c in self.cams}, feats={c: e(B, 4, 4, 512) for c in self.cams},
                masks=u8(nc, B, 4096), hmask=u8(B, HIDDEN), sle={c: e(2, B, 4096) for c in self.cams},
                enc_xhat={c: e(B, 256) for c in self.cams}, enc_rstd={c: e(B) for c in self.cams},
                X=e(2, B, F), z=e(2, B, HIDDEN), h=e(B, HIDDEN), xhat=e(B, HIDDEN), rstd=e(B), logits=e(2, B), labels=e(B),
                dlogit=e(B), dy=e(B, HIDDEN), dz=e(B, HIDDEN), dX=e(B, F), dez={c: e(B, 256) for c in self.cams},
                dey={c: e(B, 256) for c in self.cams}, d_sle=e(nc, B, 4096), err=torch.zeros(1, dtype=torch.int32, device=dev))
        return self._bufs[B]

    def _ingest(self, b, data):
        """Observation dict (host or device; (B, 1, 128, 128, 3) or unbatched (1, 128, 128, 3) frames) -> pixel buffers."""
        for cam in self.cams:
            px = data[cam]
            px = px if isinstance(px, torch.Tensor) else torch.as_tensor(np.asarray(px))
            _check_frames(px.shape, "RewardClassifier")
            b["pix"][cam].copy_(px.reshape(b["pix"][cam].shape).to(self.device, torch.uint8))

    @staticmethod
    def _rows(data, cams):
        px = data[cams[0]]
        shape = tuple(px.shape)
        _check_frames(shape, "RewardClassifier")
        return (1, True) if len(shape) == 4 else (int(np.prod(shape[:-4])), False)

    # ---- forward -------------------------------------------------------------------------------------------
    def _image_heads(self, b, B, passes):
        """passes: list of (pass index t into sle / X, masked, save).  One SLE launch, the Dense(4096 -> 256) GEMMs, one finish."""
        nc, fp32 = len(self.cams), self._cfg.precision == "fp32"
        F = 256 * nc
        S = 1 if fp32 else (b["S2"] if len(passes) == 2 else b["S1"])
        wsb = b["ws_enc"].buf
        sle, fin, gemm = [], [], []
        for i, (t, masked, save) in enumerate(passes):
            for j, cam in enumerate(self.cams):
                p = f"{ROOT}/encoder_{cam}"
                q = i * nc + j
                sle.append((b["feats"][cam].data_ptr(), self._store.P(f"{p}/SpatialLearnedEmbeddings_0/kernel"),
                            ops.at(b["masks"], j * B * 4096) if masked else None, b["sle"][cam][t].data_ptr(), 4096))
                gemm.append(ops.tgemm_problem(b["sle"][cam][t].data_ptr(), self._store.P(f"{p}/Dense_0/kernel"), sAm=4096, sAk=1, sBk=256, sBn=1))
                fin.append(dict(partials=ops.at(wsb, q * S * B * 256), S=S, bias=self._store.P(f"{p}/Dense_0/bias"), ln_scale=self._store.P(f"{p}/LayerNorm_0/scale"),
                                ln_bias=self._store.P(f"{p}/LayerNorm_0/bias"), out=ops.at(b["X"][t], 256 * j), ld_out=F, D=256,
                                xhat=b["enc_xhat"][cam].data_ptr() if save else None, rstd=b["enc_rstd"][cam].data_ptr() if save else None))
        ops.sle_fwd_multi(sle, KEEP, B, 16, 512)
        if fp32:
            # CUDA-core SGEMM, one launch per camera over its passes: partial[q] = sle[cam][t] @ W_cam (bias added by the finish)
            for j, cam in enumerate(self.cams):
                ts = [t for t, _, _ in passes]
                ops.gemm(b["ws"], b["sle"][cam][ts[0]].data_ptr(), self._store.P(f"{ROOT}/encoder_{cam}/Dense_0/kernel"), ops.at(wsb, j * B * 256),
                         B, 256, 4096, sAm=4096, sAk=1, sBk=256, sBn=1, ldc=256, Z=len(ts), sAz=B * 4096 * (ts[-1] - ts[0] if len(ts) > 1 else 0),
                         sBz=0, sCz=nc * B * 256)
        else:
            for q0 in range(0, len(gemm), L.TGEMM_MAX_PROBLEMS):        # 4 cameras x 2 passes: two launches
                chunk = gemm[q0:q0 + L.TGEMM_MAX_PROBLEMS]
                view = types.SimpleNamespace(buf=wsb[q0 * S * B * 256:], nbytes=b["ws_enc"].nbytes - 4 * q0 * S * B * 256)
                ops.tgemm(view, chunk, B, 256, 4096, epilogue=L.TGEMM_PARTIAL, splits=S, error=b["err"])
        ops.enc_finish(fin, B)

    def _dense0(self, b, B, ts):
        """z[t] = X[t] @ W0 + b0 for the passes ts: one launch."""
        F = 256 * len(self.cams)
        if self._cfg.precision == "fp32":
            ops.dense_fwd(b["ws"], b["X"][ts[0]].data_ptr(), F, self._store.P("Dense_0/kernel"), self._store.P("Dense_0/bias"), b["z"][ts[0]].data_ptr(), HIDDEN,
                          B, F, HIDDEN, Z=len(ts), x_z=B * F, w_z=0, b_z=0, out_z=B * HIDDEN)
        else:
            probs = [ops.tgemm_problem(b["X"][t].data_ptr(), self._store.P("Dense_0/kernel"), sAm=F, sAk=1, sBk=HIDDEN, sBn=1, C_=b["z"][t].data_ptr(),
                                       ldc=HIDDEN, bias=self._store.P("Dense_0/bias")) for t in ts]
            ops.tgemm(b["ws"], probs, B, HIDDEN, F, splits=1, error=b["err"])

    def _trunk_forward(self, b):
        for cam in self.cams:
            b["trunk"].forward(cam, b["pix"][cam], b["feats"][cam])

    def _eval_logits(self, b, B):
        """train=False forward of the classifier on the ingested pixels -> b["logits"][1]."""
        self._trunk_forward(b)
        self._image_heads(b, B, [(1, False, False)])
        self._dense0(b, B, [1])
        ops.ln_relu_head_fwd(b["z"][1].data_ptr(), None, KEEP, self._store.P("LayerNorm_0/scale"), self._store.P("LayerNorm_0/bias"), self._store.P("Dense_1/kernel"),
                             self._store.P("Dense_1/bias"), None, None, None, b["logits"][1].data_ptr(), B)
        return b["logits"][1]

    def __call__(self, observations, train: bool = False):
        """Logits of BinaryClassifier(obs, train=False): (B, 1) for batched observations, (1,) for one (1, 128, 128, 3) observation."""
        if train:
            raise NotImplementedError("RewardClassifier: the dropout forward runs inside train_step only")
        B, single = self._rows(observations, self.cams)
        b = self._b(B)
        self._ingest(b, observations)
        out = self._eval_logits(b, B).clone()
        return out.view(1) if single else out.view(B, 1)

    def apply_fn(self, variables, observations, train: bool = False, rngs=None):
        """classifier.apply_fn({"params": classifier.params}, obs, train=False): evaluates this classifier's own parameters."""
        if variables.get("params") is not self.params:
            raise NotImplementedError("RewardClassifier.apply_fn evaluates the classifier's own `params` tree only")
        return self(observations, train=train)

    # ---- training step (train_reward_classifier.py:121-137) -------------------------------------------------
    def _masks(self, b, B, key):
        nc = len(self.cams)
        if self.explicit_dropout is not None:
            for j, cam in enumerate(self.cams):
                b["masks"][j].copy_(torch.as_tensor(np.asarray(self.explicit_dropout["sle"][cam])).to(self.device, torch.uint8))
            b["hmask"].copy_(torch.as_tensor(np.asarray(self.explicit_dropout["hidden"])).to(self.device, torch.uint8))
            return
        self._key.copy_(torch.from_numpy(_key_array(key).view(np.int32)).view(torch.uint32))
        for j in range(nc):
            ops.dropout_mask_fill(self._key.data_ptr(), j, KEEP, b["masks"][j], B * 4096)
        ops.dropout_mask_fill(self._key.data_ptr(), nc, KEEP, b["hmask"], B * HIDDEN)

    def train_step(self, batch, key):
        from ..data.replay_buffer import refuse_nstep, refuse_prioritized
        refuse_nstep(batch, "RewardClassifier.train_step", "the classifier reads no rewards")
        refuse_prioritized(batch, "RewardClassifier.train_step")
        data, labels = batch["data"], batch["labels"]
        B, single = self._rows(data, self.cams)
        if single:
            raise ValueError("train_step: batched observations (B, 1, 128, 128, 3) expected")
        b, nc, fp32 = self._b(B), len(self.cams), self._cfg.precision == "fp32"
        F = 256 * nc
        self._ingest(b, data)
        lab = labels if isinstance(labels, torch.Tensor) else torch.as_tensor(np.asarray(labels))
        b["labels"].copy_(lab.reshape(B).to(self.device, f32))
        self._masks(b, B, key)
        P, G, ws = self._store.P, self._store.G, b["ws"]
        err = b["err"]
        # ---- forward: trunk once, then the train (dropout) and eval passes side by side ----
        self._trunk_forward(b)
        self._image_heads(b, B, [(0, True, True), (1, False, False)])
        self._dense0(b, B, [0, 1])
        ops.ln_relu_head_fwd(b["z"][0].data_ptr(), b["hmask"].data_ptr(), KEEP, P("LayerNorm_0/scale"), P("LayerNorm_0/bias"), P("Dense_1/kernel"),
                             P("Dense_1/bias"), b["h"].data_ptr(), b["xhat"].data_ptr(), b["rstd"].data_ptr(), b["logits"][0].data_ptr(), B)
        ops.ln_relu_head_fwd(b["z"][1].data_ptr(), None, KEEP, P("LayerNorm_0/scale"), P("LayerNorm_0/bias"), P("Dense_1/kernel"),
                             P("Dense_1/bias"), None, None, None, b["logits"][1].data_ptr(), B)
        ops.bce_logits_loss(b["logits"][0].data_ptr(), b["logits"][1].data_ptr(), b["labels"].data_ptr(), 1.0, b["dlogit"].data_ptr(),
                            self._info.data_ptr(), B)
        # ---- backward: Dense_1 -> LayerNorm / relu / dropout -> Dense_0 ----
        ops.ln_relu_head_bwd(b["dlogit"].data_ptr(), P("Dense_1/kernel"), b["h"].data_ptr(), b["xhat"].data_ptr(), b["rstd"].data_ptr(),
                             P("LayerNorm_0/scale"), b["hmask"].data_ptr(), KEEP, b["dy"].data_ptr(), b["dz"].data_ptr(), B)
        X0 = b["X"][0].data_ptr()
        if fp32:
            ops.dense_bwd_weight(ws, X0, F, b["dz"].data_ptr(), HIDDEN, G("Dense_0/kernel"), B, F, HIDDEN)
            ops.dense_bwd_input(ws, b["dz"].data_ptr(), HIDDEN, P("Dense_0/kernel"), b["dX"].data_ptr(), F, B, F, HIDDEN)
        else:
            ops.tgemm(ws, [ops.tgemm_problem(X0, b["dz"].data_ptr(), sAm=1, sAk=F, sBk=HIDDEN, sBn=1, C_=G("Dense_0/kernel"), ldc=HIDDEN)],
                      F, HIDDEN, B, splits=1, error=err)
            ops.tgemm(ws, [ops.tgemm_problem(b["dz"].data_ptr(), P("Dense_0/kernel"), sAm=HIDDEN, sAk=1, sBk=1, sBn=HIDDEN, C_=b["dX"].data_ptr(), ldc=F)],
                      B, F, HIDDEN, splits=1, error=err)
        jobs = [(L.SMALL_GRAD_COLSUM, b["dz"].data_ptr(), HIDDEN, None, 0, G("Dense_0/bias"), None, 1, B, HIDDEN),
                (L.SMALL_GRAD_LN, b["dy"].data_ptr(), HIDDEN, b["xhat"].data_ptr(), HIDDEN, G("LayerNorm_0/scale"), G("LayerNorm_0/bias"), 1, B, HIDDEN),
                (L.SMALL_GRAD_HEAD, b["h"].data_ptr(), HIDDEN, b["dlogit"].data_ptr(), 1, G("Dense_1/kernel"), G("Dense_1/bias"), 1, B, HIDDEN)]
        # ---- image heads: LayerNorm + tanh backward, Dense weight / input gradients, dropout, SLE kernel gradient ----
        lnb, wg, dsle = [], [], []
        for j, cam in enumerate(self.cams):
            p = f"{ROOT}/encoder_{cam}"
            dez, dey = b["dez"][cam].data_ptr(), b["dey"][cam].data_ptr()
            lnb.append(dict(dt=ops.at(b["dX"], 256 * j), ld_dt=F, t=ops.at(b["X"][0], 256 * j), ld_t=F, xhat=b["enc_xhat"][cam].data_ptr(),
                            rstd=b["enc_rstd"][cam].data_ptr(), scale=P(f"{p}/LayerNorm_0/scale"), rows_per_group=B, group_stride=0, dz=dez, dy=dey, R=B, D=256))
            jobs.append((L.SMALL_GRAD_COLSUM, dez, 256, None, 0, G(f"{p}/Dense_0/bias"), None, 1, B, 256))
            jobs.append((L.SMALL_GRAD_LN, dey, 256, b["enc_xhat"][cam].data_ptr(), 256, G(f"{p}/LayerNorm_0/scale"), G(f"{p}/LayerNorm_0/bias"), 1, B, 256))
            sle0, d_sle = b["sle"][cam][0].data_ptr(), b["d_sle"][j].data_ptr()
            if fp32:
                wg.append((sle0, dez, G(f"{p}/Dense_0/kernel")))
                dsle.append((dez, P(f"{p}/Dense_0/kernel"), d_sle))
            else:
                wg.append(ops.tgemm_problem(sle0, dez, sAm=1, sAk=4096, sBk=256, sBn=1, C_=G(f"{p}/Dense_0/kernel"), ldc=256))
                dsle.append(ops.tgemm_problem(dez, P(f"{p}/Dense_0/kernel"), sAm=256, sAk=1, sBk=1, sBn=256, C_=d_sle, ldc=4096))
        ops.ln_tanh_bwd_multi(lnb)
        if fp32:
            for (x, dz_, dw), (dz2, w, dx) in zip(wg, dsle):
                ops.dense_bwd_weight(ws, x, 4096, dz_, 256, dw, B, 4096, 256)
                ops.dense_bwd_input(ws, dz2, 256, w, dx, 4096, B, 4096, 256)
        else:
            ops.tgemm(ws, wg, 4096, 256, B, splits=1, error=err)
            ops.tgemm(ws, dsle, B, 4096, 256, splits=1, error=err)
        ops.dropout_bwd(b["d_sle"].data_ptr(), b["masks"].data_ptr(), KEEP, nc * B * 4096)      # the train pass ran with dropout
        ops.sle_bwd_multi(ws, [(b["feats"][cam].data_ptr(), b["d_sle"][j].data_ptr(), 4096, G(f"{ROOT}/encoder_{cam}/SpatialLearnedEmbeddings_0/kernel"))
                               for j, cam in enumerate(self.cams)], B, 16, 512)
        ops.small_grads(jobs)
        # ---- optax.adam(1e-4) over the trainable tree ----
        ops.adam_single(self._store, self.learning_rate)
        self.step += 1
        self._tree = None
        info = self._info.clone()
        return self, info[0], info[1]

    def check_status(self):
        for b in self._bufs.values():
            if int(b["err"].item()):
                raise L.SerlError("tgemm_tf32_kernel: pipeline barrier timeout (flagged by the kernel)")
        self._frozen_trunk.check_error()


def _register_flax_serialization():
    try:
        from flax import serialization
    except Exception:                                   # noqa: BLE001
        return False
    try:
        serialization.register_serialization_state(RewardClassifier, lambda s: s.state_dict(), lambda s, d: s.load_state_dict(d))
    except ValueError:
        pass
    return True


_register_flax_serialization()


# ---- reference API ------------------------------------------------------------------------------------------
def create_classifier(key, sample, image_keys: Iterable[str], pretrained_encoder_path: str = "./resnet10_params.pkl", *,
                      precision: str = "fp32", device=None) -> RewardClassifier:
    """networks/reward_classifier.py:31-89.  `sample`: an observation dict (batched or not); only its frame shapes are read."""
    cams = tuple(image_keys)
    for cam in cams:
        _check_frames(np.shape(sample[cam]) if not isinstance(sample[cam], torch.Tensor) else tuple(sample[cam].shape), "create_classifier")
    if precision not in ("fp32", "fp16", "bf16"):
        raise ValueError(f"create_classifier: precision {precision!r} (fp32 | fp16 | bf16)")
    L.load()
    device = torch.device(device if device is not None else "cuda")
    L.require_cuda(device)
    k = _key_array(key)
    rng = np.random.default_rng((int(k[0]) << 32) | int(k[1]))
    spec, _ = classifier_spec(cams)
    trunk = {cam: {kk: torch.as_tensor(v).to(device).contiguous() for kk, v in init_trunk(rng).items()} for cam in cams}
    clf = RewardClassifier(cams, spec, trunk, precision, device)
    clf._store.load(clf._store.params, init_leaves(rng, spec))      # flax nn.Dense / SLE defaults: lecun_normal kernels throughout
    from ..utils.train_utils import _resnet10_pickle, replace_pretrained_leaves
    encoder_params = _resnet10_pickle(pretrained_encoder_path)
    if encoder_params is not None:
        clf.replace(params=replace_pretrained_leaves(clf.params, encoder_params, cams, root=(ROOT,)))
    return clf


def train_step(classifier: RewardClassifier, batch, key):
    """The script's jitted train_step: (classifier, loss, accuracy); loss / accuracy are 0-d device tensors."""
    return classifier.train_step(batch, key)


def sample_classifier_batch(pos_buffer, neg_buffer, batch_size: int, key):
    """train_reward_classifier.py:142-157 on the device: B/2 positive NEXT observations, then B/2 negative observations, cropped by
    one batched_random_crop(key, padding=4) over the concatenated batch (frame i uses split(key, B)[i]), labels 1 then 0.
    Returns {"data": {cam: (B, 1, H, W, 3) uint8}, "labels": (B, 1) float32}, all on the device."""
    B = int(batch_size)
    if B % 2:
        raise ValueError("sample_classifier_batch: batch_size must be even")
    cams = tuple(pos_buffer.cams)
    if tuple(neg_buffer.cams) != cams or pos_buffer.T != 1 or neg_buffer.T != 1:
        raise NotImplementedError("sample_classifier_batch: both buffers hold the same cameras with obs_horizon 1")
    dev = pos_buffer.device
    H, W, Cc = pos_buffer.frame_shape
    data = {c: torch.empty(B, 1, H, W, Cc, dtype=torch.uint8, device=dev) for c in cams}
    sc = _sample_scratch(pos_buffer, neg_buffer, B)
    sc["key"].copy_(torch.from_numpy(_key_array(key).view(np.int32)).view(torch.uint32))
    sc["status"].zero_()
    for ring, row, take_next in ((pos_buffer, 0, True), (neg_buffer, B // 2, False)):
        out = L.BatchOut()
        for j, c in enumerate(cams):                  # the half of each launch the script does not keep goes to scratch
            out.obs_pix[j] = (sc["pix"] if take_next else data)[c].data_ptr()
            out.next_pix[j] = (data if take_next else sc["pix"])[c].data_ptr()
        out.obs_state, out.next_state, out.actions = sc["state"].data_ptr(), sc["state"].data_ptr(), sc["actions"].data_ptr()
        out.rewards, out.masks, out.dones, out.status = sc["r"].data_ptr(), sc["r"].data_ptr(), sc["dones"].data_ptr(), sc["status"].data_ptr()
        part = ring.sample(B // 2).parts[0]
        ring.launch_sample(part, out, crop_total=B, out_row_offset=row, key_obs=sc["key"].data_ptr(), key_next=sc["key"].data_ptr())
    if int(sc["status"].item()):
        raise L.SerlError("sample_classifier_batch: a replay draw found no valid slot within the redraw budget")
    return {"data": data, "labels": sc["labels"].clone()}


_SAMPLE_SCRATCH: Dict[tuple, dict] = {}


def _sample_scratch(pos_buffer, neg_buffer, B):
    """Per (buffers, batch size): sampler outputs the classifier batch does not use, the key and the constant labels."""
    k = (id(pos_buffer), id(neg_buffer), B)
    if k not in _SAMPLE_SCRATCH:
        dev = pos_buffer.device
        H, W, Cc = pos_buffer.frame_shape
        ns = max(pos_buffer.T * pos_buffer.S, neg_buffer.T * neg_buffer.S, 1)
        na = max(pos_buffer.A, neg_buffer.A, 1)
        e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        _SAMPLE_SCRATCH[k] = dict(pix={c: torch.empty(B, H, W, Cc, dtype=torch.uint8, device=dev) for c in pos_buffer.cams},
                                  state=e(B, ns), actions=e(B, na), r=e(B), dones=torch.empty(B, dtype=torch.uint8, device=dev),
                                  status=torch.zeros(1, dtype=torch.int32, device=dev), key=torch.zeros(2, dtype=torch.uint32, device=dev),
                                  labels=torch.cat([torch.ones(B // 2, 1), torch.zeros(B // 2, 1)]).to(dev))
    return _SAMPLE_SCRATCH[k]


def load_classifier_func(key, sample, image_keys, checkpoint_path: str, step: Optional[int] = None, *, precision: str = "fp32", device=None):
    """networks/reward_classifier.py:92-113: a callable obs -> logits of the restored classifier ((1,) for one observation)."""
    from ..utils.checkpoints import restore_checkpoint
    classifier = create_classifier(key, sample, image_keys, precision=precision, device=device)
    classifier = restore_checkpoint(checkpoint_path, target=classifier, step=step)
    return lambda obs: classifier(obs, train=False)
