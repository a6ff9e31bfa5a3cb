"""GPU: the reward classifier's train_step at its training batch and at the batch sizes where its kernels change regime, against
oracle/classifier.py fed the classifier's OWN frozen-trunk features (`oracle.classifier.features` replaced by a lookup of the
feature table the classifier's trunk wrote, after the classifier's pixel buffers are checked bit for bit against the batch).

With the trunk's rounding out of the comparison the 16-bit build's heads, which run the image-head Dense and its gradients as
3xTF32 tgemm problems, are held to the fused heads' bars (tests/test_heads_grads_b256_gpu.py) rather than the 1e-2 the fp16
trunk forces on tests/test_reward_classifier_gpu.py.  Per step: the keyed dropout masks bit-exact; train logits, eval logits and
the loss within `tol * max(|ref|, 1)` (fp32 build 1e-5, 16-bit build 1e-4); the accuracy exact except for rows whose oracle
eval logit lies within that tolerance of 0; every trainable gradient leaf non-zero and within 2e-4 of its own max; post-Adam
parameters under the noise-aware bar of DESIGN.md §5.  Two steps with different keys, then the frozen trunk bitwise unchanged,
`check_status()` clean, and a twin classifier's first step bitwise equal.

The oracle takes the hidden relu's active set from the classifier's own train pass (`hidden_live`), and every unit where the two
disagree must have a float64 pre-activation within the logit tolerance of 0.  Such a unit takes the other branch of relu's
derivative, which moves Dense_0 and every image-head leaf by about 1/B of their max.  On the 16-bit build, whose
pre-activations carry ~1e-6 of 3xTF32 rounding, one of the 262,144 units of the B = 1024 case's second step does so; without
this rule it moved Dense_0's kernel gradient by 3.05e-3 of its max (on an H100 80GB HBM3 at 700 W), and a bar that passed it
would not catch a lost row.

What each case reaches (S2 / S1: the image-head tgemm k-split of the train + eval launch / of the eval-only launch):
  script batch   fp16 and fp32, two cameras, B = 256 drawn by sample_classifier_batch from two rings (128 + 128), the reference
                 script's configuration: S2 = 16, S1 = 32, two 128-row M tiles, eight 32-row k-blocks in the weight gradients,
                 dropout_bwd's grid-stride loop (2 M elements); also a float64 trunk sample and a negative control.
  B = 2          one partial 8-row block in ln_relu_head_fwd / _bwd, a 2-row k-block.
  B = 128 / 130  one and two cameras: a 2-row second M tile, S2 falling from 32 to 16 with two cameras, R % 8 = 2.
  B = 258        a third M tile; two threads of bce_logits_loss take two rows each.
  B = 1024       S2 = 4, eight M tiles, four rows per bce_logits_loss thread.
  three cameras  B = 130: exactly SERL_TGEMM_MAX_PROBLEMS = 6 image-head problems in one launch.
  four cameras   B = 256: 8 problems in two tgemm launches, the second writing its partials through the workspace view at
                 q0 * S * B * 256; 11 small_grads jobs (the cap is 12).
  fp32 build     B = 2, 256, 1024: the SGEMM path, gemm with Z = 2 passes and dense_bwd_weight with K = B and its split-K.
Also: clf(obs) at 1, 3 and 257 rows and a checkpoint-restored load_classifier_func on one observation against the oracle's
train=False forward on the classifier's own features, and sample_classifier_batch at B = 256 and 1024 bit-exact against the replay
oracle plus the crop.  Measured errors per case: DESIGN.md §5."""
import copy
import os

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions, rel_err
from test_reward_classifier_gpu import _batch, _classifier, _flat

pytestmark = pytest.mark.gpu

BARS = {"fp32": 1e-5, "fp16": 1e-4}      # train / eval logits and loss, |got - ref| / max(|ref|, 1)
LEAF_TOL = 2e-4                          # every gradient leaf, max |got - ref| / max |ref|
TRUNK_ROWS = [0, 1, 127, 128, 129, 255]  # both M tiles' edges of the 256-row batch
TRUNK_TOL = {"fp16": 5e-3, "fp32": 2e-5}
KEYS = (np.array([0, 17], np.uint32), np.array([5, 2], np.uint32))
CAMS = ("front", "wrist", "side", "top")

#         precision, cameras, B, S2 (None: fp32 build, no k-split)
CASES = {
    "fp16-c2-b256-script": ("fp16", 2, 256, 16),
    "fp16-c2-b2": ("fp16", 2, 2, 32),
    "fp16-c1-b128": ("fp16", 1, 128, 32),
    "fp16-c1-b130": ("fp16", 1, 130, 32),
    "fp16-c2-b128": ("fp16", 2, 128, 32),
    "fp16-c2-b130": ("fp16", 2, 130, 16),
    "fp16-c2-b258": ("fp16", 2, 258, 11),
    "fp16-c2-b1024": ("fp16", 2, 1024, 4),
    "fp16-c3-b130": ("fp16", 3, 130, 11),
    "fp16-c4-b256": ("fp16", 4, 256, 8),
    "fp32-c2-b2": ("fp32", 2, 2, None),
    "fp32-c2-b256-script": ("fp32", 2, 256, None),
    "fp32-c2-b1024": ("fp32", 2, 1024, None),
}


def _scaled(got, ref):
    got, ref = np.asarray(got, np.float64).reshape(-1), np.asarray(ref, np.float64).reshape(-1)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1.0))


def _rings(cams, n):
    """A positive and a negative ring of n transitions each, with their replay oracles."""
    from oracle.replay import OracleFrameRing
    from serl_b200.utils.launcher import make_replay_buffer
    rng = np.random.default_rng(n)
    rings = []
    for seed in (21, 22):
        dev = make_replay_buffer(fake_env(cams), capacity=n, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=seed)
        ora = OracleFrameRing(n, cams, (128, 128, 3), 1, 7, 4)
        for tr in random_transitions(rng, n, cams):
            dev.insert(tr)
            ora.insert(tr)
        rings.append((dev, ora))
    return rings


def _sample_checked(rings, cams, B, key):
    """sample_classifier_batch(pos, neg, B, key) with its indices, crops and labels checked bit-exact; (device batch, host copy)."""
    from oracle import classifier as OC
    from oracle.replay import draw_indices
    from serl_b200.networks.reward_classifier import sample_classifier_batch
    (pos, opos), (neg, oneg) = rings
    steps = (pos._draw_step, neg._draw_step)
    batch = sample_classifier_batch(pos, neg, B, key)
    ip = draw_indices(pos._seed, steps[0], B // 2, opos.size, opos.valid)
    ineg = draw_indices(neg._seed, steps[1], B // 2, oneg.size, oneg.valid)
    gp, gn = opos.gather_packed(ip), oneg.gather_packed(ineg)
    ref = OC.crop_batch({c: gp["observations"][c][:, 1:] for c in cams}, {c: gn["observations"][c][:, :1] for c in cams}, key)
    host = {"data": {c: batch["data"][c].cpu().numpy() for c in cams}, "labels": batch["labels"].cpu().numpy()}
    for c in cams:
        np.testing.assert_array_equal(host["data"][c], ref[c], err_msg=c)
    np.testing.assert_array_equal(host["labels"], np.concatenate([np.ones((B // 2, 1)), np.zeros((B // 2, 1))]))
    return batch, host


def _errs(clf, b, loss, oinfo, grads):
    """Relative errors of one step against the oracle, keyed like the bars: logits and loss scaled by max(|ref|, 1), each gradient
    leaf by its own max."""
    e = {"logits": _scaled(b["logits"][0].cpu().numpy(), oinfo["_logits"].numpy()),
         "eval_logits": _scaled(b["logits"][1].cpu().numpy(), oinfo["_logits_eval"].numpy()),
         "loss": _scaled(float(loss), oinfo["loss"])}
    grad = clf._grad.cpu().numpy()
    for l in clf._spec:
        e[f"grad {l.path}"] = rel_err(grad[l.offset:l.offset + l.size].reshape(l.shape), grads[l.path].numpy())
    return e


def _over(errs, tol):
    return {k: v for k, v in errs.items() if not v <= (LEAF_TOL if k.startswith("grad ") else tol)}


@pytest.mark.parametrize("case", list(CASES))
def test_train_step_matches_float64_on_own_features(case, monkeypatch):
    from oracle import classifier as OC
    from serl_b200 import _lib as L
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    precision, nc, B, S2 = CASES[case]
    cams, tol = CAMS[:nc], BARS[precision]
    script = case.endswith("-script")
    rings = _rings(cams, 200) if script else None
    fixed = None if script else _batch(np.random.default_rng(B + nc), cams, B)
    clf, twin = _classifier(cams, precision), _classifier(cams, precision)
    trunk0 = {c: {k: v.clone() for k, v in leaves.items()} for c, leaves in clf._trunk.items()}
    trunk_features = OC.features
    fed = {}

    def own_features(params, cams_, data, dtype):
        for c in cams_:                                    # the frames the classifier's trunk encoded are the batch's
            np.testing.assert_array_equal(fed["pix"][c], np.asarray(data[c]).reshape(fed["pix"][c].shape), err_msg=c)
        return {c: fed["feats"][c].to(dtype) for c in cams_}

    monkeypatch.setattr(OC, "features", own_features)
    opt, worst = None, {}
    for step, key in enumerate(KEYS):
        batch, host = _sample_checked(rings, cams, B, np.array([9 + step, 1234], np.uint32)) if script else (fixed, fixed)
        params = {k: torch.as_tensor(np.asarray(v)) for k, v in _flat(clf.params).items()}
        if opt is None:
            z = lambda: {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items() if "pretrained_encoder" not in k}
            opt = {"count": 0, "mu": z(), "nu": z()}
        clf, loss, acc = clf.train_step(batch, key)
        b = clf._b(B)
        if precision != "fp32":
            assert b["S2"] == S2, (b["S2"], S2)
            assert (2 * nc > L.TGEMM_MAX_PROBLEMS) == (nc == 4) and (2 * nc == L.TGEMM_MAX_PROBLEMS) == (nc == 3)
        fed["pix"] = {c: b["pix"][c].cpu().numpy() for c in cams}
        fed["feats"] = {c: b["feats"][c].cpu().double() for c in cams}
        sle_m, hid_m = OC.dropout_masks(key, cams, B)
        for j, c in enumerate(cams):
            np.testing.assert_array_equal(b["masks"][j].cpu().numpy().astype(bool), np.asarray(sle_m[c], bool), err_msg=c)
        np.testing.assert_array_equal(b["hmask"].cpu().numpy().astype(bool), np.asarray(hid_m, bool))
        if step == 0:
            # a twin classifier's first step: the same loss, accuracy, logits and gradient buffer, bit for bit
            twin, tloss, tacc = twin.train_step(batch, key)
            tb = twin._b(B)
            assert float(tloss) == float(loss) and float(tacc) == float(acc)
            assert torch.equal(tb["logits"], b["logits"]) and torch.equal(twin._grad, clf._grad)
            if script:                                     # the injected features are the trunk's: a row sample in float64
                for c in cams:
                    ref = trunk_features(params, (c,), {c: host["data"][c][TRUNK_ROWS]}, torch.float64)[c].numpy()
                    e = rel_err(fed["feats"][c][TRUNK_ROWS].numpy(), ref)
                    print(f"CLF_BATCH_ERR [{case}] trunk rows {TRUNK_ROWS} of {c}: {e:.2e}")
                    assert e < TRUNK_TOL[precision], (c, e)
            opt_before = copy.deepcopy(opt)
        live = b["h"].cpu().numpy() > 0                   # the relu's active set in the classifier's train pass
        newp, opt, oinfo, grads = OC.train_step(params, opt, cams, host, masks=(sle_m, hid_m), hidden_live=live)
        pre = oinfo["_hidden_pre"].numpy()
        flips = live != (pre > 0)
        assert (np.abs(pre) <= tol * np.maximum(np.abs(pre).max(-1, keepdims=True), 1.0))[flips].all(), "a relu flipped away from 0"
        errs = _errs(clf, b, loss, oinfo, grads)
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
        leaf = max((k for k in errs if k.startswith("grad ")), key=errs.get)
        print(f"CLF_BATCH_ERR [{case}] step {step}: logits {errs['logits']:.2e} eval {errs['eval_logits']:.2e} "
              f"loss {errs['loss']:.2e} leaves {errs[leaf]:.2e} ({leaf[5:]}), relu units on the other side of 0: {int(flips.sum())}")
        for l in clf._spec:
            g = grads[l.path].numpy()
            got = clf._grad[l.offset:l.offset + l.size].cpu().numpy()
            assert np.abs(g).max() > 0 and np.abs(got).max() > 0, l.path
        assert not _over(errs, tol), _over(errs, tol)
        le_ref = oinfo["_logits_eval"].numpy().reshape(-1)
        near = int((np.abs(le_ref) <= tol * max(np.abs(le_ref).max(), 1.0)).sum())   # rows whose class may flip within tol
        assert abs(float(acc) - oinfo["accuracy"]) <= near / B + 1e-7, (float(acc), oinfo["accuracy"], near)
        now, lr = _flat(clf.params), clf.learning_rate
        for l in clf._spec:
            r, got = newp[l.path].numpy(), np.asarray(now[l.path])
            gmag = np.abs(grads[l.path].numpy())
            noisy = gmag < 2e-2 * max(gmag.max(), 1e-30)   # Adam normalises by |g|: entries at noise level move by up to ~lr either way
            allow = 1e-5 * max(np.abs(r).max(), 1e-3) + lr * np.where(noisy, 2.2, 5e-3)
            assert (np.abs(got - r) <= allow).all(), (l.path, np.abs(got - r).max())
        if step == 0 and script:
            # negative control: two camera-0 feature rows in the second M tile trade places in the oracle's table only
            swapped = dict(fed["feats"])
            swapped[cams[0]] = fed["feats"][cams[0]].clone()
            swapped[cams[0]][[200, 201]] = fed["feats"][cams[0]][[201, 200]]
            fed["feats"] = swapped
            _, _, oneg, gneg = OC.train_step(params, opt_before, cams, host, masks=(sle_m, hid_m), hidden_live=live)
            flagged = _over(_errs(clf, b, loss, oneg, gneg), tol)
            print(f"CLF_BATCH_ERR [{case}] negative control (rows 200 <-> 201 of {cams[0]}) flagged {len(flagged)} checks: "
                  + ", ".join(f"{k} {v:.1e}" for k, v in sorted(flagged.items(), key=lambda t: -t[1])[:6]))
            assert flagged, "swapping two feature rows in the second M tile went unnoticed"
    leaf = max((k for k in worst if k.startswith("grad ")), key=worst.get)
    print(f"CLF_BATCH_ERR [{case}] worst: logits {worst['logits']:.2e} eval {worst['eval_logits']:.2e} loss {worst['loss']:.2e} "
          f"leaves {worst[leaf]:.2e} ({leaf[5:]})")
    for c, leaves in clf._trunk.items():
        for k, v in leaves.items():
            assert torch.equal(v, trunk0[c][k]), (c, k)
    assert clf.step == 2
    clf.check_status()
    twin.check_status()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_eval_logits_match_float64_on_own_features(precision, tmp_path):
    """clf(obs) on the actor's single (1, 128, 128, 3) observation and on 3 and 257 rows, and a load_classifier_func restored from
    a checkpoint on one observation, against the oracle's train=False forward on the evaluating classifier's own features."""
    from oracle import classifier as OC
    from serl_b200.networks.reward_classifier import RewardClassifier, load_classifier_func
    from serl_b200.utils.checkpoints import save_checkpoint
    cams, tol = ("front", "wrist"), BARS[precision]
    rng = np.random.default_rng(8)
    clf = _classifier(cams, precision, seed=8)
    clf, _, _ = clf.train_step(_batch(rng, cams, 4), np.array([2, 3], np.uint32))
    params = {k: torch.as_tensor(np.asarray(v)).double() for k, v in _flat(clf.params).items()}
    obs = {c: rng.integers(0, 256, (257, 1, 128, 128, 3), dtype=np.uint8) for c in cams}

    def check(model, o, n, got, what):
        b = model._b(n)
        for c in cams:
            np.testing.assert_array_equal(b["pix"][c].cpu().numpy(), np.asarray(o[c]).reshape(n, 128, 128, 3), err_msg=c)
        ref = OC.forward(params, cams, {c: b["feats"][c].cpu().double() for c in cams}).numpy().reshape(-1)
        e = _scaled(got.cpu().numpy(), ref)
        print(f"CLF_BATCH_ERR eval {precision} {what}: {e:.2e}")
        assert e <= tol, (what, e)

    one = {c: obs[c][0] for c in cams}
    got = clf(one)
    assert got.shape == (1,)
    check(clf, one, 1, got, "clf(one observation)")
    for n in (3, 257):
        rows = {c: obs[c][:n] for c in cams}
        got = clf(rows)
        assert got.shape == (n, 1)
        check(clf, rows, n, got, f"clf({n} rows)")
    save_checkpoint(str(tmp_path), clf, step=1)
    f = load_classifier_func(np.array([0, 99], np.uint32), one, cams, str(tmp_path), precision=precision)
    got = f(one)
    restored = f.__closure__[0].cell_contents
    assert isinstance(restored, RewardClassifier) and got.shape == (1,)
    for k, v in _flat(restored.params).items():
        np.testing.assert_array_equal(np.asarray(v), params[k].numpy().astype(np.float32), err_msg=k)
    check(restored, one, 1, got, "load_classifier_func(one observation)")


@pytest.mark.parametrize("B", [256, 1024])
def test_sample_classifier_batch_at_training_sizes(B):
    """The device training batch at the reference's batch size and above: indices, crops and labels bit-exact, two draws."""
    cams = ("front", "wrist")
    rings = _rings(cams, B // 2 + 100)
    for i in range(2):
        _sample_checked(rings, cams, B, np.array([9, 1234 + i], np.uint32))
