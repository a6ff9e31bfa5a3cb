"""CPU: pins the autograd restatement of the reward classifier's train_step (oracle/classifier.py) to the literal formulation:
the stable BCE against torch's, finite differences of the loss for one leaf of each kind (with both dropout masks on), the
accuracy tie rule of fp32 sigmoid, the keyed dropout masks and the crop-key mapping of the training batch."""
import numpy as np
import torch
import torch.nn.functional as F

from helpers import random_transitions


def _params(rng, cams):
    from serl_b200.networks.reward_classifier import ROOT, classifier_spec
    from serl_b200.params import init_trunk, lecun_normal
    spec, _ = classifier_spec(cams)
    p = {}
    for l in spec:
        if l.path.endswith("kernel"):
            v = lecun_normal(rng, l.shape)
        elif l.path.endswith("scale"):
            v = 1 + 0.1 * rng.standard_normal(l.shape)
        else:
            v = 0.05 * rng.standard_normal(l.shape)
        p[l.path] = torch.as_tensor(np.asarray(v, np.float32))
    for cam in cams:
        for k, v in init_trunk(rng).items():
            p[f"{ROOT}/encoder_{cam}/pretrained_encoder/{k}"] = torch.as_tensor(v)
    return p


def test_bce_matches_torch_and_is_finite_at_large_logits():
    from oracle import classifier as OC
    x = torch.tensor([-100.0, -30.0, -1.5, -1e-3, 0.0, 2e-3, 0.7, 30.0, 100.0], dtype=torch.float64)
    for y in (torch.zeros_like(x), torch.ones_like(x)):
        got = OC.bce(x, y)
        ref = F.binary_cross_entropy_with_logits(x, y, reduction="none")
        assert torch.isfinite(got).all()
        assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)
    assert float(OC.bce(torch.tensor([100.0], dtype=torch.float64), torch.tensor([0.0], dtype=torch.float64))) == 100.0


def test_accuracy_follows_fp32_sigmoid_tie_rule():
    from oracle import classifier as OC
    # sigmoid(-1e-9) rounds to exactly 0.5 in fp32 -> predicted positive; sigmoid(-1e-3) < 0.5 -> predicted negative
    logits = np.array([-1e-9, -1e-3, 0.0, 3.0, -3.0], np.float32)
    labels = np.array([1.0, 1.0, 1.0, 0.0, 0.0], np.float32)
    assert OC.accuracy(logits, labels) == 3 / 5
    assert float(np.mean((logits >= 0) == labels)) == 2 / 5            # a plain sign test disagrees on the first row


def test_keyed_dropout_masks_fold_camera_then_hidden_index():
    from oracle import classifier as OC
    from oracle import jax_prng as P
    key = np.array([3, 77], np.uint32)
    sle, hid = OC.dropout_masks(key, ("a", "b"), 5)
    np.testing.assert_array_equal(sle["a"], P.bernoulli(P.fold_in(key, 0), 0.9, (5, 4096)))
    np.testing.assert_array_equal(sle["b"], P.bernoulli(P.fold_in(key, 1), 0.9, (5, 4096)))
    np.testing.assert_array_equal(hid, P.bernoulli(P.fold_in(key, 2), 0.9, (5, 256)))
    assert 0.85 < hid.mean() < 0.95


def test_train_step_gradients_match_finite_differences_with_dropout():
    from oracle import classifier as OC
    cams = ("front",)
    rng = np.random.default_rng(0)
    params = _params(rng, cams)
    B = 4
    trs = random_transitions(rng, B, cams)
    batch = {"data": {"front": np.stack([t["observations"]["front"] for t in trs])},
             "labels": np.array([[1.0], [1.0], [0.0], [0.0]], np.float32)}
    sle_m, hid_m = OC.dropout_masks(np.array([0, 5], np.uint32), cams, B)
    opt = {"count": 0, "mu": {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items() if "pretrained" not in k},
           "nu": {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items() if "pretrained" not in k}}
    newp, opt, info, grads = OC.train_step(params, opt, cams, batch, masks=(sle_m, hid_m))
    for k, g in grads.items():
        assert float(g.abs().max()) > 0.0, k                               # every trainable leaf is live (no stop_gradient)
    p64 = {k: v.double() for k, v in params.items()}
    feats = OC.features(p64, cams, batch["data"], torch.float64)
    labels = torch.as_tensor(batch["labels"]).double()

    def loss(p):
        return float(OC.bce(OC.forward(p, cams, feats, sle_m, hid_m), labels).mean())

    assert abs(loss(p64) - info["loss"]) < 1e-12
    leaves = ("encoder_def/encoder_front/SpatialLearnedEmbeddings_0/kernel", "encoder_def/encoder_front/Dense_0/kernel",
              "encoder_def/encoder_front/LayerNorm_0/scale", "encoder_def/encoder_front/Dense_0/bias", "Dense_0/kernel",
              "Dense_0/bias", "LayerNorm_0/scale", "LayerNorm_0/bias", "Dense_1/kernel", "Dense_1/bias")
    for path in leaves:
        g = grads[path].reshape(-1)
        idx = [int(torch.argmax(g.abs()))] + [int(i) for i in rng.integers(0, g.numel(), 2)]
        for i in idx:
            h = 1e-6
            vals = []
            for sgn in (+1, -1):
                p2 = dict(p64)
                t = p2[path].clone().reshape(-1)
                t[i] += sgn * h
                p2[path] = t.reshape(params[path].shape)
                vals.append(loss(p2))
            fd = (vals[0] - vals[1]) / (2 * h)
            an = float(g[i])
            assert abs(fd - an) <= 1e-5 * max(abs(an), 1e-4) + 1e-9, (path, i, fd, an)
    # the SLE kernel gradient passes the dropout mask: with every SLE unit of one feature dropped, its kernel column gets no gradient
    m0 = {"front": sle_m["front"].copy()}
    m0["front"][:, 0] = False                                              # unit c=0, f=0 dropped for every row
    _, _, _, g0 = OC.train_step(params, {"count": 0, "mu": {k: torch.zeros_like(v) for k, v in opt["mu"].items()},
                                         "nu": {k: torch.zeros_like(v) for k, v in opt["nu"].items()}}, cams, batch, masks=(m0, hid_m))
    gk = g0["encoder_def/encoder_front/SpatialLearnedEmbeddings_0/kernel"]
    assert float(gk[:, :, 0, 0].abs().max()) == 0.0 and float(gk[:, :, 0, 1].abs().max()) > 0.0
    # one Adam step from zero moments moves every entry with a non-zero gradient by lr
    k = "Dense_0/kernel"
    assert abs(float((newp[k] - params[k].double()).abs().max()) - 1e-4) < 1e-9


def test_hidden_live_is_the_relu_unless_it_flips_a_unit():
    """forward(hidden_live=pre > 0) is the plain relu bit for bit; marking one dead unit live moves only its own row's logit,
    by that unit's pre-activation times its Dense_1 weight."""
    from oracle import classifier as OC
    cams, B = ("front", "wrist"), 6
    rng = np.random.default_rng(3)
    p = {k: v.double() for k, v in _params(rng, cams).items() if "pretrained" not in k}
    feats = {c: torch.as_tensor(np.abs(rng.standard_normal((B, 4, 4, 512)))) for c in cams}
    sle_m, hid_m = OC.dropout_masks(np.array([1, 2], np.uint32), cams, B)
    saves = {}
    ref = OC.forward(p, cams, feats, sle_m, hid_m, saves=saves)
    pre = saves["hidden_pre"]
    live = (pre > 0).numpy()
    assert torch.equal(OC.forward(p, cams, feats, sle_m, hid_m, hidden_live=live), ref)
    r, d = 4, int(np.flatnonzero(~live[4])[0])
    live[r, d] = True
    got = OC.forward(p, cams, feats, sle_m, hid_m, hidden_live=live)
    moved = (got - ref).reshape(-1)
    assert abs(float(moved[r]) - float(pre[r, d] * p["Dense_1/kernel"][d, 0])) < 1e-12
    assert float(moved[r]) != 0.0 and bool((moved[torch.arange(B) != r] == 0).all())


def test_crop_batch_uses_one_key_over_the_concatenated_batch():
    from oracle import classifier as OC
    from oracle import jax_prng as P
    rng = np.random.default_rng(2)
    B = 6
    pos = {c: rng.integers(0, 256, (B // 2, 1, 128, 128, 3), dtype=np.uint8) for c in ("a", "b")}
    neg = {c: rng.integers(0, 256, (B // 2, 1, 128, 128, 3), dtype=np.uint8) for c in ("a", "b")}
    key = np.array([11, 4], np.uint32)
    out = OC.crop_batch(pos, neg, key)
    off = P.crop_offsets(key, B)
    for c in ("a", "b"):
        src = np.concatenate([pos[c], neg[c]])[:, 0]
        padded = np.pad(src, ((0, 0), (4, 4), (4, 4), (0, 0)), mode="edge")
        for i in range(B):
            cy, cx = off[i]
            np.testing.assert_array_equal(out[c][i, 0], padded[i, cy:cy + 128, cx:cx + 128])
