"""GPU: the binary reward classifier (serl_b200/networks/reward_classifier.py) against the CPU restatement of the reference's
classifier and train_step (oracle/classifier.py): loss, eval logits, accuracy, every gradient leaf (the image heads are live and
trained through their dropout), parameters after Adam, the frozen trunk; the new kernels against torch; the device-side
training batch against the replay oracle + the crop; the checkpoint round trip of load_classifier_func."""
import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

pytestmark = pytest.mark.gpu


def _flat(tree, prefix=""):
    out = {}
    for k, v in tree.items():
        p = f"{prefix}/{k}" if prefix else k
        out.update(_flat(v, p)) if isinstance(v, dict) else out.__setitem__(p, v)
    return out


def _batch(rng, cams, B):
    trs = random_transitions(rng, B, cams)
    return {"data": {c: np.stack([t["observations"][c] for t in trs]) for c in cams},
            "labels": np.concatenate([np.ones((B // 2, 1)), np.zeros((B // 2, 1))]).astype(np.float32)}


def _classifier(cams, precision, seed=3):
    from serl_b200.networks.reward_classifier import create_classifier
    sample = {c: np.zeros((1, 128, 128, 3), np.uint8) for c in cams}
    clf = create_classifier(np.array([0, seed], np.uint32), sample, cams, precision=precision)
    g = torch.Generator(device="cuda").manual_seed(seed)                # biases / scales off their init so every path is exercised
    clf._params.add_(torch.randn(clf._n, device="cuda", generator=g) * 0.05)
    clf._tree = None
    return clf


def _check_steps(cams, precision, tol, full):
    from oracle import classifier as OC
    B = 12
    rng = np.random.default_rng(1)
    batch = _batch(rng, cams, B)
    clf = _classifier(cams, precision)
    trunk0 = {c: {k: v.clone() for k, v in leaves.items()} for c, leaves in clf._trunk.items()}
    opt = None
    for step, key in enumerate((np.array([0, 17], np.uint32), np.array([5, 2], np.uint32))):
        params = {k: torch.as_tensor(np.asarray(v)) for k, v in _flat(clf.params).items()}
        if opt is None:
            z = lambda: {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items() if "pretrained_encoder" not in k}
            opt = {"count": 0, "mu": z(), "nu": z()}
        clf, loss, acc = clf.train_step(batch, key)
        newp, opt, oinfo, grads = OC.train_step(params, opt, cams, batch, key=key)
        assert loss.dim() == 0 and acc.dim() == 0 and f"{loss:.4f}" and f"{acc:.4f}"
        ref = oinfo["loss"]
        assert abs(float(loss) - ref) <= tol * max(abs(ref), 1.0), (step, float(loss), ref)
        le = clf._b(B)["logits"][1].cpu().numpy().astype(np.float64)
        le_ref = oinfo["_logits_eval"].numpy().reshape(-1)
        assert np.abs(le - le_ref).max() <= tol * max(np.abs(le_ref).max(), 1.0), (step, np.abs(le - le_ref).max())
        near = int((np.abs(le_ref) <= tol * max(np.abs(le_ref).max(), 1.0)).sum())   # rows whose class flips within the tolerance
        assert abs(float(acc) - oinfo["accuracy"]) <= near / B + 1e-7, (float(acc), oinfo["accuracy"])
        if not full:
            continue
        for l in clf._spec:
            got = clf._grad[l.offset:l.offset + l.size].view(l.shape).cpu().numpy()
            g = grads[l.path].numpy()
            assert np.abs(g).max() > 0 and np.abs(got).max() > 0, l.path
            assert np.abs(got - g).max() <= 2e-4 * np.abs(g).max(), (l.path, np.abs(got - g).max() / np.abs(g).max())
        now = _flat(clf.params)
        lr = clf.learning_rate
        for l in clf._spec:
            r, got = newp[l.path].numpy(), np.asarray(now[l.path])
            gmag = np.abs(grads[l.path].numpy())
            noisy = gmag < 2e-2 * max(gmag.max(), 1e-30)       # Adam normalises by |g|: entries at noise level move by up to ~lr either way
            allow = 1e-5 * max(np.abs(r).max(), 1e-3) + lr * np.where(noisy, 2.2, 5e-3)
            assert (np.abs(got - r) <= allow).all(), (l.path, np.abs(got - r).max())
    for c, leaves in clf._trunk.items():
        for k, v in leaves.items():
            assert torch.equal(v, trunk0[c][k]), (c, k)
    assert clf.step == 2
    clf.check_status()


@pytest.mark.parametrize("cams", [("front",), ("front", "wrist")])
def test_train_step_fp32_matches_oracle(cams):
    _check_steps(cams, "fp32", 1e-5, full=True)


def test_train_step_fp16_matches_oracle():
    _check_steps(("front", "wrist"), "fp16", 1e-2, full=False)


def test_ln_relu_head_kernels_match_torch():
    from serl_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    R, D, keep = 37, 256, 0.9
    z = torch.randn(R, D, device="cuda", generator=g) * 2 + 0.3
    mask = (torch.rand(R, D, device="cuda", generator=g) < keep).to(torch.uint8)
    sc = 1 + 0.2 * torch.randn(D, device="cuda", generator=g)
    bi = 0.1 * torch.randn(D, device="cuda", generator=g)
    w = torch.randn(D, device="cuda", generator=g) * 0.1
    b = torch.randn(1, device="cuda", generator=g)
    dl = torch.randn(R, device="cuda", generator=g)
    for m in (None, mask):
        h, xh, rs, lo = (torch.empty(R, D, device="cuda"), torch.empty(R, D, device="cuda"), torch.empty(R, device="cuda"),
                         torch.empty(R, device="cuda"))
        ops.ln_relu_head_fwd(z.data_ptr(), None if m is None else m.data_ptr(), keep, sc.data_ptr(), bi.data_ptr(), w.data_ptr(), b.data_ptr(),
                             h.data_ptr(), xh.data_ptr(), rs.data_ptr(), lo.data_ptr(), R)
        dy, dz = torch.empty(R, D, device="cuda"), torch.empty(R, D, device="cuda")
        ops.ln_relu_head_bwd(dl.data_ptr(), w.data_ptr(), h.data_ptr(), xh.data_ptr(), rs.data_ptr(), sc.data_ptr(),
                             None if m is None else m.data_ptr(), keep, dy.data_ptr(), dz.data_ptr(), R)
        zz = z.double().clone().requires_grad_(True)
        x = zz if m is None else torch.where(m.bool(), zz / keep, torch.zeros_like(zz))
        mean = x.mean(-1, keepdim=True)
        var = ((x * x).mean(-1, keepdim=True) - mean * mean).clamp_min(0)
        y = (x - mean) * torch.rsqrt(var + 1e-6) * sc.double() + bi.double()
        hr = torch.relu(y)
        logit = hr @ w.double() + b.double()
        (gz,) = torch.autograd.grad((logit * dl.double()).sum(), zz)
        assert (h.double() - hr).abs().max() < 1e-5
        logit = logit.detach()
        assert (lo.double() - logit).abs().max() < 1e-5 * max(float(logit.abs().max()), 1.0)
        assert (dz.double() - gz).abs().max() < 1e-5 * float(gz.abs().max())
        if m is not None:
            assert float(dz[~m.bool()].abs().max()) == 0.0
        dyr = (dl.double()[:, None] * w.double()[None, :]) * (hr > 0)
        assert (dy.double() - dyr).abs().max() < 1e-6


def test_bce_kernel_large_logits_and_gradient():
    from serl_b200 import ops
    x = torch.tensor([-100.0, -20.0, -1e-9, -1e-3, 0.0, 0.5, 20.0, 100.0], device="cuda")
    y = torch.tensor([1.0, 0.0, 1.0, 1.0, 0.0, 1.0, 0.0, 1.0], device="cuda")
    dl, info = torch.empty(8, device="cuda"), torch.zeros(2, device="cuda")
    ops.bce_logits_loss(x.data_ptr(), x.data_ptr(), y.data_ptr(), 2.0, dl.data_ptr(), info.data_ptr(), 8)
    xd = x.double().clone().requires_grad_(True)
    ref = torch.nn.functional.binary_cross_entropy_with_logits(xd, y.double())
    (g,) = torch.autograd.grad(ref * 2.0, xd)
    ref = ref.detach()
    assert torch.isfinite(info).all() and torch.isfinite(dl).all()
    assert abs(float(info[0]) - float(ref)) <= 1e-6 * float(ref)
    assert (dl.double() - g).abs().max() < 1e-7
    # predictions (label): -100 neg (1, wrong), -20 neg (0, right), -1e-9 -> sigmoid rounds to 0.5 -> pos (1, right),
    # -1e-3 neg (1, wrong), 0 pos (0, wrong), 0.5 pos (1, right), 20 pos (0, wrong), 100 pos (1, right)
    assert float(info[1]) == 4 / 8


def test_dropout_bwd_kernel():
    from serl_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    n = 3 * 4096 + 7
    dx = torch.randn(n, device="cuda", generator=g)
    m = (torch.rand(n, device="cuda", generator=g) < 0.9).to(torch.uint8)
    keep = torch.tensor(0.9, dtype=torch.float32).double()               # correctly rounded fp32 division, like the forward's x / keep
    ref = torch.where(m.bool(), (dx.double() / keep).float(), torch.zeros_like(dx))
    ops.dropout_bwd(dx.data_ptr(), m.data_ptr(), 0.9, n)
    assert torch.equal(dx, ref)


def test_sample_classifier_batch_matches_replay_oracle_and_crop():
    from oracle import classifier as OC
    from oracle.replay import OracleFrameRing, draw_indices
    from serl_b200.networks.reward_classifier import sample_classifier_batch
    from serl_b200.utils.launcher import make_replay_buffer
    cams, B = ("front", "wrist"), 10
    rng = np.random.default_rng(7)
    rings = []
    for seed in (21, 22):
        dev = make_replay_buffer(fake_env(cams), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=seed)
        ora = OracleFrameRing(40, cams, (128, 128, 3), 1, 7, 4)
        for tr in random_transitions(rng, 30, cams):
            dev.insert(tr)
            ora.insert(tr)
        rings.append((dev, ora))
    (pos, opos), (neg, oneg) = rings
    key = np.array([9, 1234], np.uint32)
    for _ in range(2):
        steps = (pos._draw_step, neg._draw_step)
        batch = sample_classifier_batch(pos, neg, B, key)
        ip = draw_indices(pos._seed, steps[0], B // 2, opos.size, opos.valid)
        ineg = draw_indices(neg._seed, steps[1], B // 2, oneg.size, oneg.valid)
        gp, gn = opos.gather_packed(ip), oneg.gather_packed(ineg)
        ref = OC.crop_batch({c: gp["observations"][c][:, 1:] for c in cams}, {c: gn["observations"][c][:, :1] for c in cams}, key)
        for c in cams:
            np.testing.assert_array_equal(batch["data"][c].cpu().numpy(), ref[c])
        np.testing.assert_array_equal(batch["labels"].cpu().numpy(), np.concatenate([np.ones((B // 2, 1)), np.zeros((B // 2, 1))]))
        key = np.array([3, 3], np.uint32)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_checkpoint_roundtrip_load_classifier_func(tmp_path, precision):
    """fp32 build: bitwise.  fp16 build: the restored parameters are bitwise the trained ones; the logits of two passes agree to
    the trunk's run-to-run noise (its GroupNorm sums are accumulated with atomics, so an fp16 activation can round either way)."""
    from serl_b200.networks.reward_classifier import load_classifier_func
    from serl_b200.utils.checkpoints import save_checkpoint
    cams = ("front", "wrist")
    rng = np.random.default_rng(5)
    batch = _batch(rng, cams, 8)
    clf = _classifier(cams, precision)
    clf, _, _ = clf.train_step(batch, np.array([1, 1], np.uint32))
    clf, _, _ = clf.train_step(batch, np.array([1, 2], np.uint32))
    one = {c: batch["data"][c][3] for c in cams}                           # the actor's unbatched (1, 128, 128, 3) observation
    want_b, want_1 = clf(batch["data"]).clone(), clf(one).clone()
    assert want_b.shape == (8, 1) and want_1.shape == (1,)
    same = torch.equal if precision == "fp32" else (lambda a, b: bool((a - b).abs().max() <= 5e-3 * max(float(b.abs().max()), 1.0)))
    assert same(clf.apply_fn({"params": clf.params}, batch["data"], train=False), want_b)
    save_checkpoint(str(tmp_path), clf, step=2)
    f = load_classifier_func(np.array([0, 99], np.uint32), one, cams, str(tmp_path), precision=precision)
    from serl_b200.networks.reward_classifier import create_classifier
    from serl_b200.utils.checkpoints import restore_checkpoint
    r = restore_checkpoint(str(tmp_path), create_classifier(np.array([0, 98], np.uint32), one, cams, precision=precision))
    got_p = _flat(r.params)
    for k, v in _flat(clf.params).items():
        np.testing.assert_array_equal(np.asarray(got_p[k]), np.asarray(v), err_msg=k)
    assert r.step == 2 and r.opt_state["count"] == 2
    got_b, got_1 = f(batch["data"]), f(one)
    assert same(got_b, want_b)
    assert got_1.shape == (1,) and same(got_1, want_1)
    assert isinstance(got_1.item(), float)
    if precision == "fp32":
        assert got_1.item() == want_1.item()
