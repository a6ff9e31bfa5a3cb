"""CPU: the VICE classifier's layout, refused configurations, the update_vice key chain, and the float64 restatement
(tests/vice_oracle.py): its penalty gradient against central finite differences of its own loss, and the reference semantics
it keeps on purpose (last camera's labels, per-(camera, row) norms, per-camera mixup draws) each changing the result with two cameras."""
import numpy as np
import pytest
import torch

import vice_oracle as V

CAMS = ("wrist", "side")


def _params(seed=0):
    from serl_b200.agents.continuous.vice import init_vice, vice_spec
    spec, _ = vice_spec(CAMS)
    rng = np.random.default_rng(seed)
    p = init_vice(rng, spec)
    return {k: v + 0.05 * rng.standard_normal(v.shape) for k, v in p.items()}


def _raw(B, seed=1):
    rng = np.random.default_rng(seed)
    return {c: 0.5 * rng.standard_normal((2 * B, 4, 4, 512)) for c in CAMS}


def test_layout_and_trunk_clones():
    from serl_b200.agents.continuous.vice import trunk_clone_paths, vice_spec
    spec, n = vice_spec(CAMS)
    shapes = {l.path: l.shape for l in spec}
    assert shapes["modules_vice/encoder/encoder_side/Dense_0/kernel"] == (4096, 512)
    assert shapes["modules_vice/encoder/encoder_wrist/SpatialLearnedEmbeddings_0/kernel"] == (4, 4, 512, 8)
    assert shapes["modules_vice/network/Dense_0/kernel"] == (1024, 256)
    assert shapes["modules_vice/network/LayerNorm_0/scale"] == (256,)
    assert shapes["modules_vice/Dense_0/kernel"] == (256, 1) and shapes["modules_vice/Dense_0/bias"] == (1,)
    assert all(l.offset % 4 == 0 for l in spec) and n >= sum(l.size for l in spec)
    assert trunk_clone_paths(CAMS) == ["modules_vice/pretrained_encoder", "modules_vice/encoder/encoder_wrist/pretrained_encoder",
                                       "modules_vice/encoder/encoder_side/pretrained_encoder"]


@pytest.mark.parametrize("nk", [{"hidden_dims": [256, 256]}, {"activations": "relu"}, {"dropout_rate": 0.0},
                                {"use_layer_norm": False}])
def test_unsupported_vice_network_kwargs_raise(nk):
    from serl_b200.agents.continuous.vice import check_vice_network_kwargs
    with pytest.raises(NotImplementedError):
        check_vice_network_kwargs(nk)
    check_vice_network_kwargs({"activations": "leaky_relu", "use_layer_norm": True, "hidden_dims": [256], "dropout_rate": 0.1,
                               "activate_final": True})


def test_key_chain_and_permutation_rounds():
    from oracle import jax_prng as P
    from serl_b200.agents.continuous.vice import permutation_rounds, update_vice_keys
    rng = np.array([7, 11], np.uint32)
    got, ref = update_vice_keys(rng, 2), V.keys(rng, 2)
    for k in ("aug", "drop", "vice", "final"):
        assert np.array_equal(got[k], ref[k]), k
    for a, b in zip(got["cams"], ref["cams"]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    # restated by hand: key, rng = split(rng) ...; apply_loss_fns splits the ORIGINAL key five ways, the vice loss takes the last
    r = P.split(rng)[1]
    for _ in range(2):
        r = P.split(r)[1]
        r = P.split(r, 3)[2]
        r = P.split(r)[1]
    assert np.array_equal(ref["final"], P.split(r)[1])
    assert np.array_equal(ref["vice"], P.split(rng, 5)[4])
    assert permutation_rounds(1625) == 1 and permutation_rounds(2048) == 2
    perm = V.permutation(P.split(rng)[0], 512)
    assert sorted(perm.tolist()) == list(range(512))


def test_penalty_gradient_matches_finite_differences():
    B = 2
    params = _params()
    k = V.keys(np.array([0, 5], np.uint32), len(CAMS))
    raw = _raw(B)
    grads, _ = V.update_vice_grads(params, CAMS, raw, k)

    def total(p):
        with torch.enable_grad():
            t, _ = V.loss({n: torch.as_tensor(v, dtype=torch.float64) for n, v in p.items()}, CAMS, raw, k)
        return float(t)

    rng = np.random.default_rng(3)
    for path in ("modules_vice/network/LayerNorm_0/scale", "modules_vice/encoder/encoder_side/LayerNorm_0/bias",
                 "modules_vice/network/Dense_0/kernel", "modules_vice/Dense_0/kernel"):
        g = grads[path].numpy()
        for _ in range(2):
            idx = tuple(int(rng.integers(0, s)) for s in g.shape)
            h = 1e-5
            pp, pm = dict(params), dict(params)
            pp[path], pm[path] = params[path].copy(), params[path].copy()
            pp[path][idx] += h
            pm[path][idx] -= h
            fd = (total(pp) - total(pm)) / (2 * h)
            assert abs(fd - g[idx]) <= 1e-5 * max(1.0, abs(fd)), (path, idx, fd, g[idx])


def test_reference_semantics_change_the_result():
    B = 4
    params = {n: torch.as_tensor(v, dtype=torch.float64) for n, v in _params(2).items()}
    k = V.keys(np.array([1, 9], np.uint32), len(CAMS))
    raw = _raw(B, 4)
    base, info = V.loss(params, CAMS, raw, k)
    other_labels, _ = V.loss(params, CAMS, raw, k, last_camera_labels=False)
    joint_norms, _ = V.loss(params, CAMS, raw, k, per_camera_norms=False)
    shared_draws, _ = V.loss(params, CAMS, raw, k, per_camera_draws=False)
    assert abs(float(base) - float(other_labels)) > 1e-6
    assert abs(float(base) - float(joint_norms)) > 1e-6
    assert abs(float(base) - float(shared_draws)) > 1e-6
    (l0, p0, _), (l1, p1, _) = info["draws"]                 # each camera mixes with its own lam and permutation
    assert l0 != l1 and not np.array_equal(p0, p1)
