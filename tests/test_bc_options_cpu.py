"""CPU: BCAgent.create's option resolution, the leaf spec per configuration, the float64 restatement of the options
(tests/bc_options_oracle.py) and the host call sequence of a non-launcher BC update with the kernels replaced by a recorder."""
import math

import numpy as np
import pytest
import torch

from helpers import random_transitions

SWISH = {"activations": "swish", "use_layer_norm": False, "hidden_dims": [256, 256]}


def _opts(nk=None, pk=None):
    from serl_b200.agents.continuous.bc import bc_options
    return bc_options(nk, pk)


def test_resolution_accepts():
    from serl_b200.agents.continuous.bc import BC_LAUNCHER_MLP
    from serl_b200.params import MlpArch
    assert _opts() == (BC_LAUNCHER_MLP, "exp", 1e-5, 10.0, False)
    assert _opts({"activations": "tanh", "use_layer_norm": False, "hidden_dims": [256, 256], "dropout_rate": None, "activate_final": False})[0] == BC_LAUNCHER_MLP
    assert _opts({"hidden_dims": [256, 256], "dropout_rate": 0})[0] == BC_LAUNCHER_MLP
    assert _opts(SWISH)[0] == MlpArch((256, 256), "swish", False, 0.0)
    arch, std, lo, hi, sq = _opts({"activations": "tanh", "use_layer_norm": True, "hidden_dims": [512, 512, 512], "dropout_rate": 0.1},
                                  {"std_parameterization": "uniform", "tanh_squash_distribution": True, "std_min": 1e-3, "std_max": 2})
    assert arch == MlpArch((512, 512, 512), "tanh", True, 0.1) and (std, lo, hi, sq) == ("uniform", 1e-3, 2.0, True)
    assert _opts(None, {"std_parameterization": "softplus"})[1] == "softplus"


@pytest.mark.parametrize("nk,pk,exc", [
    ({"hidden": [256]}, None, TypeError),
    (None, {"std": "exp"}, TypeError),
    ({"hidden_dims": [512, 512]}, None, ValueError),                                   # no activations / use_layer_norm
    ({"activations": "relu"}, None, ValueError),                                       # no use_layer_norm
    ({"dropout_rate": 0.1}, None, ValueError),
    ({"activations": "relu", "use_layer_norm": False, "hidden_dims": [100]}, None, ValueError),
    ({"activations": "relu", "use_layer_norm": False, "hidden_dims": [2048]}, None, ValueError),
    ({"activations": "relu", "use_layer_norm": False, "dropout_rate": 1.0}, None, ValueError),
    ({"activations": "elu", "use_layer_norm": False}, None, NotImplementedError),
    (None, {"std_parameterization": "fixed"}, NotImplementedError),
    (None, {"fixed_std": [0.1, 0.1]}, NotImplementedError),
    (None, {"std_parameterization": "tanh"}, NotImplementedError),
])
def test_resolution_refuses(nk, pk, exc):
    with pytest.raises(exc):
        _opts(nk, pk)


def test_missing_keys_name_the_flax_defaults():
    with pytest.raises(ValueError, match="flax defaults"):
        _opts({"hidden_dims": [64]})


def test_sac_keeps_refusing_dropout():
    from serl_b200.agents.continuous.sac import _mlp_arch
    with pytest.raises(NotImplementedError):
        _mlp_arch("policy_network_kwargs", {"activations": "tanh", "use_layer_norm": True, "dropout_rate": 0.1})


def test_other_encoders_refused():
    from serl_b200.agents.continuous.bc import BCAgent
    trs = random_transitions(np.random.default_rng(0), 1, ("front",), 16)
    for enc in ("small", "resnet"):
        with pytest.raises(NotImplementedError):
            BCAgent.create(0, trs[0]["observations"], trs[0]["actions"], encoder_type=enc, image_keys=("front",), device="cpu")


@pytest.mark.parametrize("std", ["exp", "softplus", "uniform"])
@pytest.mark.parametrize("proprio", [True, False])
def test_leaf_spec(std, proprio):
    from serl_b200.agents.continuous.bc import bc_spec
    from serl_b200.params import ENC, MlpArch
    arch = MlpArch((512, 128, 64), "gelu", True, 0.1)
    spec, n = bc_spec(("a", "b"), 7, 4, arch, std, proprio)
    paths = {l.path: l.shape for l in spec}
    F = 512 + (64 if proprio else 0)
    assert paths["modules_actor/network/Dense_0/kernel"] == (F, 512) and paths["modules_actor/network/Dense_2/kernel"] == (128, 64)
    assert paths["modules_actor/network/LayerNorm_1/scale"] == (128,) and "modules_actor/network/LayerNorm_3/scale" not in paths
    assert paths["modules_actor/Dense_0/kernel"] == (64, 4)
    assert ("modules_actor/log_stds" in paths) == (std == "uniform") and ("modules_actor/Dense_1/kernel" in paths) == (std != "uniform")
    if std == "uniform":
        assert paths["modules_actor/log_stds"] == (4,)
    assert (f"{ENC}/Dense_0/kernel" in paths) == proprio and (f"{ENC}/LayerNorm_0/scale" in paths) == proprio
    assert all(l.offset % 4 == 0 for l in spec) and n >= spec[-1].offset + spec[-1].size
    spec2, _ = bc_spec(("a", "b"), 7, 4, MlpArch((256, 256), "tanh", False), "exp", True)
    assert not any("LayerNorm" in l.path and "network" in l.path for l in spec2)


def test_launcher_spec_unchanged():
    """make_bc_agent's leaves keep their order and offsets (checkpoints and the parent's parameters)."""
    from serl_b200.agents.continuous.bc import bc_spec
    spec, n = bc_spec(("front", "wrist"), 7, 4)
    tail = [l.path for l in spec[-8:]]
    assert tail == ["modules_actor/network/Dense_0/kernel", "modules_actor/network/Dense_0/bias", "modules_actor/network/Dense_1/kernel",
                    "modules_actor/network/Dense_1/bias", "modules_actor/Dense_0/kernel", "modules_actor/Dense_0/bias",
                    "modules_actor/Dense_1/kernel", "modules_actor/Dense_1/bias"]


def test_oracle_squashed_log_prob_matches_torch():
    from bc_options_oracle import log_prob
    g = torch.Generator().manual_seed(0)
    mu, sd = torch.randn(50, 5, generator=g, dtype=torch.float64), torch.rand(50, 5, generator=g, dtype=torch.float64) + 0.1
    a = torch.tanh(mu + sd * torch.randn(50, 5, generator=g, dtype=torch.float64))
    d = torch.distributions.TransformedDistribution(torch.distributions.Normal(mu, sd), [torch.distributions.TanhTransform()])
    torch.testing.assert_close(log_prob(mu, sd, a, True), d.log_prob(a).sum(-1), rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(log_prob(mu, sd, a, False), torch.distributions.Normal(mu, sd).log_prob(a).sum(-1))


def test_oracle_masks_follow_the_fold_convention():
    from bc_options_oracle import mlp_masks
    from oracle.jax_prng import bernoulli, fold_in, prng_key
    key = prng_key(5)
    m = mlp_masks(key, 2, 6, (64, 128), 0.25)
    assert [x.shape for x in m] == [(6, 64), (6, 128)]
    np.testing.assert_array_equal(m[1], bernoulli(fold_in(key, 3), 0.75, (6, 128)))
    assert not np.array_equal(m[0][:, :64], bernoulli(fold_in(key, 0), 0.75, (6, 64)))       # not the cameras' folds


def test_oracle_policy_architectures_and_masks():
    """Dropout before LayerNorm: the dropped-out rows of layer 0 enter the LayerNorm as zeros, scaled by 1 / (1 - rate)."""
    from bc_options_oracle import policy
    from oracle.drq import layer_norm
    from serl_b200.params import MlpArch
    g = torch.Generator().manual_seed(1)
    arch = MlpArch((64,), "relu", True, 0.5)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    p = {"modules_actor/network/Dense_0/kernel": r(8, 64), "modules_actor/network/Dense_0/bias": r(64),
         "modules_actor/network/LayerNorm_0/scale": r(64), "modules_actor/network/LayerNorm_0/bias": r(64),
         "modules_actor/Dense_0/kernel": r(64, 3), "modules_actor/Dense_0/bias": r(3), "modules_actor/log_stds": r(3)}
    x = r(5, 8)
    mask = np.random.default_rng(0).random((5, 64)) < 0.5
    mu, sd = policy(p, x, arch, "uniform", 1e-5, 10.0, [mask], temperature=0.25)
    z = x @ p["modules_actor/network/Dense_0/kernel"] + p["modules_actor/network/Dense_0/bias"]
    h = torch.relu(layer_norm(torch.where(torch.as_tensor(mask), z * 2, torch.zeros_like(z)), p["modules_actor/network/LayerNorm_0/scale"],
                              p["modules_actor/network/LayerNorm_0/bias"]))
    torch.testing.assert_close(mu, h @ p["modules_actor/Dense_0/kernel"] + p["modules_actor/Dense_0/bias"])
    torch.testing.assert_close(sd, (torch.exp(p["modules_actor/log_stds"]) * 0.5).expand(5, 3))
    mu0, _ = policy(p, x, arch, "uniform", 1e-5, 10.0, None)                                  # train=False: no dropout
    assert not torch.allclose(mu0, mu)


def test_oracle_gradient_matches_finite_differences():
    """The restated loss's gradient of a squashed, uniform-std, dropout + LayerNorm policy against central differences."""
    from bc_options_oracle import log_prob, policy
    from serl_b200.params import MlpArch
    g = torch.Generator().manual_seed(2)
    arch = MlpArch((64,), "swish", True, 0.2)
    r = lambda *s: 0.3 * torch.randn(*s, generator=g, dtype=torch.float64)
    p = {"modules_actor/network/Dense_0/kernel": r(6, 64), "modules_actor/network/Dense_0/bias": r(64),
         "modules_actor/network/LayerNorm_0/scale": 1 + r(64), "modules_actor/network/LayerNorm_0/bias": r(64),
         "modules_actor/Dense_0/kernel": r(64, 2), "modules_actor/Dense_0/bias": r(2), "modules_actor/log_stds": r(2)}
    x, a = r(4, 6), torch.tanh(r(4, 2) * 3)
    mask = [np.random.default_rng(1).random((4, 64)) < 0.8]

    def loss(pp):
        mu, sd = policy(pp, x, arch, "uniform", 1e-5, 10.0, mask)
        return -log_prob(mu, sd, a, True).mean()
    leaf = "modules_actor/log_stds"
    q = {k: v.clone().requires_grad_(k == leaf) for k, v in p.items()}
    (gr,) = torch.autograd.grad(loss(q), [q[leaf]])
    for j in range(2):
        e = torch.zeros(2, dtype=torch.float64)
        e[j] = 1e-6
        fd = (loss({**p, leaf: p[leaf] + e}) - loss({**p, leaf: p[leaf] - e})) / 2e-6
        assert abs(fd.item() - gr[j].item()) < 1e-6 * max(1.0, abs(gr[j].item()))


@pytest.fixture()
def dry(monkeypatch):
    from serl_b200 import _lib as L
    calls = []
    real_call = L.call

    def fake_call(name, *args):
        if name.startswith("serl_host_"):
            return real_call(name, *args)
        calls.append(name)
        return 0

    monkeypatch.setattr(L, "call", fake_call)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    return calls


def test_options_call_sequence(dry):
    """A pixel-only, squashed, uniform-std BC update with a dropout + LayerNorm MLP: no proprio launches, one keyed mask per camera
    and per hidden layer, the dropout layer kernels, serl_bc_loss_std instead of serl_bc_loss, and no serl_tanh_fwd / _bwd."""
    from serl_b200.agents.continuous.bc import BCAgent
    cams = ("front", "wrist")
    trs = random_transitions(np.random.default_rng(0), 6, cams, 128)
    agent = BCAgent.create(1, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet-pretrained", image_keys=cams, use_proprio=False,
                           network_kwargs={"activations": "gelu", "use_layer_norm": True, "hidden_dims": [128, 64, 64], "dropout_rate": 0.1},
                           policy_kwargs={"std_parameterization": "uniform", "tanh_squash_distribution": True}, device="cpu")
    assert agent._cfg.enc_dim == 512
    obs = {**{c: np.stack([t["observations"][c] for t in trs]) for c in cams}, "state": np.stack([t["observations"]["state"] for t in trs])}
    batch = {"observations": obs, "actions": np.stack([t["actions"] for t in trs]).astype(np.float32)}
    del dry[:]
    agent.update(batch)
    assert dry.count("serl_dropout_mask_fill") == 2 + 3 and dry.count("serl_bc_loss_std") == 1 and "serl_bc_loss" not in dry
    assert dry.count("serl_ln_act_dropout_fwd") == 3 and dry.count("serl_ln_act_dropout_bwd") == 3
    assert dry.count("serl_layernorm_param_grad") == 3 and "serl_tanh_fwd" not in dry and "serl_tanh_bwd" not in dry
    assert dry.count("serl_layernorm_tanh_fwd") == 2 and "serl_layernorm_tanh_bwd" not in dry       # image heads only, no proprio
    tree = agent.state.params["modules_actor"]
    assert tree["log_stds"].shape == (4,) and (tree["log_stds"] == 0).all() and "Dense_1" not in tree
    assert tree["network"]["Dense_0"]["kernel"].shape == (512, 128)
    del dry[:]
    agent.sample_actions({k: v for k, v in obs.items() if k != "state"}, argmax=True)
    assert "serl_dropout_mask_fill" not in dry and "serl_ln_act_dropout_fwd" not in dry and dry.count("serl_layernorm_act_fwd") == 3
