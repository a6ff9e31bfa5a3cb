"""GPU: BCAgent.create's network / policy / proprio options against the float64 restatement (tests/bc_options_oracle.py) fed the
agent's own trunk features, on the fp32 build: loss and mse within 1e-5, every trainable gradient leaf within 2e-4 of its max,
post-Adam parameters under the noise-aware bar of DESIGN.md §5 over 3 updates, SLE / MLP dropout masks and the key chain
bit-exact, sample_actions and get_debug_metrics within 1e-5, a checkpoint round trip bitwise; the fp16 build, also on its own
trunk features, loss and mse within 1e-4 and every trainable gradient leaf within 2e-4 of its max.

Each option appears in at least two configurations; among them the reference constructor's defaults (use_proprio=False, swish
[256, 256], no LayerNorm, "exp" std) and [512, 512, 512] + LayerNorm + dropout 0.1 + tanh squash + "uniform" std."""
import numpy as np
import pytest
import torch

from bc_options_oracle import log_prob, mode, policy, update as oracle_update, encode as oracle_encode
from helpers import random_transitions, rel_err

pytestmark = pytest.mark.gpu

# The fp16 build on its own trunk features: the heads run the 3xTF32 per-op chain, held to the fused heads' loss bar
FP16_LOSS_TOL = 1e-4
SWISH = {"activations": "swish", "use_layer_norm": False, "hidden_dims": [256, 256]}
LARGE = {"activations": "tanh", "use_layer_norm": True, "hidden_dims": [512, 512, 512], "dropout_rate": 0.1}
CONFIGS = {
    # name: (network_kwargs, policy_kwargs, use_proprio, cams, B)
    "reference_defaults": (SWISH, {}, False, ("front",), 2),
    "large_squash_uniform": (LARGE, {"tanh_squash_distribution": True, "std_parameterization": "uniform"}, True, ("front", "wrist"), 256),
    "gelu_ln_drop_softplus_squash": ({"activations": "gelu", "use_layer_norm": True, "hidden_dims": [192, 128], "dropout_rate": 0.2},
                                     {"tanh_squash_distribution": True, "std_parameterization": "softplus", "std_max": 5.0}, False,
                                     ("front", "wrist"), 100),
    "relu_drop_uniform": ({"activations": "relu", "use_layer_norm": False, "hidden_dims": [256], "dropout_rate": 0.1},
                          {"std_parameterization": "uniform", "std_min": 0.05}, True, ("front",), 256),
    "leaky_ln_softplus": ({"activations": "leaky_relu", "use_layer_norm": True, "hidden_dims": [64, 64]},
                          {"std_parameterization": "softplus"}, True, ("front",), 2),
    "tanh_ln_exp_squash": ({"activations": "tanh", "use_layer_norm": True, "hidden_dims": [256, 256]},
                           {"tanh_squash_distribution": True, "std_max": 5.0}, True, ("front", "wrist"), 100),
}


def _flat(tree, prefix=""):
    out = {}
    for k, v in tree.items():
        p = f"{prefix}/{k}" if prefix else k
        out.update(_flat(v, p)) if isinstance(v, dict) else out.__setitem__(p, v)
    return out


def _make(name, precision="fp32", seed=3):
    from serl_b200.agents.continuous.bc import BCAgent
    nk, pk, proprio, cams, B = CONFIGS[name]
    rng = np.random.default_rng(seed)
    trs = random_transitions(rng, B, cams)
    agent = BCAgent.create(seed, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet-pretrained", image_keys=cams,
                           use_proprio=proprio, network_kwargs=nk, policy_kwargs=pk, precision=precision)
    g = torch.Generator(device="cuda").manual_seed(1)               # biases / log_stds off zero so that every path is exercised
    agent._params.add_(torch.randn(agent._n, device="cuda", generator=g) * 0.05)
    batch = {"observations": {**{c: np.stack([t["observations"][c] for t in trs]) for c in cams},
                              "state": np.stack([t["observations"]["state"] for t in trs])},
             "actions": np.stack([t["actions"] for t in trs]).astype(np.float32)}
    return agent, batch


def _opts(agent):
    return dict(arch=agent.arch, std=agent.std_parameterization, std_min=agent.std_min, std_max=agent.std_max, squash=agent.tanh_squash,
                use_proprio=agent._cfg.use_proprio)


def _feats(agent, B):
    return {c: agent._bufs[B]["feats"][c].detach().cpu().double() for c in agent._cfg.cams}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_bc_options_update_matches_oracle(name):
    agent, batch = _make(name)
    cams, B = tuple(agent._cfg.cams), batch["actions"].shape[0]
    state = batch["observations"]["state"] if agent._cfg.use_proprio else None
    opt = None
    for step in range(3):
        params = {k: torch.as_tensor(np.asarray(v)) for k, v in _flat(agent.state.params).items()}
        if opt is None:
            z = lambda v: torch.zeros_like(v, dtype=torch.float64)
            opt = {"count": 0, "mu": {k: z(v) for k, v in params.items() if "pretrained_encoder" not in k},
                   "nu": {k: z(v) for k, v in params.items() if "pretrained_encoder" not in k}}
        rng0 = agent.state.rng
        agent, info = agent.update(batch)
        b = agent._bufs[B]
        newp, opt, new_rng, oinfo, grads, masks = oracle_update(params, opt, rng0, cams, _feats(agent, B), state, batch["actions"], _opts(agent))
        np.testing.assert_array_equal(agent.state.rng, new_rng)
        for c in cams:
            np.testing.assert_array_equal(b["masks"][c].cpu().numpy().astype(bool), masks["sle"][c])
        if agent.arch.dropout:
            for got, ref in zip(b["mlp_masks"], masks["mlp"]):
                np.testing.assert_array_equal(got.cpu().numpy().astype(bool), ref)
        for k in ("actor_loss", "mse"):
            assert abs(float(info[k]) - oinfo[k]) <= 1e-5 * max(abs(oinfo[k]), 1.0), (k, float(info[k]), oinfo[k])
        for l in agent._spec:
            got = agent._grad[l.offset:l.offset + l.size].view(l.shape).cpu().numpy()
            ref = grads[l.path].numpy()
            if "/encoder_" in l.path:                               # image heads: behind stop_gradient (encoding.py:48-49)
                assert np.abs(ref).max() == 0 and np.abs(got).max() == 0, l.path
            else:
                assert np.abs(ref).max() > 0, l.path
                assert np.abs(got - ref).max() <= 2e-4 * np.abs(ref).max(), (l.path, np.abs(got - ref).max() / np.abs(ref).max())
        now = _flat(agent.state.params)
        lr = agent.learning_rate
        for l in agent._spec:
            ref, got = newp[l.path].numpy(), np.asarray(now[l.path])
            gmag = np.abs(grads[l.path].numpy())
            noisy = gmag < 2e-2 * max(gmag.max(), 1e-30)
            allow = 1e-5 * max(np.abs(ref).max(), 1e-3) + lr * np.where(noisy, 2.2, 5e-3)
            assert (np.abs(got - ref) <= allow).all(), (l.path, np.abs(got - ref).max())
    assert agent.state.step == 3


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_bc_options_inference_matches_oracle(name):
    from oracle.jax_prng import normal
    agent, batch = _make(name, seed=5)
    obs, cams, B, A = batch["observations"], tuple(agent._cfg.cams), batch["actions"].shape[0], batch["actions"].shape[1]
    o = _opts(agent)
    a = agent.sample_actions(obs, argmax=True)
    params = {k: torch.as_tensor(np.asarray(v)).double() for k, v in _flat(agent.state.params).items()}
    st = torch.as_tensor(obs["state"]).double() if o["use_proprio"] else None
    enc = oracle_encode(params, cams, _feats(agent, B), st, None, o["use_proprio"])
    mu, sd = policy(params, enc, o["arch"], o["std"], o["std_min"], o["std_max"])
    assert rel_err(a, mode(mu, o["squash"]).numpy()) < 1e-5
    seed = np.array([0, 11], np.uint32)
    s = agent.sample_actions(obs, seed=seed, temperature=0.5)
    _, sd5 = policy(params, enc, o["arch"], o["std"], o["std_min"], o["std_max"], temperature=0.5)
    assert rel_err(s, mode(mu + sd5 * torch.as_tensor(normal(seed, (B, A))).double(), o["squash"]).numpy()) < 1e-5
    one = agent.sample_actions({k: v[0] for k, v in obs.items()}, argmax=True)
    assert one.shape == (A,) and rel_err(one, mode(mu, o["squash"]).numpy()[0]) < 1e-5
    m = agent.get_debug_metrics(batch)
    act = torch.as_tensor(batch["actions"]).double()
    assert rel_err(m["mse"].cpu().numpy(), ((mode(mu, o["squash"]) - act) ** 2).sum(-1).numpy()) < 1e-5
    assert rel_err(m["log_probs"].cpu().numpy(), log_prob(mu, sd, act, o["squash"]).numpy()) < 1e-5
    assert rel_err(m["pi_actions"].cpu().numpy(), mode(mu, o["squash"]).numpy()) < 1e-5


@pytest.mark.parametrize("name", ["reference_defaults", "large_squash_uniform"])
def test_bc_options_checkpoint_round_trip(name, tmp_path):
    from serl_b200.utils.checkpoints import restore_checkpoint, save_checkpoint
    agent, batch = _make(name)
    agent, _ = agent.update(batch)
    save_checkpoint(str(tmp_path), agent.state.params, step=1)
    fresh, _ = _make(name, seed=9)
    fresh.state.replace(params=restore_checkpoint(str(tmp_path), None))
    a, b = _flat(agent.state.params), _flat(fresh.state.params)
    assert a.keys() == b.keys()
    for k in a:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=k)
    np.testing.assert_array_equal(agent.sample_actions(batch["observations"], argmax=True), fresh.sample_actions(batch["observations"], argmax=True))


@pytest.mark.parametrize("name", ["large_squash_uniform", "gelu_ln_drop_softplus_squash"])
def test_bc_options_fp16_loss(name):
    agent, batch = _make(name, precision="fp16")
    cams, B = tuple(agent._cfg.cams), batch["actions"].shape[0]
    state = batch["observations"]["state"] if agent._cfg.use_proprio else None
    params = {k: torch.as_tensor(np.asarray(v)) for k, v in _flat(agent.state.params).items()}
    opt = {"count": 0, "mu": {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items() if "pretrained_encoder" not in k},
           "nu": {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items() if "pretrained_encoder" not in k}}
    rng0 = agent.state.rng
    agent, info = agent.update(batch)
    _, _, _, oinfo, grads, _ = oracle_update(params, opt, rng0, cams, _feats(agent, B), state, batch["actions"], _opts(agent))
    for k in ("actor_loss", "mse"):
        err = abs(float(info[k]) - oinfo[k]) / max(abs(oinfo[k]), 1.0)
        print(f"BC_FP16_ERR {name} {k} {err:.2e}")
        assert err <= FP16_LOSS_TOL, (k, float(info[k]), oinfo[k])
    worst = 0.0
    for l in agent._spec:
        got = agent._grad[l.offset:l.offset + l.size].view(l.shape).cpu().numpy()
        ref = grads[l.path].numpy()
        if "/encoder_" in l.path:                                   # image heads: behind stop_gradient (encoding.py:48-49)
            assert np.abs(ref).max() == 0 and np.abs(got).max() == 0, l.path
        else:
            assert np.abs(ref).max() > 0, l.path
            err = np.abs(got - ref).max() / np.abs(ref).max()
            worst = max(worst, err)
            assert err <= 2e-4, (l.path, err)
    print(f"BC_FP16_ERR {name} grad_leaves {worst:.2e}")
