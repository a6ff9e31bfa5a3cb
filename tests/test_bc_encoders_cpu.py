"""CPU: BCAgent with the trainable "small" / "resnet" encoders and the fixed std, without a GPU.

- the float64 oracle (tests/bc_encoders_oracle.py): its gradients against central differences, and exactly zero on every encoder
  leaf (the policy's stop_gradient), although the loss does move with those leaves;
- the state tree's paths and shapes per encoder type (the reference's: no pretrained_encoder level), the same encoder subtree as
  DrQ's, and the initialisers;
- `bc_options` / `BCAgent.create` for the fixed std: accepted, and the error cases;
- the host side of an update with the kernels replaced by a recorder: the encoder forward launches, no encoder backward, no std
  head with a fixed std;
- a checkpoint round trip of the whole state, on the recorder.
"""
import pickle

import numpy as np
import pytest
import torch

from bc_encoders_oracle import keyed_masks, loss_fn, policy, update
from helpers import random_transitions

CAMS = ("front", "wrist")
TANH = {"activations": "tanh", "use_layer_norm": True, "hidden_dims": [128, 64], "dropout_rate": 0.1}


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


def _flat(tree, prefix=""):
    out = {}
    for k, v in tree.items():
        p = f"{prefix}/{k}" if prefix else k
        out.update(_flat(v, p)) if isinstance(v, dict) else out.__setitem__(p, v)
    return out


def _agent(encoder, seed=1, hw=None, cams=CAMS, **kw):
    from serl_b200.agents.continuous.bc import BCAgent
    hw = hw or (128 if encoder == "resnet" else 48)
    trs = random_transitions(np.random.default_rng(0), 1, cams, hw)
    return BCAgent.create(seed, trs[0]["observations"], trs[0]["actions"], encoder_type=encoder, image_keys=cams, device="cpu", **kw)


# ---- the oracle ------------------------------------------------------------------------------------------------------------
def _oracle_problem(encoder, std="exp", proprio=True, B=3, seed=0):
    """A small random parameter tree (encoder leaves from the agent's own spec) and batch."""
    from serl_b200.agents.continuous.bc import bc_spec
    from serl_b200.params import MlpArch, init_leaves, kaiming_in_resnet_encoder, xavier_outside_encoders
    arch = MlpArch((32, 16), "tanh", True, 0.25)
    hw = 128 if encoder == "resnet" else 40
    rng = np.random.default_rng(seed)
    spec, _ = bc_spec(("c0",), 5, 3, arch, "exp" if std == "fixed" else std, proprio, encoder)
    if std == "fixed":
        spec = [l for l in spec if not l.path.startswith("modules_actor/Dense_1")]
    params = {k: torch.as_tensor(v).double() for k, v in init_leaves(rng, spec, xavier_outside_encoders, kaiming=kaiming_in_resnet_encoder).items()}
    for k in params:                                  # biases, scales and heads off their initial values
        params[k] = params[k] + 0.05 * torch.as_tensor(rng.standard_normal(params[k].shape))
    opts = dict(encoder=encoder, arch=arch, std=std, std_min=1e-5, std_max=10.0, squash=False, use_proprio=proprio,
                fixed_std=np.array([0.3, 0.7, 1.2], np.float32))
    images = {"c0": rng.integers(0, 256, (B, hw, hw, 3), dtype=np.uint8)}
    state = rng.standard_normal((B, 5)) if proprio else None
    actions = np.clip(rng.standard_normal((B, 3)) * 0.5, -0.9, 0.9)
    sle, mlp = keyed_masks(np.array([0, 7], np.uint32), encoder, ("c0",), B, arch)
    return params, opts, images, state, actions, sle, mlp


@pytest.mark.parametrize("encoder,std,proprio", [("small", "exp", True), ("small", "fixed", False), ("resnet", "softplus", True),
                                                 ("resnet", "fixed", True)])
def test_oracle_gradients_match_finite_differences_and_vanish_on_the_encoder(encoder, std, proprio):
    params, opts, images, state, actions, sle, mlp = _oracle_problem(encoder, std, proprio)
    train = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    loss, _ = loss_fn(train, opts, ("c0",), images, state, actions, sle, mlp)
    grads = dict(zip(train, torch.autograd.grad(loss, list(train.values()), allow_unused=True)))
    enc = [k for k in params if "/encoder_" in k]
    assert enc and all(grads[k] is None or not grads[k].any() for k in enc)
    rng = np.random.default_rng(1)

    def at(k, idx, h):
        return loss_fn({**params, k: params[k] + h * _unit(params[k], idx)}, opts, ("c0",), images, state, actions, sle, mlp)[0].item()

    # every trained leaf: autograd against central differences at two entries
    trained = [k for k in params if "/encoder_" not in k]
    assert any(k.startswith("modules_actor/encoder/Dense_0") for k in trained) == proprio
    assert ("modules_actor/Dense_1/kernel" in trained) == (std != "fixed")
    for k in trained:
        for idx in {tuple(rng.integers(0, s) for s in params[k].shape), tuple(np.unravel_index(int(grads[k].abs().argmax()), params[k].shape))}:
            fd = (at(k, idx, 1e-6) - at(k, idx, -1e-6)) / 2e-6
            assert abs(fd - grads[k][idx].item()) <= 1e-6 * max(1.0, abs(fd)), (k, idx, fd, grads[k][idx].item())
    # the encoder's zero gradient is the stop_gradient, not a dead leaf: its last Dense moves the loss
    k = "modules_actor/encoder/encoder_c0/Dense_0/bias"
    assert abs(at(k, (0,), 1e-3) - at(k, (0,), -1e-3)) > 1e-9


def _unit(t, idx):
    e = torch.zeros_like(t)
    e[idx] = 1.0
    return e


def test_oracle_update_leaves_the_encoder_and_its_moments_at_zero():
    params, opts, images, state, actions, _, _ = _oracle_problem("small")
    z = {k: torch.zeros_like(v) for k, v in params.items()}
    opt = {"count": 0, "mu": dict(z), "nu": dict(z)}
    for _ in range(2):
        new, opt, _, info, grads, masks = update(params, opt, np.array([0, 7], np.uint32), ("c0",), images, state, actions, opts)
        assert masks["sle"] is None and len(masks["mlp"]) == 2            # the small encoder has no Dropout
        for k in params:
            if "/encoder_" in k:
                assert torch.equal(new[k], params[k]) and not opt["mu"][k].any() and not opt["nu"][k].any(), k
            else:
                assert not torch.equal(new[k], params[k]), k
        params = new
    assert np.isfinite(info["actor_loss"]) and info["mse"] > 0


def test_oracle_fixed_std_is_clipped_and_scaled():
    params, opts, images, state, *_ = _oracle_problem("small", "fixed")
    from bc_encoders_oracle import encode
    enc = encode(params, "small", ("c0",), images, torch.as_tensor(state), None)
    _, sd = policy(params, enc, dict(opts, std_min=0.5, std_max=1.0), temperature=0.25)
    torch.testing.assert_close(sd, torch.tensor([0.5, 0.7, 1.0], dtype=torch.float64).mul(0.5).expand(3, 3), rtol=1e-7, atol=0)


# ---- the state tree --------------------------------------------------------------------------------------------------------
def _expected_encoder(encoder):
    if encoder == "small":
        out = {}
        for i, (ci, co) in enumerate(((3, 32), (32, 64), (64, 128), (128, 256))):
            out[f"Conv_{i}/kernel"], out[f"Conv_{i}/bias"] = (3, 3, ci, co), (co,)
        return {**out, "Dense_0/kernel": (256, 256), "Dense_0/bias": (256,), "LayerNorm_0/scale": (256,), "LayerNorm_0/bias": (256,)}
    out = {"conv_init/kernel": (7, 7, 3, 64), "norm_init/scale": (64,), "norm_init/bias": (64,)}
    cin = 64
    for i, f in enumerate((64, 128, 256, 512)):
        b = f"ResNetBlock_{i}"
        out.update({f"{b}/Conv_0/kernel": (3, 3, cin, f), f"{b}/Conv_1/kernel": (3, 3, f, f)})
        out.update({f"{b}/MyGroupNorm_{j}/{s}": (f,) for j in (0, 1) for s in ("scale", "bias")})
        if cin != f:
            out.update({f"{b}/conv_proj/kernel": (1, 1, cin, f), f"{b}/norm_proj/scale": (f,), f"{b}/norm_proj/bias": (f,)})
        cin = f
    return {**out, "SpatialLearnedEmbeddings_0/kernel": (4, 4, 512, 8), "Dense_0/kernel": (4096, 256), "Dense_0/bias": (256,),
            "LayerNorm_0/scale": (256,), "LayerNorm_0/bias": (256,)}


@pytest.mark.parametrize("encoder", ["small", "resnet"])
@pytest.mark.parametrize("proprio", [True, False])
def test_state_tree_per_encoder_type(dry, encoder, proprio):
    from serl_b200.params import ENC, trainable_spec
    agent = _agent(encoder, use_proprio=proprio)
    want = {f"{ENC}/encoder_{c}/{k}": v for c in CAMS for k, v in _expected_encoder(encoder).items()}
    want.update({"modules_actor/network/Dense_0/kernel": (512 + 64 * proprio, 256), "modules_actor/network/Dense_0/bias": (256,),
                 "modules_actor/network/Dense_1/kernel": (256, 256), "modules_actor/network/Dense_1/bias": (256,),
                 "modules_actor/Dense_0/kernel": (256, 4), "modules_actor/Dense_0/bias": (4,),
                 "modules_actor/Dense_1/kernel": (256, 4), "modules_actor/Dense_1/bias": (4,)})
    if proprio:
        want.update({f"{ENC}/Dense_0/kernel": (7, 64), f"{ENC}/Dense_0/bias": (64,), f"{ENC}/LayerNorm_0/scale": (64,),
                     f"{ENC}/LayerNorm_0/bias": (64,)})
    d = agent.state.state_dict()
    for key in ("params", "target_params"):
        assert {k: tuple(v.shape) for k, v in _flat(d[key]).items()} == want, key
    for key in ("mu", "nu"):
        assert {k: tuple(v.shape) for k, v in _flat(d["opt_states"][key]).items()} == want, key
    assert not agent._frozen_trunk.leaves
    # the same encoder subtree (names, shapes, order) as DrQ's agent with that encoder
    drq = [(l.path, l.shape) for l in trainable_spec(CAMS, 7, 4, 2, True, use_proprio=proprio, encoder=encoder) if "/encoder_" in l.path]
    assert [(l.path, l.shape) for l in agent._spec if "/encoder_" in l.path] == drq
    # initialisers: kaiming-normal ResNet convs, lecun-normal small convs / SLE / bottleneck Dense, zero biases, unit scales
    p = _flat(d["params"])
    kern = {"small": ("Conv_3/kernel", 1.0), "resnet": ("ResNetBlock_2/Conv_1/kernel", 2.0)}[encoder]
    w = p[f"{ENC}/encoder_front/{kern[0]}"]
    fan_in = int(np.prod(w.shape[:-1]))
    assert abs(w.std() / np.sqrt(kern[1] / fan_in) - 1) < 0.05
    assert not p[f"{ENC}/encoder_front/Dense_0/bias"].any() and (p[f"{ENC}/encoder_wrist/LayerNorm_0/scale"] == 1).all()
    assert not np.array_equal(p[f"{ENC}/encoder_front/Dense_0/kernel"], p[f"{ENC}/encoder_wrist/Dense_0/kernel"])


def test_launcher_defaults_build_a_small_agent(dry):
    from serl_b200.utils.launcher import make_bc_agent
    trs = random_transitions(np.random.default_rng(0), 1, ("image",), 64)
    agent = make_bc_agent(0, trs[0]["observations"], trs[0]["actions"], device="cpu")
    assert agent._cfg.encoder == "small" and agent._cfg.image_hw == 64 and agent._cfg.use_proprio
    assert "Conv_0" in agent.state.params["modules_actor"]["encoder"]["encoder_image"]


def test_frame_sizes(dry):
    from serl_b200.agents.continuous.bc import BCAgent
    _agent("small", hw=31, cams=("image",))                                    # the fourth conv keeps one position
    for enc, hw in (("small", 30), ("resnet", 64), ("resnet", 96)):
        trs = random_transitions(np.random.default_rng(0), 1, ("image",), hw)
        with pytest.raises(NotImplementedError):
            BCAgent.create(0, trs[0]["observations"], trs[0]["actions"], encoder_type=enc, image_keys=("image",), device="cpu")
    with pytest.raises(NotImplementedError):
        _agent("resnet-18")


# ---- the fixed std ---------------------------------------------------------------------------------------------------------
def test_fixed_std_options():
    from serl_b200.agents.continuous.bc import BC_LAUNCHER_MLP, bc_options, resolve_fixed_std
    assert bc_options(None, {"std_parameterization": "fixed", "fixed_std": [0.1, 0.2]}) == (BC_LAUNCHER_MLP, "fixed", 1e-5, 10.0, False)
    pk = {"std_parameterization": "fixed", "fixed_std": np.array([0.1, 0.2]), "tanh_squash_distribution": True, "std_max": 1.0}
    assert bc_options(None, pk)[1:] == ("fixed", 1e-5, 1.0, True)
    np.testing.assert_array_equal(resolve_fixed_std(pk), np.array([0.1, 0.2], np.float32))
    for bad, exc in (({"std_parameterization": "fixed"}, NotImplementedError),                     # no fixed_std
                     ({"fixed_std": [0.1, 0.2]}, NotImplementedError),                             # the reference's assert
                     ({"std_parameterization": "exp", "fixed_std": [0.1]}, NotImplementedError),
                     ({"std_parameterization": "fixed", "fixed_std": [[0.1, 0.2]]}, ValueError),
                     ({"std_parameterization": "fixed", "fixed_std": 0.1}, ValueError),
                     ({"std_parameterization": "fixed", "fixed_std": [0.1, np.nan]}, ValueError),
                     ({"std_parameterization": "fixed", "fixed_std": []}, ValueError)):
        with pytest.raises(exc):
            bc_options(None, bad)


def test_fixed_std_create_and_sac_refusal(dry):
    from serl_b200.agents.continuous.sac import architecture_settings
    with pytest.raises(ValueError, match="action dimensions"):
        _agent("small", policy_kwargs={"std_parameterization": "fixed", "fixed_std": [0.5] * 3})
    agent = _agent("small", policy_kwargs={"std_parameterization": "fixed", "fixed_std": [0.5, 0.6, 0.7, 0.8]})
    assert agent.std_parameterization == "fixed" and agent.fixed_std.tolist() == pytest.approx([0.5, 0.6, 0.7, 0.8])
    tree = agent.state.params["modules_actor"]
    assert "Dense_1" not in tree and "log_stds" not in tree and tree["Dense_0"]["kernel"].shape == (256, 4)
    with pytest.raises(NotImplementedError):                                  # SAC / DrQ keep refusing a fixed std
        architecture_settings({"std_parameterization": "fixed", "fixed_std": [0.5] * 4}, {}, pixel=True, allow_dropout=True)


# ---- the host side of a step -----------------------------------------------------------------------------------------------
def _batch(encoder, B=6, cams=CAMS):
    trs = random_transitions(np.random.default_rng(0), B, cams, 128 if encoder == "resnet" else 48)
    obs = {**{c: np.stack([t["observations"][c] for t in trs]) for c in cams}, "state": np.stack([t["observations"]["state"] for t in trs])}
    return {"observations": obs, "actions": np.stack([t["actions"] for t in trs]).astype(np.float32)}


ENCODER_BACKWARD = ("wgrad", "dgrad", "groupnorm_bwd", "maxpool3x3s2_bwd", "sconv_mean_bwd", "sle_bwd", "sle_input")


@pytest.mark.parametrize("encoder", ["small", "resnet"])
def test_update_call_sequence(dry, encoder):
    """Per camera the encoder forward (small: four convs and the mean pool; resnet: the stem prep and the SLE head), no frozen trunk,
    no launch of any encoder backward, the keyed SLE masks for "resnet" only, and one Adam step over the whole store."""
    agent = _agent(encoder, network_kwargs=TANH, use_proprio=True)
    batch = _batch(encoder)
    del dry[:]
    agent.update(batch)
    n = len(CAMS)
    assert not [c for c in dry if any(s in c for s in ENCODER_BACKWARD)], dry
    assert not [c for c in dry if "trunk" in c or "stem_pool" in c or "conv3x3" in c]
    if encoder == "small":
        assert dry.count("serl_sconv_fwd") == 4 * n and dry.count("serl_sconv_mean_fwd") == n and "serl_sle_fwd" not in dry
        assert dry.count("serl_dropout_mask_fill") == 2                      # the MLP's two layers only
    else:
        assert dry.count("serl_rconv_stem_prep") == n and dry.count("serl_sle_fwd") == n
        assert dry.count("serl_dropout_mask_fill") == n + 2
    assert dry.count("serl_layernorm_tanh_fwd") == n + 1                      # the image heads and the proprio block
    assert dry.count("serl_layernorm_tanh_bwd") == 1                          # the proprio block only
    assert len([c for c in dry if c.startswith("serl_adam")]) == 1
    assert agent.state.step == 1


def test_fixed_std_call_sequence(dry):
    agent = _agent("small", policy_kwargs={"std_parameterization": "fixed", "fixed_std": [0.5] * 4})
    batch = _batch("small")
    del dry[:]
    agent.update(batch)
    assert dry.count("serl_bc_loss_std") == 1 and "serl_bc_loss" not in dry
    del dry[:]
    agent.sample_actions({k: v for k, v in batch["observations"].items()}, argmax=True)
    assert dry.count("serl_tanh_gaussian_fwd_std") == 1


# ---- checkpoints -----------------------------------------------------------------------------------------------------------
def _perturb(agent, seed):
    g = torch.Generator().manual_seed(seed)
    st = agent._store
    for buf in (st.params, st.target, st.m, st.v):
        buf.add_(torch.rand(buf.shape, generator=g))
    st.counts.fill_(17)
    agent.state.replace(rng=np.array([seed, 3 * seed + 1], np.uint32), step=17)


@pytest.mark.parametrize("encoder", ["small", "resnet"])
def test_checkpoint_round_trip(dry, tmp_path, encoder):
    from serl_b200.utils.checkpoints import restore_checkpoint, save_checkpoint
    a = _agent(encoder, seed=1)
    _perturb(a, 5)
    path = save_checkpoint(str(tmp_path), a.state, step=17)

    class NumpyOnly(pickle.Unpickler):
        def find_class(self, module, name):
            assert module.split(".")[0] in ("numpy", "builtins"), (module, name)
            return super().find_class(module, name)

    with open(path, "rb") as f:
        payload = NumpyOnly(f).load()
    assert not [k for k in _flat(payload["params"]) if "pretrained_encoder" in k]
    b = _agent(encoder, seed=2)
    b._graphs["stale"] = "warm"
    assert not torch.equal(b._store.params, a._store.params)
    b.replace(state=restore_checkpoint(str(tmp_path), None))
    for name in ("params", "target", "m", "v", "counts"):
        assert torch.equal(getattr(a._store, name), getattr(b._store, name)), name
    assert torch.equal(a._rng, b._rng) and b.state.step == 17 and not b._graphs
    c = _agent(encoder, seed=3)
    c = c.replace(state=restore_checkpoint(str(tmp_path), c.state, step=17))
    assert torch.equal(a._store.params, c._store.params) and torch.equal(a._store.v, c._store.v)
