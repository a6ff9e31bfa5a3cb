"""GPU: BCAgent with the trainable "small" and "resnet" encoders and with a fixed std, against the float64 oracle
(tests/bc_encoders_oracle.py: tests/small_encoder_oracle.py / tests/resnet_encoder_oracle.py composed with
tests/bc_options_oracle.py), which runs each camera's encoder on the same uint8 frames.

- `update` at the batch sizes where the encoder kernels change regime (tests/test_trainable_encoder_batches_gpu.py: 1 row, the
  9 / 18 rows of its partial M tiles, 256), with and without proprio, on every build, with explicit dropout masks: the loss and
  mse (fp32 build 1e-5; 16-bit builds 1e-4, 2e-4 below 64 rows, that file's bars), every trained leaf's gradient (of its max:
  fp32 build 1e-5, 16-bit builds 2e-4),
  the post-Adam parameters (tests/test_bc_options_gpu.py's noise-aware bar), and every encoder leaf: zero gradient, parameters
  bitwise unchanged, Adam moments exactly zero;
- a replay-ring batch replayed as a CUDA graph bitwise equal to the eager step, the encoder untouched after several steps;
- `sample_actions(argmax=True)` and `get_debug_metrics` against the oracle; a checkpoint round trip; make_bc_agent's defaults;
- the fixed std: update and inference against the oracle, with and without the tanh squash.
"""
import os

import numpy as np
import pytest
import torch

from bc_encoders_oracle import encode, log_prob, mode, policy, update as oracle_update
from helpers import fake_env, random_transitions, rel_err

pytestmark = pytest.mark.gpu

LAUNCHER = None                                                       # make_bc_agent's MLP: [256, 256] tanh, no LayerNorm
DROPOUT = {"activations": "tanh", "use_layer_norm": True, "hidden_dims": [256, 256], "dropout_rate": 0.1}
LOSS_TOL = {"fp32": 1e-5, "fp16": 1e-4, "bf16": 1e-4}
FEW_ROWS_16_LOSS_TOL = 2e-4                                           # 16-bit builds below 64 rows
GRAD_TOL = {"fp32": 1e-5, "fp16": 2e-4, "bf16": 2e-4}              # of each trained leaf's max

#         encoder, precision, cameras, B, use_proprio, network_kwargs
CASES = {
    "small-fp32-b1-proprio": ("small", "fp32", 2, 1, True, LAUNCHER),
    "small-fp16-b1-pixels": ("small", "fp16", 2, 1, False, DROPOUT),
    "small-bf16-b9-proprio": ("small", "bf16", 1, 9, True, DROPOUT),
    "small-fp16-b18-pixels": ("small", "fp16", 1, 18, False, LAUNCHER),
    "small-fp16-b256-proprio": ("small", "fp16", 2, 256, True, LAUNCHER),
    "small-fp32-b256-pixels": ("small", "fp32", 1, 256, False, DROPOUT),
    "resnet-fp32-b1-pixels": ("resnet", "fp32", 2, 1, False, DROPOUT),
    "resnet-fp16-b1-proprio": ("resnet", "fp16", 2, 1, True, LAUNCHER),
    "resnet-bf16-b9-pixels": ("resnet", "bf16", 1, 9, False, LAUNCHER),
    "resnet-fp16-b18-proprio": ("resnet", "fp16", 2, 18, True, DROPOUT),
    "resnet-fp16-b256-pixels": ("resnet", "fp16", 2, 256, False, DROPOUT),
    "resnet-fp32-b256-proprio": ("resnet", "fp32", 1, 256, True, LAUNCHER),
}


def _flat(tree, prefix=""):
    out = {}
    for k, v in tree.items():
        p = f"{prefix}/{k}" if prefix else k
        out.update(_flat(v, p)) if isinstance(v, dict) else out.__setitem__(p, v)
    return out


def _make(encoder, precision="fp32", cams=("front", "wrist"), use_proprio=True, mlp=LAUNCHER, policy_kwargs=None, seed=3, perturb=True):
    from serl_b200.agents.continuous.bc import BCAgent
    tr = random_transitions(np.random.default_rng(0), 1, cams)[0]
    pk = {"std_parameterization": "exp", "std_min": 1e-5, "std_max": 5} if policy_kwargs is None else policy_kwargs
    agent = BCAgent.create(seed, tr["observations"], tr["actions"], encoder_type=encoder, image_keys=cams, use_proprio=use_proprio,
                           network_kwargs=mlp, policy_kwargs=pk, precision=precision)
    if perturb:                                                      # every leaf off its initial value, as training would
        g = torch.Generator(device="cuda").manual_seed(seed)
        agent._params.add_(torch.randn(agent._n, device="cuda", generator=g) * 0.05)
    return agent


def _batch(cams, B, seed):
    trs = random_transitions(np.random.default_rng(seed), B, cams)
    obs = {**{c: np.stack([t["observations"][c] for t in trs]) for c in cams}, "state": np.stack([t["observations"]["state"] for t in trs])}
    return {"observations": obs, "actions": np.stack([t["actions"] for t in trs]).astype(np.float32)}


def _opts(agent):
    return dict(encoder=agent._cfg.encoder, arch=agent.arch, std=agent.std_parameterization, std_min=agent.std_min, std_max=agent.std_max,
                squash=agent.tanh_squash, use_proprio=agent._cfg.use_proprio,
                fixed_std=None if agent.fixed_std is None else agent.fixed_std.cpu().numpy())


def _images(batch, cams):
    return {c: batch["observations"][c][:, 0] for c in cams}


def _slices(agent, buf, pred):
    return {l.path: buf[l.offset:l.offset + l.size].view(l.shape) for l in agent._spec if pred(l.path)}


def _is_enc(path):
    return "/encoder_" in path


def _step_against_oracle(agent, batch, opt, bars, explicit_rng=None):
    """One agent.update against oracle_update on the same parameters, masks and frames; returns (opt, worst errors)."""
    cams, B = tuple(agent._cfg.cams), batch["actions"].shape[0]
    o = _opts(agent)
    state = batch["observations"]["state"] if o["use_proprio"] else None
    params = {k: torch.as_tensor(np.asarray(v)) for k, v in _flat(agent.state.params).items()}
    sle = mlp = None
    if explicit_rng is not None:
        sle = {c: explicit_rng.random((B, 4096)) < 0.9 for c in cams} if o["encoder"] == "resnet" else None
        mlp = [explicit_rng.random((B, H)) < 1 - o["arch"].dropout for H in o["arch"].hidden] if o["arch"].dropout else None
        agent.explicit_dropout = {**(sle or {}), "mlp": mlp or []}
    if opt is None:
        opt = {"count": 0, "mu": {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items()},
               "nu": {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items()}}
    st = agent._store
    enc_before = {k: v.clone() for k, v in _slices(agent, st.params, _is_enc).items()}
    rng0 = agent.state.rng
    agent, info = agent.update(batch)
    newp, opt, new_rng, oinfo, grads, masks = oracle_update(params, opt, rng0, cams, _images(batch, cams), state, batch["actions"], o,
                                                            sle_masks=sle, hidden_masks=mlp, lr=agent.learning_rate)
    np.testing.assert_array_equal(agent.state.rng, new_rng)
    worst = {}
    for k in ("actor_loss", "mse"):
        worst[k] = abs(float(info[k]) - oinfo[k]) / max(abs(oinfo[k]), 1.0)
        assert worst[k] <= bars["loss"], (k, float(info[k]), oinfo[k])
    got_g = _slices(agent, agent._grad, lambda p: True)
    for path, g in got_g.items():
        ref = grads[path].numpy()
        got = g.cpu().numpy()
        if _is_enc(path):                                   # behind the policy's stop_gradient (actor_critic_nets.py:185)
            assert not np.abs(ref).any() and not np.abs(got).any(), path
        else:
            assert np.abs(ref).max() > 0, path
            worst[path] = np.abs(got - ref).max() / np.abs(ref).max()
            assert worst[path] <= GRAD_TOL[agent._cfg.precision], (path, worst[path])
    for path, v in _slices(agent, st.params, _is_enc).items():
        assert torch.equal(v, enc_before[path]), f"{path}: an encoder leaf moved"
        assert not _slices(agent, st.m, lambda p: p == path)[path].any() and not _slices(agent, st.v, lambda p: p == path)[path].any(), path
    now, lr = _flat(agent.state.params), agent.learning_rate
    for path in got_g:
        if _is_enc(path):
            continue
        ref, got = newp[path].numpy(), np.asarray(now[path])
        gmag = np.abs(grads[path].numpy())
        noisy = gmag < 2e-2 * max(gmag.max(), 1e-30)
        allow = 1e-5 * max(np.abs(ref).max(), 1e-3) + lr * np.where(noisy, 2.2, 5e-3)
        assert (np.abs(got - ref) <= allow).all(), (path, np.abs(got - ref).max())
    return opt, worst


@pytest.mark.parametrize("case", list(CASES))
def test_update_matches_float64(case):
    encoder, precision, ncam, B, proprio, mlp = CASES[case]
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams = ("front", "wrist")[:ncam]
    agent = _make(encoder, precision, cams, proprio, mlp)
    bars = {"loss": FEW_ROWS_16_LOSS_TOL if precision != "fp32" and B < 64 else LOSS_TOL[precision]}
    opt, worst = None, {}
    rng = np.random.default_rng(B)
    for step in range(2):
        opt, w = _step_against_oracle(agent, _batch(cams, B, 10 + step), opt, bars, explicit_rng=rng)
        for k, v in w.items():
            worst[k] = max(worst.get(k, 0.0), v)
    assert agent.state.step == 2
    grads = {k: v for k, v in worst.items() if "/" in k}
    k = max(grads, key=grads.get)
    print(f"[{case}] actor_loss {worst['actor_loss']:.2e}, mse {worst['mse']:.2e}, worst gradient leaf {grads[k]:.2e} ({k})")


def test_keyed_masks_match_the_oracle():
    """Without explicit_dropout the step keys its masks on the device: resnet's SLE masks fold the camera index, the MLP's fold
    ncams + i (bc_encoders_oracle.keyed_masks)."""
    from bc_encoders_oracle import keyed_masks
    for encoder in ("small", "resnet"):
        cams, B = ("front", "wrist"), 5
        agent = _make(encoder, "fp32", cams, True, DROPOUT)
        rng0 = agent.state.rng
        _step_against_oracle(agent, _batch(cams, B, 1), None, {"loss": 1e-5})
        sle, mlp = keyed_masks(rng0, encoder, cams, B, agent.arch)
        b = agent._bufs[B]
        assert set(b["masks"]) == (set(cams) if encoder == "resnet" else set())
        for c in b["masks"]:
            np.testing.assert_array_equal(b["masks"][c].cpu().numpy().astype(bool), sle[c])
        for got, ref in zip(b["mlp_masks"], mlp):
            np.testing.assert_array_equal(got.cpu().numpy().astype(bool), ref)


# ---- replay rings and CUDA graphs ------------------------------------------------------------------------------------------
def _ring(cams, trs, seed=11):
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(cams), capacity=64, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=seed)
    for tr in trs:
        rb.insert(tr)
    return rb


@pytest.mark.parametrize("encoder,precision,proprio,mlp", [("small", "fp16", True, DROPOUT), ("small", "fp32", False, LAUNCHER),
                                                           ("resnet", "fp16", False, LAUNCHER), ("resnet", "fp32", True, DROPOUT)])
def test_graph_replay_equals_eager_and_keeps_the_encoder(encoder, precision, proprio, mlp):
    cams, B = ("front", "wrist"), 32
    trs = random_transitions(np.random.default_rng(0), 60, cams)
    agents = [_make(encoder, precision, cams, proprio, mlp) for _ in range(2)]
    agents[1].use_cuda_graphs = False
    its = [_ring(cams, trs).get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True}) for _ in range(2)]
    p0 = agents[0]._store.params.clone()
    for _ in range(5):                                               # eager, capture + replay, replays
        infos = [a.update(next(it))[1] for a, it in zip(agents, its)]
        for k in ("actor_loss", "mse"):
            assert torch.equal(infos[0][k], infos[1][k]), k
    assert len(agents[0]._graphs) == 1 and not agents[1]._graphs
    sa, sb = agents[0]._store, agents[1]._store
    for name in ("params", "target", "m", "v", "counts"):
        assert torch.equal(getattr(sa, name), getattr(sb, name)), name
    assert np.array_equal(agents[0].state.rng, agents[1].state.rng) and agents[0].state.step == agents[1].state.step == 5
    before = _slices(agents[0], p0, lambda p: True)
    for path, v in _slices(agents[0], sa.params, lambda p: True).items():
        assert torch.equal(v, before[path]) == _is_enc(path), path          # the encoder untouched, every other leaf trained
    for buf in (sa.m, sa.v):
        assert not any(v.any() for v in _slices(agents[0], buf, _is_enc).values())
    for a in agents:
        a.check_status()


# ---- inference, checkpoints, the launcher ----------------------------------------------------------------------------------
def _oracle_dist(agent, batch, temperature=1.0):
    o = _opts(agent)
    cams = tuple(agent._cfg.cams)
    params = {k: torch.as_tensor(np.asarray(v)).double() for k, v in _flat(agent.state.params).items()}
    st = torch.as_tensor(batch["observations"]["state"]).double() if o["use_proprio"] else None
    enc = encode(params, o["encoder"], cams, _images(batch, cams), st, None)
    return (*policy(params, enc, o, temperature=temperature), o)


def _check_inference(agent, batch, tol=1e-5):
    from oracle.jax_prng import normal
    obs, B, A = batch["observations"], batch["actions"].shape[0], batch["actions"].shape[1]
    mu, sd, o = _oracle_dist(agent, batch)
    a = agent.sample_actions(obs, argmax=True)
    assert rel_err(a, mode(mu, o["squash"]).numpy()) < tol
    seed = np.array([0, 11], np.uint32)
    s = agent.sample_actions(obs, seed=seed, temperature=0.5)
    mu5, sd5, _ = _oracle_dist(agent, batch, 0.5)
    assert rel_err(s, mode(mu5 + sd5 * torch.as_tensor(normal(seed, (B, A))).double(), o["squash"]).numpy()) < tol
    one = agent.sample_actions({k: v[0] for k, v in obs.items()}, argmax=True)
    assert one.shape == (A,) and rel_err(one, mode(mu, o["squash"]).numpy()[0]) < tol
    m = agent.get_debug_metrics(batch)
    act = torch.as_tensor(batch["actions"]).double()
    assert rel_err(m["mse"].cpu().numpy(), ((mode(mu, o["squash"]) - act) ** 2).sum(-1).numpy()) < tol
    assert rel_err(m["log_probs"].cpu().numpy(), log_prob(mu, sd, act, o["squash"]).numpy()) < tol
    assert rel_err(m["pi_actions"].cpu().numpy(), mode(mu, o["squash"]).numpy()) < tol


@pytest.mark.parametrize("encoder", ["small", "resnet"])
@pytest.mark.parametrize("proprio", [True, False])
def test_inference_matches_float64(encoder, proprio):
    cams = ("front", "wrist")
    agent = _make(encoder, "fp32", cams, proprio, DROPOUT, seed=5)
    _check_inference(agent, _batch(cams, 6, 2))


@pytest.mark.parametrize("encoder", ["small", "resnet"])
def test_checkpoint_round_trip(encoder, tmp_path):
    from serl_b200.utils.checkpoints import restore_checkpoint, save_checkpoint
    cams = ("front", "wrist")
    agent = _make(encoder, "fp16", cams, True, DROPOUT)
    batch = _batch(cams, 8, 3)
    for _ in range(2):
        agent, _ = agent.update(batch)
    save_checkpoint(str(tmp_path), agent.state, step=2)
    fresh = _make(encoder, "fp16", cams, True, DROPOUT, seed=9)
    fresh = fresh.replace(state=restore_checkpoint(str(tmp_path), fresh.state, step=2))
    for name in ("params", "target", "m", "v", "counts"):
        assert torch.equal(getattr(agent._store, name), getattr(fresh._store, name)), name
    assert np.array_equal(agent.state.rng, fresh.state.rng) and fresh.state.step == 2
    np.testing.assert_array_equal(agent.sample_actions(batch["observations"], argmax=True), fresh.sample_actions(batch["observations"], argmax=True))
    _, ia = agent.update(batch)
    _, ib = fresh.update(batch)
    assert all(torch.equal(ia[k], ib[k]) for k in ia)


def test_make_bc_agent_defaults_train_a_small_agent():
    from serl_b200.utils.launcher import make_bc_agent
    tr = random_transitions(np.random.default_rng(0), 1, ("image",))[0]
    agent = make_bc_agent(0, tr["observations"], tr["actions"])
    assert agent._cfg.encoder == "small" and agent._cfg.precision == "fp32"
    batch = _batch(("image",), 16, 4)
    enc0 = {k: v.clone() for k, v in _slices(agent, agent._store.params, _is_enc).items()}
    p0 = agent._store.params.clone()
    losses = []
    for _ in range(3):
        agent, info = agent.update(batch)
        losses.append(float(info["actor_loss"]))
    assert all(np.isfinite(losses)) and not torch.equal(p0, agent._store.params)
    assert all(torch.equal(v, enc0[k]) for k, v in _slices(agent, agent._store.params, _is_enc).items())
    assert agent.sample_actions(batch["observations"], argmax=True).shape == (16, batch["actions"].shape[1])


# ---- the fixed std ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("squash", [False, True])
def test_fixed_std_update_and_inference(squash):
    cams, B = ("front",), 40
    # one std below std_min and one above std_max: both clipped
    pk = {"std_parameterization": "fixed", "fixed_std": [0.2, 0.5, 1e-7, 9.0], "std_min": 1e-3, "std_max": 2.0,
          "tanh_squash_distribution": squash}
    agent = _make("small", "fp32", cams, True, DROPOUT, policy_kwargs=pk)
    opt = None
    rng = np.random.default_rng(7)
    for step in range(2):
        batch = _batch(cams, B, 20 + step)
        opt, _ = _step_against_oracle(agent, batch, opt, {"loss": 1e-5}, explicit_rng=rng)
    agent.explicit_dropout = None
    _check_inference(agent, _batch(cams, 5, 30))
    _, sd, _ = _oracle_dist(agent, _batch(cams, 5, 30))
    np.testing.assert_allclose(sd[0].numpy(), [0.2, 0.5, 1e-3, 2.0], rtol=1e-7)
