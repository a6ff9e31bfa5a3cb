"""GPU: the reference's network architecture options (MLP widths / depth / activation / LayerNorm, "exp" / "softplus" /
"uniform" std) through the public API against the float64 oracle with the same networks (tests/arch_oracle.py), on the
fp32 build, with the bars of the existing oracle tests (DESIGN.md section 5): Q, targets, losses and actions within 1e-5,
gradient leaves within 2e-4 of their max, post-Adam parameters with the noise-aware bar.  Plus replay / determinism, a
checkpoint round trip, clipping with "uniform", and the fp16 build's losses."""
import numpy as np
import pytest
import torch

from helpers import fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, rel_err, to_numpy_tree
from test_agent_gpu import G_TOL, Q_TOL, _compare_state, _perturb

pytestmark = pytest.mark.gpu

REF_NET = {"hidden_dims": [256, 256], "activations": "swish", "use_layer_norm": False}
CASES = {
    # the reference constructors' own defaults (sac.py:486-504, drq.py:104-131)
    "reference_defaults": (REF_NET, REF_NET, "uniform"),
    "512x3_relu_ln_softplus": ({"hidden_dims": [512, 512, 512], "activations": "relu", "use_layer_norm": True},) * 2 + ("softplus",),
    # critic and policy differ; one uses gelu, one leaky_relu without LayerNorm
    "mixed_gelu": ({"hidden_dims": [512, 128], "activations": "gelu", "use_layer_norm": True},
                   {"hidden_dims": [192], "activations": "leaky_relu", "use_layer_norm": False}, "exp"),
}
TXS = ("critic", "actor", "temperature")


def _kw(case, **extra):
    c, p, std = CASES[case]
    return dict(critic_network_kwargs=dict(c), policy_network_kwargs=dict(p),
                policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": std, "std_min": 1e-5, "std_max": 5}, **extra)


def _drq(cams, seed, case, precision="fp32", **extra):
    """DrQAgent.create_drq with the launcher's hyper-parameters (utils/launcher.py:79-116) and the case's networks."""
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(cams), capacity=200, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
    trs = random_transitions(np.random.default_rng(seed), 260, cams)
    for tr in trs:
        rb.insert(tr)
    agent = DrQAgent.create_drq(seed, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet-pretrained", use_proprio=True,
                                image_keys=cams, temperature_init=1e-2, discount=0.96, backup_entropy=False, critic_ensemble_size=10,
                                critic_subsample_size=2, precision=precision, **_kw(case, **extra))
    _perturb(agent, seed=seed)
    return agent, rb


def _host(batch):
    from oracle.replay import unpack
    return unpack(to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"}))


# relu and leaky_relu have a kink at 0: a pre-activation within fp32 rounding of it (the fp32 trunk features alone differ from
# the float64 oracle's by ~1e-6) takes the other branch in one of the two runs, and that single unit moves every gradient leaf
# upstream of it by up to ~2e-3 of the leaf's max.  Losses, Q-values and actions are continuous there and keep their bar.
KINK_G_TOL = 5e-3


def _check_grads(agent, oinfo, groups):
    st, c = agent._store, agent._cfg
    tol = KINK_G_TOL if {c.critic_arch.act, c.policy_arch.act} & {"relu", "leaky_relu"} else G_TOL
    for leaf in st.spec:
        if leaf.group not in groups:
            continue
        ref = oinfo["_grads"][TXS[leaf.group]][leaf.path].numpy()
        got = st.view(st.grad, leaf.path).cpu().numpy()
        assert np.abs(got - ref).max() <= tol * max(np.abs(ref).max(), 1e-8), leaf.path


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("cams", [("front",), ("front", "wrist")], ids=["cam1", "cam2"])
def test_drq_steps_match_oracle(case, cams):
    from arch_oracle import networks_of
    from oracle import drq as O
    from oracle import jax_prng as P
    B = 12
    agent, rb = _drq(cams, 7, case)
    agent.use_cuda_graphs = False
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    eng = agent._engine(B)
    with networks_of(agent):
        for step in range(2):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            agent, info = agent.update_critics(batch)
            oinfo = O.update_critics(ostate, ocfg, _host(batch))
            assert rel_err(eng.q.cpu().numpy(), oinfo["critic"]["_q"].numpy()) < Q_TOL
            assert rel_err(eng.target_q.cpu().numpy(), oinfo["critic"]["_target_q"].numpy()) < Q_TOL
            for k in ("critic_loss", "predicted_qs", "target_qs"):
                np.testing.assert_allclose(float(info["critic"][k]), oinfo["critic"][k], rtol=Q_TOL, atol=1e-6)
            if step == 0:
                _check_grads(agent, oinfo, (0,))
            _compare_state(agent, ostate, oinfo, f"update_critics {step}")
        for nets in ({"critic"}, {"actor"}, {"temperature"}, {"actor", "temperature"}, {"critic", "actor", "temperature"}):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            rnd, new_rng = O.derive_update_randomness(ostate.rng, B, 4, cams, True, ocfg.ensemble, ocfg.subsample or 0, nets=tuple(sorted(nets)))
            agent, info = agent.update(batch, networks_to_update=frozenset(nets))
            oinfo = O.update(ostate, ocfg, _host(batch), rnd, frozenset(nets), torch.float64, new_rng)
            if "critic" in nets:
                np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL, atol=1e-6)
            if "actor" in nets:
                for k in ("actor_loss", "temperature", "entropy"):
                    np.testing.assert_allclose(float(info["actor"][k]), oinfo["actor"][k], rtol=Q_TOL, atol=1e-6)
            if "temperature" in nets:
                np.testing.assert_allclose(float(info["temperature"]["temperature_loss"]), oinfo["temperature"]["temperature_loss"],
                                           rtol=Q_TOL, atol=1e-7)
            _check_grads(agent, oinfo, tuple(TXS.index(n) for n in nets))
            _compare_state(agent, ostate, oinfo, f"update {sorted(nets)}")
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        agent, info = agent.update_high_utd(batch, utd_ratio=1)
        oinfo = O.update_high_utd(ostate, ocfg, _host(batch), 1)
        for k in ("critic_loss", "predicted_qs", "target_qs"):
            np.testing.assert_allclose(float(info["critic"][k]), oinfo["critic"][k], rtol=Q_TOL, atol=1e-6)
        np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-6)
        _compare_state(agent, ostate, oinfo, "update_high_utd")
        # sample_actions: seeded and argmax, unbatched and batched
        ostate = oracle_state_from_agent(agent)
        rng = np.random.default_rng(0)
        obs = {c: rng.integers(0, 256, (3, 1, 128, 128, 3), dtype=np.uint8) for c in cams}
        obs["state"] = rng.standard_normal((3, 1, 7)).astype(np.float32)
        key = P.prng_key(2024)
        assert rel_err(agent.sample_actions(obs, seed=key), O.sample_actions(ostate, ocfg, obs, seed=key).numpy()) < Q_TOL
        assert rel_err(agent.sample_actions(obs, argmax=True), O.sample_actions(ostate, ocfg, obs, argmax=True).numpy()) < Q_TOL
        one = {k: v[0] for k, v in obs.items()}
        a = agent.sample_actions(one, seed=key)
        assert a.shape == (4,) and rel_err(a, O.sample_actions(ostate, ocfg, {k: v[None] for k, v in one.items()}, seed=key)[0].numpy()) < Q_TOL
    agent.check_status()


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("utd", [1, 4])
def test_state_sac_high_utd_matches_oracle(case, utd):
    from arch_oracle import networks_of
    from oracle import drq as O
    from serl_b200.agents.continuous.sac import SACAgent
    S, A, B = 10, 4, 32
    rng = np.random.default_rng(0)
    agent = SACAgent.create_states(42, rng.standard_normal(S).astype(np.float32), rng.uniform(-1, 1, A).astype(np.float32),
                                   temperature_init=1e-2, discount=0.99, critic_ensemble_size=10, critic_subsample_size=2, **_kw(case))
    _perturb(agent, seed=4)
    agent._store.counts.fill_(700)            # inside the 2000-step warm-up ramp so lr != 0
    ostate, ocfg = oracle_state_from_agent(agent), oracle_cfg_from_agent(agent)
    batch = dict(observations=rng.standard_normal((B, S)).astype(np.float32), next_observations=rng.standard_normal((B, S)).astype(np.float32),
                 actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.random(B).astype(np.float32),
                 masks=(rng.random(B) > 0.1).astype(np.float32), dones=np.zeros(B, bool))
    agent, info = agent.update_high_utd(batch, utd_ratio=utd)
    ob = dict(batch, observations={"state": batch["observations"]}, next_observations={"state": batch["next_observations"]})
    with networks_of(agent):
        oinfo = O.update_high_utd(ostate, ocfg, ob, utd, augment=False)
        np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL)
        np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-6)
        _check_grads(agent, oinfo, (1, 2))
        _compare_state(agent, ostate, oinfo, f"state sac {case} utd {utd}")
        ostate = oracle_state_from_agent(agent)
        x = rng.standard_normal((5, S)).astype(np.float32)
        assert rel_err(agent.sample_actions(x, argmax=True), O.sample_actions(ostate, ocfg, {"state": x}, argmax=True).numpy()) < Q_TOL


def test_uniform_std_with_actor_clipping_matches_oracle():
    """clip_grad_norm on the actor tx: its global norm covers log_stds (a leaf of the actor tx's group)."""
    from arch_oracle import networks_of
    from oracle import optim
    cams, B = ("front",), 12
    agent, rb = _drq(cams, 5, "reference_defaults", actor_optimizer_kwargs={"clip_grad_norm": 1e-3})
    agent.use_cuda_graphs = False
    c = agent._cfg
    oopts = optim.OptimizerOptions(lr=dict(zip(TXS, c.lr)), cosine_decay_steps=dict(zip(TXS, c.decay)), clip_grad_norm=dict(zip(TXS, c.clip)))
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    with networks_of(agent):
        for _ in range(2):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            agent, info = agent.update_high_utd(batch, utd_ratio=1)
            oinfo = optim.update_high_utd(ostate, ocfg, _host(batch), 1, oopts)
            np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-6)
            ref = float(oinfo["_grad_norm"]["actor"])
            assert abs(float(agent._engine(B).grad_norms[1]) - ref) <= G_TOL * ref
            assert ref > 1e-3                                           # it clips
            g = oinfo["_grads"]["actor"]["modules_actor/log_stds"].numpy()
            got = agent._store.view(agent._store.grad, "modules_actor/log_stds").cpu().numpy()
            assert np.abs(g).max() > 0 and np.abs(got - g).max() <= G_TOL * np.abs(g).max()
            _compare_state(agent, ostate, oinfo, "uniform + clip")


@pytest.mark.parametrize("case", ["reference_defaults", "mixed_gelu"])
def test_graph_replay_pipeline_and_reruns_are_bitwise_equal(case):
    cams, B = ("front", "wrist"), 8
    runs = {}
    for name in ("eager", "graph", "graph2", "pipeline"):
        agent, rb = _drq(cams, 11, case)
        agent.use_cuda_graphs = name != "eager"
        agent.pipeline_critic_steps = name == "pipeline"
        it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
        snaps = []
        for _ in range(4):
            agent.update_critics(next(it))
            snaps.append(agent._store.params.clone())
        for _ in range(3):
            agent.update_high_utd(next(it), utd_ratio=1)
            snaps.append(agent._store.params.clone())
        runs[name] = snaps
    for name in ("graph", "graph2", "pipeline"):
        for i, (p, pe) in enumerate(zip(runs[name], runs["eager"])):
            assert torch.equal(p, pe), f"{name}: step {i} parameters differ from the eager run"


def test_checkpoint_round_trip_is_bitwise(tmp_path):
    from serl_b200.utils import checkpoints
    cams, B = ("front",), 8
    agent, rb = _drq(cams, 3, "512x3_relu_ln_softplus")
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    for _ in range(2):
        agent.update_high_utd(next(it), utd_ratio=1)
    checkpoints.save_checkpoint(str(tmp_path), agent.state, step=1)
    fresh, _ = _drq(cams, 99, "512x3_relu_ln_softplus")
    fresh.state = checkpoints.restore_checkpoint(str(tmp_path), fresh.state)
    fresh.replace(state=fresh.state)
    for buf in ("params", "target", "m", "v"):                      # every leaf (the padding between leaves is no state)
        got, ref = fresh._store.dump(getattr(fresh._store, buf)), agent._store.dump(getattr(agent._store, buf))
        assert got.keys() == ref.keys() and all(np.array_equal(got[k], ref[k]) for k in ref), buf
        if buf in ("m", "v"):
            got, ref = fresh._store.dump_aux(getattr(fresh._store, buf)), agent._store.dump_aux(getattr(agent._store, buf))
            assert all(np.array_equal(got[k], ref[k]) for k in ref), buf
    assert torch.equal(fresh._store.counts, agent._store.counts)
    np.testing.assert_array_equal(fresh.state.rng, agent.state.rng)
    tree = fresh.state.params
    assert tree["modules_critic"]["network"]["Dense_2"]["kernel"].shape == (10, 512, 512)
    assert tree["modules_actor"]["Dense_1"]["kernel"].shape == (512, 4)
    b = next(it)
    agent.update_high_utd(b, utd_ratio=1)
    fresh.update_high_utd(b, utd_ratio=1)
    got, ref = fresh._store.dump(fresh._store.params), agent._store.dump(agent._store.params)
    assert all(np.array_equal(got[k], ref[k]) for k in ref)


@pytest.mark.parametrize("case", ["reference_defaults", "512x3_relu_ln_softplus"])
def test_fp16_build_losses(case):
    from arch_oracle import networks_of
    from oracle import drq as O
    cams, B = ("front", "wrist"), 16
    agent, rb = _drq(cams, 5, case, precision="fp16")
    assert agent._engine(B).fused is None                               # a non-launcher architecture runs the per-op chain
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    with networks_of(agent):
        for _ in range(2):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            agent, info = agent.update_high_utd(batch, utd_ratio=1)
            oinfo = O.update_high_utd(ostate, ocfg, _host(batch), 1)
            np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=1e-2)
            np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=1e-2, atol=1e-3)
    assert torch.isfinite(agent._store.params).all()
    agent.check_status()
