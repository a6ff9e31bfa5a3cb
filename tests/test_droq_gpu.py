"""GPU: SAC / DrQ agents with the critic and policy MLPs' dropout_rate (dropout Q-functions) against the float64 oracle of
tests/droq_oracle.py, which draws the same masks from the same keys (DESIGN.md §4).  The bars are those of
test_architecture_options_gpu.py: Q, targets, losses and actions within 1e-5, gradient leaves within 2e-4 of their max (5e-3 with
relu), post-Adam parameters with the noise-aware bar.  Plus the public forward passes, replay / pipeline determinism, a checkpoint
round trip and the 16-bit builds."""
import contextlib

import numpy as np
import pytest
import torch

from helpers import fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, rel_err, to_numpy_tree
from test_agent_gpu import G_TOL, Q_TOL, _compare_state, _perturb

pytestmark = pytest.mark.gpu

DROQ = {"hidden_dims": [256, 256], "activations": "tanh", "use_layer_norm": True, "dropout_rate": 0.01}
RELU = {"hidden_dims": [512, 128], "activations": "relu", "use_layer_norm": False, "dropout_rate": 0.2}
TXS = ("critic", "actor", "temperature")
KINK_G_TOL = 5e-3


def _drq(cams, seed, nets, encoder="resnet-pretrained", subsample=2, precision="fp32", ensemble=None):
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(cams), capacity=200, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
    trs = random_transitions(np.random.default_rng(seed), 260, cams)
    for tr in trs:
        rb.insert(tr)
    agent = DrQAgent.create_drq(seed, trs[0]["observations"], trs[0]["actions"], encoder_type=encoder, use_proprio=True, image_keys=cams,
                                temperature_init=1e-2, discount=0.96, backup_entropy=False,
                                critic_ensemble_size=ensemble or (10 if subsample else 2), critic_subsample_size=subsample,
                                precision=precision, **nets)
    _perturb(agent, seed=seed)
    return agent, rb


def _host(batch):
    from oracle.replay import unpack
    return unpack(to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"}))


def _oracles(agent):
    from droq_oracle import networks_of
    stack = contextlib.ExitStack()
    stack.enter_context(networks_of(agent))
    if agent._cfg.small:
        from small_encoder_oracle import small_encoder_oracle
        stack.enter_context(small_encoder_oracle())
    return stack


def _check_grads(agent, oinfo, groups):
    st, c = agent._store, agent._cfg
    tol = KINK_G_TOL if {c.critic_arch.act, c.policy_arch.act} & {"relu", "leaky_relu"} else G_TOL
    for leaf in st.spec:
        if leaf.group not in groups:
            continue
        ref = oinfo["_grads"][TXS[leaf.group]][leaf.path].numpy()
        got = st.view(st.grad, leaf.path).cpu().numpy()
        bar = max(tol, KINK_G_TOL) if "/Conv_" in leaf.path else tol      # the small encoder's ReLU convs (test_small_encoder_gpu.py)
        assert np.abs(got - ref).max() <= bar * max(np.abs(ref).max(), 1e-8), leaf.path


def _mlp_grads_nonzero(agent, groups):
    st = agent._store
    for leaf in st.spec:
        if leaf.group in groups and ("modules_critic" in leaf.path if leaf.group == 0 else "modules_actor" in leaf.path):
            assert torch.count_nonzero(st.view(st.grad, leaf.path)) > 0, leaf.path


CASES = [(("front",), "resnet-pretrained", 2, DROQ), (("front", "wrist"), "resnet-pretrained", None, DROQ),
         (("front",), "small", None, RELU), (("front", "wrist"), "small", 2, DROQ)]


@pytest.mark.parametrize("cams,encoder,subsample,nk", CASES, ids=["cam1-resnet-sub2", "cam2-resnet-nosub", "cam1-small-relu", "cam2-small-sub2"])
def test_drq_steps_match_oracle(cams, encoder, subsample, nk):
    from oracle import drq as O
    B = 12
    agent, rb = _drq(cams, 7, dict(critic_network_kwargs=nk, policy_network_kwargs=nk), encoder, subsample)
    agent.use_cuda_graphs = False
    trunk = None if agent._frozen_trunk is None else {c: {k: v.clone() for k, v in d.items()} for c, d in agent._trunk.items()}
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    eng = agent._engine(B)
    with _oracles(agent):
        for step in range(2):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            agent, info = agent.update_critics(batch)
            oinfo = O.update_critics(ostate, ocfg, _host(batch))
            assert rel_err(eng.q.cpu().numpy(), oinfo["critic"]["_q"].numpy()) < Q_TOL
            assert rel_err(eng.target_q.cpu().numpy(), oinfo["critic"]["_target_q"].numpy()) < Q_TOL
            for k in ("critic_loss", "predicted_qs", "target_qs"):
                np.testing.assert_allclose(float(info["critic"][k]), oinfo["critic"][k], rtol=Q_TOL, atol=1e-6)
            # the device's masks are the oracle's: online critic, target critic
            calls = oinfo["_mlp_masks"]
            for got, ref in zip(eng.c_mask + eng.c_mask_tgt, calls[2][1] + calls[1][1]):
                np.testing.assert_array_equal(got.cpu().numpy().astype(bool), ref)
            if step == 0:
                _check_grads(agent, oinfo, (0,))
                _mlp_grads_nonzero(agent, (0,))
            _compare_state(agent, ostate, oinfo, f"update_critics {step}")
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        rnd, new_rng = O.derive_update_randomness(ostate.rng, B, 4, cams, True, ocfg.ensemble, ocfg.subsample or 0)
        agent, info = agent.update(batch)
        oinfo = O.update(ostate, ocfg, _host(batch), rnd, frozenset(TXS), torch.float64, new_rng)
        np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL, atol=1e-6)
        for k in ("actor_loss", "temperature", "entropy"):
            np.testing.assert_allclose(float(info["actor"][k]), oinfo["actor"][k], rtol=Q_TOL, atol=1e-6)
        np.testing.assert_allclose(float(info["temperature"]["temperature_loss"]), oinfo["temperature"]["temperature_loss"], rtol=Q_TOL, atol=1e-7)
        _check_grads(agent, oinfo, (0, 1, 2))
        _mlp_grads_nonzero(agent, (1,))
        _compare_state(agent, ostate, oinfo, "update")
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        agent, info = agent.update_high_utd(batch, utd_ratio=2)
        oinfo = O.update_high_utd(ostate, ocfg, _host(batch), 2)
        for k in ("critic_loss", "predicted_qs", "target_qs"):
            np.testing.assert_allclose(float(info["critic"][k]), oinfo["critic"][k], rtol=Q_TOL, atol=1e-6)
        # the actor loss reads the critic after two minibatch Adam steps, whose entries with fp32-noise gradients may move by up to
        # ~2 lr in either direction (the allowance of _compare_state): a ~1e-6 absolute shift of Q
        np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-5)
        _compare_state(agent, ostate, oinfo, "update_high_utd")
    if trunk is not None:                                                # the frozen trunk is bitwise unchanged
        assert all(torch.equal(agent._trunk[c][k], v) for c, d in trunk.items() for k, v in d.items())
    agent.check_status()


@pytest.mark.parametrize("subsample", [2, None])
@pytest.mark.parametrize("nk", [DROQ, RELU], ids=["tanh_ln", "relu"])
def test_state_sac_matches_oracle(subsample, nk):
    from droq_oracle import networks_of
    from oracle import drq as O
    from serl_b200.agents.continuous.sac import SACAgent
    S, A, B = 10, 4, 32
    rng = np.random.default_rng(0)
    agent = SACAgent.create_states(42, rng.standard_normal(S).astype(np.float32), rng.uniform(-1, 1, A).astype(np.float32),
                                   temperature_init=1e-2, discount=0.99, critic_ensemble_size=10 if subsample else 2,
                                   critic_subsample_size=subsample, critic_network_kwargs=nk, policy_network_kwargs=nk)
    _perturb(agent, seed=4)
    agent._store.counts.fill_(700)
    mk = lambda: dict(observations=rng.standard_normal((B, S)).astype(np.float32), next_observations=rng.standard_normal((B, S)).astype(np.float32),
                      actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.random(B).astype(np.float32),
                      masks=(rng.random(B) > 0.1).astype(np.float32), dones=np.zeros(B, bool))
    ob = lambda b: dict(b, observations={"state": b["observations"]}, next_observations={"state": b["next_observations"]})
    with networks_of(agent):
        for utd in (2, 1):
            ostate, ocfg = oracle_state_from_agent(agent), oracle_cfg_from_agent(agent)
            batch = mk()
            agent, info = agent.update_high_utd(batch, utd_ratio=utd)
            oinfo = O.update_high_utd(ostate, ocfg, ob(batch), utd, augment=False)
            np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL)
            np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-6)
            _check_grads(agent, oinfo, (1, 2))
            _compare_state(agent, ostate, oinfo, f"state sac utd {utd}")
        ostate = oracle_state_from_agent(agent)
        batch = mk()
        rnd, new_rng = O.derive_update_randomness(ostate.rng, B, A, (), False, ocfg.ensemble, ocfg.subsample or 0)
        agent, info = agent.update(batch)
        oinfo = O.update(ostate, ocfg, ob(batch), rnd, frozenset(TXS), torch.float64, new_rng)
        np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL)
        _check_grads(agent, oinfo, (0, 1, 2))
        _mlp_grads_nonzero(agent, (0, 1))
        _compare_state(agent, ostate, oinfo, "state sac update")


def test_forward_passes_train_and_eval():
    """train=True draws the masks from the given rng (fold_in(rng, ncams + i)) and matches the oracle; train=False is bitwise the
    forward of the same agent without dropout."""
    from droq_oracle import critic_forward, mlp_masks, policy_forward
    from oracle import drq as O
    from oracle import jax_prng as P
    cams, B = ("front", "wrist"), 5
    agent, _ = _drq(cams, 9, dict(critic_network_kwargs=DROQ, policy_network_kwargs=DROQ))
    plain, _ = _drq(cams, 9, {})
    assert torch.equal(agent._store.params, plain._store.params)
    rng = np.random.default_rng(1)
    obs = {c: rng.integers(0, 256, (B, 1, 128, 128, 3), dtype=np.uint8) for c in cams}
    obs["state"] = rng.standard_normal((B, 1, 7)).astype(np.float32)
    act = rng.uniform(-1, 1, (B, 4)).astype(np.float32)
    key = P.prng_key(31)
    assert torch.equal(agent.forward_critic(obs, act, key, train=False), plain.forward_critic(obs, act, key, train=False))
    assert torch.equal(agent.forward_critic(obs, act[:, None].repeat(3, 1), key, train=False),
                       plain.forward_critic(obs, act[:, None].repeat(3, 1), key, train=False))
    assert torch.equal(agent.forward_policy(obs, key, train=False).mode(), plain.forward_policy(obs, key, train=False).mode())
    with pytest.raises(NotImplementedError, match="multi-action kernel"):
        agent.forward_critic(obs, act[:, None].repeat(3, 1), key, train=True)
    ostate, ocfg = oracle_state_from_agent(agent), oracle_cfg_from_agent(agent)
    arch = agent._cfg.critic_arch
    with torch.no_grad():
        feats = O._features(ostate, ocfg, obs, torch.float64)
        enc = O._enc(ostate.params, ocfg, feats, obs["state"], None)
        q = critic_forward(ostate.params, enc, torch.as_tensor(act), arch, True, mlp_masks(key, 2, B, arch))
        qt = critic_forward(ostate.target_params, O._enc(ostate.target_params, ocfg, feats, obs["state"], None), torch.as_tensor(act), arch,
                            True, mlp_masks(key, 2, B, arch))
        enc_p = O._enc(ostate.params, ocfg, feats, obs["state"], O._dropout_masks(key, cams, B))
        mu, _ = policy_forward(ostate.params, enc_p, agent._cfg.policy_arch, "exp", agent._cfg.std_min, agent._cfg.std_max,
                               mlp_masks(key, 2, B, agent._cfg.policy_arch))
    assert rel_err(agent.forward_critic(obs, act, key).cpu().numpy(), q.numpy()) < Q_TOL
    assert rel_err(agent.forward_target_critic(obs, act, key).cpu().numpy(), qt.numpy()) < Q_TOL
    assert rel_err(agent.forward_policy(obs, key).loc.cpu().numpy(), mu.numpy()) < Q_TOL
    assert not torch.equal(agent.forward_critic(obs, act, key), agent.forward_critic(obs, act, key, train=False))


def test_graph_replay_pipeline_and_reruns_are_bitwise_equal():
    cams, B = ("front", "wrist"), 8
    runs = {}
    for name in ("eager", "graph", "graph2", "pipeline"):
        agent, rb = _drq(cams, 11, dict(critic_network_kwargs=DROQ, policy_network_kwargs=DROQ), subsample=None)
        agent.use_cuda_graphs = name != "eager"
        agent.pipeline_critic_steps = name == "pipeline"
        it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
        snaps = []
        for _ in range(4):
            agent.update_critics(next(it))
            snaps.append(agent._store.params.clone())
        for _ in range(3):
            agent.update_high_utd(next(it), utd_ratio=2)
            snaps.append(agent._store.params.clone())
        runs[name] = snaps
    for name in ("graph", "graph2", "pipeline"):
        for i, (p, pe) in enumerate(zip(runs[name], runs["eager"])):
            assert torch.equal(p, pe), f"{name}: step {i} parameters differ from the eager run"


def test_checkpoint_round_trip_is_bitwise(tmp_path):
    from serl_b200.utils import checkpoints
    cams, B = ("front",), 8
    nets = dict(critic_network_kwargs=RELU, policy_network_kwargs=DROQ)
    agent, rb = _drq(cams, 3, nets)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    for _ in range(2):
        agent.update_high_utd(next(it), utd_ratio=1)
    checkpoints.save_checkpoint(str(tmp_path), agent.state, step=1)
    fresh, _ = _drq(cams, 99, nets)
    fresh.state = checkpoints.restore_checkpoint(str(tmp_path), fresh.state)
    fresh.replace(state=fresh.state)
    for buf in ("params", "target", "m", "v"):
        got, ref = fresh._store.dump(getattr(fresh._store, buf)), agent._store.dump(getattr(agent._store, buf))
        assert got.keys() == ref.keys() and all(np.array_equal(got[k], ref[k]) for k in ref), buf
    np.testing.assert_array_equal(fresh.state.rng, agent.state.rng)
    b = next(it)
    agent.update_high_utd(b, utd_ratio=1)
    fresh.update_high_utd(b, utd_ratio=1)
    got, ref = fresh._store.dump(fresh._store.params), agent._store.dump(agent._store.params)
    assert all(np.array_equal(got[k], ref[k]) for k in ref)


def test_fp16_droq_losses_and_rate_zero_bits():
    """The 16-bit build at the launcher widths: a dropout agent runs the fused heads within 1e-2 of the oracle; a rate-0 dict is the
    launcher agent, bit for bit."""
    from oracle import drq as O
    cams, B = ("front", "wrist"), 16
    agent, rb = _drq(cams, 5, dict(critic_network_kwargs=DROQ, policy_network_kwargs=DROQ), subsample=None, precision="fp16")
    assert agent._engine(B).fused is not None
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    with _oracles(agent):
        for _ in range(2):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            agent, info = agent.update_high_utd(batch, utd_ratio=1)
            oinfo = O.update_high_utd(ostate, ocfg, _host(batch), 1)
            np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=1e-2)
            np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=1e-2, atol=1e-3)
    agent.check_status()
    zero = dict(DROQ, dropout_rate=0.0)
    runs = []
    for nets in ({}, dict(critic_network_kwargs=zero, policy_network_kwargs=zero)):
        a, rb = _drq(cams, 6, nets, precision="fp16")
        assert a._engine(B).fused is not None
        it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
        for _ in range(3):
            a.update_critics(next(it))
        a.update_high_utd(next(it), utd_ratio=1)
        runs.append(a._store.params.clone())
    assert torch.equal(runs[0], runs[1])


@pytest.mark.parametrize("subsample,B", [(None, 12), (2, 160)])
def test_fused_heads_match_the_per_op_chain_with_the_same_masks(subsample, B, monkeypatch):
    """fp16 DroQ at the launcher widths: the fused tgemm heads (masked LayerNorm epilogues, masked ln_tanh_bwd_multi) against the
    per-op chain (SERL_FUSED_HEADS=0) from the same state, keys and batch, so with the same masks; the bars of
    test_fused_heads_gpu.py (5e-3 relative on Q, targets, pi(s), log-probs and the losses; gradient leaves within 1e-2 of their
    max, TF32 vs 3xTF32 heads)."""
    cams = ("front", "wrist")
    nets = dict(critic_network_kwargs=DROQ, policy_network_kwargs=dict(DROQ, dropout_rate=0.1))
    agent, rb = _drq(cams, 13, nets, subsample=subsample, precision="fp16")
    agent.use_cuda_graphs = False
    monkeypatch.setenv("SERL_FUSED_HEADS", "0")
    ref, _ = _drq(cams, 13, nets, subsample=subsample, precision="fp16")
    ref.use_cuda_graphs = False
    ref._engine(B)
    monkeypatch.delenv("SERL_FUSED_HEADS")
    eng, reng = agent._engine(B), ref._engine(B)
    assert eng.fused is not None and reng.fused is None
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    for call in ("update_critics", "update"):
        st, rs = agent._store, ref._store
        for buf in ("params", "target", "m", "v", "counts"):
            getattr(rs, buf).copy_(getattr(st, buf))
        ref.state._rng.copy_(agent.state._rng)
        batch = next(it)
        bd = {k: v for k, v in batch.to_dict().items() if k != "_indices"}
        if call == "update_critics":
            agent, info = agent.update_critics(batch)
            ref, rinfo = ref.update_critics(bd)
        else:
            agent, info = agent.update(bd)
            ref, rinfo = ref.update(bd)
        for got, want in zip(eng.c_mask + eng.c_mask_tgt, reng.c_mask + reng.c_mask_tgt):
            assert torch.equal(got, want)                               # the same masks on both paths
        if call == "update_critics":
            assert all(torch.equal(g, w) for g, w in zip(eng.p_mask, reng.p_mask))
            assert rel_err(eng.q.cpu().numpy(), reng.q.cpu().numpy()) < 5e-3
            assert rel_err(eng.target_q.cpu().numpy(), reng.target_q.cpu().numpy()) < 5e-3
            np.testing.assert_allclose(float(info["critic"]["critic_loss"]), float(rinfo["critic"]["critic_loss"]), rtol=5e-3)
        else:
            for k in ("actor_loss", "entropy"):
                np.testing.assert_allclose(float(info["actor"][k]), float(rinfo["actor"][k]), rtol=5e-3, atol=1e-4)
            np.testing.assert_allclose(float(info["temperature"]["temperature_loss"]), float(rinfo["temperature"]["temperature_loss"]),
                                       rtol=5e-3, atol=1e-6)
            # the temperature pass's log-probs (the per-op chain runs it last into the engine's buffers; the fused path keeps its own)
            assert rel_err(eng.fused.logp_t.cpu().numpy(), reng.logp.cpu().numpy()) < 5e-3
        groups = (0,) if call == "update_critics" else (0, 1, 2)
        for leaf in st.spec:
            if leaf.group in groups and ("modules_critic" in leaf.path or "modules_actor/network" in leaf.path):
                g, r = st.view(st.grad, leaf.path).cpu().numpy(), rs.view(rs.grad, leaf.path).cpu().numpy()
                assert np.abs(g - r).max() <= 1e-2 * max(np.abs(r).max(), 1e-8), (call, leaf.path)
    agent.check_status()
