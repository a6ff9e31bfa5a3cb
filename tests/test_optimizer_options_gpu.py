"""GPU: per-network optimizer options (clip_grad_norm, cosine_decay_steps, per-tx learning rates) through the public API
against the float64 oracle, on the fp32 build (DESIGN.md section 5 bars), plus replay / determinism checks and the fp16 build.

Norms: the device's per-tx global norm must be within 1e-6 relative of a float64 sum over the same gradient buffer (what the
kernel computes); against the oracle's float64 gradients the gradient bar (2e-4) applies."""
import numpy as np
import pytest
import torch

from helpers import fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, to_numpy_tree
from test_agent_gpu import Q_TOL, _compare_state, _perturb

pytestmark = pytest.mark.gpu
NORM_TOL, G_TOL = 1e-6, 2e-4
TXS = ("critic", "actor", "temperature")
# the critic tx clips, the actor and temperature txs do not (their thresholds are far above any gradient norm here) ...
CRITIC_CLIPS = dict(critic_optimizer_kwargs={"clip_grad_norm": 1e-3}, actor_optimizer_kwargs={"clip_grad_norm": 1e6, "learning_rate": 1e-4},
                    temperature_optimizer_kwargs={"clip_grad_norm": 1e6})
# ... and the other way round, with a cosine schedule on the temperature tx
ACTOR_CLIPS = dict(critic_optimizer_kwargs={"clip_grad_norm": 1e6}, actor_optimizer_kwargs={"clip_grad_norm": 1e-3},
                   temperature_optimizer_kwargs={"clip_grad_norm": 1e-4, "cosine_decay_steps": 6, "warmup_steps": 2})


def _drq(cams, seed, precision="fp32", **opt):
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    rb = make_replay_buffer(fake_env(cams), capacity=200, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
    trs = random_transitions(np.random.default_rng(seed), 260, cams)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(seed, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained",
                           precision=precision, **opt)
    _perturb(agent, seed=seed)
    return agent, rb


def _opts(agent):
    from oracle.optim import OptimizerOptions
    c = agent._cfg
    return OptimizerOptions(lr=dict(zip(TXS, c.lr)), cosine_decay_steps=dict(zip(TXS, c.decay)), clip_grad_norm=dict(zip(TXS, c.clip)))


def _host(batch):
    from oracle.replay import unpack
    return unpack(to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"}))


def _check_norms(agent, eng, oinfo, nets):
    """Device norms vs float64 over the same buffer (the slots each tx sees) and vs the oracle's norm of its gradient tree."""
    from serl_b200.params import INFO_GAP
    st, c = agent._store, agent._cfg
    g = st.grad.detach().double().cpu().numpy()
    s0, s1, s2, gap = st.seg_end[0], st.seg_end[1], st.seg_end[2], st.info_off + INFO_GAP
    slots = {"critic": [g[:s0]], "actor": [g[gap:s1], g[st.n_main:st.n]], "temperature": [g[s1:s2]]}
    got = eng.grad_norms.cpu().numpy()
    checked = 0
    for i, tx in enumerate(TXS):
        if c.clip[i] is None or tx not in nets:
            continue
        ref = np.sqrt(sum(float((x ** 2).sum()) for x in slots[tx]))
        assert abs(got[i] - ref) <= NORM_TOL * ref, (tx, got[i], ref)
        assert abs(got[i] - float(oinfo["_grad_norm"][tx])) <= G_TOL * float(oinfo["_grad_norm"][tx]), tx
        checked += 1
    if "critic" in nets:                                        # the info scalars in the gap are in no norm
        assert np.abs(g[s0:gap]).max() > 0
    return checked


@pytest.mark.parametrize("opts", [CRITIC_CLIPS, ACTOR_CLIPS], ids=["critic_clips", "actor_clips"])
def test_drq_steps_with_clipping_match_oracle(opts):
    from oracle import drq as O
    from oracle import optim
    cams, B = ("front",), 16
    agent, rb = _drq(cams, 7, **opts)
    agent.use_cuda_graphs = False
    ocfg, oopts = oracle_cfg_from_agent(agent), _opts(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    eng = agent._engine(B)
    for step in range(2):
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        agent, info = agent.update_critics(batch)
        oinfo = optim.update_critics(ostate, ocfg, _host(batch), oopts)
        np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL, atol=1e-6)
        _check_norms(agent, eng, oinfo, {"critic"})
        _compare_state(agent, ostate, oinfo, f"update_critics {step}")
        for tx in TXS:
            np.testing.assert_allclose(float(info[f"{tx}_lr"]), oinfo[f"{tx}_lr"], rtol=1e-6, atol=1e-12)
    for nets in ({"critic"}, {"actor"}, {"temperature"}, {"actor", "temperature"}, {"critic", "actor", "temperature"}):
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        host = _host(batch)
        rnd, new_rng = O.derive_update_randomness(ostate.rng, B, 4, cams, True, ocfg.ensemble, ocfg.subsample or 0, nets=tuple(sorted(nets)))
        agent, info = agent.update(batch, networks_to_update=frozenset(nets))
        oinfo = optim.update(ostate, ocfg, host, rnd, frozenset(nets), torch.float64, new_rng, opts=oopts)
        if "critic" in nets:
            np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL, atol=1e-6)
        if "actor" in nets:
            np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-6)
        _check_norms(agent, eng, oinfo, nets)
        _compare_state(agent, ostate, oinfo, f"update {sorted(nets)}")
        for tx in TXS:
            np.testing.assert_allclose(float(info[f"{tx}_lr"]), oinfo[f"{tx}_lr"], rtol=1e-6, atol=1e-12)
    ostate = oracle_state_from_agent(agent)
    batch = next(it)
    agent, info = agent.update_high_utd(batch, utd_ratio=1)
    oinfo = optim.update_high_utd(ostate, ocfg, _host(batch), 1, oopts)
    np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-6)
    _check_norms(agent, eng, oinfo, {"actor", "temperature"})
    _compare_state(agent, ostate, oinfo, "update_high_utd")
    for tx in TXS:
        np.testing.assert_allclose(float(info[f"{tx}_lr"]), oinfo[f"{tx}_lr"], rtol=1e-6, atol=1e-12)
    agent.check_status()


@pytest.mark.parametrize("opts", [CRITIC_CLIPS, ACTOR_CLIPS], ids=["critic_clips", "actor_clips"])
@pytest.mark.parametrize("utd", [1, 4])
def test_state_sac_high_utd_with_clipping_matches_oracle(opts, utd):
    from oracle import optim
    from serl_b200.utils.launcher import make_sac_agent
    S, A, B = 10, 4, 32
    rng = np.random.default_rng(0)            # the batch of test_agent_gpu's state-SAC test, whose default step meets the bar
    agent = make_sac_agent(42, rng.standard_normal(S).astype(np.float32), rng.uniform(-1, 1, A).astype(np.float32), **opts)
    _perturb(agent, seed=4)
    agent._store.counts.fill_(700)            # inside the 2000-step warm-up ramp so lr != 0
    ostate, ocfg, oopts = oracle_state_from_agent(agent), oracle_cfg_from_agent(agent), _opts(agent)
    ocfg.discount = 0.99
    batch = dict(observations=rng.standard_normal((B, S)).astype(np.float32), next_observations=rng.standard_normal((B, S)).astype(np.float32),
                 actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.random(B).astype(np.float32),
                 masks=(rng.random(B) > 0.1).astype(np.float32), dones=np.zeros(B, bool))
    agent, info = agent.update_high_utd(batch, utd_ratio=utd)
    ob = dict(batch, observations={"state": batch["observations"]}, next_observations={"state": batch["next_observations"]})
    oinfo = optim.update_high_utd(ostate, ocfg, ob, utd, oopts, augment=False)
    np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL)
    np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=Q_TOL, atol=1e-6)
    assert _check_norms(agent, agent._engine(B), oinfo, {"actor", "temperature"}) >= 1
    _compare_state(agent, ostate, oinfo, f"state sac utd {utd}")
    for tx in TXS:
        np.testing.assert_allclose(float(info[f"{tx}_lr"]), oinfo[f"{tx}_lr"], rtol=1e-6, atol=1e-12)


def test_graph_replay_pipeline_and_reruns_are_bitwise_equal():
    """Eager steps, CUDA-graph replays, the cross-step pipeline and a second run give the same bits with clipping on."""
    cams, B = ("front",), 8
    runs = {}
    for name in ("eager", "graph", "graph2", "pipeline"):
        agent, rb = _drq(cams, 11, **CRITIC_CLIPS)
        agent.use_cuda_graphs = name != "eager"
        agent.pipeline_critic_steps = name == "pipeline"
        it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
        snaps = []
        for _ in range(4):
            agent.update_critics(next(it))
            snaps.append((agent._store.params.clone(), agent._engine(B).grad_norms.clone() if name != "pipeline" else None))
        agent.update_high_utd(next(it), utd_ratio=1)
        snaps.append((agent._store.params.clone(), None))
        runs[name] = snaps
    for name in ("graph", "graph2", "pipeline"):
        for i, ((p, nrm), (pe, ne)) in enumerate(zip(runs[name], runs["eager"])):
            assert torch.equal(p, pe), f"{name}: step {i} parameters differ from the eager run"
            if nrm is not None and ne is not None:
                assert torch.equal(nrm, ne), f"{name}: step {i} norms differ"


def test_cosine_schedule_reaches_zero():
    from oracle.optim import lr_schedule
    from serl_b200.utils.launcher import make_sac_agent
    S, A, B, w, D = 6, 2, 16, 2, 8
    rng = np.random.default_rng(0)
    kw = {"warmup_steps": w, "cosine_decay_steps": D, "clip_grad_norm": 0.1}
    agent = make_sac_agent(3, rng.standard_normal(S).astype(np.float32), rng.uniform(-1, 1, A).astype(np.float32),
                           critic_optimizer_kwargs=kw, actor_optimizer_kwargs={**kw, "learning_rate": 1e-3},
                           temperature_optimizer_kwargs={"cosine_decay_steps": D})
    batch = dict(observations=rng.standard_normal((B, S)).astype(np.float32), next_observations=rng.standard_normal((B, S)).astype(np.float32),
                 actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.random(B).astype(np.float32),
                 masks=np.ones(B, np.float32), dones=np.zeros(B, bool))
    for count in range(D + 5):
        before = agent._store.params.clone()
        agent, info = agent.update(batch)
        for tx, lr, warm in (("critic", 3e-4, w), ("actor", 1e-3, w), ("temperature", 3e-4, 0)):
            np.testing.assert_allclose(float(info[f"{tx}_lr"]), lr_schedule(count, lr, warm, D), rtol=1e-6, atol=1e-12)
    assert all(float(info[f"{tx}_lr"]) == 0.0 for tx in TXS)
    assert torch.equal(agent._store.params, before)                 # lr 0: the last step leaves every parameter where it was


@pytest.mark.parametrize("opts", [CRITIC_CLIPS, ACTOR_CLIPS], ids=["critic_clips", "actor_clips"])
def test_fp16_build_losses_with_clipping(opts):
    from oracle import optim
    cams, B = ("front", "wrist"), 16
    agent, rb = _drq(cams, 5, precision="fp16", **opts)
    ocfg, oopts = oracle_cfg_from_agent(agent), _opts(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    for _ in range(2):
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        agent, info = agent.update_high_utd(batch, utd_ratio=1)
        oinfo = optim.update_high_utd(ostate, ocfg, _host(batch), 1, oopts)
        np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=1e-2)
        np.testing.assert_allclose(float(info["actor"]["actor_loss"]), oinfo["actor"]["actor_loss"], rtol=1e-2, atol=1e-3)
    assert torch.isfinite(agent._store.params).all()
    agent.check_status()
