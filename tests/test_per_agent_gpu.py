"""GPU: SAC / DrQ gradient steps on batches drawn from a prioritized ring.

An RLPD batch concatenates a prioritized online ring and a uniform demo ring.  Each step's draw of the online part must be
oracle/per.py's draw over the tree as the device left it, its weights (p_min / p)^beta over that part (1 on the demo rows),
info["critic"]["critic_loss"] the weighted loss of the step's own Q and targets, and the drawn slots' leaves
(|delta| + eps)^alpha of the step's TD errors, with the tree bitwise a function of its leaves.  With beta = 0 the step is bit for
bit the uniform step on the same rows; eager, captured and replayed steps agree bit for bit, and pipeline_critic_steps falls back
to the serial step.
"""
import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

pytestmark = pytest.mark.gpu

CAMS = ("front", "wrist")


def _ring(alpha, seed=3, cap=200, n_fill=260, beta=0.4):
    from serl_b200.utils.launcher import make_replay_buffer
    kw = {} if alpha is None else dict(priority_alpha=alpha, priority_beta=beta)
    rb = make_replay_buffer(fake_env(CAMS), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(CAMS), seed=seed, **kw)
    rng = np.random.default_rng(seed)
    trs = random_transitions(rng, n_fill, CAMS, mean_ep=8)
    for tr in trs:
        rb.insert(tr)
    rb.flush()
    return rb, trs


def _agent(trs, precision="fp32", encoder="resnet-pretrained"):
    from serl_b200.utils.launcher import make_drq_agent
    return make_drq_agent(42, trs[0]["observations"], trs[0]["actions"], image_keys=CAMS, encoder_type=encoder, precision=precision)


def _host(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("fp16", 1e-2)])
def test_update_critics_weights_losses_and_write_back(precision, tol):
    from oracle import per as P
    from serl_b200.utils.train_utils import concat_batches
    online, trs = _ring(0.6)
    demo, _ = _ring(None, seed=5, cap=120, n_fill=150)
    agent = _agent(trs, precision)
    B = 32
    cap = online._capacity
    for step in range(3):                                     # eager, capture + replay, replay
        tree0 = _host(online.tree)
        valid = _host(online.valid).astype(bool)
        h = concat_batches(online.sample(B // 2, pack_obs_and_next_obs=True), demo.sample(B // 2, pack_obs_and_next_obs=True), axis=0)
        agent, info = agent.update_critics(h)
        eng = agent._engines[B]
        idx = _host(eng.idx)[: B // 2]
        np.testing.assert_array_equal(idx, P.draw(tree0, cap, online._seed, h.parts[0]["step"], B // 2, valid=valid))
        w = _host(eng.weights)
        np.testing.assert_allclose(w[: B // 2], P.weights(tree0[idx], 0.4), rtol=1e-6, atol=0)
        assert (w[B // 2:] == 1).all()
        q, y = _host(eng.q).reshape(-1, B), _host(eng.target_q)
        loss, _, delta = P.critic_loss(q, y, w)
        np.testing.assert_allclose(float(info["critic"]["critic_loss"]), loss, rtol=tol)
        d_dev = _host(eng.delta)
        np.testing.assert_allclose(d_dev, delta, rtol=1e-5, atol=1e-6)
        tree1 = _host(online.tree)
        np.testing.assert_array_equal(tree1.view(np.uint32), P.build(tree1[:cap]).view(np.uint32))
        want, _ = P.set_leaves(tree0[:cap], 1.0, idx, td=d_dev[: B // 2], ring_valid=valid, alpha=0.6, eps=1e-6)
        np.testing.assert_allclose(tree1[:cap], want, rtol=1e-6, atol=0)       # the drawn slots, last row winning
        untouched = np.setdiff1d(np.arange(cap), idx)
        np.testing.assert_array_equal(tree1[untouched], tree0[untouched])
    agent.check_status()


def test_beta_zero_is_the_uniform_step_and_execution_modes_agree():
    from serl_b200.utils.train_utils import concat_batches
    B = 32
    rings = [_ring(0.6, beta=0.0) for _ in range(3)]             # graphs, eager, pipelined
    uni, trs = _ring(None)
    demos = [_ring(None, seed=5, cap=120, n_fill=150)[0] for _ in range(4)]
    agents = [_agent(trs) for _ in range(4)]
    agents[1].use_cuda_graphs = False
    agents[2].pipeline_critic_steps = True
    for step in range(4):
        hs = [concat_batches(r.sample(B // 2, pack_obs_and_next_obs=True), d.sample(B // 2, pack_obs_and_next_obs=True), axis=0)
              for (r, _), d in zip(rings, demos)]
        for k in range(3):
            agents[k], info = agents[k].update_critics(hs[k])
        idx = _host(agents[0]._engines[B].idx)
        hu = concat_batches(uni.sample(B // 2, indx=idx[: B // 2], pack_obs_and_next_obs=True),
                            demos[3].sample(B // 2, indx=idx[B // 2:], pack_obs_and_next_obs=True), axis=0)
        agents[3], iu = agents[3].update_critics(hu)
        for k in (1, 2, 3):
            assert torch.equal(agents[k]._store.params, agents[0]._store.params), (step, k)
        for k in (1, 2):
            assert torch.equal(rings[k][0].tree, rings[0][0].tree), (step, k)
        assert float(info["critic"]["critic_loss"]) == float(iu["critic"]["critic_loss"])


@pytest.mark.parametrize("encoder", ["resnet-pretrained", "small"])
def test_high_utd_writes_every_minibatch(encoder):
    from oracle import per as P
    online, trs = _ring(0.6)
    agent = _agent(trs, encoder=encoder)
    B, cap = 32, online._capacity
    for _ in range(2):
        tree0 = _host(online.tree)
        agent, info = agent.update_high_utd(online.sample(B, pack_obs_and_next_obs=True), utd_ratio=4)
        idx = _host(agent._engines[B].idx)
        tree1 = _host(online.tree)
        np.testing.assert_array_equal(tree1.view(np.uint32), P.build(tree1[:cap]).view(np.uint32))
        changed = np.flatnonzero(tree1[:cap] != tree0[:cap])
        assert set(changed) <= set(idx.tolist()) and len(changed) > 0
        assert np.isfinite(float(info["critic"]["critic_loss"]))
    agent.check_status()


def test_state_sac_on_a_prioritized_replay_buffer():
    from oracle import per as P
    from helpers import Box
    from serl_b200.data.replay_buffer import ReplayBuffer
    from serl_b200.utils.launcher import make_sac_agent
    rb = ReplayBuffer(Box((7,)), Box((4,)), 300, seed=1, priority_alpha=0.5)
    rng = np.random.default_rng(0)
    for _ in range(250):
        rb.insert(dict(observations=rng.standard_normal(7).astype(np.float32), next_observations=rng.standard_normal(7).astype(np.float32),
                       actions=rng.uniform(-1, 1, 4).astype(np.float32), rewards=float(rng.standard_normal()), masks=1.0, dones=False))
    agent = make_sac_agent(0, np.zeros(7, np.float32), np.zeros(4, np.float32))
    for step in range(3):
        # critic only: a full update's actor pass reuses the engine's Q buffer after the critic loss
        agent, info = agent.update(rb.sample(64), networks_to_update=frozenset({"critic"}))
        eng = agent._engines[64]
        q, y, w = _host(eng.q).reshape(-1, 64), _host(eng.target_q), _host(eng.weights)
        np.testing.assert_allclose(float(info["critic"]["critic_loss"]), P.critic_loss(q, y, w)[0], rtol=1e-5)
        assert w.max() == 1.0 and (step == 0 or w.min() < 1.0)      # every leaf is m = 1 until the first write-back
    tree0 = _host(rb.tree)
    agent, info = agent.update(rb.sample(64))                      # all three networks: the critic part writes back
    idx = _host(agent._engines[64].idx)
    changed = np.flatnonzero(_host(rb.tree)[:300] != tree0[:300])
    assert len(changed) > 0 and set(changed) <= set(idx.tolist())
    agent.check_status()


def test_resume_from_a_saved_ring_equals_an_uninterrupted_run(tmp_path):
    """Save the prioritized ring after two steps, load it into a new ring and continue: the same parameters and tree, bit for bit,
    as four steps without the interruption (fp32)."""
    from serl_b200.utils.train_utils import concat_batches
    B = 32
    (ra, trs), (rb_, _) = _ring(0.6), _ring(0.6)
    da, db = _ring(None, seed=5, cap=120, n_fill=150)[0], _ring(None, seed=5, cap=120, n_fill=150)[0]
    a, b = _agent(trs), _agent(trs)
    step = lambda agent, r, d: agent.update_critics(concat_batches(r.sample(B // 2, pack_obs_and_next_obs=True),
                                                                   d.sample(B // 2, pack_obs_and_next_obs=True), axis=0))[0]
    for _ in range(4):
        a = step(a, ra, da)
    for _ in range(2):
        b = step(b, rb_, db)
    rb_.save(tmp_path / "online.npz")
    rc, _ = _ring(0.6, seed=9, n_fill=10)
    rc.load(tmp_path / "online.npz")
    for _ in range(2):
        b = step(b, rc, db)
    assert torch.equal(a._store.params, b._store.params)
    assert torch.equal(ra.tree, rc.tree) and torch.equal(ra.max_priority_dev, rc.max_priority_dev)
