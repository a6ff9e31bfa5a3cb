"""GPU: VICEAgent (serl_b200/agents/continuous/vice.py) against the float64 restatement of update_vice / vice_reward
(tests/vice_oracle.py), fed the agent's own trunk features, on the fp32 and fp16 builds: the draws and crops bit-exact, the infos,
every vice gradient leaf and the post-Adam vice parameters; the relabelled rewards (eager, replayed CUDA graph, utd_ratio 4);
the zero-gradient drift of the four txs; the checkpoint round trip; the learner loop through the serl_launcher shim."""
import numpy as np
import pytest
import torch

from helpers import random_transitions

pytestmark = pytest.mark.gpu

CAMS = ("wrist", "side")


def _agent(precision, seed=0):
    from serl_b200.agents.continuous.vice import VICEAgent
    obs = {c: np.zeros((1, 128, 128, 3), np.uint8) for c in CAMS}
    obs["state"] = np.zeros((1, 7), np.float32)
    agent = VICEAgent.create_vice(seed, obs, np.zeros(4, np.float32), encoder_type="resnet-pretrained", image_keys=CAMS,
                                  precision=precision)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)           # biases / scales off their init so every path is exercised
    agent._vice.params.add_(torch.randn(agent._vice.n, device="cuda", generator=g) * 0.05)
    agent._vice.target.copy_(agent._vice.params)
    return agent


def _batch(rng, B):
    trs = random_transitions(rng, B, CAMS)
    st = lambda k: {**{c: np.stack([t[k][c] for t in trs]) for c in CAMS}, "state": np.stack([t[k]["state"] for t in trs])}
    return {"observations": st("observations"), "next_observations": st("next_observations"),
            "actions": np.stack([t["actions"] for t in trs]), "rewards": np.array([t["rewards"] for t in trs], np.float32),
            "masks": np.array([t["masks"] for t in trs], np.float32), "dones": np.array([t["dones"] for t in trs])}


# heads, loss and penalty run in fp32 in every build; the oracle takes the build's own trunk features, so the bars stay fp32-class
BARS = {"fp32": (1e-5, 2e-4), "fp16": (1e-4, 1e-3)}


def _adam_bar_ok(got, ref, g, lr):
    """Post-Adam parameters: 1e-5 of the leaf's scale where the gradient is well above fp32 noise; elsewhere Adam's step
    -lr m/(sqrt(v)+eps) may take either sign in any fp32 implementation, so those entries are bounded by 2.2 lr (DESIGN.md §5)."""
    scale = max(np.abs(ref).max(), 1e-3)
    live = np.abs(g) > 1e-3 * np.abs(g).max()
    return np.abs(got - ref)[live].max(initial=0.0) <= 1e-5 * scale and np.abs(got - ref)[~live].max(initial=0.0) <= 2.2 * lr


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_update_vice_matches_oracle(precision):
    import vice_oracle as V
    from oracle import drq as O
    from oracle import jax_prng as P
    from oracle.replay import random_shift
    B = 8
    tol, gtol = BARS[precision]
    agent = _agent(precision)
    batch = _batch(np.random.default_rng(2), B)
    vp = agent._vice
    params = vp.dump(vp.params)
    rng0 = agent.state.rng
    actor0 = agent._store.dump(agent._store.params)["modules_actor/Dense_0/kernel"].copy()
    agent, info = agent.update_vice(batch)
    assert set(info) == {"actor", "critic", "temperature", "vice"} and set(info["vice"]) == {"bce_loss", "grad_norm"}
    k = V.keys(rng0, len(CAMS))
    assert np.array_equal(agent.state.rng, k["final"])
    b = agent._vice_scratch(B)
    # crops: [goal, goal crop, obs, obs crop] of the next observations, crop offsets split(k_aug, B)
    off = P.crop_offsets(k["aug"], B)
    H = B // 2
    for cam in CAMS:
        nxt = batch["next_observations"][cam][:, 0]
        crop = random_shift(nxt, off)
        want = np.concatenate([nxt[H:], crop[H:], nxt[:H], crop[:H]])
        assert np.array_equal(b["pix"][cam].cpu().numpy(), want), cam
    raw = {cam: b["raw"][j].view(2 * B, 4, 4, 512).cpu().numpy().astype(np.float64) for j, cam in enumerate(CAMS)}
    grads, oinfo = V.update_vice_grads(params, CAMS, raw, k)
    for j, (lam, perm, eps) in enumerate(oinfo["draws"]):
        assert np.float32(lam) == b["lam"][j].item()
        assert np.array_equal(b["perm"][j].cpu().numpy(), perm)
        assert np.array_equal(b["eps"][j].cpu().numpy(), eps)
    for key, got in (("bce", info["vice"]["bce_loss"]), ("grad_norm", info["vice"]["grad_norm"]), ("total", vp.info[3])):
        ref = float(oinfo[key])
        assert abs(float(got) - ref) <= tol * max(abs(ref), 1.0), (key, float(got), ref)
    g = vp.dump(vp.grad)
    for path, ref in grads.items():
        ref = ref.numpy()
        scale = np.abs(ref).max()
        assert scale > 0, path
        err = np.abs(g[path] - ref).max() / scale
        assert err <= gtol, (path, err)
    # the vice tx: one Adam step from zero moments, lr 3e-4
    opt = {"count": 0, "mu": {k: torch.zeros_like(v) for k, v in grads.items()}, "nu": {k: torch.zeros_like(v) for k, v in grads.items()}}
    upd = O.adam_tx_update(grads, opt, 3e-4)
    new = vp.dump(vp.params)
    for path in grads:
        assert _adam_bar_ok(new[path], params[path] + upd[path].numpy(), grads[path].numpy(), 3e-4), path
    # the other three txs ticked with zero gradients: counts advance; the actor has zero moments, so it does not move yet
    assert agent._store.counts.cpu().tolist() == [1, 1, 1] and vp.counts[0].item() == 1
    assert np.array_equal(agent._store.dump(agent._store.params)["modules_actor/Dense_0/kernel"], actor0)


def test_sac_leaves_drift_under_update_vice_fp32():
    """After a critic step the critic tx has non-zero moments: update_vice's zero-gradient tick moves the critic leaves by
    -lr m_hat / (sqrt(v_hat) + eps), exactly as the float64 Adam of a zero gradient predicts."""
    from oracle import drq as O
    B = 8
    agent = _agent("fp32", seed=11)
    batch = _batch(np.random.default_rng(12), B)
    agent, _ = agent.update_critics(batch)
    st = agent._store
    path = "modules_critic/network/Dense_0/kernel"
    p0, m0, v0 = (st.dump(buf)[path].astype(np.float64) for buf in (st.params, st.m, st.v))
    count = int(st.counts[0].item())
    agent, _ = agent.update_vice(batch)
    p1 = st.dump(st.params)[path]
    assert not np.array_equal(p1, p0.astype(np.float32))
    opt = {"count": count, "mu": {path: torch.as_tensor(m0)}, "nu": {path: torch.as_tensor(v0)}}
    upd = O.adam_tx_update({path: torch.zeros_like(torch.as_tensor(m0))}, opt, 3e-4)[path].numpy()
    assert np.abs(p1 - (p0 + upd)).max() <= 1e-6 + 1e-5 * np.abs(upd).max()


def test_relabelled_rewards_and_drift_fp32():
    import vice_oracle as V
    B = 8
    agent = _agent("fp32", seed=4)
    batch = _batch(np.random.default_rng(5), B)
    agent, _ = agent.update_vice(batch)
    vice0 = agent._vice.dump(agent._vice.params)
    agent, info = agent.update_critics(batch)
    eng = agent._engine(B)
    feats = {c: eng.feats[c][B:].cpu().numpy() for c in CAMS}
    p = vice0
    logits = V.forward({k: torch.as_tensor(v).double() for k, v in p.items()}, CAMS,
                       {c: torch.as_tensor(f).double() for c, f in feats.items()}).numpy()
    want = (1 / (1 + np.exp(-logits)) >= 0.5).astype(np.float32)
    got = eng.rewards.cpu().numpy()
    near = np.abs(logits) <= 1e-5 * max(np.abs(logits).max(), 1.0)
    assert np.array_equal(got[~near], want[~near])
    # the vice tx ticked with a zero gradient during the critic step: its leaves drift by the momentum of update_vice
    assert agent._vice.counts[0].item() == 2
    assert not np.array_equal(agent._vice.dump(agent._vice.params)["modules_vice/Dense_0/kernel"], vice0["modules_vice/Dense_0/kernel"])
    r = agent.vice_reward(batch["next_observations"])
    assert r.shape == (B,) and torch.isfinite(r).all()


def _relabel_ref(vice_params, feats):
    import vice_oracle as V
    logits = V.forward({k: torch.as_tensor(v).double() for k, v in vice_params.items()}, CAMS,
                       {c: torch.as_tensor(f).double() for c, f in feats.items()}).numpy()
    near = np.abs(logits) <= 1e-5 * max(np.abs(logits).max(), 1.0)
    return (1 / (1 + np.exp(-logits)) >= 0.5).astype(np.float32), near


def _ring(agent_cams, n, seed):
    from helpers import fake_env
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(agent_cams, 128), capacity=64, type="memory_efficient_replay_buffer", image_keys=list(agent_cams), seed=seed)
    for tr in random_transitions(np.random.default_rng(seed), n, agent_cams):
        rb.insert(tr)
    return rb


def test_relabel_in_replayed_graph_survives_update_vice_fp32():
    """update_vice moves the key chain on the device only: the captured update_critics graph is kept and replayed afterwards, and
    its relabelling reads the vice parameters of that moment."""
    B = 8
    agent = _agent("fp32", seed=21)
    rb = _ring(CAMS, 40, 22)
    for _ in range(3):                                      # eager warm-up, capture + replay, replay
        agent.update_critics(rb.sample(B, pack_obs_and_next_obs=True))
    keys = [k for k, v in agent._graphs.items() if isinstance(v, tuple)]
    assert keys, "update_critics was not captured"
    agent.update_vice(_batch(np.random.default_rng(23), B))
    vice0 = agent._vice.dump(agent._vice.params)
    l0 = agent.kernel_launches
    agent.update_critics(rb.sample(B, pack_obs_and_next_obs=True))
    assert all(isinstance(agent._graphs.get(k), tuple) for k in keys) and agent._graphs_version == agent._store.version
    assert agent.kernel_launches - l0 > 0
    eng = agent._engine(B)
    want, near = _relabel_ref(vice0, {c: eng.feats[c][B:].cpu().numpy() for c in CAMS})
    got = eng.rewards.cpu().numpy()
    assert np.array_equal(got[~near], want[~near])


def test_update_high_utd_4_relabels_before_the_minibatches_fp32():
    B = 8
    agent = _agent("fp32", seed=31)
    batch = _batch(np.random.default_rng(32), B)
    agent, _ = agent.update_vice(batch)
    vice0 = agent._vice.dump(agent._vice.params)
    c0 = agent._vice.counts[0].item()
    agent, info = agent.update_high_utd(batch, utd_ratio=4)
    assert agent._vice.counts[0].item() == c0 + 5            # four critic steps and one actor / temperature step tick the vice tx
    full = agent._engine(B)
    want, near = _relabel_ref(vice0, {c: full.feats[c][B:].cpu().numpy() for c in CAMS})
    got = full.rewards.cpu().numpy()
    assert np.array_equal(got[~near], want[~near])
    mb = agent._engine(B // 4)                               # the last minibatch engine holds its rows of the relabelled rewards
    assert np.array_equal(mb.rewards.cpu().numpy(), got[3 * B // 4:])
    assert abs(float(info["vice_rewards"]) - float(got.mean())) <= 1e-7


def test_checkpoint_round_trip_fp16():
    B = 8
    a = _agent("fp16", seed=41)
    batch = _batch(np.random.default_rng(42), B)
    a.update_vice(batch)
    a.update_critics(batch)
    sd = a.state.state_dict()
    b = _agent("fp16", seed=43)
    b.state.load_state_dict(sd)
    b.invalidate_graphs()
    same = lambda da, db: da.keys() == db.keys() and all(np.array_equal(da[k], db[k]) for k in da)     # leaves (not the alignment padding)
    for x, y in ((a._vice.params, b._vice.params), (a._vice.target, b._vice.target), (a._vice.m, b._vice.m), (a._vice.v, b._vice.v)):
        assert same(a._vice.dump(x), b._vice.dump(y))
    assert a._vice.counts[0].item() == b._vice.counts[0].item()
    assert same(a._store.dump(a._store.params), b._store.dump(b._store.params))
    assert set(sd["opt_states"]) == {"actor", "critic", "temperature", "vice"}
    assert set(sd["opt_states"]["vice"]["mu"]) == set(sd["opt_states"]["critic"]["mu"])
    _, ia = a.update_vice(batch)
    _, ib = b.update_vice(batch)
    assert same(a._vice.dump(a._vice.params), b._vice.dump(b._vice.params)) and float(ia["vice"]["bce_loss"]) == float(ib["vice"]["bce_loss"])


def test_learner_loop_through_the_shim_with_a_goal_ring_fp16():
    from serl_launcher.utils.launcher import make_vice_agent
    from serl_launcher.utils.train_utils import concat_batches
    B = 16
    obs = {c: np.zeros((1, 128, 128, 3), np.uint8) for c in CAMS}
    obs["state"] = np.zeros((1, 7), np.float32)
    agent = make_vice_agent(0, obs, np.zeros(4, np.float32), None, image_keys=CAMS, vice_image_keys=CAMS,
                            encoder_type="resnet-pretrained", precision="fp16")
    rb, goals = _ring(CAMS, 40, 51), _ring(CAMS, 20, 52)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    vit = rb.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True})
    git = goals.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True})
    for _ in range(3):
        agent, vi = agent.update_vice(concat_batches(next(vit), next(git), axis=0))
        agent, ci = agent.update_critics(next(it))
        agent, hi = agent.update_high_utd(next(it), utd_ratio=1)
    agent.check_status()
    for v in (vi["vice"]["bce_loss"], vi["vice"]["grad_norm"], ci["critic"]["critic_loss"], hi["actor"]["actor_loss"]):
        assert np.isfinite(float(v))
    assert 0.0 <= float(hi["vice_rewards"]) <= 1.0


def test_learner_loop_fp16():
    B = 16
    agent = _agent("fp16", seed=7)
    rng = np.random.default_rng(8)
    for _ in range(2):
        batch = _batch(rng, B)
        agent, ci = agent.update_critics(batch)
        agent, hi = agent.update_high_utd(batch, utd_ratio=1)
        agent, vi = agent.update_vice(batch)
        for v in (ci["critic"]["critic_loss"], hi["vice_rewards"], vi["vice"]["bce_loss"], vi["vice"]["grad_norm"]):
            assert np.isfinite(float(v))
    assert 0.0 <= float(hi["vice_rewards"]) <= 1.0
    tree = agent.state.params
    assert "modules_vice" in tree and "pretrained_encoder" in tree["modules_vice"]
    assert set(agent.state.opt_states) == {"actor", "critic", "temperature", "vice"}
