"""GPU: the pixel-only DrQ agent (use_proprio=False: the encoder is the camera embeddings alone, common/encoding.py:26-72) against
the float64 oracle with that encoder (tests/pixel_only.py), with the bars of DESIGN.md section 5: Q, losses and actions within
1e-5, gradient leaves within 2e-4 of their max, post-Adam parameters with the noise-aware bar (fp32 build); on the 16-bit build
the fused heads, their losses, the benchmark-batch gradients with the oracle fed the engine's own trunk features, CUDA-graph
replay, the cross-step pipeline, checkpoints and replay files without a state vector.  Plus an oracle-independent check: a
pixel-only agent equals a proprio agent whose first-layer proprio rows are zero."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import injected_features, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, rel_err, to_numpy_tree
from pixel_only import make_agent, pixel_only_env, pixel_only_oracle, pixel_only_transitions, strip_state, with_empty_state
from test_agent_gpu import G_TOL, Q_TOL, _compare_state, _perturb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TXS = ("critic", "actor", "temperature")
SUBSETS = [{"critic"}, {"actor"}, {"temperature"}, {"actor", "temperature"}, {"critic", "actor"}, {"critic", "temperature"},
           {"critic", "actor", "temperature"}]


def _setup(cams, seed=7, precision="fp32", cap=200, n_fill=260):
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(pixel_only_env(cams), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
    trs = pixel_only_transitions(np.random.default_rng(seed), n_fill, cams)
    for tr in trs:
        rb.insert(tr)
    agent = make_agent(seed, trs[0]["observations"], trs[0]["actions"], cams, precision=precision)
    _perturb(agent, seed=seed)
    return agent, rb


def _host(batch):
    from oracle.replay import unpack
    d = to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"})
    assert "state" not in d["observations"] and "state" not in d["next_observations"]
    return with_empty_state(unpack(d))


def _check_grads(agent, oinfo, groups, tol=G_TOL):
    st = agent._store
    for leaf in st.spec:
        if leaf.group in groups:
            ref = oinfo["_grads"][TXS[leaf.group]][leaf.path].numpy()
            got = st.view(st.grad, leaf.path).cpu().numpy()
            assert np.abs(got - ref).max() <= tol * max(np.abs(ref).max(), 1e-8), leaf.path


@pytest.mark.parametrize("cams", [("front",), ("front", "wrist")], ids=["cam1", "cam2"])
def test_pixel_only_steps_match_oracle(cams):
    from oracle import drq as O
    from oracle import jax_prng as P
    B = 12
    agent, rb = _setup(cams)
    assert agent._store.n == agent._store.n_main
    agent.use_cuda_graphs = False
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    eng = agent._engine(B)
    assert eng.fused is None and eng.F == 256 * len(cams)
    with pixel_only_oracle():
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
        for nets in SUBSETS:
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            rnd, new_rng = O.derive_update_randomness(ostate.rng, B, 4, cams, True, ocfg.ensemble, ocfg.subsample or 0, nets=tuple(sorted(nets)))
            st = agent._store
            if nets == {"actor"}:
                st.grad[:st.seg_end[0]].zero_()          # what the actor step writes into group 0 is checked below: nothing
            agent, info = agent.update(batch, networks_to_update=frozenset(nets))
            oinfo = O.update(ostate, ocfg, _host(batch), rnd, frozenset(nets), torch.float64, new_rng)
            if "critic" in nets:
                np.testing.assert_allclose(float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"], rtol=Q_TOL, atol=1e-6)
            if "actor" in nets:
                for k in ("actor_loss", "temperature", "entropy"):
                    np.testing.assert_allclose(float(info["actor"][k]), oinfo["actor"][k], rtol=Q_TOL, atol=1e-6)
            if "temperature" in nets:
                np.testing.assert_allclose(float(info["temperature"]["temperature_loss"]), oinfo["temperature"]["temperature_loss"],
                                           rtol=Q_TOL, atol=1e-6)
            _check_grads(agent, oinfo, tuple(TXS.index(n) for n in nets))
            if nets == {"actor"}:
                # the policy's stop_gradient covers every image embedding: the actor loss reaches no encoder leaf
                for leaf in st.spec:
                    if leaf.path.startswith("modules_actor/encoder/"):
                        assert float(oinfo["_grads"]["actor"][leaf.path].abs().max()) == 0.0, leaf.path
                        assert float(st.view(st.grad, leaf.path).abs().max()) == 0.0, leaf.path
            _compare_state(agent, ostate, oinfo, f"update {sorted(nets)}")
        for utd in (1, 4):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            agent, info = agent.update_high_utd(batch, utd_ratio=utd)
            oinfo = O.update_high_utd(ostate, ocfg, _host(batch), utd)
            for k in ("critic_loss", "predicted_qs", "target_qs"):
                np.testing.assert_allclose(float(info["critic"][k]), oinfo["critic"][k], rtol=Q_TOL, atol=1e-6)
            for k in ("actor_loss", "temperature", "entropy"):
                np.testing.assert_allclose(float(info["actor"][k]), oinfo["actor"][k], rtol=Q_TOL, atol=1e-6)
            np.testing.assert_allclose(float(info["temperature"]["temperature_loss"]), oinfo["temperature"]["temperature_loss"],
                                       rtol=Q_TOL, atol=1e-6)
            _compare_state(agent, ostate, oinfo, f"update_high_utd({utd})")
        # sample_actions: seeded and argmax, batched and unbatched; observations without a state vector
        ostate = oracle_state_from_agent(agent)
        rng = np.random.default_rng(0)
        obs = {c: rng.integers(0, 256, (3, 1, 128, 128, 3), dtype=np.uint8) for c in cams}
        oobs = dict(obs, state=np.zeros((3, 1, 0), np.float32))
        key = P.prng_key(2024)
        assert rel_err(agent.sample_actions(obs, seed=key), O.sample_actions(ostate, ocfg, oobs, seed=key).numpy()) < Q_TOL
        assert rel_err(agent.sample_actions(obs, argmax=True), O.sample_actions(ostate, ocfg, oobs, argmax=True).numpy()) < Q_TOL
        one = {k: v[0] for k, v in obs.items()}
        ref1 = O.sample_actions(ostate, ocfg, {k: v[:1] for k, v in oobs.items()}, seed=key)[0].numpy()
        a = agent.sample_actions(one, seed=key)
        assert a.shape == (4,) and rel_err(a, ref1) < Q_TOL
        am = agent.sample_actions(one, argmax=True)
        assert am.shape == (4,) and rel_err(am, O.sample_actions(ostate, ocfg, {k: v[:1] for k, v in oobs.items()}, argmax=True)[0].numpy()) < Q_TOL
    agent.check_status()


@pytest.mark.parametrize("cams", [("front",), ("front", "wrist")], ids=["cam1", "cam2"])
def test_pixel_only_forward_passes_match_oracle(cams):
    import forward_oracle as FO
    from oracle import jax_prng as P
    agent, _ = _setup(cams, seed=5, n_fill=10)
    params = {k: torch.as_tensor(np.asarray(v)).double() for k, v in _flat_params(agent.state.params).items()}
    target = {k: torch.as_tensor(np.asarray(v)).double() for k, v in _flat_params(agent.state.target_params).items()}
    B, N, A = 12, 3, 4
    rng = np.random.default_rng(1)
    obs = {c: rng.integers(0, 256, (B, 1, 128, 128, 3), dtype=np.uint8) for c in cams}
    oobs = dict(obs, state=np.zeros((B, 1, 0), np.float32))
    acts = rng.uniform(-0.99, 0.99, (B, A)).astype(np.float32)
    multi = rng.uniform(-0.99, 0.99, (B, N, A)).astype(np.float32)
    key = P.prng_key(3)
    with pixel_only_oracle():
        q = agent.forward_critic(obs, acts, key)
        assert tuple(q.shape) == (10, B) and rel_err(q.cpu().numpy(), FO.critic(agent, params, oobs, acts).numpy()) < Q_TOL
        qm = agent.forward_critic(obs, multi, key)
        assert tuple(qm.shape) == (10, B, N) and rel_err(qm.cpu().numpy(), FO.critic(agent, params, oobs, multi).numpy()) < Q_TOL
        qt = agent.forward_target_critic(obs, acts, key)
        assert rel_err(qt.cpu().numpy(), FO.critic(agent, target, oobs, acts).numpy()) < Q_TOL
        q1 = agent.forward_critic({c: v[0] for c, v in obs.items()}, acts[0], key)
        assert tuple(q1.shape) == (10,) and rel_err(q1.cpu().numpy(), q.cpu().numpy()[:, 0]) < Q_TOL
        for train, dkey in ((True, key), (False, None)):
            dist = agent.forward_policy(obs, key, train=train)
            mu, sd = FO.policy(agent, params, oobs, dropout_key=dkey)
            assert rel_err(dist.loc.cpu().numpy(), mu.numpy()) < Q_TOL
            assert rel_err(dist.scale_diag.cpu().numpy(), sd.numpy()) < Q_TOL


def _flat_params(tree):
    from serl_b200.params import flatten
    return flatten(tree)


# ---- oracle-independent: pixel-only == proprio agent with zero proprio rows in both first layers ---------------------------
def _pair(cams, precision, seed=11):
    """A pixel-only agent and a proprio agent with the same trunk, image heads, MLPs and rng, whose critic / policy Dense_0 rows
    for the 64 proprio features are zero; two identical rings (with a state vector) feed them the same draws."""
    from serl_b200.params import flatten, nest
    from serl_b200.utils.launcher import make_replay_buffer
    from helpers import fake_env
    trs = random_transitions(np.random.default_rng(seed), 260, cams)
    rings = []
    for _ in range(2):
        rb = make_replay_buffer(fake_env(cams), capacity=200, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
        for tr in trs:
            rb.insert(tr)
        rings.append(rb)
    px = make_agent(seed, trs[0]["observations"], trs[0]["actions"], cams, use_proprio=False, precision=precision)
    pr = make_agent(seed + 1, trs[0]["observations"], trs[0]["actions"], cams, use_proprio=True, precision=precision)
    _perturb(px, seed=seed)
    _perturb(pr, seed=seed + 1)                               # (moves the proprio leaves off their init too)
    Fi = 256 * len(cams)

    def widen(flat_px, flat_pr):
        out = dict(flat_pr)
        for k, v in flat_px.items():
            v = np.asarray(v)
            if k == "modules_critic/network/Dense_0/kernel":
                v = np.concatenate([v[:, :Fi], np.zeros((v.shape[0], 64, v.shape[2]), np.float32), v[:, Fi:]], axis=1)
            elif k == "modules_actor/network/Dense_0/kernel":
                v = np.concatenate([v[:Fi], np.zeros((64, v.shape[1]), np.float32)], axis=0)
            out[k] = v
        return nest(out)

    pr.state.replace(params=widen(flatten(px.state.params), flatten(pr.state.params)),
                     target_params=widen(flatten(px.state.target_params), flatten(pr.state.target_params)), rng=px.state.rng)
    pr.invalidate_graphs()
    return px, pr, rings, Fi


def _zero_proprio_rows(agent, Fi):
    st = agent._store
    for buf in (st.params, st.target):
        st.view(buf, "modules_critic/network/Dense_0/kernel")[:, Fi:Fi + 64].zero_()
        st.view(buf, "modules_actor/network/Dense_0/kernel")[Fi:Fi + 64].zero_()
    st.version += 1


def _image_path_grads_equal(px, pr, Fi, groups, tol):
    sx, sr = px._store, pr._store
    for leaf in sx.spec:
        if leaf.group not in groups:
            continue
        a, b = sx.view(sx.grad, leaf.path), sr.view(sr.grad, leaf.path)
        if leaf.path == "modules_critic/network/Dense_0/kernel":
            b = torch.cat([b[:, :Fi], b[:, Fi + 64:]], dim=1)
        elif leaf.path == "modules_actor/network/Dense_0/kernel":
            b = b[:Fi]
        err = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-12)
        assert err <= tol, (leaf.path, err)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_pixel_only_equals_proprio_with_zero_proprio_rows(precision):
    cams, B = ("front", "wrist"), 16
    px, pr, rings, Fi = _pair(cams, precision)
    assert (px._engine(B).fused is None) == (precision == "fp32") and (pr._engine(B).fused is None) == (precision == "fp32")
    tol = 1e-5 if precision == "fp32" else 1e-4
    its = [r.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True}) for r in rings]
    for step in range(2):
        _zero_proprio_rows(pr, Fi)
        _, ix = px.update_critics(next(its[0]))
        _, ir = pr.update_critics(next(its[1]))
        ex, er = px._engine(B), pr._engine(B)
        assert torch.equal(ex.idx, er.idx) and all(torch.equal(ex.pix[c], er.pix[c]) for c in cams)
        assert rel_err(ex.q.cpu().numpy(), er.q.cpu().numpy()) <= tol
        for k in ("critic_loss", "predicted_qs", "target_qs"):
            np.testing.assert_allclose(float(ix["critic"][k]), float(ir["critic"][k]), rtol=tol, atol=tol * 0.1)
        _image_path_grads_equal(px, pr, Fi, (0,), 2e-4 if precision == "fp32" else 1e-3)
        # the actor and temperature losses on their own: update_high_utd's critic step would move the proprio rows first
        _zero_proprio_rows(pr, Fi)
        nets = frozenset({"actor", "temperature"})
        _, ix = px.update(next(its[0]), networks_to_update=nets)
        _, ir = pr.update(next(its[1]), networks_to_update=nets)
        for k in ("actor_loss", "temperature", "entropy"):
            np.testing.assert_allclose(float(ix["actor"][k]), float(ir["actor"][k]), rtol=tol, atol=tol * 0.1)
        np.testing.assert_allclose(float(ix["temperature"]["temperature_loss"]), float(ir["temperature"]["temperature_loss"]),
                                   rtol=tol, atol=tol * 0.1)
        _image_path_grads_equal(px, pr, Fi, (1, 2), 2e-4 if precision == "fp32" else 1e-3)
        np.testing.assert_array_equal(px.state.rng, pr.state.rng)
    px.check_status(); pr.check_status()


# ---- 16-bit build ---------------------------------------------------------------------------------------------------------
def test_fp16_runs_fused_heads_and_matches_oracle_losses():
    from oracle import drq as O
    from serl_b200.heads_fused import FusedCritic
    cams, B = ("front", "wrist"), 16
    agent, rb = _setup(cams, precision="fp16")
    assert isinstance(agent._engine(B).fused, FusedCritic)
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    with pixel_only_oracle():
        for _ in range(2):
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            agent, info = agent.update_critics(batch)
            oinfo = O.update_critics(ostate, ocfg, _host(batch))
            got, ref = float(info["critic"]["critic_loss"]), oinfo["critic"]["critic_loss"]
            assert abs(got - ref) <= 1e-2 * max(abs(ref), 1e-3), (got, ref)
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        agent, info = agent.update_high_utd(batch, utd_ratio=1)
        oinfo = O.update_high_utd(ostate, ocfg, _host(batch), 1)
        for k, grp in (("critic_loss", "critic"), ("actor_loss", "actor")):
            got, ref = float(info[grp][k]), oinfo[grp][k]
            assert abs(got - ref) <= 1e-2 * max(abs(ref), 1e-3), (k, got, ref)
    agent.check_status()


def test_fp16_benchmark_batch_gradients_with_injected_features():
    """B = 256, two cameras: fused-head Q, infos and gradients against the float64 oracle fed the engine's own trunk features,
    at the fp32-class bars of tests/test_heads_grads_b256_gpu.py (Q 1e-4, infos 1e-4, gradient leaves 2e-4)."""
    sys.path.insert(0, ROOT)
    from bench import fill_ring_synthetic
    from oracle import drq as O
    from oracle.replay import unpack
    from serl_b200.utils.launcher import make_replay_buffer
    cams, B = ("front", "wrist"), 256
    rb = make_replay_buffer(pixel_only_env(cams), capacity=2000, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=11)
    fill_ring_synthetic(rb, seed=1)
    tr = pixel_only_transitions(np.random.default_rng(0), 1, cams)[0]
    agent = make_agent(42, tr["observations"], tr["actions"], cams, precision="fp16")
    _perturb(agent, seed=0)
    assert agent._engine(B).fused is not None
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    scalar = lambda got, ref: abs(float(got) - float(ref)) / (abs(float(ref)) + 0.1)
    with pixel_only_oracle():
        for step in range(3):                                    # eager, capture, replay
            ostate = oracle_state_from_agent(agent)
            batch = next(it)
            host = with_empty_state(unpack(to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"})))
            agent, info = agent.update_critics(batch)
            eng = agent._engines[B]
            with injected_features({c: eng.pix[c] for c in cams}, {c: eng.feats[c] for c in cams}):
                oinfo = O.update_critics(ostate, ocfg, host)
            assert rel_err(eng.q.cpu().numpy(), oinfo["critic"]["_q"].numpy()) < 1e-4, step
            for k in ("critic_loss", "predicted_qs", "target_qs"):
                assert scalar(info["critic"][k], oinfo["critic"][k]) < 1e-4, (step, k)
            _check_grads(agent, oinfo, (0,), tol=2e-4)
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        host = with_empty_state(unpack(to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"})))
        agent, info = agent.update_high_utd(batch, utd_ratio=1)
        eng = agent._engines[B]
        with injected_features({c: eng.pix[c] for c in cams}, {c: eng.feats[c] for c in cams}):
            oinfo = O.update_high_utd(ostate, ocfg, host, 1)
        for k in ("actor_loss", "temperature", "entropy"):
            assert scalar(info["actor"][k], oinfo["actor"][k]) < 1e-4, k
        _check_grads(agent, oinfo, (1, 2), tol=2e-4)
    agent.check_status()


def _run_steps(agent, its, n, pipelined=False):
    agent.pipeline_critic_steps = pipelined
    out = []
    for _ in range(n):
        agent, i = agent.update_critics(next(its[0]))
        out.append(float(i["critic"]["critic_loss"]))
    agent, i = agent.update_high_utd(next(its[0]), utd_ratio=1)
    out.append(float(i["actor"]["actor_loss"]))
    return out


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_graphs_pipeline_and_second_run_equal_eager(precision):
    """CUDA-graph replay, the cross-step pipeline and a second identical run against eager steps, each run on a fresh agent from the
    same seeds.  The draws and the key chain are bit-exact on every build.  The fp32 build has no floating-point atomics: its
    losses, parameters and Adam moments are bitwise equal in all four runs.  The 16-bit trunk accumulates GroupNorm statistics
    with float atomicAdd (csrc/stem_pool.cu, the stem's per-image sums; csrc/conv_tcgen05.cu, the stage heads' projection branch),
    whose order varies from run to run, so two fp16 runs are not guaranteed to agree bit for bit (as for the proprio agent,
    INTEGRATION.md); there they are held to the summation-order bar of tests/test_pipeline_gpu.py."""
    cams, B = ("front", "wrist"), 32
    runs = {}
    for name, graphs, pipe in (("eager", False, False), ("graph", True, False), ("pipe", True, True), ("graph2", True, False)):
        agent, rb = _setup(cams, precision=precision)
        agent.use_cuda_graphs = graphs
        its = [rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})]
        losses = _run_steps(agent, its, 6, pipe)
        agent.check_status()
        eng = agent._engines[B]                                     # the last call, update_high_utd, ran here
        st = agent._store
        runs[name] = (losses, st.params.clone(), st.m.clone(), st.v.clone(), agent.state.rng, eng.idx.clone(),
                      {c: eng.pix[c].clone() for c in cams})
    ref = runs["eager"]
    for name in ("graph", "pipe", "graph2"):
        losses, params, m, v, rng, idx, pix = runs[name]
        np.testing.assert_array_equal(rng, ref[4])
        assert torch.equal(idx, ref[5]) and all(torch.equal(pix[c], ref[6][c]) for c in cams), name
        if precision == "fp32":
            assert losses == ref[0], (name, losses, ref[0])
            assert torch.equal(params, ref[1]) and torch.equal(m, ref[2]) and torch.equal(v, ref[3]), name
        else:
            np.testing.assert_allclose(losses, ref[0], rtol=2e-3, atol=1e-6)
            assert float((params - ref[1]).abs().max()) <= 2e-3 * float(ref[1].abs().max()), name


def test_fp16_checkpoint_round_trip_bitwise(tmp_path):
    from serl_b200.utils import checkpoints
    cams, B = ("front", "wrist"), 16
    agent, rb = _setup(cams, precision="fp16")
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
    for _ in range(3):
        agent.update_high_utd(next(it), utd_ratio=1)
    checkpoints.save_checkpoint(str(tmp_path / "ckpt"), agent.state, step=3)
    fresh = make_agent(99, {c: np.zeros((1, 128, 128, 3), np.uint8) for c in cams}, np.zeros(4, np.float32), cams, precision="fp16")
    fresh = fresh.replace(state=checkpoints.restore_checkpoint(str(tmp_path / "ckpt"), fresh.state))
    st, sf = agent._store, fresh._store
    assert st.n == st.n_main == sf.n
    own = torch.zeros(st.n, dtype=torch.bool, device=st.params.device)      # the leaves (not the alignment padding or info gap)
    for l in st.spec:
        own[l.offset:l.offset + l.size] = True
    for name in ("params", "target", "m", "v"):
        assert torch.equal(getattr(st, name)[own], getattr(sf, name)[own]), name
    assert torch.equal(st.counts, sf.counts) and fresh.state.step == agent.state.step
    np.testing.assert_array_equal(agent.state.rng, fresh.state.rng)
    for cam in cams:
        for k, t in agent._trunk[cam].items():
            assert torch.equal(t, fresh._trunk[cam][k]), k
    batch = rb.sample(B, pack_obs_and_next_obs=True)
    d = to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"})
    agent.update_high_utd(d, utd_ratio=1)
    fresh.update_high_utd(d, utd_ratio=1)
    assert torch.equal(st.params[own], sf.params[own])


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_ring_save_load_resume_matches_an_uninterrupted_run(tmp_path, precision):
    """A pixel-only learner that saves its checkpoint and rings (zero-width state members, S = 0 in the meta), restarts from them
    and continues inserting and training gives the uninterrupted run's losses and parameters (bitwise on the fp32 build)."""
    from serl_b200.data import replay_io as RIO
    from serl_b200.utils import checkpoints
    from serl_b200.utils.launcher import make_replay_buffer
    cams, B, PER = ("front",), 8, 4
    trs = pixel_only_transitions(np.random.default_rng(0), 40 + 8 * PER, cams, mean_ep=7)

    def fresh(seed, ring_seed=5):
        rb = make_replay_buffer(pixel_only_env(cams), capacity=64, type="memory_efficient_replay_buffer", image_keys=list(cams),
                                seed=ring_seed)
        return make_agent(seed, trs[0]["observations"], trs[0]["actions"], cams, precision=precision), rb

    def loop(agent, rb, lo, n, log):
        for i in range(n):
            for tr in trs[lo + i * PER:lo + (i + 1) * PER]:
                rb.insert(tr)
            agent, ci = agent.update_critics(rb.sample(B, pack_obs_and_next_obs=True))
            agent, ui = agent.update_high_utd(rb.sample(B, pack_obs_and_next_obs=True), utd_ratio=1)
            log.append((float(ci["critic"]["critic_loss"]), float(ui["actor"]["actor_loss"])))
        return agent

    agent_a, rb_a = fresh(42)
    for tr in trs[:40]:
        rb_a.insert(tr)
    log_a = []
    agent_a = loop(agent_a, rb_a, 40, 8, log_a)
    agent, rb = fresh(42)
    for tr in trs[:40]:
        rb.insert(tr)
    log_b = []
    agent = loop(agent, rb, 40, 4, log_b)
    checkpoints.save_checkpoint(str(tmp_path / "ckpt"), agent.state, step=4)
    path = tmp_path / "ring.npz"
    rb.save(path)
    meta = RIO.read_meta(path)
    assert meta["S"] == 0
    with np.load(path) as z:
        assert z["state"].shape == (len(rb), 0) and z["next_state"].shape == (len(rb), 0)
    agent_b, rb_b = fresh(7, ring_seed=None)
    agent_b = agent_b.replace(state=checkpoints.restore_checkpoint(str(tmp_path / "ckpt"), agent_b.state))
    rb_b.load(path)
    agent_b = loop(agent_b, rb_b, 40 + 4 * PER, 4, log_b)
    agent_a.check_status(); agent_b.check_status()
    if precision == "fp32":
        assert log_a == log_b
        assert torch.equal(agent_a._store.params, agent_b._store.params)
    else:
        np.testing.assert_allclose(np.array(log_b), np.array(log_a), rtol=2e-3, atol=1e-5)


def test_classifier_batch_from_rings_without_state():
    """sample_classifier_batch on two rings without a state vector gives the batch it gives on rings holding the same frames
    with one: same draws, crops and labels."""
    from oracle import jax_prng as P
    from serl_b200.networks.reward_classifier import sample_classifier_batch
    from serl_b200.utils.launcher import make_replay_buffer
    from helpers import fake_env
    cams = ("front", "wrist")
    trs = random_transitions(np.random.default_rng(4), 120, cams)
    out = {}
    for name, env, strip in (("pixel_only", pixel_only_env(cams), True), ("with_state", fake_env(cams), False)):
        rings = []
        for seed, part in ((21, trs[:60]), (22, trs[60:])):
            rb = make_replay_buffer(env, capacity=80, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=seed)
            for tr in part:
                rb.insert(strip_state(tr) if strip else tr)
            rings.append(rb)
        assert (rings[0].S == 0) == strip
        out[name] = [sample_classifier_batch(rings[0], rings[1], 16, P.prng_key(k)) for k in (0, 1)]
    for a, b in zip(out["pixel_only"], out["with_state"]):
        assert tuple(a["data"]["front"].shape) == (16, 1, 128, 128, 3)
        for c in cams:
            assert torch.equal(a["data"][c], b["data"][c]), c
        assert torch.equal(a["labels"], b["labels"]) and float(a["labels"][:8].min()) == 1.0 and float(a["labels"][8:].max()) == 0.0
