"""CPU: the pixel-only DrQ agent (use_proprio=False) and replay rings without a state vector - parameter layout (no proprio
leaves, empty aux tail), construction, ring bookkeeping with S = 0 against oracle/replay.py, the data-parallel exchange and the
reference learner loop.  Kernels are replaced by a recorder (host logic only)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from helpers import random_transitions
from pixel_only import make_agent, pixel_only_env, pixel_only_transitions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMS = ("front", "wrist")


def _dry(monkeypatch):
    from serl_b200 import _lib as L
    real_call = L.call
    monkeypatch.setattr(L, "call", lambda name, *a: real_call(name, *a) if name.startswith("serl_host_") else 0)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    ev = types.SimpleNamespace(record=lambda: None, synchronize=lambda: None, make_current_stream_wait=lambda: None)
    monkeypatch.setattr(L, "new_event", lambda: ev)
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: 0)


@pytest.mark.parametrize("cams", [("front",), CAMS])
def test_spec_without_proprio_leaves(cams):
    from serl_b200.params import ENC, PROPRIO_LEAVES, ParamStore, trainable_spec
    full = trainable_spec(cams, 7, 4, 10, True)
    px = trainable_spec(cams, 0, 4, 10, True, use_proprio=False)
    assert [l.path for l in px] == [l.path for l in full if l.path not in PROPRIO_LEAVES]
    assert not any(l.path.startswith(f"{ENC}/Dense_0") or l.path.startswith(f"{ENC}/LayerNorm_0") for l in px)
    F = 256 * len(cams)
    shapes = {l.path: l.shape for l in px}
    for l in full:
        if l.path == "modules_critic/network/Dense_0/kernel":
            assert l.shape == (10, F + 64 + 4, 256) and shapes[l.path] == (10, F + 4, 256)
        elif l.path == "modules_actor/network/Dense_0/kernel":
            assert l.shape == (F + 64, 256) and shapes[l.path] == (F, 256)
        elif l.path not in PROPRIO_LEAVES:
            assert shapes[l.path] == l.shape, l.path
    assert [l.group for l in px] == [l.group for l in full if l.path not in PROPRIO_LEAVES]
    st = ParamStore(px, "cpu")
    assert st.n == st.n_main and st.aux_lo == st.aux_hi == 0
    assert not any(st.two_tx(l.path) for l in px)
    assert st.dump_aux(st.m) == {}
    assert ParamStore(full, "cpu").n > ParamStore(full, "cpu").n_main        # the proprio agent keeps its aux tail


def test_enc_dim_and_fused_rule():
    from serl_b200 import heads_fused
    from serl_b200.engine import AgentConfig
    px = AgentConfig(cams=CAMS, state_in=0, action_dim=4, use_proprio=False, precision="fp16")
    pr = AgentConfig(cams=CAMS, state_in=7, action_dim=4, precision="fp16")
    assert px.enc_dim == 512 and pr.enc_dim == 576 and not px.proprio and pr.proprio
    assert heads_fused.enabled(px) and heads_fused.enabled(pr)
    # the 64-input limit of enc_finish's small dense applies to the proprio block only
    assert heads_fused.enabled(AgentConfig(cams=CAMS, state_in=100, action_dim=4, use_proprio=False, precision="fp16"))
    assert not heads_fused.enabled(AgentConfig(cams=CAMS, state_in=100, action_dim=4, precision="fp16"))
    # 16-byte row strides: (enc_dim + A) % 4 == 0, else the per-op chain
    assert not heads_fused.enabled(AgentConfig(cams=CAMS, state_in=0, action_dim=3, use_proprio=False, precision="fp16"))
    assert not heads_fused.enabled(AgentConfig(cams=CAMS, state_in=0, action_dim=4, use_proprio=False, precision="fp32"))


def test_construction(monkeypatch):
    _dry(monkeypatch)
    from serl_b200.utils.launcher import make_drq_agent
    tr = pixel_only_transitions(np.random.default_rng(0), 1, CAMS)[0]
    full = random_transitions(np.random.default_rng(0), 1, CAMS)[0]
    agent = make_agent(1, tr["observations"], tr["actions"], CAMS, device="cpu")
    assert agent._cfg.state_in == 0 and not agent._cfg.use_proprio and agent._cfg.enc_dim == 512
    enc = agent.state.params["modules_actor"]["encoder"]
    assert set(enc) == {"encoder_front", "encoder_wrist"}
    assert agent.state.params["modules_critic"]["network"]["Dense_0"]["kernel"].shape == (10, 512 + 4, 256)
    assert agent.state.params["modules_actor"]["network"]["Dense_0"]["kernel"].shape == (512, 256)
    # a "state" entry is ignored: same layout, same initial values
    agent2 = make_agent(1, full["observations"], full["actions"], CAMS, device="cpu")
    assert agent2._cfg.state_in == 0
    assert torch.equal(agent._store.params, agent2._store.params)
    # the reference's import path
    from serl_launcher.agents.continuous.drq import DrQAgent
    a3 = DrQAgent.create_drq(2, tr["observations"], tr["actions"], encoder_type="resnet-pretrained", use_proprio=False,
                             image_keys=CAMS, device="cpu")
    assert a3._store.n == a3._store.n_main
    # proprio agent without a state vector: ValueError naming the key (the launcher passes use_proprio=True)
    with pytest.raises(ValueError, match="'state'"):
        make_agent(1, tr["observations"], tr["actions"], CAMS, use_proprio=True, device="cpu")
    with pytest.raises(ValueError, match="'state'"):
        make_drq_agent(1, tr["observations"], tr["actions"], image_keys=CAMS, encoder_type="resnet-pretrained", device="cpu")
    # the proprio agent is built as before
    pr = make_drq_agent(1, full["observations"], full["actions"], image_keys=CAMS, encoder_type="resnet-pretrained", device="cpu")
    assert pr._cfg.use_proprio and pr._cfg.state_in == 7 and pr._store.n > pr._store.n_main
    # full-tree Adam states and their re-expansion with an empty aux tail
    os_ = agent.state.opt_states
    assert "Dense_0" not in os_["actor"]["mu"]["modules_actor"]["encoder"]
    agent._store.m.copy_(torch.arange(agent._store.n, dtype=torch.float32))
    m0 = agent._store.m.clone()
    os_ = agent.state.opt_states
    agent._store.m.zero_()
    agent.state.replace(opt_states=os_)
    own = torch.zeros(agent._store.n, dtype=torch.bool)
    for l in agent._store.spec:
        own[l.offset:l.offset + l.size] = True
    assert torch.equal(agent._store.m[own], m0[own])


def test_ring_bookkeeping_without_state_matches_oracle_through_a_wrap(monkeypatch):
    _dry(monkeypatch)
    from oracle.replay import OracleFrameRing
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
    from serl_b200.utils.launcher import make_replay_buffer
    cap, hw = 37, 16
    env = pixel_only_env(CAMS, hw)
    rb = make_replay_buffer(env, capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(CAMS), device="cpu", seed=4)
    assert isinstance(rb, MemoryEfficientReplayBuffer) and rb.S == 0 and tuple(rb.state.shape) == (cap, 0)
    ora = OracleFrameRing(cap, CAMS, (hw, hw, 3), 1, 0, 4)
    trs = pixel_only_transitions(np.random.default_rng(1), 3 * cap + 5, CAMS, hw, mean_ep=7)
    for i, tr in enumerate(trs):
        rb.insert(tr)
        ora.insert({**tr, "observations": {**tr["observations"], "state": np.zeros((1, 0), np.float32)},
                    "next_observations": {**tr["next_observations"], "state": np.zeros((1, 0), np.float32)}})
        assert (len(rb), rb._insert_index, rb._first) == (ora.size, ora.cursor, ora.episode_start), i
        np.testing.assert_array_equal(rb._valid_host[:ora.size], ora.valid[:ora.size])
    assert rb._stn[0]["state"].shape == (rb.STAGE, 0)
    rb.flush()
    # other observation layouts are still refused
    bad = pixel_only_env(CAMS, hw)
    bad.observation_space.spaces["joints"] = bad.observation_space.spaces[CAMS[0]]
    with pytest.raises(NotImplementedError):
        make_replay_buffer(bad, capacity=cap, type="memory_efficient_replay_buffer", image_keys=[CAMS[0]], device="cpu")


def _gloo_worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from serl_b200 import _lib as L
    real = L.call
    L.call = lambda name, *a: real(name, *a) if name.startswith("serl_host_") else 0
    ev = types.SimpleNamespace(record=lambda: None, synchronize=lambda: None, make_current_stream_wait=lambda: None)
    L.require_cuda, L.stream_ptr, L.new_event, L.pin = (lambda d: None), (lambda: 0), (lambda: ev), (lambda t: t)
    from pixel_only import make_agent, pixel_only_env, pixel_only_transitions
    from serl_b200.utils.launcher import make_replay_buffer
    cams = ("front",)
    rb = make_replay_buffer(pixel_only_env(cams), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams),
                            device="cpu", seed=100 + rank)
    trs = pixel_only_transitions(np.random.default_rng(rank), 30, cams)
    for tr in trs:
        rb.insert(tr)
    agent = make_agent(7, trs[0]["observations"], trs[0]["actions"], cams, device="cpu")
    agent.data_parallel = True
    agent.use_cuda_graphs = False
    st = agent._store
    agent._engine(4)                                         # (a new engine zeroes the info scalars in the gradient buffer)
    n_coll = []
    real_ar = dist.all_reduce
    dist.all_reduce = lambda t, *a, **k: (n_coll.append(t.numel()), real_ar(t, *a, **k))[1]
    res = {}
    for name, call in (("critic", lambda b: agent.update_critics(b)), ("utd", lambda b: agent.update_high_utd(b, utd_ratio=1)),
                       ("all", lambda b: agent.update(b, pmap_axis="devices"))):
        del n_coll[:]
        st.grad.copy_(torch.arange(st.n, dtype=torch.float32) * (rank + 1))
        call(rb.sample(4, pack_obs_and_next_obs=True))
        res[name] = (list(n_coll), st.grad.clone())
    torch.save(dict(n=st.n, n_main=st.n_main, info_off=st.info_off, res=res), out.format(rank))
    dist.destroy_process_group()


def test_data_parallel_one_collective_with_an_empty_aux_tail(tmp_path):
    import torch.multiprocessing as mp
    world, port = 2, 33000 + os.getpid() % 2000
    out = str(tmp_path / "rank{}.pt")
    mp.spawn(_gloo_worker, args=(world, port, out), nprocs=world, join=True)
    r0, r1 = torch.load(out.format(0)), torch.load(out.format(1))
    n, cut = r0["n"], r0["info_off"] + 4
    assert n == r0["n_main"]
    base = torch.arange(n, dtype=torch.float32)
    n_crit, g_crit = r0["res"]["critic"]
    assert n_crit == [cut]
    torch.testing.assert_close(g_crit[:cut], 3.0 * base[:cut])
    torch.testing.assert_close(g_crit[cut:], base[cut:])
    n_utd, g_utd = r0["res"]["utd"]
    assert n_utd == [cut, n - cut]                         # critic step, then actor / temperature step up to n == n_main
    torch.testing.assert_close(g_utd, 3.0 * base)
    n_all, g_all = r0["res"]["all"]
    assert n_all == [n]
    torch.testing.assert_close(g_all, 3.0 * base)
    for k in ("critic", "utd", "all"):
        torch.testing.assert_close(r0["res"][k][1][:cut], r1["res"][k][1][:cut], rtol=0, atol=0)


def test_learner_loop_host_logic_pixel_only_cpu(monkeypatch, tmp_path):
    """The learner loop of the reference's async_drq_sim.py (as tests/test_learner_loop_conformance.py drives it) on an environment
    whose observations are camera images only, with a pixel-only agent: RLPD concat, update_critics, update_high_utd, publishing
    the parameter tree and checkpoints."""
    _dry(monkeypatch)
    from serl_b200.utils import checkpoints
    from serl_launcher.data.data_store import MemoryEfficientReplayBufferDataStore
    from serl_launcher.utils.launcher import make_replay_buffer
    from serl_launcher.utils.train_utils import concat_batches
    env = pixel_only_env(CAMS)
    trs = pixel_only_transitions(np.random.default_rng(0), 60, CAMS)
    agent = make_agent(42, trs[0]["observations"], trs[0]["actions"], CAMS, device="cpu")
    replay_buffer = make_replay_buffer(env, capacity=200, type="memory_efficient_replay_buffer", image_keys=list(CAMS), device="cpu")
    demo_buffer = make_replay_buffer(env, capacity=200, type="memory_efficient_replay_buffer", image_keys=list(CAMS), device="cpu")
    assert isinstance(replay_buffer, MemoryEfficientReplayBufferDataStore)
    for tr in trs[:25]:
        demo_buffer.insert(tr)
    for tr in trs:
        replay_buffer.insert(tr)
    published = [agent.state.params]
    demo_it = demo_buffer.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    replay_it = replay_buffer.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    max_steps = 3
    for step in range(max_steps):
        for _ in range(3):
            batch = concat_batches(next(replay_it), next(demo_it), axis=0)
            agent, critics_info = agent.update_critics(batch)
        batch = concat_batches(next(replay_it), next(demo_it), axis=0)
        agent, update_info = agent.update_high_utd(batch, utd_ratio=1)
        if step > 0 and step % 2 == 0:
            published.append(agent.state.params)
        checkpoints.save_checkpoint(str(tmp_path / "ckpt"), agent.state, step=step, keep=20)
    assert set(critics_info) == {"critic", "critic_lr", "actor_lr", "temperature_lr"}
    assert set(update_info["actor"]) == {"actor_loss", "temperature", "entropy"}
    assert agent.state.step == max_steps * 5
    tree = published[-1]
    assert set(tree["modules_actor"]["encoder"]) == {"encoder_front", "encoder_wrist"}
    assert tree["modules_critic"]["network"]["Dense_0"]["kernel"].shape == (10, 512 + 4, 256)
    restored = checkpoints.restore_checkpoint(str(tmp_path / "ckpt"), None)
    assert "Dense_0" not in restored["opt_states"]["actor"]["mu"]["modules_actor"]["encoder"]

