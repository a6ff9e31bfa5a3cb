"""GPU, world size 2 (NCCL default group for the gradients + the replay store's gloo group; skipped below 2 devices):
`DataParallelDataStore` in the learner loop.  An actor thread inserts on rank 0 while both ranks train; afterwards the ring
replicas and the agents (parameters, target parameters, Adam moments) are bitwise equal across ranks.  Rank r's draws are
bit-exact to a standalone ring seeded base + r with the same contents, and on the fp32 build a run that checkpoints and saves
its rings after N iterations and resumes in a fresh 2-rank job matches an uninterrupted run of N + M iterations bitwise."""
import datetime
import os
import sys
import threading
import time
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMS, CAP, BATCH = ("front", "wrist"), 200, 16          # BATCH: global, half from the online ring and half from the demo ring
SEEDS = (21, 22)                                        # base sampler seeds of the online and demo rings


def _state_transitions(rng, n, S=10, A=4):
    return [dict(observations=rng.standard_normal(S).astype(np.float32), next_observations=rng.standard_normal(S).astype(np.float32),
                 actions=rng.uniform(-1, 1, A).astype(np.float32), rewards=np.float32(rng.random()), masks=np.float32(1.0),
                 dones=bool(rng.random() < 0.1)) for _ in range(n)]


def _setup(kind, precision="fp32", agent_seed=42, ring_seeds=SEEDS, n=400):
    from helpers import Box, fake_env, random_transitions
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer, make_sac_agent
    rng = np.random.default_rng(0)
    if kind == "drq":
        trs = random_transitions(rng, n, CAMS, mean_ep=9)
        env, rb_kw = fake_env(CAMS), dict(type="memory_efficient_replay_buffer", image_keys=list(CAMS))
        agent = make_drq_agent(agent_seed, trs[0]["observations"], trs[0]["actions"], image_keys=CAMS, encoder_type="resnet-pretrained",
                               precision=precision)
    else:
        trs = _state_transitions(rng, n)
        env, rb_kw = types.SimpleNamespace(observation_space=Box((10,)), action_space=Box((4,))), dict(type="replay_buffer")
        agent = make_sac_agent(agent_seed, trs[0]["observations"], trs[0]["actions"])
    agent.data_parallel = True
    rb, demo = (make_replay_buffer(env, capacity=CAP, seed=s, data_parallel=True, **rb_kw) for s in ring_seeds)
    return agent, rb, demo, trs


def _fill(rank, rb, demo, trs, n_online=60, n_demo=40):
    """The learner's fill loop: rank 0 receives, every rank waits on sync()."""
    if rank == 0:
        for tr in trs[:n_demo]:
            demo.insert(tr)
        for tr in trs[n_demo:n_demo + n_online]:
            rb.insert(tr)
    demo.sync()
    while rb.sync() < n_online:
        time.sleep(0.01)
    return n_demo + n_online


def _loop(kind, agent, rb, demo, iters, before_each=None):
    from serl_b200.utils.train_utils import concat_batches
    half = {"batch_size": BATCH // 2, "pack_obs_and_next_obs": True}
    it, dit = rb.get_iterator(sample_args=half), demo.get_iterator(sample_args=half)
    nxt = lambda: concat_batches(next(it), next(dit), axis=0)
    for i in range(iters):
        if before_each is not None:
            before_each(i)
        for _ in range(3):
            if kind == "drq":
                agent, _ = agent.update_critics(nxt())
            else:
                agent, _ = agent.update(nxt(), networks_to_update=frozenset({"critic"}))
        agent, _ = agent.update_high_utd(nxt(), utd_ratio=1 if kind == "drq" else 2)
    return agent


def _agent_snapshot(agent) -> dict:
    st = agent._store
    torch.cuda.synchronize()
    mask = torch.ones_like(st.params, dtype=torch.bool)
    mask[st.info_off:st.info_off + 16] = False          # the info gap holds no parameters
    main = mask.clone()
    main[st.n_main:] = False                            # params / target have no aux part
    out = {name: getattr(st, name)[m].cpu() for name, m in (("params", main), ("target", main), ("m", mask), ("v", mask))}
    out.update(counts=st.counts.cpu(), step=np.asarray(agent.state.step), rng=np.asarray(agent.state.rng))
    return out


def _ring_snapshot(dp) -> dict:
    from test_replay_persistence_gpu import _snapshot
    snap = _snapshot(dp.store)
    snap["_seed"] = None                                # the one field the replicas do not share
    return snap


def _close(agent):
    agent._graphs.clear()                               # captured NCCL kernels must not outlive the process group
    torch.cuda.synchronize()


# ---- workers ------------------------------------------------------------------------------------------------------------
def _actor_run(rank, world, tmp, kind):
    """An actor thread inserts into rank 0's online ring while both ranks run the learner loop."""
    from test_replay_persistence_gpu import _assert_same, _draw, _snapshot
    precision = "fp16" if kind == "drq" else "fp32"
    agent, rb, demo, trs = _setup(kind, precision)
    if kind == "drq":
        agent.pipeline_critic_steps = True               # the cross-step pipeline prefetches the next draw one call early
    done = _fill(rank, rb, demo, trs)
    th = None
    if rank == 0:
        def actor():
            for tr in trs[done:]:
                rb.insert(tr)
                time.sleep(0.002)
        th = threading.Thread(target=actor)
        th.start()
    agent = _loop(kind, agent, rb, demo, 6)
    if th is not None:
        th.join(timeout=120)
        assert not th.is_alive()
    rb.sync()
    agent.check_status()
    assert len(rb) == CAP and rb.store._seed == SEEDS[0] + rank and demo.store._seed == SEEDS[1] + rank
    res = {"agent": _agent_snapshot(agent), "rb": _ring_snapshot(rb), "demo": _ring_snapshot(demo), "got": rb.sync_bytes}
    if kind == "drq":
        # rank r draws exactly what a standalone ring seeded base + r, holding the same transitions, draws
        from serl_b200.utils.launcher import make_replay_buffer
        from helpers import fake_env
        alone = make_replay_buffer(fake_env(CAMS), capacity=CAP, type="memory_efficient_replay_buffer", image_keys=list(CAMS),
                                   seed=SEEDS[0] + rank)
        for tr in trs[40:]:
            alone.insert(tr)
        alone._draw_step = rb.store._draw_step
        a, b = _snapshot(alone), _snapshot(rb.store)
        for k in ("step_dev", "_dev_step_mirror"):
            a.pop(k), b.pop(k)
        _assert_same(a, b)
        keys = np.random.default_rng(5).integers(0, 2 ** 32, (3, 4), dtype=np.uint64).astype(np.uint32)
        draws = []
        for k in keys:
            x = _draw(rb.store, rb.sample(BATCH, pack_obs_and_next_obs=True), k)
            _assert_same(x, _draw(alone, alone.sample(BATCH // world, pack_obs_and_next_obs=True), k))
            draws.append(x["idx"])
        res["idx"] = np.stack(draws)
    _close(agent)
    torch.save(res, os.path.join(tmp, f"{kind}{rank}.pt"))


N, M, PER = 3, 3, 5


def _deterministic_actor(rank, rb, trs, start):
    """Inserts PER transitions on rank 0 at the start of every iteration: the same schedule in every run."""
    def before_each(i):
        if rank == 0:
            for tr in trs[start + i * PER:start + (i + 1) * PER]:
                rb.insert(tr)
    return before_each


def _resume_first(rank, world, tmp):
    """The uninterrupted N + M run, then a run that stops after N, checkpoints on rank 0 and saves both rings."""
    from serl_b200.utils import checkpoints
    agent, rb, demo, trs = _setup("drq")
    done = _fill(rank, rb, demo, trs)
    agent = _loop("drq", agent, rb, demo, N + M, _deterministic_actor(rank, rb, trs, done))
    rb.sync()
    torch.save({"agent": _agent_snapshot(agent), "rb": _ring_snapshot(rb), "demo": _ring_snapshot(demo), "seed": rb.store._seed},
               os.path.join(tmp, f"whole{rank}.pt"))
    _close(agent)
    agent, rb, demo, trs = _setup("drq")
    done = _fill(rank, rb, demo, trs)
    agent = _loop("drq", agent, rb, demo, N, _deterministic_actor(rank, rb, trs, done))
    if rank == 0:
        checkpoints.save_checkpoint(os.path.join(tmp, "ckpt"), agent.state, step=N, keep=10)
    rb.save(os.path.join(tmp, "replay.npz"))
    demo.save(os.path.join(tmp, "demo.npz"))
    _close(agent)


def _resume_second(rank, world, tmp):
    """A fresh 2-rank job: other agent seed, entropy-seeded rings; restores the checkpoint and both rings, runs M more."""
    import torch.distributed as dist
    from serl_b200.utils import checkpoints
    agent, rb, demo, trs = _setup("drq", agent_seed=7, ring_seeds=(None, None))
    dist.barrier()
    agent = agent.replace(state=checkpoints.restore_checkpoint(os.path.join(tmp, "ckpt"), agent.state))
    rb.load(os.path.join(tmp, "replay.npz"))
    demo.load(os.path.join(tmp, "demo.npz"))
    agent = _loop("drq", agent, rb, demo, M, _deterministic_actor(rank, rb, trs, 100 + N * PER))
    rb.sync()
    torch.save({"agent": _agent_snapshot(agent), "rb": _ring_snapshot(rb), "demo": _ring_snapshot(demo), "seed": rb.store._seed},
               os.path.join(tmp, f"resumed{rank}.pt"))
    _close(agent)


def _worker(rank, world, port, tmp, case, *args):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank),
                            timeout=datetime.timedelta(seconds=300))
    try:
        globals()[case](rank, world, tmp, *args)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _spawn(tmp_path, case, *args, timeout=600):
    """Runs `case` on two ranks; every worker is joined, or killed and joined, before this returns."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    port = 33000 + (os.getpid() * 7 + len(case) + len(args)) % 2000
    ctx = mp.spawn(_worker, args=(2, port, str(tmp_path), case, *args), nprocs=2, join=False)
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=5):
            assert time.monotonic() < deadline, f"{case}: workers still running after {timeout} s"
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join()


def _assert_equal_trees(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, torch.Tensor):
            assert torch.equal(x, y), f"{what}: {k}"
        else:
            np.testing.assert_array_equal(np.asarray(x), np.asarray(y), err_msg=f"{what}: {k}")


# ---- tests --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["drq", "sac"])
def test_replicas_and_agents_stay_bitwise_equal_with_an_actor_inserting(tmp_path, kind):
    _spawn(tmp_path, "_actor_run", kind)
    r0, r1 = (torch.load(tmp_path / f"{kind}{r}.pt", weights_only=False) for r in (0, 1))
    for part in ("rb", "demo", "agent"):
        _assert_equal_trees(r0[part], r1[part], f"{kind} {part}")
    assert r0["got"] > 0 and r0["got"] == r1["got"]
    if kind == "drq":
        assert not np.array_equal(r0["idx"], r1["idx"])   # the ranks' sampler streams differ


def test_resumed_run_matches_an_uninterrupted_one_bitwise(tmp_path):
    _spawn(tmp_path, "_resume_first")
    _spawn(tmp_path, "_resume_second")
    for r in (0, 1):
        whole, resumed = (torch.load(tmp_path / f"{name}{r}.pt", weights_only=False) for name in ("whole", "resumed"))
        assert whole["seed"] == resumed["seed"] == SEEDS[0] + r
        for part in ("rb", "demo", "agent"):
            _assert_equal_trees(resumed[part], whole[part], f"rank {r} {part}")
