"""CPU, gloo: `DataParallelDataStore` host logic - rank 0's pending list and its order under a concurrent inserting thread,
replicas whose host bookkeeping equals a single ring fed the same transitions after every sync, the global-batch split,
per-rank sampler seeds, save on rank 0 / load on every rank, and the world-size-1 pass-through.  Kernels are stubbed as in
test_dp_gloo_cpu.py, so device arrays stay untouched and only host state is compared."""
import contextlib
import datetime
import os
import sys
import threading
import time
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMS, HW = ("front", "wrist"), 16


class _Ev:
    def record(self): pass
    def synchronize(self): pass
    def make_current_stream_wait(self): pass


def _stub(setattr_):
    """No-op kernels and CUDA plumbing; ring files go through replay_io's HostStager."""
    from serl_b200 import _lib as L
    from serl_b200.data import replay_buffer as RB
    from serl_b200.data import replay_io as RIO
    real = L.call

    class HostStager(RIO.HostStager):
        def __init__(self, stream, chunk_bytes):
            super().__init__(chunk_bytes)
            self.pinned_bytes = 2 * self.chunk_bytes

        @staticmethod
        def _bytes(a):
            return a.numpy() if isinstance(a, torch.Tensor) else a.reshape(-1).view(np.uint8)

    setattr_(L, "call", lambda name, *a: real(name, *a) if name.startswith("serl_host_") else 0)
    setattr_(L, "require_cuda", lambda d: None)
    setattr_(L, "stream_ptr", lambda: 0)
    setattr_(L, "new_event", lambda: _Ev())
    setattr_(L, "pin", lambda t: t)
    setattr_(RB, "_CudaStager", HostStager)
    setattr_(RB.DeviceRing, "_io_copy_stream", lambda self: types.SimpleNamespace(synchronize=lambda: None))
    setattr_(torch.cuda, "stream", lambda s: contextlib.nullcontext())


def _frame_env():
    from helpers import fake_env
    return fake_env(CAMS, HW)


def _state_env(S=7, A=4):
    from helpers import Box
    return types.SimpleNamespace(observation_space=Box((S,)), action_space=Box((A,)))


def _state_transitions(rng, n, S=7, A=4):
    return [dict(observations=rng.standard_normal(S).astype(np.float32), next_observations=rng.standard_normal(S).astype(np.float32),
                 actions=rng.uniform(-1, 1, A).astype(np.float32), rewards=np.float32(i), masks=np.float32(1.0),
                 dones=bool(rng.random() < 0.1)) for i in range(n)]


def _ring(kind, cap, seed=None, data_parallel=False):
    from serl_b200.utils.launcher import make_replay_buffer
    if kind == "frames":
        return make_replay_buffer(_frame_env(), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(CAMS),
                                  device="cpu", seed=seed, data_parallel=data_parallel)
    return make_replay_buffer(_state_env(), capacity=cap, type="replay_buffer", device="cpu", seed=seed, data_parallel=data_parallel)


def _transitions(kind, n, seed=0):
    from helpers import random_transitions
    rng = np.random.default_rng(seed)
    return random_transitions(rng, n, CAMS, HW, mean_ep=7) if kind == "frames" else _state_transitions(rng, n)


def _book(ring) -> dict:
    return {"_insert_index": ring._insert_index, "_size": ring._size, "_first": getattr(ring, "_first", None),
            "valid": ring._valid_host.copy()}


def _assert_book(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=f"{what}: {k}")


def _draw(ring) -> dict:
    return {"_seed": ring._seed, "_draw_step": ring._draw_step, "_dev_step_mirror": ring._dev_step_mirror,
            "step_dev": int(ring.step_dev.item())}


# ---- workers ------------------------------------------------------------------------------------------------------------
def _order(rank, world, tmp):
    from serl_b200.data.data_parallel import DataParallelDataStore
    n = 200
    trs = _transitions("state", n)
    dp = _ring("state", 64, seed=5, data_parallel=True)
    assert isinstance(dp, DataParallelDataStore)
    seen, real_insert = [], dp.store.insert
    dp.store.insert = lambda tr: (seen.append(int(tr["rewards"])), real_insert(tr))
    ref = _ring("state", 64)
    if rank == 0:
        def actor():
            for tr in trs:
                dp.insert(tr)
                time.sleep(0.001)
        th = threading.Thread(target=actor)
        th.start()
    lens, received = [], []
    for i in range(42):                                # collective: both ranks sync the same number of times
        if i == 41 and rank == 0:
            th.join(timeout=60)
            assert not th.is_alive()
        before = dp.sync_bytes
        lens.append(dp.sync())
        received.append(dp.sync_bytes > before)
        time.sleep(0.01)
    assert seen == list(range(n)), seen[:20]            # every transition, once, in insertion order, on every rank
    for tr in trs:
        ref.insert(tr)
    _assert_book(_book(dp.store), _book(ref), f"rank {rank}")
    torch.save({"lens": lens, "received": received}, os.path.join(tmp, f"order{rank}.pt"))


def _replicas(rank, world, tmp, kind):
    cap = 40 if kind == "frames" else 32
    trs = _transitions(kind, 100)
    dp = _ring(kind, cap, seed=3, data_parallel=True)
    ref = _ring(kind, cap)
    books, lo = [], 0
    for n in (0, 1, 7, 13, 30, 2, 47):                 # wraps the ring twice and starts episodes inside chunks
        if rank == 0:
            for tr in trs[lo:lo + n]:
                dp.insert(tr)
        assert len(dp) == len(ref)                      # nothing lands before the sync
        for tr in trs[lo:lo + n]:
            ref.insert(tr)
        lo += n
        assert dp.sync() == len(ref)
        _assert_book(_book(dp.store), _book(ref), f"rank {rank} after {lo} transitions")
        books.append(_book(dp.store))
    assert lo == 100 and len(dp) == cap
    if kind == "frames":
        assert not all(b["_first"] for b in books) and not books[-1]["valid"].all()
    torch.save(books, os.path.join(tmp, f"books_{kind}{rank}.pt"))


def _roles(rank, world, tmp):
    from serl_b200.data.data_parallel import DataParallelDataStore
    from serl_b200.data.replay_buffer import BatchHandle
    trs = _transitions("frames", 30)
    dp = _ring("frames", 40, seed=77, data_parallel=True)
    assert dp.store._seed == 77 + rank                  # base + rank
    drawn = _ring("frames", 40, seed=None if rank == 0 else 5, data_parallel=True)
    seeds = [None] * world
    dist.all_gather_object(seeds, drawn.store._seed)
    assert seeds[1] == seeds[0] + 1                     # rank 0 drew the base; rank 1's own seed was replaced
    if rank == 0:
        for tr in trs:
            dp.insert(tr)
    else:
        with pytest.raises(RuntimeError, match="rank 1"):
            dp.insert(trs[0])
    ref = _ring("frames", 40)
    for tr in trs:
        ref.insert(tr)
    h = dp.sample(8, pack_obs_and_next_obs=True)        # syncs first: the transitions arrive on rank 1
    assert isinstance(h, BatchHandle) and len(dp) == len(ref) and h.batch_size == 4
    assert h.parts[0]["ring"] is dp.store and h.parts[0]["seed"] == 77 + rank and h.parts[0]["step"] == 0
    with pytest.raises(ValueError, match="global batch 7"):
        dp.sample(7)
    it = dp.get_iterator(sample_args={"batch_size": 6, "pack_obs_and_next_obs": True})
    assert [next(it).parts[0]["batch"] for _ in range(2)] == [3, 3] and dp.store._draw_step == 3
    assert dp.latest_data_id() == dp.store._insert_index
    assert isinstance(drawn, DataParallelDataStore)


def _persist(rank, world, tmp):
    from serl_b200.data import replay_io as RIO
    from serl_b200.data.data_parallel import META_KEY
    writes = []
    real_write = RIO.write_ring_file
    RIO.write_ring_file = lambda *a, **k: (writes.append(a[0]), real_write(*a, **k))[1]
    trs = _transitions("frames", 50)
    dp = _ring("frames", 40, seed=11, data_parallel=True)
    if rank == 0:
        for tr in trs:
            dp.insert(tr)
    dp.sample(4)
    for _ in range(rank + 2):                           # local draws: the ranks' draw counters differ
        dp.store.sample(2)
    dp.store.step_dev.fill_(30 + rank)
    dp.store._dev_step_mirror = 30 + rank
    path = os.path.join(tmp, "dp.npz")
    assert dp.save(path) == os.path.getsize(path)
    assert len(writes) == (1 if rank == 0 else 0)       # one writer: the replicas are identical
    want, book = _draw(dp.store), _book(dp.store)
    assert want == {"_seed": 11 + rank, "_draw_step": 3 + rank, "_dev_step_mirror": 30 + rank, "step_dev": 30 + rank}
    meta = RIO.read_meta(path)[META_KEY]
    assert meta["world"] == 2 and [r["_draw_step"] for r in meta["ranks"]] == [3, 4]
    fresh = _ring("frames", 40, seed=900, data_parallel=True)
    assert fresh.load(path) is fresh
    assert _draw(fresh.store) == want                   # each rank restores its own seed and draw counters
    got = _book(fresh.store)
    assert {k: got[k] for k in ("_insert_index", "_size", "_first")} == {k: book[k] for k in ("_insert_index", "_size", "_first")}
    # a single-process file: every rank loads it; rank r continues with the saved seed + r
    single = os.path.join(tmp, "single.npz")
    plain = _ring("frames", 40, seed=500)
    for tr in trs[:20]:
        plain.insert(tr)
    plain.sample(2)
    if rank == 0:
        plain.save(single)
    dist.barrier()
    fresh.load(single)
    assert len(fresh) == len(plain) and fresh.store._seed == 500 + rank and fresh.store._draw_step == 1
    # a file from another world size raises on every rank
    other = os.path.join(tmp, "world3.npz")
    if rank == 0:
        dp.store.save(other, extra_meta={META_KEY: {"world": 3, "ranks": [want] * 3}})
    dist.barrier()
    with pytest.raises(ValueError, match="3 data-parallel ranks"):
        fresh.load(other)
    # one rank failing makes every rank raise (none is left waiting in a collective)
    if rank == 0:
        with pytest.raises(RuntimeError, match="another rank failed"):
            fresh.load(path)
    else:
        with pytest.raises(OSError):
            fresh.load(os.path.join(tmp, "missing.npz"))


def _worker(rank, world, port, tmp, case, *args):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    _stub(setattr)
    globals()[case](rank, world, tmp, *args)
    dist.barrier()
    dist.destroy_process_group()


def _spawn(tmp_path, case, *args, timeout=300):
    """Runs `case` on two gloo ranks; every worker is joined or killed before this returns."""
    port = 32000 + (os.getpid() * 7 + len(case)) % 2000
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


# ---- tests --------------------------------------------------------------------------------------------------------------
def test_pending_list_keeps_insertion_order_under_a_concurrent_inserting_thread(tmp_path):
    _spawn(tmp_path, "_order")
    r0, r1 = (torch.load(tmp_path / f"order{r}.pt") for r in (0, 1))
    assert r0 == r1 and r0["lens"][-1] == 64            # both replicas grew at the same syncs
    assert sum(r0["received"]) >= 2                     # transitions arrived at several syncs while the actor inserted


@pytest.mark.parametrize("kind", ["frames", "state"])
def test_replica_bookkeeping_equals_a_single_ring_after_every_sync(tmp_path, kind):
    _spawn(tmp_path, "_replicas", kind)
    b0, b1 = (torch.load(tmp_path / f"books_{kind}{r}.pt", weights_only=False) for r in (0, 1))
    assert len(b0) == len(b1) == 7
    for i, (x, y) in enumerate(zip(b0, b1)):
        _assert_book(x, y, f"sync {i}")


def test_insert_on_rank_1_raises_and_the_global_batch_splits_over_ranks(tmp_path):
    _spawn(tmp_path, "_roles")


def test_save_on_rank_0_and_load_on_every_rank(tmp_path):
    _spawn(tmp_path, "_persist")


def test_world_size_1_is_a_pass_through(tmp_path, monkeypatch):
    from serl_b200.data import replay_io as RIO
    from serl_b200.data.data_parallel import META_KEY, DataParallelDataStore
    _stub(monkeypatch.setattr)
    trs = _transitions("frames", 30)
    for use_group in (False, True):                     # no process group, and a gloo group of one rank
        if use_group:
            dist.init_process_group("gloo", rank=0, world_size=1, store=dist.HashStore())
        try:
            dp, ref = _ring("frames", 40, seed=9, data_parallel=True), _ring("frames", 40, seed=9)
            assert isinstance(dp, DataParallelDataStore) and dp.world == 1 and dp.store._seed == 9
            for tr in trs:
                dp.insert(tr)                           # straight into the ring: no sync needed
                ref.insert(tr)
                assert len(dp) == len(ref)
            _assert_book(_book(dp.store), _book(ref), "world 1")
            assert dp.sync() == len(ref) and dp.sync_bytes == 0
            assert dp.sample(7).batch_size == 7
            path = tmp_path / "w1.npz"
            dp.save(path)
            assert META_KEY not in RIO.read_meta(path)
            again = _ring("frames", 40, seed=1, data_parallel=True).load(path)
            assert len(again) == len(ref) and _draw(again.store) == _draw(dp.store)
            dp.store.save(tmp_path / "w2.npz", extra_meta={META_KEY: {"world": 2, "ranks": [_draw(dp.store)] * 2}})
            with pytest.raises(ValueError, match="2 data-parallel ranks"):
                again.load(tmp_path / "w2.npz")
        finally:
            if use_group:
                dist.destroy_process_group()
