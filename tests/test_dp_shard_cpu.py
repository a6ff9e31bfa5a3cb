"""CPU: frame-sharded replay host logic (serl_b200/data/frame_shards.py, data_parallel.py with shard_frames).

- slot ranges and halos, capacities that do not divide by the world size, and the layouts the kernels cannot follow;
- which frames each rank's scatter keeps: the staged slot writes of a frame-dedup ring (episode starts, wrap-around re-insert
  at the front) are applied through `FrameShards.locals`, and every window the sampler reads, taken from the owner the kernels
  pick, must equal the window of a replica fed the same writes;
- on two gloo ranks with the kernels and CUDA IPC stubbed (as test_dp_replay_cpu.py stubs them): the shard table each rank
  hands the sampler, the refusal without peer access, and that a sharded store's ring file carries a replicated store's meta.
"""
import contextlib
import ctypes as C
import datetime
import os
import sys
import time
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMS, HW = ("front", "wrist"), 8


def test_ranges_and_halos():
    from serl_b200.data.frame_shards import FrameShards
    for cap, world, T in ((41, 2, 1), (50, 3, 2), (64, 8, 1), (10, 1, 3), (23, 4, 2)):
        sh = [FrameShards(cap, T, r, world) for r in range(world)]
        spr = -(-cap // world)
        assert all(s.slots_per_rank == spr and s.local_slots == spr + T for s in sh)
        owned = [x for s in sh for x in range(*s.range())]
        assert owned == list(range(cap))                       # contiguous, disjoint, in rank order
        for r, s in enumerate(sh):
            lo, hi = s.range()
            assert (lo, hi) == (r * spr, min(cap, (r + 1) * spr)) and all(s.owner(x) == r for x in range(lo, hi))
            halo = [(lo - d) % cap for d in range(T, 0, -1)]     # T slots in front, wrapping below slot 0
            for l, x in enumerate(halo):
                assert l in s.locals(x)
            for x in range(lo, hi):
                assert x - lo + T in s.locals(x)
            stored = {x for x in range(cap) if s.locals(x)}
            assert stored == set(range(lo, hi)) | set(halo)
    with pytest.raises(ValueError, match="without slots"):
        FrameShards(17, 1, 0, 8)                               # 3 slots per rank: rank 6 would start at 18
    with pytest.raises(ValueError, match="twice the frame stack"):
        FrameShards(12, 4, 0, 2)
    with pytest.raises(ValueError, match="1 to 8 ranks"):
        FrameShards(100, 1, 0, 9)


def _staged_writes(cap, T, n, seed=0):
    """(dst, src, frame id) slot writes a frame-dedup ring stages for n transitions, read from its host staging records."""
    from serl_b200 import _lib as L
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
    from helpers import Box, DictSpace
    space = DictSpace({"cam": Box((T, 2, 2, 1), np.uint8), "state": Box((T, 1))})
    writes = []
    real = L.call

    def call(name, *a):
        if name == "serl_replay_scatter":
            rq = a[1]._obj
            for k in range(rq.n):
                rec = lambda ptr: ptr + k * rq.row_stride
                dst = C.c_int32.from_address(rec(rq.dst_slot)).value
                src = C.c_int32.from_address(rec(rq.src_slot)).value
                frame = bytes((C.c_uint8 * 4).from_address(rec(rq.frames[0])))
                writes.append((dst, src, frame))
            return 0
        return real(name, *a) if name.startswith("serl_host_") else 0

    saved = (L.call, L.require_cuda, L.stream_ptr, L.new_event, L.pin)
    L.call, L.require_cuda, L.stream_ptr, L.pin = call, (lambda d: None), (lambda: 0), (lambda t: t)
    L.new_event = lambda: types.SimpleNamespace(record=lambda: None, synchronize=lambda: None, make_current_stream_wait=lambda: None)
    try:
        ring = MemoryEfficientReplayBuffer(space, Box((1,)), cap, pixel_keys=("cam",), device="cpu")
        rng = np.random.default_rng(seed)
        fid = 0
        for i in range(n):
            frames = np.arange(fid, fid + T + 1, dtype=np.uint32).view(np.uint8).reshape(T + 1, 2, 2, 1)
            fid += T + 1
            done = bool(rng.random() < 0.15)
            ring.insert(dict(observations={"cam": frames[:T], "state": np.zeros((T, 1), np.float32)},
                             next_observations={"cam": frames[1:], "state": np.zeros((T, 1), np.float32)},
                             actions=np.zeros(1, np.float32), rewards=np.float32(0), masks=np.float32(1), dones=done))
        ring.flush()
    finally:
        L.call, L.require_cuda, L.stream_ptr, L.new_event, L.pin = saved
    return writes, ring


@pytest.mark.parametrize("cap,world,T", [(41, 2, 1), (40, 2, 3), (50, 3, 2), (64, 8, 1), (30, 1, 2)])
def test_sharded_scatter_keeps_every_window_the_sampler_reads(cap, world, T):
    from serl_b200.data.frame_shards import FrameShards
    writes, ring = _staged_writes(cap, T, 3 * cap)
    assert any(src >= 0 for _, src, _ in writes)                # the mid-episode wrap re-inserted frames at the front
    replica = [None] * cap
    sh = [FrameShards(cap, T, r, world) for r in range(world)]
    local = [[None] * s.local_slots for s in sh]
    for dst, src, frame in writes:                              # in staging order, like the scatter launches
        for r, s in enumerate(sh):                              # each rank: its copies only, the source from its own copy
            if not s.locals(dst):
                continue
            val = frame if src < 0 else local[r][s.locals(src)[0]]
            assert src < 0 or val == replica[src]
            for l in s.locals(dst):
                local[r][l] = val
        replica[dst] = frame if src < 0 else replica[src]
    for idx in range(cap):                                      # every window the sampler can read (serl_replay_sample_crop)
        w0 = idx - T + (cap - T if idx - T < 0 else 0)
        o, l0 = sh[0].window_source(w0)
        assert [local[o][l0 + t] for t in range(T + 1)] == replica[w0:w0 + T + 1], (idx, o)


# ---- two gloo ranks ---------------------------------------------------------------------------------------------------
def _stub(setattr_, calls):
    from serl_b200 import _lib as L
    from serl_b200.data import data_parallel as DP
    from serl_b200.data import replay_buffer as RB
    real = L.call

    def call(name, *a):
        calls.append((name, a))
        if name == "serl_ipc_export":                            # handle = the pointer's bytes; offset 16
            C.memmove(a[1], C.c_uint64(a[0].value - 16).value.to_bytes(8, "little") + b"\0" * 56, 64)
            a[2]._obj.value = 16
        elif name == "serl_ipc_open":
            a[1]._obj.value = int.from_bytes(bytes(a[0])[:8], "little")
        elif name.startswith("serl_host_"):
            return real(name, *a)
        return 0

    setattr_(L, "call", call)
    setattr_(L, "require_cuda", lambda d: None)
    setattr_(L, "stream_ptr", lambda: 0)
    setattr_(L, "new_event", lambda: types.SimpleNamespace(record=lambda: None, synchronize=lambda: None,
                                                           make_current_stream_wait=lambda: None))
    setattr_(L, "pin", lambda t: t)
    setattr_(RB.DeviceRing, "_io_copy_stream", lambda self: types.SimpleNamespace(synchronize=lambda: None))
    setattr_(torch.cuda, "synchronize", lambda *a: None)
    setattr_(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    setattr_(torch.cuda, "current_device", lambda: 0)
    setattr_(torch.cuda, "device_count", lambda: 1)
    setattr_(torch.cuda, "get_device_properties", lambda d: types.SimpleNamespace(uuid="GPU-0"))
    return DP


def _shard_job(rank, world, tmp):
    from helpers import fake_env, random_transitions
    from serl_b200.data import replay_io as RIO
    from serl_b200.utils.launcher import make_replay_buffer
    calls = []
    peer_ok = []
    DP = _stub(setattr, calls)
    import serl_b200._lib as L
    L.load = lambda: types.SimpleNamespace(serl_can_access_peer=lambda a, b: peer_ok[0] if peer_ok else 1)
    kw = dict(capacity=41, type="memory_efficient_replay_buffer", image_keys=list(CAMS), device="cpu", seed=3)
    env = fake_env(CAMS, HW)
    dp = make_replay_buffer(env, data_parallel="shard_frames", **kw)
    rep = make_replay_buffer(env, data_parallel=True, **kw)
    assert dp.sharded and dp.store.shards.range() == ((0, 21) if rank == 0 else (21, 41))
    fb = HW * HW * 3
    assert all(dp.store.frames[c].numel() == 22 * fb for c in CAMS)
    ptrs = [None] * world
    dist.all_gather_object(ptrs, [dp.store.frames[c].data_ptr() for c in CAMS])
    t = dp.store.shard_table()
    assert (t.slots_per_rank, t.halo, t.world, t.rank) == (21, 1, 2, rank)
    assert [[t.frames[j][r] for r in range(world)] for j in range(len(CAMS))] == [[ptrs[r][j] for r in range(world)]
                                                                                  for j in range(len(CAMS))]
    trs = random_transitions(np.random.default_rng(0), 60, CAMS, HW, mean_ep=7)
    if rank == 0:
        for tr in trs:
            dp.insert(tr)
            rep.insert(tr)
    calls.clear()
    dp.sample(8).to_dict()                                  # syncs (inserts + flush), then one sharded sampler launch
    names = [n for n, _ in calls]
    assert "serl_replay_scatter_sharded" in names and "serl_replay_scatter" not in names
    (_, args), = [c for c in calls if c[0] == "serl_replay_sample_crop_sharded"]
    got = args[1]._obj
    assert (got.slots_per_rank, got.rank) == (21, rank) and got.frames[1][1 - rank] == ptrs[1 - rank][1]
    rep.sample(8)
    metas = []
    real_write = RIO.write_ring_file
    RIO.write_ring_file = lambda path, meta, fields, stager: (metas.append(meta), 0)[1]
    for s in (dp, rep):
        s.save(os.path.join(tmp, "x.npz"))
    RIO.write_ring_file = real_write
    if rank == 0:
        assert len(metas) == 2 and metas[0] == metas[1]    # the same file meta as a replicated store's
    # a job whose GPUs cannot reach each other is refused on every rank
    peer_ok.append(0)
    with pytest.raises(RuntimeError, match="peer access"):
        make_replay_buffer(env, data_parallel="shard_frames", **kw)


def _worker(rank, world, port, tmp, case):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    globals()[case](rank, world, tmp)
    dist.barrier()
    dist.destroy_process_group()


def test_shard_table_peer_refusal_and_file_meta_on_two_ranks(tmp_path):
    port = 36000 + os.getpid() % 2000
    ctx = mp.spawn(_worker, args=(2, port, str(tmp_path), "_shard_job"), nprocs=2, join=False)
    deadline = time.monotonic() + 300
    try:
        while not ctx.join(timeout=5):
            assert time.monotonic() < deadline, "workers still running after 300 s"
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join()
