"""GPU, world size 2 over gloo: a frame-sharded `DataParallelDataStore` (make_replay_buffer(data_parallel="shard_frames")) draws
the batches of a replicated one bit for bit.

Both ranks run a sharded and a replicated store side by side, with the same seeds and the same transitions, inserted on rank 0
by an actor thread.  After every sync each rank draws from both (n_step 1 and 3) and the materialised batches must be bitwise
equal.  The frame shapes are those of test_replay_sampler_paths_gpu.py that select each sampler kernel.  Then `save` must write
the replicated file's arrays, a fresh sharded store loading it must draw the replicated store's next batches, and each rank must hold (ceil(C / 2) + T) / C of a replica's frame bytes.
With both ranks on cuda:0 the peer frames are another process's allocation on the same device (CUDA IPC); with two devices
the same test reads them over peer-to-peer links."""
import datetime
import os
import sys
import threading
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP, BATCH, SEED = 40, 8, 7


def _env(ncam, T, H, W, C):
    import types
    from helpers import Box, DictSpace
    cams = tuple(f"cam{j}" for j in range(ncam))
    space = DictSpace({**{c: Box((T, H, W, C), np.uint8) for c in cams}, "state": Box((T, 5))})
    return types.SimpleNamespace(observation_space=space, action_space=Box((3,))), cams


def _transitions(n, cams, T, H, W, C, seed=0):
    """Episodes whose frames shift by one per step (next_obs of t == obs of t + 1), mean length 9."""
    rng = np.random.default_rng(seed)
    out, cur = [], None
    for _ in range(n):
        if cur is None:
            cur = {c: rng.integers(0, 256, (T, H, W, C), dtype=np.uint8) for c in cams}
            cur["state"] = rng.standard_normal((T, 5)).astype(np.float32)
        nxt = {c: np.concatenate([cur[c][1:], rng.integers(0, 256, (1, H, W, C), dtype=np.uint8)]) for c in cams}
        nxt["state"] = rng.standard_normal((T, 5)).astype(np.float32)
        done = bool(rng.random() < 1 / 9)
        out.append(dict(observations=cur, next_observations=nxt, actions=rng.uniform(-1, 1, 3).astype(np.float32),
                        rewards=np.float32(rng.random()), masks=np.float32(0.0 if done else 1.0), dones=done))
        cur = None if done else nxt
    return out


def _flat(d, prefix=""):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out.update(_flat(v, prefix + k + "/"))
        else:
            out[prefix + k] = v.cpu().numpy()
    return out


def _assert_same_batch(a, b, what):
    fa, fb = _flat(a.to_dict()), _flat(b.to_dict())
    assert fa.keys() == fb.keys(), what
    for k in fa:
        assert fa[k].tobytes() == fb[k].tobytes(), f"{what}: {k}"


def _draw_same(ref, *stores, what):
    """One draw from every store (n_step 1, then 3); each batch must equal `ref`'s."""
    for n_step in (1, 3):
        kw = dict(pack_obs_and_next_obs=True) if n_step == 1 else dict(n_step=3, discount=0.9)
        want = ref.sample(BATCH, **kw)
        for k, st in enumerate(stores):
            _assert_same_batch(st.sample(BATCH, **kw), want, f"{what} store {k} n_step={n_step}")


def _case(rank, world, tmp, shape):
    import torch.distributed as dist
    from serl_b200.utils.launcher import make_replay_buffer
    ncam, T, H, W, C = shape
    env, cams = _env(*shape)
    kw = dict(capacity=CAP, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=SEED)
    sh = make_replay_buffer(env, data_parallel="shard_frames", **kw)
    rep = make_replay_buffer(env, data_parallel=True, **kw)
    assert sh.sharded and not rep.sharded and sh.store._seed == rep.store._seed == SEED + rank
    fb = H * W * C
    for c in cams:                                      # (ceil(C / 2) + T) / C of a replica
        assert sh.store.frames[c].numel() == (-(-CAP // 2) + T) * fb and rep.store.frames[c].numel() == CAP * fb
    trs = _transitions(130, cams, T, H, W, C)
    lock = threading.Lock()                             # both stores see the same pending transitions at every sync
    th = None
    if rank == 0:
        def actor():
            for tr in trs:
                with lock:
                    sh.insert(tr)
                    rep.insert(tr)
                time.sleep(0.002)
        th = threading.Thread(target=actor)
        th.start()
    for i in range(40):                                 # collective: both ranks go through the same syncs
        if i == 39 and th is not None:
            th.join(timeout=120)
            assert not th.is_alive()
        with lock:                                      # sample() syncs again: no insert may land in one store only
            sh.sync()
            rep.sync()
            if len(rep) > T + 1:
                _draw_same(rep, sh, what=f"rank {rank} sync {i}")
        time.sleep(0.005)
    assert len(sh) == len(rep) == CAP and not sh.store._valid_host.all()   # wrapped, with re-inserted front slots
    # save: the replicated file's arrays; load: the replicated store's next draws
    p_sh, p_rep = os.path.join(tmp, f"sh{rank}.npz"), os.path.join(tmp, f"rep{rank}.npz")
    sh.save(p_sh)
    rep.save(p_rep)
    if rank == 0:
        a, b = np.load(p_sh), np.load(p_rep)
        assert sorted(a.files) == sorted(b.files)
        for k in a.files:
            if k != "meta":
                assert a[k].tobytes() == b[k].tobytes(), k
    dist.barrier()
    fresh = make_replay_buffer(env, data_parallel="shard_frames", **{**kw, "seed": 1})
    fresh.load(os.path.join(tmp, "sh0.npz"))
    fresh_rep = make_replay_buffer(env, data_parallel=True, **{**kw, "seed": 1})
    fresh_rep.load(os.path.join(tmp, "sh0.npz"))        # a sharded file seeds a replicated store: the files are interchangeable
    for j in range(3):                                  # the sharded file restores both kinds of store
        _draw_same(rep, fresh, fresh_rep, what=f"rank {rank} after load, draw {j}")
    for s in (sh, fresh):
        s.close()


def _worker(rank, world, port, tmp, devices, shape):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.cuda.set_device(rank if devices == "two" else 0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        _case(rank, world, tmp, shape)
        dist.barrier()
    finally:
        dist.destroy_process_group()


SHAPES = [
    pytest.param((2, 1, 128, 128, 3), id="frames-128x128x3-2cam"),
    pytest.param((1, 3, 64, 64, 3), id="frames-64x64x3-T3"),
    pytest.param((1, 1, 128, 128, 3), id="frames-128x128x3-1cam"),
    pytest.param((1, 1, 256, 128, 3), id="banded-256x128x3"),
    pytest.param((1, 9, 32, 32, 3), id="banded-32x32x3-T9"),
    pytest.param((1, 1, 84, 84, 3), id="bytewise-84x84x3"),
]


@pytest.mark.parametrize("devices", ["one", "two"])
@pytest.mark.parametrize("shape", SHAPES)
def test_sharded_store_draws_the_replicated_batches(tmp_path, shape, devices):
    import torch.multiprocessing as mp
    if devices == "two" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    port = 34000 + (os.getpid() * 13 + hash((shape, devices)) % 997) % 2000
    ctx = mp.spawn(_worker, args=(2, port, str(tmp_path), devices, shape), nprocs=2, join=False)
    deadline = time.monotonic() + 600
    try:
        while not ctx.join(timeout=5):
            assert time.monotonic() < deadline, "workers still running after 600 s"
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join()
