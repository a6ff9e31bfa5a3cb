"""Replay for a data-parallel learner: every rank holds a replica of the ring (by default a full one), fed by the one actor that
talks to rank 0.

In SERL's learner the actor sends transitions to a single agentlace `TrainerServer`, whose thread calls `insert` on a single
data store in a single process.  `DataParallelDataStore` wraps one of the stores of data_store.py so that a learner started
with `torchrun --nproc-per-node N` trains on those transitions on every rank:

- `insert` (rank 0 only, any thread) pickles the transition onto a pending list and returns.
- `sync` (collective, every rank's main thread) broadcasts rank 0's pending list over a gloo group of the wrapper's own and
  inserts it, in order, through every rank's ring.  Transitions take effect only at sync points, so the replicas stay bitwise
  identical.  The transfer stays off NCCL: the gradient all-reduce owns the NCCL communicator, and a gloo call is synchronous
  on the host, so it cannot interleave with NCCL kernels already queued on a stream.
- `sample` / `get_iterator` sync, then draw `batch_size // world` rows from the local ring: `batch_size` is the global batch.
  Ranks differ only in their sampler seed: rank r draws with `base + r`, where `base` is rank 0's ring seed.

Replicas by default: replication needs no episode routing, has no empty shards early in a run and keeps one `len()` for the
whole job.  When a replica's frames do not fit in one GPU's HBM (two 500 k-slot two-camera rings are ~98 GB), the store
shards them (`shard_frames=True`, make_replay_buffer's data_parallel="shard_frames"; frame_shards.py): every field but the
frames stays a replica, so index draws, crops, n-step windows and the insert order are those of the replicated store and rank
r draws bitwise the batch it would draw from a replica, but rank r stores only the frames of slots [lo_r, hi_r) plus a halo of
T slots in front, (ceil(C / N) + T) / C of a replica.  Each rank maps the others' frame allocations with CUDA IPC at
construction (refused without peer access between every pair of devices), and the sampler reads each row's frames from their
owner, over NVLink when that is another GPU.  Inserts travel as before; each rank's scatter keeps the frames it stores.

Ordering in a frame-sharded store: a rank's sampler may read a peer's frames, so a sync that carries inserts first waits for
the rank's outstanding device work (sampler launches, prefetches, graph replays), meets every rank at a barrier, inserts and
flushes, waits for the flush, and meets every rank at a second barrier.  No rank overwrites a slot a peer is still reading,
and no rank reads a frame before its owner has written it.  A sync without inserts adds nothing.

With world size 1, or without an initialised process group, the wrapper passes every call straight to the store.
"""
from __future__ import annotations

import ctypes as C
import pickle
import socket
import threading
import weakref
from typing import Optional

import torch
import torch.distributed as dist

from .. import _lib as L
from . import replay_io as RIO

try:                                                   # optional: real agentlace base class (see data_store.py)
    from agentlace.data.data_store import DataStoreBase as _Base
except Exception:                                      # noqa: BLE001
    _Base = None

META_KEY = "data_parallel"                             # ring-file meta entry: {"world": N, "ranks": [draw state of rank r, ...]}
SHARD_FRAMES = "shard_frames"                          # make_replay_buffer(data_parallel=...) for a frame-sharded store


def dp_rank_world():
    """(rank, world) of the default process group, or (0, 1) without one."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _close_ipc(bases):
    for b in bases:
        L.call("serl_ipc_close", C.c_void_p(b))
    bases.clear()


class DataParallelDataStore:
    """`store` replicated on every rank of the default process group.

    group: a gloo group over every rank that carries the transitions; None creates one (`dist.new_group` is collective, so
    every rank constructs its wrappers in the same order).  Construction broadcasts rank 0's ring seed and reseeds rank r's
    ring with that seed + r.

    shard_frames: `store` was built with frame_shard=(rank, world) (only its share of the frames); construction maps every
    other rank's frame allocation into this process.  A state ring has no frames and stays a replica."""

    def __init__(self, store, *, group=None, shard_frames: bool = False):
        if getattr(store, "prioritized", False):
            raise NotImplementedError("a prioritized ring (priority_alpha) cannot be a data-parallel store: each rank would have to "
                                      "carry its written priorities to every replica")
        self.store = store
        self._pending = []                             # pickled transitions inserted on rank 0 since the last sync
        self._pending_lock = threading.Lock()
        self.sync_bytes = 0                            # payload bytes received by sync() so far
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            self.rank, self.world = dist.get_rank(), dist.get_world_size()
            self._group = group if group is not None else dist.new_group(backend="gloo")
            base = [store._seed]
            dist.broadcast_object_list(base, src=0, group=self._group)
            store.seed(int(base[0]) + self.rank)
        else:
            self.rank, self.world, self._group = 0, 1, None
        self.sharded = bool(shard_frames) and getattr(store, "shards", None) is not None
        self._ipc = []                                 # bases of the peers' allocations mapped into this process
        if shard_frames and getattr(store, "cams", ()) and not self.sharded:
            raise ValueError("shard_frames: build the ring with frame_shard=(rank, world) (make_replay_buffer(data_parallel="
                             f"{SHARD_FRAMES!r}))")
        if self.sharded:
            sh = store.shards
            if (sh.rank, sh.world) != (self.rank, self.world):
                raise ValueError(f"ring sharded for rank {sh.rank} of {sh.world}; this is rank {self.rank} of {self.world}")
            if self.world > 1:
                self._map_peers()
            self._finalizer = weakref.finalize(self, _close_ipc, self._ipc)

    # ---- frame sharding --------------------------------------------------------------------------------------------
    def _map_peers(self):
        """Collective: exports this rank's frame allocations, opens every other rank's (CUDA IPC), fills the shard table."""
        store = self.store
        dev = store.device.index if store.device.index is not None else torch.cuda.current_device()
        mine = {"host": socket.gethostname(), "uuid": str(torch.cuda.get_device_properties(dev).uuid), "frames": []}
        for c in store.cams:
            h, off = (C.c_char * L.IPC_HANDLE_BYTES)(), C.c_uint64()
            L.call("serl_ipc_export", C.c_void_p(store.frames[c].data_ptr()), h, C.byref(off))
            mine["frames"].append((bytes(h), int(off.value)))
        everyone = [None] * self.world
        dist.all_gather_object(everyone, mine, group=self._group)
        err = None
        uuids = {str(torch.cuda.get_device_properties(d).uuid): d for d in range(torch.cuda.device_count())}
        for r, peer in enumerate(everyone):
            if peer["host"] != mine["host"] or peer["uuid"] not in uuids:
                err = f"rank {r}'s GPU is not visible to rank {self.rank} (host {peer['host']})"
            elif L.load().serl_can_access_peer(dev, uuids[peer["uuid"]]) != 1:
                err = f"GPU {dev} of rank {self.rank} cannot access rank {r}'s GPU {uuids[peer['uuid']]} (no peer access)"
            if err:
                break
        failed = [None] * self.world
        dist.all_gather_object(failed, err, group=self._group)
        errs = [f for f in failed if f]
        if errs:
            raise RuntimeError("frame-sharded replay needs peer access between every pair of the job's GPUs: " + "; ".join(errs))
        peers = {j: [None] * self.world for j in range(len(store.cams))}
        for r, peer in enumerate(everyone):
            for j, (h, off) in enumerate(peer["frames"]):
                if r == self.rank:
                    continue
                base = C.c_void_p()
                L.call("serl_ipc_open", C.create_string_buffer(h, L.IPC_HANDLE_BYTES), C.byref(base))
                self._ipc.append(base.value)
                peers[j][r] = base.value + off
        store.shards.peer_frames = peers

    def close(self):
        """Collective: unmaps the peers' frame allocations once no rank reads them any more.  The store samples no more."""
        if self.sharded and self._ipc:
            torch.cuda.synchronize(self.store.device)
            dist.barrier(group=self._group)
            self._finalizer()
            dist.barrier(group=self._group)

    def _quiesce(self):
        """Every rank's device work (its sampler reads of peers' frames included) is complete when this returns."""
        torch.cuda.synchronize(self.store.device)
        dist.barrier(group=self._group)

    # ---- agentlace data-store interface ----------------------------------------------------------------------------
    def insert(self, data_dict: dict):
        """Queues a transition for the next `sync`.  Rank 0 only; safe to call from any thread."""
        if self.world == 1:
            return self.store.insert(data_dict)
        if self.rank != 0:
            raise RuntimeError(f"DataParallelDataStore.insert on rank {self.rank}: transitions enter on rank 0 and reach the "
                               "other ranks at sync()")
        blob = pickle.dumps(data_dict, protocol=pickle.HIGHEST_PROTOCOL)     # a copy now, like the ring's staging write
        with self._pending_lock:
            self._pending.append(blob)

    def __len__(self) -> int:
        return len(self.store)

    def latest_data_id(self):
        return self.store.latest_data_id()

    def get_latest_data(self, from_id: int):
        return self.store.get_latest_data(from_id)

    # ---- replication -----------------------------------------------------------------------------------------------
    def sync(self) -> int:
        """Collective: moves rank 0's pending transitions into every rank's ring, in insertion order.  Returns the new len()."""
        if self.world == 1:
            return len(self.store)
        n = torch.zeros(1, dtype=torch.int64)
        if self.rank == 0:
            with self._pending_lock:
                pending, self._pending = self._pending, []
            payload = pickle.dumps(pending, protocol=pickle.HIGHEST_PROTOCOL) if pending else b""
            n[0] = len(payload)
        dist.broadcast(n, src=0, group=self._group)
        nbytes = int(n.item())
        if nbytes:
            buf = torch.frombuffer(bytearray(payload), dtype=torch.uint8) if self.rank == 0 else torch.empty(nbytes, dtype=torch.uint8)
            dist.broadcast(buf, src=0, group=self._group)
            if self.sharded:                           # no rank still reads a slot the inserts overwrite
                self._quiesce()
            for blob in pickle.loads(memoryview(buf.numpy())):   # every rank, rank 0 included, inserts the same bytes
                self.store.insert(pickle.loads(blob))
            if self.sharded:                           # every rank's frames have landed before any rank samples them
                self.store.flush()
                self._quiesce()
            self.sync_bytes += nbytes
        return len(self.store)

    def sample(self, batch_size: int, *args, **kwargs):
        """Syncs, then draws this rank's `batch_size // world` rows: `batch_size` is the global batch."""
        if batch_size % self.world:
            raise ValueError(f"global batch {batch_size} does not split evenly over {self.world} ranks")
        self.sync()
        return self.store.sample(batch_size // self.world, *args, **kwargs)

    def get_iterator(self, queue_size: int = 2, sample_args: dict = {}, device=None):
        while True:
            yield self.sample(**sample_args)

    # ---- persistence -----------------------------------------------------------------------------------------------
    def _draw_state(self) -> dict:
        s = self.store
        return {"_seed": s._seed, "_draw_step": s._draw_step, "_dev_step_mirror": s._dev_step_mirror,
                "step_dev": int(s.step_dev.item())}

    def save(self, path, chunk_bytes: Optional[int] = None) -> int:
        """Collective: syncs, then rank 0 writes its replica (the ring file format of `DeviceRing.save`, atomic and CRC-checked),
        with every rank's sampler seed and draw counters in the file's meta.  Returns the file's size on every rank."""
        if self.world == 1:
            return self.store.save(path, chunk_bytes)
        self.sync()
        if self.sharded:                               # rank 0 reads every rank's frames
            self.store.flush()
            self._quiesce()
        draws = [None] * self.world
        dist.all_gather_object(draws, self._draw_state(), group=self._group)
        size = torch.full((1,), -1, dtype=torch.int64)
        try:
            if self.rank == 0:
                size[0] = self.store.save(path, chunk_bytes, extra_meta={META_KEY: {"world": self.world, "ranks": draws}})
        finally:                                       # the other ranks learn whether the file exists instead of waiting on it
            dist.broadcast(size, src=0, group=self._group)
        if int(size.item()) < 0:
            raise RuntimeError(f"rank 0 could not write the replay file {path!r}")
        return int(size.item())

    def load(self, path, chunk_bytes: Optional[int] = None):
        """Collective: every rank loads the file into its ring and restores its own sampler seed and draw counters.

        A file saved by a data-parallel store must come from the same world size (ValueError otherwise).  A file saved by a
        single-process ring seeds a data-parallel run as well: every rank loads the same contents and rank r continues with the
        saved seed + r and the saved draw counters.  When any rank fails, every rank raises.  Returns self."""
        err = None
        if self.sharded and self.world > 1:            # no rank still reads the frames a load replaces
            self._quiesce()
        try:
            dp = RIO.read_meta(path).get(META_KEY)
            if dp is not None and int(dp["world"]) != self.world:
                raise ValueError(f"replay file {path!r} was saved by {dp['world']} data-parallel ranks; this job has {self.world}")
            self.store.load(path, chunk_bytes)
            if dp is not None:
                st = dp["ranks"][self.rank]
                s = self.store
                s._seed, s._draw_step, s._dev_step_mirror = int(st["_seed"]), int(st["_draw_step"]), int(st["_dev_step_mirror"])
                s.step_dev.fill_(int(st["step_dev"]))
            elif self.world > 1:
                self.store.seed(self.store._seed + self.rank)
        except Exception as e:                         # noqa: BLE001
            err = e
        if self.world > 1:
            failed = torch.tensor([int(err is not None)], dtype=torch.int64)
            dist.all_reduce(failed, op=dist.ReduceOp.MAX, group=self._group)     # a sharded load has landed on every rank
            if err is None and int(failed.item()):
                raise RuntimeError(f"another rank failed to load the replay file {path!r}")
        if err is not None:
            raise err
        return self


if _Base is not None and hasattr(_Base, "register"):
    _Base.register(DataParallelDataStore)
