"""HBM-resident replay ring + lazy batch handles.

Mirrors the reference's `ReplayBuffer` (data/replay_buffer.py:40-90: ring storage, `insert`,
`__len__`, `get_iterator`) on top of a device ring: storage lives in HBM, inserts are staged in
pinned host memory and applied by a scatter kernel, and `sample` / the iterator return a
`BatchHandle` - indices are drawn, gathered and (for pixels) DrQ-shifted by ONE kernel when the agent
consumes the handle, so the reference's host gather + `jax.device_put` (replay_buffer.py:82-85)
disappears.  Index draws follow this repo's counter-based spec (oracle/replay.py::draw_indices).
`save` / `load` write and restore a ring as one `.npz` (replay_io.py), for the reference's
`replay_buffer.save(...)` in its learner's pause-and-save branch.
`sample(..., n_step=n, discount=g)` draws the same rows and crops and gives each row the n-step window that starts at its
slot (rewards, masks, dones and next observation; serl_replay_sample_crop_nstep in include/serl_b200.h, oracle/nstep.py).
`priority_alpha=a` makes a ring prioritized (Schaul et al. 2016): rows are drawn in proportion to per-slot priorities kept in a
device sum tree, `update_priorities` sets them from TD errors, and a materialised batch carries importance weights
(serl_replay_sample_crop_prio in include/serl_b200.h, oracle/per.py).
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _lib as L
from .. import ops
from . import replay_io as RIO
from .frame_shards import FrameShards, ShardedFrameArray


def _space_shape(space):
    return tuple(space.shape)


def _is_dict_space(space):
    return hasattr(space, "spaces")


MAX_NSTEP = L.MAX_NSTEP


def _tree_nodes(capacity: int) -> int:
    """Floats of the sum tree over `capacity` leaves (serl_priority_tree in include/serl_b200.h)."""
    n, total = int(capacity), 0
    while n > 1:
        total += n
        n = (n + L.PRIO_FANOUT - 1) // L.PRIO_FANOUT
    return total + 1


def check_nstep(n_step, discount):
    """Validated (n_step, discount) of a sample request: discount is None for n_step = 1 (the one-step batch needs none)."""
    if isinstance(n_step, bool) or int(n_step) != n_step or not 1 <= int(n_step) <= MAX_NSTEP:
        raise ValueError(f"n_step={n_step!r}: must be an integer in 1..{MAX_NSTEP}")
    if int(n_step) == 1:
        return 1, None
    if discount is None:
        raise ValueError(f"n_step={n_step} needs the agent's discount (sample_args {{'n_step': {n_step}, 'discount': ...}})")
    discount = float(discount)
    if not np.isfinite(discount):
        raise ValueError(f"discount={discount!r} is not finite")
    return int(n_step), discount


def refuse_nstep(batch, what: str, why: str):
    """NotImplementedError for a consumer that has no n-step meaning, when `batch` is a handle drawn with n_step > 1."""
    if isinstance(batch, BatchHandle) and batch.n_step[0] > 1:
        raise NotImplementedError(f"{what} does not take n-step batches (n_step={batch.n_step[0]}): {why}")


def check_priority_args(alpha, beta, eps):
    """ValueError when a prioritized ring's argument is out of range (alpha None: a uniform ring)."""
    def num(v):
        return isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool) and bool(np.isfinite(v))
    if alpha is not None and not (num(alpha) and alpha >= 0):
        raise ValueError(f"priority_alpha={alpha!r}: must be a finite float >= 0, or None for uniform draws")
    if not (num(beta) and 0 <= beta <= 1):
        raise ValueError(f"priority_beta={beta!r}: must be in [0, 1]")
    if not (num(eps) and eps > 0):
        raise ValueError(f"priority_eps={eps!r}: must be a finite float > 0")


def is_prioritized(batch) -> bool:
    return isinstance(batch, BatchHandle) and any(p["ring"].prioritized for p in batch.parts)


def refuse_prioritized(batch, what: str):
    """NotImplementedError for a consumer that neither weights its loss nor writes priorities back, when `batch` is a handle
    with a part drawn from a prioritized ring (its dict form, `batch.to_dict()`, carries `_weights` for a custom learner)."""
    if is_prioritized(batch):
        raise NotImplementedError(f"{what} does not take batches drawn from a prioritized ring (priority_alpha): it does not "
                                  "weight its loss or write priorities back; use batch.to_dict()['_weights'] and "
                                  "ring.update_priorities in a custom learner, or a uniform ring")


def nstep_of(part: dict):
    """(n_step, discount) recorded in a handle part; parts made without the option are one-step."""
    return part.get("n_step", 1), part.get("discount")


class BatchHandle:
    """A not-yet-materialised minibatch: (ring, seed, step, rows) parts, in concat order.  A part may carry `n_step` and
    `discount`; every part of one handle has the same pair."""

    def __init__(self, parts: List[dict], pack_obs_and_next_obs: bool = True):
        self.parts = parts
        self.pack = pack_obs_and_next_obs
        self._dict = None

    @property
    def batch_size(self) -> int:
        return sum(p["batch"] for p in self.parts)

    @property
    def n_step(self):
        """(n_step, discount) of the handle's rows."""
        return nstep_of(self.parts[0])

    def concat(self, other: "BatchHandle") -> "BatchHandle":
        if self.n_step != other.n_step:
            raise ValueError(f"concatenating batches with different n-step targets: (n_step, discount) {self.n_step} and "
                             f"{other.n_step}; draw both with the same sample_args")
        return BatchHandle(self.parts + other.parts, self.pack)

    # dict-style access materialises an un-augmented copy in the reference's layout
    def to_dict(self) -> dict:
        if self._dict is None:
            outs = [p["ring"]._gather_dict(p, self.pack) for p in self.parts]
            self._dict = outs[0] if len(outs) == 1 else _cat_dicts(outs)
        return self._dict

    def __getitem__(self, k):
        return self.to_dict()[k]

    def keys(self):
        return self.to_dict().keys()


def _cat_dicts(ds):
    out = {}
    for k, v in ds[0].items():
        out[k] = _cat_dicts([d[k] for d in ds]) if isinstance(v, dict) else torch.cat([d[k] for d in ds], dim=0)
    return out


class _CudaStager:
    """replay_io's `Stager` for HBM rings: two pinned chunks and one copy stream; events order each chunk's copy against the
    host's use of its buffer."""

    def __init__(self, stream, chunk_bytes: int):
        self.chunk_bytes = int(chunk_bytes)
        self.stream = stream
        self._pin = [L.pin(torch.empty(self.chunk_bytes, dtype=torch.uint8)) for _ in range(2)]
        self._np = [p.numpy() for p in self._pin]
        self._evt = [None, None]
        self._len = [0, 0]
        self.pinned_bytes = 2 * self.chunk_bytes

    def _copy(self, k, dst, src):
        with torch.cuda.stream(self.stream):
            dst.copy_(src, non_blocking=True)
            evt = torch.cuda.Event()
            evt.record(self.stream)
        self._evt[k] = evt

    def _sharded(self, k, copy):
        with torch.cuda.stream(self.stream):
            copy(self._pin[k].data_ptr(), self.stream.cuda_stream)
            evt = torch.cuda.Event()
            evt.record(self.stream)
        self._evt[k] = evt

    def d2h(self, k, src, lo, hi):
        if isinstance(src, ShardedFrameArray):
            self._sharded(k, lambda p, st: src.copy_out(p, lo, hi, st))
        else:
            self._copy(k, self._pin[k][:hi - lo], src[lo:hi])
        self._len[k] = hi - lo

    def wait(self, k):
        self._evt[k].synchronize()
        return memoryview(self._np[k][:self._len[k]])

    def host(self, k, n):
        if self._evt[k] is not None:          # the H2D out of this buffer two chunks ago
            self._evt[k].synchronize()
            self._evt[k] = None
        return memoryview(self._np[k][:n])

    def h2d(self, k, dst, lo, hi):
        if isinstance(dst, ShardedFrameArray):
            self._sharded(k, lambda p, st: dst.copy_in(p, lo, hi, st))
        else:
            self._copy(k, dst[lo:hi], self._pin[k][:hi - lo])

    def finish(self):
        self.stream.synchronize()


class DeviceRing:
    """Ring storage in HBM + host bookkeeping shared by both buffer flavours.

    frame_shard=(rank, world): this process stores only rank's share of the frames (frame_shards.py); every other field is
    whole.  The ring samples once the other ranks' frame allocations are mapped (data_parallel.py)."""

    STAGE = 512
    _RING_CLASS = "DeviceRing"          # the flavour a saved file records and a load checks
    _IO_EMPTY: dict = {}                # flavour-specific host bookkeeping saved in the file, with its empty-ring value

    def __init__(self, capacity: int, cams: Sequence[str], frame_shape, num_stack: int, state_dim: int, action_dim: int,
                 device=None, seed: Optional[int] = None, frame_shard: Optional[Tuple[int, int]] = None,
                 priority_alpha: Optional[float] = None, priority_beta: float = 0.4, priority_eps: float = 1e-6):
        check_priority_args(priority_alpha, priority_beta, priority_eps)
        if priority_alpha is not None and frame_shard is not None:
            raise NotImplementedError("a prioritized ring (priority_alpha) cannot shard its frames across data-parallel ranks")
        self.device = torch.device(device if device is not None else "cuda")
        L.require_cuda(self.device)
        L.load()
        self._capacity = int(capacity)
        self.cams = tuple(cams)
        self.frame_shape = tuple(frame_shape) if cams else (1, 1, 1)
        self.T, self.S, self.A = int(num_stack), int(state_dim), int(action_dim)
        dev, cap = self.device, self._capacity
        self.shards = FrameShards(cap, self.T, *frame_shard) if frame_shard is not None and self.cams else None
        rows = self.shards.local_slots if self.shards is not None else cap
        self.frames = {c: torch.zeros((rows, *self.frame_shape), dtype=torch.uint8, device=dev) for c in self.cams}
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        self.state, self.next_state = f(cap, self.T * self.S), f(cap, self.T * self.S)
        self.actions, self.rewards, self.masks = f(cap, self.A), f(cap), f(cap)
        self.dones = torch.zeros(cap, dtype=torch.uint8, device=dev)
        self.valid = torch.zeros(cap, dtype=torch.uint8, device=dev)
        self.size_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.head_dev = torch.zeros(1, dtype=torch.int32, device=dev)     # insert index, read by n-step draws (graph replays too)
        self._head_mirror = 0                                             # value last written to head_dev
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=dev)     # graph-replay draw counter
        # prioritized: the sum tree (leaves first, include/serl_b200.h), the running maximum m given to new slots, and beta,
        # all in device memory so replayed CUDA graphs read their current values
        self.prioritized = priority_alpha is not None
        if self.prioritized:
            self.priority_alpha, self.priority_eps = float(priority_alpha), float(priority_eps)
            self.tree = torch.zeros(_tree_nodes(cap), dtype=torch.float32, device=dev)
            self.max_priority_dev = torch.ones(1, dtype=torch.float32, device=dev)
            self.beta_dev = torch.full((1,), float(priority_beta), dtype=torch.float32, device=dev)
            self._beta = float(priority_beta)
        self._valid_host = np.zeros(cap, dtype=bool)
        self._size = 0
        self._insert_index = 0
        self._seed = int(seed) if seed is not None else int(np.random.SeedSequence().entropy % (1 << 63))
        self._draw_step = 0
        self._dev_step_mirror = 0                                         # host mirror of step_dev (graph replays)
        self._lock = threading.RLock()
        # Pinned staging, one interleaved record per staged slot write, behind a small header holding the validity changes:
        #   [touched slots int32 x 4n | touched values u8 x 4n | record 0 | record 1 | ...]
        # so a flush is ONE host->device copy of the used prefix, one scatter launch and one commit launch.  Two host
        # buffers alternate: the copy out of one overlaps the inserts into the other (no host sync per flush).
        n = self.STAGE
        fb = int(np.prod(self.frame_shape)) if self.cams else 0
        ns = self.T * self.S
        off, fields = 0, {}
        for c in self.cams:
            fields[("frames", c)] = (off, np.uint8, self.frame_shape); off += (fb + 15) // 16 * 16
        for name, cnt in (("state", ns), ("next_state", ns), ("actions", self.A), ("rewards", 1), ("masks", 1)):
            fields[name] = (off, np.float32, (cnt,)); off += 4 * cnt
        for name in ("dst", "src"):
            fields[name] = (off, np.int32, (1,)); off += 4
        for name in ("dones", "valid"):
            fields[name] = (off, np.uint8, (1,)); off += 1
        self._row_bytes = (off + 15) // 16 * 16
        self._hdr_bytes = (4 * n * 4 + 4 * n + 15) // 16 * 16
        self._fields = fields
        total = self._hdr_bytes + n * self._row_bytes
        self._stage_host = [L.pin(torch.zeros(total, dtype=torch.uint8)) for _ in range(2)]
        self._stage_dev = torch.empty(total, dtype=torch.uint8, device=dev)
        self._stage_evt = [None, None]                                   # copy-out completion of each host buffer
        self._cur = 0
        self._stn = [self._stage_views(b.numpy()) for b in self._stage_host]
        self._n_pending = 0
        self._pending_dst = set()
        self._touched = set()
        self._sample_evt = None
        self.h2d_bytes = 0
        self._io_stream = None
        self.io_pinned_bytes = 0                                          # pinned staging held by the last save / load

    def _stage_views(self, base: np.ndarray) -> dict:
        """Strided numpy views of one staging buffer: field -> (STAGE, ...) array whose row k lives in record k."""
        n, rb, hb = self.STAGE, self._row_bytes, self._hdr_bytes
        out = {"touched": base[:4 * n * 4].view(np.int32), "touched_val": base[4 * n * 4:4 * n * 4 + 4 * n], "frames": {}}
        for key, (off, dt, shape) in self._fields.items():
            item = np.dtype(dt).itemsize
            inner = tuple(int(np.prod(shape[i + 1:])) * item for i in range(len(shape)))
            v = np.ndarray((n, *shape), dtype=dt, buffer=base, offset=hb + off, strides=(rb, *inner))
            if isinstance(key, tuple):
                out["frames"][key[1]] = v
            else:
                out[key] = v[:, 0] if shape == (1,) else v
        return out

    # ---- reference API ---------------------------------------------------------------------------
    def __len__(self) -> int:
        return self._size

    def seed(self, seed: Optional[int] = None):
        if seed is not None:
            self._seed = int(seed)
        return [self._seed]

    # ---- staging ---------------------------------------------------------------------------------
    def _stage_write(self, dst: int, *, src_slot: int = -1, frames=None, state=None, next_state=None, action=None,
                     reward=0.0, mask=0.0, done=False, valid=False):
        """Queue one slot write (replay_buffer.py:71-75 semantics for the slot at `dst`)."""
        if (self._n_pending == self.STAGE or dst in self._pending_dst or (src_slot >= 0 and src_slot in self._pending_dst)
                or len(self._touched) > 3 * self.STAGE):
            self.flush()
        k = self._n_pending
        if k == 0 and self._stage_evt[self._cur] is not None:   # this buffer's previous copy-out (two flushes ago) must be over
            self._stage_evt[self._cur].synchronize()
            self._stage_evt[self._cur] = None
        st = self._stn[self._cur]
        st["dst"][k], st["src"][k] = dst, src_slot
        if src_slot < 0:
            for c in self.cams:
                st["frames"][c][k] = frames[c]
            st["state"][k] = np.asarray(state, np.float32).reshape(-1)
            st["next_state"][k] = np.asarray(next_state, np.float32).reshape(-1)
            st["actions"][k] = np.asarray(action, np.float32).reshape(-1)
            st["rewards"][k], st["masks"][k], st["dones"][k] = float(reward), float(mask), int(bool(done))
        st["valid"][k] = int(valid)
        self._valid_host[dst] = valid
        self._pending_dst.add(dst)
        self._touched.add(dst)
        self._n_pending = k + 1

    def _advance(self):
        self._insert_index = (self._insert_index + 1) % self._capacity
        self._size = min(self._size + 1, self._capacity)

    def _mark(self, slot: int, valid: bool):
        self._valid_host[slot] = valid
        self._touched.add(slot)

    def view(self) -> L.ReplayView:
        v = L.ReplayView()
        for j, c in enumerate(self.cams):
            v.frames[j] = self.frames[c].data_ptr()
        v.state, v.next_state, v.actions = self.state.data_ptr(), self.next_state.data_ptr(), self.actions.data_ptr()
        v.rewards, v.masks, v.dones, v.valid = (self.rewards.data_ptr(), self.masks.data_ptr(), self.dones.data_ptr(),
                                                self.valid.data_ptr())
        v.num_cams = len(self.cams)
        v.height, v.width, v.channels = self.frame_shape
        v.num_stack, v.state_dim, v.action_dim = self.T, self.S, self.A
        v.capacity, v.size = self._capacity, self._size
        return v

    # ---- prioritized replay -------------------------------------------------------------------------------------------
    @property
    def priority_beta(self) -> float:
        """Importance-weight exponent of batches materialised from now on (settable: anneal it towards 1)."""
        self._require_prioritized("priority_beta")
        return self._beta

    @priority_beta.setter
    def priority_beta(self, beta: float):
        self._require_prioritized("priority_beta")
        check_priority_args(None, beta, self.priority_eps)
        self._beta = float(beta)
        self.beta_dev.fill_(self._beta)

    def _require_prioritized(self, what: str):
        if not self.prioritized:
            raise ValueError(f"{what}: this ring draws uniformly; build it with priority_alpha to prioritize it")

    def priority_tree(self) -> L.PriorityTree:
        return ops.priority_tree(self.tree, self.max_priority_dev, self._capacity, self.valid)

    def update_priorities(self, indices, td_errors):
        """Sets the priority of slots `indices` to (|td_errors| + priority_eps) ^ priority_alpha on the current stream, and
        raises the running maximum given to new slots to the largest value written.  A slot named twice takes its last
        entry.  Device or host arrays of equal length; host indices outside [0, capacity) raise, device ones are skipped
        (checking them would wait for the device)."""
        self._require_prioritized("update_priorities")
        if not torch.is_tensor(indices):
            indices = np.asarray(indices).reshape(-1)
            if indices.size and (indices.min() < 0 or indices.max() >= self._capacity):
                raise ValueError(f"update_priorities: indices outside [0, {self._capacity})")
        idx = torch.as_tensor(indices).to(self.device, torch.int32).reshape(-1).contiguous()
        td = torch.as_tensor(np.asarray(td_errors) if not torch.is_tensor(td_errors) else td_errors)
        td = td.to(self.device, torch.float32).reshape(-1).contiguous()
        if idx.shape != td.shape:
            raise ValueError(f"update_priorities: {idx.numel()} indices, {td.numel()} TD errors")
        with self._lock:
            t = self.priority_tree()
            for lo in range(0, idx.numel(), L.PRIO_SET_MAX):       # in order: a later piece overrides an earlier one
                n = min(L.PRIO_SET_MAX, idx.numel() - lo)
                ops.priority_set(t, idx[lo:], n, td=td[lo:], alpha=self.priority_alpha, eps=self.priority_eps)

    def shard_table(self) -> L.ReplayShards:
        """The sharded kernels' descriptor (serl_replay_shards) of a frame-sharded ring."""
        return self.shards.table([self.frames[c].data_ptr() for c in self.cams])

    def flush(self):
        """Apply staged slot writes + validity changes on the current stream."""
        with self._lock:
            n = self._n_pending
            stream_ptr = L.stream_ptr()
            if self._sample_evt is not None:
                self._sample_evt.make_current_stream_wait()   # never overwrite slots a sampling kernel still reads
            if n or self._touched:
                cur = self._cur
                if self._stage_evt[cur] is not None:          # only reachable when a flush carries validity changes alone
                    self._stage_evt[cur].synchronize()
                    self._stage_evt[cur] = None
                st, host, dv = self._stn[cur], self._stage_host[cur], self._stage_dev
                m = len(self._touched)
                if m:
                    slots = np.fromiter(self._touched, dtype=np.int32, count=m)
                    st["touched"][:m] = slots
                    st["touched_val"][:m] = self._valid_host[slots]
                nbytes = self._hdr_bytes + n * self._row_bytes
                dv[:nbytes].copy_(host[:nbytes], non_blocking=True)       # the ONE host->device copy of this flush
                self.h2d_bytes += nbytes
                base = dv.data_ptr() + self._hdr_bytes
                if n:
                    rq = L.ScatterRequest()
                    rq.n, rq.row_stride = n, self._row_bytes
                    f = self._fields
                    rq.dst_slot, rq.src_slot = base + f["dst"][0], base + f["src"][0]
                    for j, c in enumerate(self.cams):
                        rq.frames[j] = base + f[("frames", c)][0]
                    rq.state, rq.next_state, rq.actions = base + f["state"][0], base + f["next_state"][0], base + f["actions"][0]
                    rq.rewards, rq.masks, rq.dones, rq.valid = (base + f["rewards"][0], base + f["masks"][0], base + f["dones"][0],
                                                                base + f["valid"][0])
                    v = self.view()
                    if self.shards is not None:
                        L.call("serl_replay_scatter_sharded", C.byref(v), C.byref(self.shard_table()), C.byref(rq), stream_ptr)
                    else:
                        L.call("serl_replay_scatter", C.byref(v), C.byref(rq), stream_ptr)
                # validity changes (applied after the slot writes, like the host ring logic orders them) + the new size
                L.call("serl_replay_commit", self.valid.data_ptr(), dv.data_ptr(), dv.data_ptr() + 4 * self.STAGE * 4, m,
                       self.size_dev.data_ptr(), self._size, stream_ptr)
                if self.prioritized and m:                     # touched slots: m when valid, 0 when not
                    L.call("serl_replay_priority_set", C.byref(self.priority_tree()), dv.data_ptr(), None,
                           dv.data_ptr() + 4 * self.STAGE * 4, m, 0.0, 0.0, stream_ptr)
                evt = L.new_event()
                evt.record()
                self._stage_evt[cur] = evt
                self._cur = cur ^ 1
            if self._head_mirror != self._insert_index:
                self.head_dev.fill_(self._insert_index)
                self._head_mirror = self._insert_index
            self._n_pending = 0
            self._pending_dst.clear()
            self._touched.clear()

    # ---- persistence (replay_io.py: one .npz per ring) ----------------------------------------------------------------
    def _io_layout(self) -> dict:
        return {"version": RIO.FORMAT_VERSION, "class": self._RING_CLASS, "capacity": self._capacity, "cams": self.cams,
                "frame_shape": self.frame_shape, "T": self.T, "S": self.S, "A": self.A}

    def _io_arrays(self) -> List[tuple]:
        named = [(f"frames/{c}", self.frames[c]) for c in self.cams]
        named += [(k, getattr(self, k)) for k in ("state", "next_state", "actions", "rewards", "masks", "dones", "valid")]
        return named + ([("priorities", self.tree[:self._capacity])] if self.prioritized else [])   # the leaves; load rebuilds the rest

    _IO_PRIORITY = ("priority_alpha", "priority_beta", "priority_eps", "max_priority")

    def _io_check_priorities(self, path, meta: dict):
        """ValueError naming the field where a prioritized file meets a uniform ring, or the priority rule differs."""
        if ("priority_alpha" in meta) != self.prioritized:
            raise ValueError(f"replay file does not fit this buffer: priority_alpha is {meta.get('priority_alpha')!r} in the file, "
                             f"{self.priority_alpha if self.prioritized else None!r} here")
        if self.prioritized:
            missing = [k for k in self._IO_PRIORITY if k not in meta]
            if missing:
                raise ValueError(f"replay file {path!r}: meta lacks {missing}")
            for k in ("priority_alpha", "priority_eps"):
                if float(meta[k]) != getattr(self, k):
                    raise ValueError(f"replay file does not fit this buffer: {k} is {meta[k]!r} in the file, {getattr(self, k)!r} here")

    def _io_fields(self, n: int) -> List[RIO.Field]:
        """The file's arrays over slots [0, n); each field's `src` is the flat byte view of those rows in HBM (a frame-sharded
        ring's frames: a ShardedFrameArray, which reads each slot from its owner and writes only the slots this rank stores)."""
        dt = {torch.uint8: np.uint8, torch.float32: np.float32}
        fb = int(np.prod(self.frame_shape))
        return [RIO.Field(name, dt[t.dtype], (n, *t.shape[1:]),
                          ShardedFrameArray(self.shards, self.cams.index(name[7:]), t.data_ptr(), fb)
                          if self.shards is not None and name.startswith("frames/") else t[:n].reshape(-1).view(torch.uint8))
                for name, t in self._io_arrays()]

    def _io_copy_stream(self):
        """The copy stream, made to wait for every scatter / sampler launch already enqueued on the ring."""
        if self._io_stream is None:
            self._io_stream = torch.cuda.Stream(self.device)
        cs = self._io_stream
        cs.wait_stream(torch.cuda.current_stream(self.device))
        for evt in (*self._stage_evt, self._sample_evt):
            if evt is not None:
                cs.wait_event(evt.e)
        return cs

    def save(self, path, chunk_bytes: Optional[int] = None, extra_meta: Optional[dict] = None) -> int:
        """Writes the ring to `path` (replay_io.py format), atomically: a failed save leaves an existing file as it was.
        Staged inserts are applied first, and the ring's lock is held throughout, so the file is one point in time and an
        `insert` from another thread lands after it.  Host memory: two pinned chunks of `chunk_bytes` (default
        replay_io.CHUNK_BYTES).  `extra_meta` (JSON-serialisable) is stored in the file's meta next to the ring's own
        entries; `load` ignores it.  Returns the file's size in bytes."""
        with self._lock:
            self.flush()
            cs = self._io_copy_stream()
            with torch.cuda.stream(cs):
                step_dev = int(self.step_dev.item())
                prio = ({"priority_alpha": self.priority_alpha, "priority_beta": self._beta, "priority_eps": self.priority_eps,
                         "max_priority": float(self.max_priority_dev.item())} if self.prioritized else {})
            meta = {**self._io_layout(), "_size": self._size, "_insert_index": self._insert_index, "_seed": self._seed,
                    "_draw_step": self._draw_step, "_dev_step_mirror": self._dev_step_mirror, "step_dev": step_dev,
                    **{k: getattr(self, k) for k in self._IO_EMPTY}, **prio, **(extra_meta or {})}
            stager = _CudaStager(cs, chunk_bytes or RIO.CHUNK_BYTES)
            self.io_pinned_bytes = stager.pinned_bytes
            return RIO.write_ring_file(path, meta, self._io_fields(self._size), stager)

    def _io_clear(self, cs):
        """Empty ring: nothing valid, size 0, host bookkeeping of a fresh ring (seed and draw counter are kept)."""
        with torch.cuda.stream(cs):
            self.valid.zero_()
            self.size_dev.zero_()
            self.head_dev.zero_()
            if self.prioritized:                        # no valid slot: every node 0, m back to 1
                self.tree.zero_()
                self.max_priority_dev.fill_(1.0)
        cs.synchronize()
        self._head_mirror = 0
        self._valid_host[:] = False
        self._size = self._insert_index = 0
        for k, v in self._IO_EMPTY.items():
            setattr(self, k, v)

    def load(self, path, chunk_bytes: Optional[int] = None):
        """Restores a file written by `save` into this ring, which must have the same class, capacity, cameras and shapes
        (ValueError naming the field otherwise, and on a damaged or truncated file).  Afterwards inserts and draws continue
        exactly as they would have in the saved ring.  On any error the ring is left empty.  Returns self."""
        with self._lock:
            self.flush()
            cs = self._io_copy_stream()
            try:
                meta = RIO.read_meta(path)
                RIO.check_meta(meta, self._io_layout())
                self._io_check_priorities(path, meta)
                missing = [k for k in ("_size", "_insert_index", "_seed", "_draw_step", "_dev_step_mirror", "step_dev",
                                       *self._IO_EMPTY) if k not in meta]
                if missing:
                    raise ValueError(f"replay file {path!r}: meta lacks {missing}")
                n, cap = int(meta["_size"]), self._capacity
                if not (0 <= n <= cap and 0 <= int(meta["_insert_index"]) < cap):
                    raise ValueError(f"replay file {path!r}: _size {n} / _insert_index {meta['_insert_index']} outside capacity {cap}")
                self._io_clear(cs)
                if self.shards is not None:
                    with torch.cuda.stream(cs):
                        for t in self.frames.values():
                            t.zero_()
                stager = _CudaStager(cs, chunk_bytes or RIO.CHUNK_BYTES)
                self.io_pinned_bytes = stager.pinned_bytes
                RIO.read_ring_file(path, self._io_fields(n), stager)
                with torch.cuda.stream(cs):
                    for name, t in self._io_arrays():        # slots past the file's rows hold zeros, as in a ring that never used them
                        if self.shards is None or not name.startswith("frames/"):   # sharded frames: zeroed before the read
                            t[n:].zero_()
                    self.size_dev.fill_(n)
                    self.head_dev.fill_(int(meta["_insert_index"]))
                    self.step_dev.fill_(int(meta["step_dev"]))
                    if self.prioritized:
                        ops.priority_rebuild(self.priority_tree())
                        self.max_priority_dev.fill_(float(meta["max_priority"]))
                        self.beta_dev.fill_(float(meta["priority_beta"]))
                    valid = self.valid.cpu()
                self._valid_host[:] = valid.numpy().astype(bool)
                self._size, self._insert_index = n, int(meta["_insert_index"])
                self._head_mirror = self._insert_index
                self._seed, self._draw_step = int(meta["_seed"]), int(meta["_draw_step"])
                self._dev_step_mirror = int(meta["_dev_step_mirror"])
                for k in self._IO_EMPTY:
                    setattr(self, k, meta[k])
                if self.prioritized:
                    self._beta = float(meta["priority_beta"])
                self._sample_evt = None
            except BaseException:
                self._io_clear(cs)
                raise
        return self

    # ---- insert / sample (state-only flavour; the frame-dedup flavour overrides insert) -----------------
    def insert(self, data_dict: dict):
        """replay_buffer.py:71-75."""
        with self._lock:
            self._stage_write(self._insert_index, frames={}, state=data_dict["observations"], next_state=data_dict["next_observations"],
                              action=data_dict["actions"], reward=data_dict["rewards"], mask=data_dict["masks"], done=data_dict["dones"],
                              valid=True)
            self._advance()

    def sample(self, batch_size: int, keys: Optional[Iterable[str]] = None, indx=None, pack_obs_and_next_obs: bool = False,
               n_step: int = 1, discount: Optional[float] = None) -> BatchHandle:
        """n_step > 1 (up to MAX_NSTEP, with the agent's `discount`): each row carries the n-step window that starts at its slot
        (see include/serl_b200.h, serl_replay_sample_crop_nstep).  Index draws and crops are those of n_step = 1."""
        n_step, discount = check_nstep(n_step, discount)
        with self._lock:
            self.flush()
            if self._size <= (self.T if self.cams else 0):
                raise L.SerlError(f"replay buffer holds {self._size} slots; cannot sample")
            part = dict(ring=self, seed=self._seed, step=self._draw_step, batch=int(batch_size),
                        indx=None if indx is None else torch.as_tensor(np.asarray(indx), dtype=torch.int32, device=self.device),
                        n_step=n_step, discount=discount)
            self._draw_step += 1
            return BatchHandle([part], pack_obs_and_next_obs)

    def get_iterator(self, queue_size: int = 2, sample_args: dict = {}, device=None):
        """replay_buffer.py:77-90.  No prefetch queue is needed: handles are lazy and the data never leaves HBM."""
        while True:
            yield self.sample(**sample_args)

    # ---- kernel launch used by the agents ---------------------------------------------------------
    def arm_draw_counter(self, step: int, draws: int) -> None:
        """Points the device draw counter (`step_dev`) at `step` before a captured step graph that makes `draws` draws from this
        ring is captured or replayed; the graph's own counter increments leave it at step + draws."""
        if self._dev_step_mirror != step:
            self.step_dev.fill_(step)
        self._dev_step_mirror = step + draws

    def launch_sample(self, part: dict, out: L.BatchOut, *, crop_total: int, out_row_offset: int, key_obs=None, key_next=None,
                      explicit_off=None, padding: int = 4, step_dev=None, record_event: bool = True, nstep_out=None,
                      prio_out=None):
        """One sampler launch for `part`: serl_replay_sample_crop, or serl_replay_sample_crop_nstep when the part has
        n_step > 1, or serl_replay_sample_crop_prio on a prioritized ring.  nstep_out: optional (m, next slot) int32 device
        tensors of the launch's output rows.  prio_out: (B_total) float32 device tensor receiving each row's priority; a
        prioritized ring requires it (its rows are only usable with their importance weights)."""
        if self.prioritized and prio_out is None:
            raise NotImplementedError("this consumer does not take batches drawn from a prioritized ring (priority_alpha): it does "
                                      "not weight its loss or write priorities back")
        with self._lock:
            rq = L.SampleRequest()
            rq.seed, rq.step, rq.lane_offset, rq.batch = part["seed"], part["step"], 0, part["batch"]
            rq.step_dev = None if step_dev is None else step_dev.data_ptr()
            rq.size_dev = self.size_dev.data_ptr()
            rq.explicit_idx = None if part.get("indx") is None else part["indx"].data_ptr()
            rq.key_obs, rq.key_next = key_obs, key_next
            if explicit_off is not None:
                rq.explicit_off_obs, rq.explicit_off_next = explicit_off[0].data_ptr(), explicit_off[1].data_ptr()
            rq.crop_total, rq.out_row_offset, rq.padding = crop_total, out_row_offset, padding
            v = self.view()
            n_step, discount = nstep_of(part)
            sh = () if self.shards is None else (C.byref(self.shard_table()),)
            sfx = "" if self.shards is None else "_sharded"
            if self.prioritized:
                ns = None
                if n_step > 1:
                    ns = L.NStepDesc()
                    ns.n, ns.discount, ns.head_dev = n_step, discount, self.head_dev.data_ptr()
                    if nstep_out is not None:
                        ns.m_out, ns.next_idx_out = nstep_out[0].data_ptr(), nstep_out[1].data_ptr()
                L.call("serl_replay_sample_crop_prio", C.byref(v), C.byref(rq), C.byref(self.priority_tree()),
                       None if ns is None else C.byref(ns), C.byref(out), prio_out.data_ptr(), L.stream_ptr())
            elif n_step > 1:
                ns = L.NStepDesc()
                ns.n, ns.discount, ns.head_dev = n_step, discount, self.head_dev.data_ptr()
                if nstep_out is not None:
                    ns.m_out, ns.next_idx_out = nstep_out[0].data_ptr(), nstep_out[1].data_ptr()
                L.call("serl_replay_sample_crop_nstep" + sfx, C.byref(v), *sh, C.byref(rq), C.byref(ns), C.byref(out), L.stream_ptr())
            else:
                L.call("serl_replay_sample_crop" + sfx, C.byref(v), *sh, C.byref(rq), C.byref(out), L.stream_ptr())
            if record_event:
                evt = L.new_event()
                evt.record()
                self._sample_evt = evt

    def _gather_dict(self, part: dict, pack: bool) -> dict:
        """Un-augmented materialisation in the reference's batch layout (memory_efficient_replay_buffer.py:126-164).  An n-step
        part returns its n-step rewards, masks, dones and next observations, plus `_n_step_lengths` (m of each row) and
        `_next_indices` (the slot whose next observation the row holds); its frames stay packed only for one-frame
        observations (a stack of T > 1 next frames is not the obs stack shifted by one)."""
        B, dev, T = part["batch"], self.device, self.T
        nstep = nstep_of(part)[0] > 1
        pack = pack and (not nstep or T == 1)
        e = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=dev)
        obs_pix = {c: e(B, T, *self.frame_shape, dt=torch.uint8) for c in self.cams}
        next_pix = {c: e(B, T, *self.frame_shape, dt=torch.uint8) for c in self.cams}
        out = L.BatchOut()
        for j, c in enumerate(self.cams):
            out.obs_pix[j], out.next_pix[j] = obs_pix[c].data_ptr(), next_pix[c].data_ptr()
        st, nst, ac, rw, mk = e(B, T * self.S), e(B, T * self.S), e(B, self.A), e(B), e(B)
        dn = e(B, dt=torch.uint8)
        idx = e(B, dt=torch.int32)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        out.obs_state, out.next_state, out.actions, out.rewards, out.masks = (st.data_ptr(), nst.data_ptr(), ac.data_ptr(),
                                                                              rw.data_ptr(), mk.data_ptr())
        out.dones, out.idx, out.status = dn.data_ptr(), idx.data_ptr(), status.data_ptr()
        ident = torch.full((B * T, 2), 4, dtype=torch.int32, device=dev)          # centre offset = identity shift
        nstep_out = (e(B, dt=torch.int32), e(B, dt=torch.int32)) if nstep else None
        prio = e(B) if self.prioritized else None
        self.launch_sample(part, out, crop_total=B * T, out_row_offset=0, explicit_off=(ident, ident), nstep_out=nstep_out,
                           prio_out=prio)
        if self.prioritized:
            weights = e(B)
            ops.priority_weights(prio, B, self.beta_dev, weights)
        if int(status.item()):
            raise L.SerlError("replay draw failed: no valid slot within the redraw budget")
        state_shape = (B, T, self.S) if self.cams else (B, self.S)
        obs = ({"state": st.view(state_shape)} if self.S else {}) if self.cams else st.view(state_shape)       # pixel ring without
        nobs = ({"state": nst.view(state_shape)} if self.S else {}) if self.cams else nst.view(state_shape)   # a state vector: no "state"
        for c in self.cams:
            if pack:                                    # frames [idx-T .. idx]: obs frames then the newest next frame
                obs[c] = torch.cat([obs_pix[c], next_pix[c][:, -1:]], dim=1)
            else:
                obs[c], nobs[c] = obs_pix[c], next_pix[c]
        res = {"observations": obs, "next_observations": nobs, "actions": ac, "rewards": rw, "masks": mk,
               "dones": dn.bool(), "_indices": idx}
        if nstep:
            res["_n_step_lengths"], res["_next_indices"] = nstep_out
        if self.prioritized:                          # importance weights over this part's rows (oracle/per.py::weights)
            res["_weights"] = weights
        return res


class ReplayBuffer(DeviceRing):
    """State-observation ring (reference data/replay_buffer.py:40-75), storage in HBM."""

    _RING_CLASS = "ReplayBuffer"

    def __init__(self, observation_space, action_space, capacity: int, next_observation_space=None, device=None, seed=None,
                 priority_alpha: Optional[float] = None, priority_beta: float = 0.4, priority_eps: float = 1e-6):
        if _is_dict_space(observation_space):
            raise TypeError("ReplayBuffer holds flat observations; use MemoryEfficientReplayBuffer for pixel dicts")
        S = int(np.prod(_space_shape(observation_space)))
        A = int(np.prod(_space_shape(action_space)))
        super().__init__(capacity, (), (1, 1, 1), 1, S, A, device=device, seed=seed, priority_alpha=priority_alpha,
                         priority_beta=priority_beta, priority_eps=priority_eps)
