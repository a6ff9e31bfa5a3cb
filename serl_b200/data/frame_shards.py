"""Frame sharding of a replay ring over the ranks of a data-parallel learner (include/serl_b200.h, serl_replay_shards).

Rank r of N owns the slots [lo_r, hi_r), lo_r = r * ceil(C / N), and also stores the T slots in front of lo_r,
(lo_r - T .. lo_r - 1) mod C: its halo.  Its frame allocation holds ceil(C / N) + T slots, local index (s - lo_r + T) mod C
for slot s.  A sampled row reads the T + 1 frames w0 .. w0 + T of its window from the owner of w0 + T, where the halo makes
them contiguous.  Rank 0's halo wraps to slots C - T .. C - 1: the sampler never reads it (a window never ends below slot T),
but the frame-dedup ring's wrap-around re-insert copies exactly those slots to the front, so rank 0 finds the source frames
of that copy in its own allocation.

Everything here is host-side bookkeeping; the frames themselves move through the sharded scatter and sampler kernels, and
peers' allocations are mapped with CUDA IPC by data_parallel.py.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterator, List, Optional, Tuple

from .. import _lib as L


class FrameShards:
    """Rank `rank` of `world`'s share of a ring of `capacity` slots with frame stack `T`.  ValueError for a layout the kernels
    cannot follow: a rank without slots, or (world > 1) a rank range shorter than 2T, which would put a rank other than 0 in
    the way of the wrap-around re-insert at the front."""

    def __init__(self, capacity: int, T: int, rank: int, world: int):
        self.capacity, self.T, self.rank, self.world = int(capacity), int(T), int(rank), int(world)
        if not 1 <= self.world <= L.MAX_SHARD_RANKS or not 0 <= self.rank < self.world:
            raise ValueError(f"frame sharding: rank {rank} of {world} (1 to {L.MAX_SHARD_RANKS} ranks)")
        self.slots_per_rank = -(-self.capacity // self.world)
        if (self.world - 1) * self.slots_per_rank >= self.capacity:
            raise ValueError(f"frame sharding: capacity {capacity} leaves a rank of {world} without slots "
                             f"({self.slots_per_rank} slots per rank)")
        if self.world > 1 and self.slots_per_rank < 2 * self.T:
            raise ValueError(f"frame sharding: {self.slots_per_rank} slots per rank is less than twice the frame stack {self.T}")
        self.halo = self.T
        self.local_slots = self.slots_per_rank + self.halo        # rows of each rank's frame allocation
        self.peer_frames: Optional[dict] = None                    # cam index -> [frame pointer of rank r for r < world]

    def range(self, rank: Optional[int] = None) -> Tuple[int, int]:
        """[lo, hi) of the slots `rank` (default: this rank) owns."""
        r = self.rank if rank is None else rank
        lo = r * self.slots_per_rank
        return lo, min(self.capacity, lo + self.slots_per_rank)

    def owner(self, slot: int) -> int:
        return slot // self.slots_per_rank

    def locals(self, slot: int, rank: Optional[int] = None) -> List[int]:
        """Local indices at which `rank` stores `slot`: its range copy and its halo copy, either or both (both at world 1, where
        rank 0's halo wraps into its own range).  The sharded scatter writes a slot's frame at exactly these."""
        lo, hi = self.range(rank)
        out = []
        if lo <= slot < hi:
            out.append(slot - lo + self.halo)
        d = (lo - slot) % self.capacity
        if 1 <= d <= self.halo:
            out.append(self.halo - d)
        return out

    def window_source(self, w0: int) -> Tuple[int, int]:
        """(rank, local index of slot w0) the sampler reads the window w0 .. w0 + T from."""
        o = self.owner(w0 + self.T)
        return o, w0 - o * self.slots_per_rank + self.halo

    def runs(self, s0: int, s1: int, rank: Optional[int] = None) -> Iterator[Tuple[int, int, int]]:
        """(first slot, local index, count) runs of the slots in [s0, s1) that `rank` stores, each contiguous in both."""
        run = None
        for s in range(s0, s1):
            for l in self.locals(s, rank):
                if run is not None and s == run[0] + run[2] and l == run[1] + run[2]:
                    run[2] += 1
                    continue
                if run is not None:
                    yield tuple(run)
                run = [s, l, 1]
        if run is not None:
            yield tuple(run)

    def table(self, local_frames: List[int]) -> L.ReplayShards:
        """The kernels' shard table; `local_frames` are this rank's frame pointers, one per camera.  Until the peers' allocations
        are mapped (world > 1), the other ranks' entries are null and the library refuses the table."""
        t = L.ReplayShards()
        t.slots_per_rank, t.halo, t.world, t.rank = self.slots_per_rank, self.halo, self.world, self.rank
        for c, p in enumerate(local_frames):
            ptrs = self.peer_frames[c] if self.peer_frames is not None else [None] * self.world
            for r in range(self.world):
                t.frames[c][r] = p if r == self.rank else ptrs[r]
        return t


class ShardedFrameArray:
    """Field source of one camera's frames in a ring file (replay_io.Field.src), for the ring's CUDA stager: bytes [lo, hi)
    of the (n, H, W, C) array over slots [0, n) are gathered from their owners' allocations (save), or scattered into the
    copies this rank stores (load)."""

    def __init__(self, shards: FrameShards, cam: int, local_ptr: int, frame_bytes: int):
        self.shards, self.cam, self.local_ptr, self.fb = shards, cam, int(local_ptr), int(frame_bytes)

    def _pieces(self, lo: int, hi: int, runs) -> Iterator[Tuple[int, int, int]]:
        """(byte offset into [lo, hi), byte offset into the allocation, bytes) for each stored run overlapping [lo, hi)."""
        fb = self.fb
        for s, l, n in runs(lo // fb, -(-hi // fb)):
            a, b = max(lo, s * fb), min(hi, (s + n) * fb)
            if a < b:
                yield a - lo, l * fb + (a - s * fb), b - a

    def copy_out(self, dst: int, lo: int, hi: int, stream: int):
        """Device-to-host (pinned `dst`) copy of bytes [lo, hi), each slot read from its owner."""
        sh, fb = self.shards, self.fb
        s, end = lo // fb, -(-hi // fb)
        while s < end:                                      # one copy per owner
            o = sh.owner(s)
            lo_o, hi_o = sh.range(o)
            e = min(end, hi_o)
            base = self.local_ptr if o == sh.rank else sh.peer_frames[self.cam][o]
            a, b = max(lo, s * fb), min(hi, e * fb)
            L.call("serl_copy_async", C.c_void_p(dst + a - lo), C.c_void_p(base + (s - lo_o + sh.halo) * fb + a - s * fb),
                   b - a, C.c_void_p(stream))
            s = e

    def copy_in(self, src: int, lo: int, hi: int, stream: int):
        """Host (pinned `src`) to device copy of bytes [lo, hi) into every local copy of their slots on this rank."""
        for off, dev, n in self._pieces(lo, hi, self.shards.runs):
            L.call("serl_copy_async", C.c_void_p(self.local_ptr + dev), C.c_void_p(src + off), n, C.c_void_p(stream))
