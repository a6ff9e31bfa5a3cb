"""Frame-deduplicating replay ring in HBM.

Mirrors `MemoryEfficientReplayBuffer` (reference data/memory_efficient_replay_buffer.py:12-164):
one camera frame per slot, episode-start filler slots, `_is_correct_index` validity, wrap-around
re-insert, and `sample(..., pack_obs_and_next_obs=True)`.  The host keeps only the ring bookkeeping
(cursor, size, episode flag, validity bits); frames and fields are staged through pinned memory into
HBM (serl_replay_scatter).  Layout semantics are pinned against the real reference class by
tests/golden/replay_*.npz (via oracle/replay.py) and tests/test_replay_device.py.
"""
from __future__ import annotations

from typing import Iterable, Optional, Tuple

import numpy as np

from .replay_buffer import BatchHandle, DeviceRing, _space_shape, check_priority_args


class MemoryEfficientReplayBuffer(DeviceRing):
    _RING_CLASS = "MemoryEfficientReplayBuffer"
    _IO_EMPTY = {"_first": True}                       # mid-episode flag: saved, restored, and reset by a failed load

    def __init__(self, observation_space, action_space, capacity: int, pixel_keys: Tuple[str, ...] = ("pixels",),
                 device=None, seed=None, frame_shard=None, priority_alpha: Optional[float] = None, priority_beta: float = 0.4,
                 priority_eps: float = 1e-6):
        check_priority_args(priority_alpha, priority_beta, priority_eps)
        self.pixel_keys = tuple(pixel_keys)
        spaces = observation_space.spaces
        stacks = {int(_space_shape(spaces[k])[0]) for k in self.pixel_keys}
        assert len(stacks) == 1, "all pixel keys must share the frame-stack length"          # (:25-28)
        self._num_stack = stacks.pop()
        frame_shape = _space_shape(spaces[self.pixel_keys[0]])[1:]
        other = [k for k in spaces if k not in self.pixel_keys]
        if other not in (["state"], []):
            raise NotImplementedError(f"non-pixel observation keys must be exactly ['state'] or none, got {other}")
        if other:
            st_shape = _space_shape(spaces["state"])
            S = int(np.prod(st_shape[1:])) if len(st_shape) > 1 else int(st_shape[0])
        else:                       # camera images only: zero-width state records, and batches without a "state" entry
            S = 0
        A = int(np.prod(_space_shape(action_space)))
        super().__init__(capacity, self.pixel_keys, frame_shape, self._num_stack, S, A, device=device, seed=seed,
                         frame_shard=frame_shard, priority_alpha=priority_alpha, priority_beta=priority_beta, priority_eps=priority_eps)
        self._first = True

    def insert(self, data_dict: dict):
        T = self._num_stack
        with self._lock:
            # (:54-59) wrapping a full buffer mid-episode: re-insert the last T slots at the front as invalid copies
            if self._insert_index == 0 and self._capacity == self._size and not self._first:
                for src in range(self._size - T, self._size):
                    self._stage_write(self._insert_index, src_slot=src, valid=False)
                    self._advance()
            obs, nobs = data_dict["observations"], data_dict["next_observations"]
            no_state = np.zeros(0, np.float32)
            common = dict(state=obs["state"] if self.S else no_state, next_state=nobs["state"] if self.S else no_state,
                          action=data_dict["actions"],
                          reward=data_dict["rewards"], mask=data_dict["masks"], done=data_dict["dones"])
            if self._first:                                                                  # (:71-77)
                for i in range(T):
                    self._stage_write(self._insert_index, frames={k: np.asarray(obs[k])[i] for k in self.pixel_keys},
                                      valid=False, **common)
                    self._advance()
            self._first = bool(data_dict["dones"])                                           # (:82)
            self._stage_write(self._insert_index, frames={k: np.asarray(nobs[k])[-1] for k in self.pixel_keys},
                              valid=True, **common)                                          # (:79-85)
            self._advance()
            for i in range(T):                                                               # (:87-89)
                self._mark((self._insert_index + i) % self._size, False)

    def sample(self, batch_size: int, keys: Optional[Iterable[str]] = None, indx=None,
               pack_obs_and_next_obs: bool = False, n_step: int = 1, discount: Optional[float] = None) -> BatchHandle:
        if keys is not None:
            assert "observations" in keys                                                    # (:128-129)
        return super().sample(batch_size, keys, indx, pack_obs_and_next_obs, n_step=n_step, discount=discount)
