"""Thread-safe data stores the agentlace TrainerServer inserts into.

Mirrors reference data/data_store.py:26-145 (`ReplayBufferDataStore`,
`MemoryEfficientReplayBufferDataStore`, `populate_data_store*`).  The reference subclasses
`agentlace.data.data_store.DataStoreBase`; agentlace is not installable here, so the same four-method
interface (`insert`, `__len__`, `latest_data_id`, `get_latest_data`) is duck-typed and, when agentlace
IS importable, the classes are registered as virtual subclasses so `isinstance` checks pass.
The ring's own re-entrant lock serialises insert (server thread) against sample (learner thread),
like the reference's `threading.Lock` (:36,44-45,70-71).
"""
from __future__ import annotations

import pickle as pkl
from typing import Iterable, Optional

from .memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
from .replay_buffer import ReplayBuffer

try:                                                   # optional: real agentlace base class
    from agentlace.data.data_store import DataStoreBase as _Base
except Exception:                                      # noqa: BLE001
    _Base = None


class _DataStoreMixin:
    def latest_data_id(self):                          # data_store.py:75-76,139-140
        return self._insert_index

    def get_latest_data(self, from_id: int):           # data_store.py:79-80,143-144
        raise NotImplementedError


class ReplayBufferDataStore(_DataStoreMixin, ReplayBuffer):
    def __init__(self, observation_space, action_space, capacity: int, rlds_logger=None, device=None, seed=None,
                 priority_alpha: Optional[float] = None, priority_beta: float = 0.4, priority_eps: float = 1e-6):
        ReplayBuffer.__init__(self, observation_space, action_space, capacity, device=device, seed=seed, priority_alpha=priority_alpha, priority_beta=priority_beta, priority_eps=priority_eps)
        if rlds_logger is not None:
            raise NotImplementedError("RLDS logging (oxe_envlogger) is outside the learner hot path")


class MemoryEfficientReplayBufferDataStore(_DataStoreMixin, MemoryEfficientReplayBuffer):
    def __init__(self, observation_space, action_space, capacity: int, image_keys: Iterable[str] = ("image",),
                 rlds_logger=None, device=None, seed=None, frame_shard=None, priority_alpha: Optional[float] = None,
                 priority_beta: float = 0.4, priority_eps: float = 1e-6):
        MemoryEfficientReplayBuffer.__init__(self, observation_space, action_space, capacity, pixel_keys=tuple(image_keys),
                                             device=device, seed=seed, frame_shard=frame_shard, priority_alpha=priority_alpha, priority_beta=priority_beta, priority_eps=priority_eps)
        if rlds_logger is not None:
            raise NotImplementedError("RLDS logging (oxe_envlogger) is outside the learner hot path")


if _Base is not None:
    _Base.register(ReplayBufferDataStore) if hasattr(_Base, "register") else None
    _Base.register(MemoryEfficientReplayBufferDataStore) if hasattr(_Base, "register") else None


def populate_data_store(data_store, demos_path):
    """data_store.py:147-162: load pickled demo transitions (lists of transition dicts)."""
    for demo_path in demos_path:
        with open(demo_path, "rb") as f:
            for transition in pkl.load(f):
                data_store.insert(transition)
        print(f"Loaded {len(data_store)} transitions.")
    return data_store
