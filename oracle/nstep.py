"""ORACLE (test infrastructure, not product): NumPy restatement of the n-step replay targets that
`serl_replay_sample_crop_nstep` (serl_b200/csrc/sampler.cu) gathers, over the host arrays of an `OracleFrameRing`
(oracle/replay.py; a state-only ring is one with no image keys).

Drawn slot i, window bound n, discount g, ring insert index `head` (the newest written slot is head - 1):
  m     = the largest m <= n such that slots i, i+1, ..., i+m-1 (mod capacity) are written - at or behind head - 1 in
          insertion order - and valid, and none of i, ..., i+m-2 has dones = 1.  The window stops at the first episode end
          (terminated or truncated) and at the newest slot.  A written slot after i is invalid only where the frame-dedup
          ring re-inserted the last T frames at the front on a mid-episode wrap; those copies are not the next transition.
  rewards = sum_{k<m} g^k r[i+k];  masks = g^(m-1) masks[i+m-1];  dones = dones[i+m-1]
  next observation (frames and state) = slot i+m-1's; observations and actions = slot i's.

`scalars` gives both the float64 values and the fp32 restatement in the kernel's documented order
(g_0 = 1, R = r[i]; for k = 1..m-1: g_k = g_{k-1} * g, R = R + g_k * r[i+k], each product and sum rounded to fp32;
masks = g_{m-1} * masks[i+m-1]).
"""
from __future__ import annotations

import numpy as np

MAX_NSTEP = 16


def window(idx, n: int, *, capacity: int, head: int, dones, valid):
    """(m, j) int64 arrays: window length and last slot of each drawn slot in `idx`."""
    if not 1 <= n <= MAX_NSTEP:
        raise ValueError(f"n_step={n}: must be in 1..{MAX_NSTEP}")
    idx = np.asarray(idx, np.int64)
    dones, valid = np.asarray(dones, bool), np.asarray(valid, bool)
    avail = (head - idx - 1) % capacity + 1                      # slots idx .. head-1 in insertion order
    lim = np.minimum(n, avail)
    m = np.ones_like(idx)
    j = idx.copy()
    live = m < lim
    for _ in range(n - 1):
        nxt = (j + 1) % capacity
        live &= (m < lim) & ~dones[j] & valid[nxt]
        j = np.where(live, nxt, j)
        m = np.where(live, m + 1, m)
    return m, j


def scalars(idx, m, *, capacity: int, rewards, masks, dones, discount: float) -> dict:
    """The row scalars of windows (idx, m): float64 `rewards` / `masks`, their fp32 restatement `rewards32` / `masks32`, `dones`."""
    idx, m = np.asarray(idx, np.int64), np.asarray(m, np.int64)
    rewards, masks = np.asarray(rewards, np.float32), np.asarray(masks, np.float32)
    j = (idx + m - 1) % capacity
    k = np.arange(int(m.max()) if m.size else 1)
    slots = (idx[:, None] + k[None, :]) % capacity
    inside = k[None, :] < m[:, None]
    r64 = np.where(inside, rewards[slots].astype(np.float64) * float(discount) ** k[None, :], 0.0).sum(axis=1)
    m64 = float(discount) ** (m - 1) * masks[j].astype(np.float64)
    g32, d32 = np.ones(len(idx), np.float32), np.float32(discount)
    r32 = rewards[idx].copy()
    for kk in range(1, len(k)):
        on = kk < m
        g_next = (g32 * d32).astype(np.float32)
        r_next = (r32 + (g_next * rewards[slots[:, kk]]).astype(np.float32)).astype(np.float32)
        g32, r32 = np.where(on, g_next, g32), np.where(on, r_next, r32)
    return {"rewards": r64, "masks": m64, "rewards32": r32, "masks32": (g32 * masks[j]).astype(np.float32),
            "dones": np.asarray(dones, bool)[j]}


def nstep_batch(ring, idx, n: int, discount: float, head=None) -> dict:
    """The n-step batch of slots `idx` of an OracleFrameRing, un-augmented and unpacked: observations of idx, next observations
    of the window's last slot (frame windows as `gather_packed` builds them), plus `m` and `next_idx`."""
    head = ring.cursor if head is None else head
    idx = np.asarray(idx, np.int64)
    m, j = window(idx, n, capacity=ring.capacity, head=head, dones=ring.dones, valid=ring.valid)
    sc = scalars(idx, m, capacity=ring.capacity, rewards=ring.rewards, masks=ring.masks, dones=ring.dones, discount=discount)
    at_i, at_j = ring.gather_packed(idx), ring.gather_packed(j)
    obs = {"state": at_i["observations"]["state"]}
    nobs = {"state": at_j["next_observations"]["state"]}
    for k in ring.image_keys:
        obs[k] = at_i["observations"][k][:, :-1]
        nobs[k] = at_j["observations"][k][:, 1:]
    return {"observations": obs, "next_observations": nobs, "actions": at_i["actions"], "m": m, "next_idx": j, **sc}
