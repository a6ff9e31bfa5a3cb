"""ORACLE (test infrastructure, not product): NumPy restatement of proportional prioritized replay (Schaul et al. 2016) as
the replay rings implement it (serl_b200/csrc/sampler.cu; layout and draw stated in include/serl_b200.h).

Sum tree, fan-out 32, every level in one float32 array, leaves first:
  count[0] = capacity, count[l] = ceil(count[l-1] / 32) until a level of one node (the root; capacity 1: the leaf is the root);
  offset[0] = 0, offset[l] = offset[l-1] + count[l-1].
  Leaf i = priority p_i of slot i, 0 while the slot is not valid.  Node j of level l >= 1 = float32 sum, from 0 in ascending
  order, of children 32j .. min(32j+31, count[l-1]-1).  Nodes are recomputed from their children, never incremented, so the
  tree is a pure function of its leaves (`build`).

Leaves:
  * a slot written or made valid by a ring flush gets the running maximum m (1.0 in a new ring); a slot made invalid gets 0;
  * update_priorities(slots, td) sets p = (|td| + eps)^alpha (float32 add, then powf on the device) and m = max(m, written p);
    a slot that is not valid gets 0, and an entry with a non-finite td is skipped;
  * a slot named twice in one write takes its LAST entry.

Draw of row b of a part of B rows (stratified, proportional), attempt a = 0, 1, ...:
  x = word 0 of philox4x32((lane_offset + b, a, step_lo, step_hi), (seed_lo, seed_hi))   (the uniform draw's counter)
  u = fl(fl(fl(b + fl(x) * 2^-32) / B) * root)                                            (fl: float32 round to nearest)
  at each node, over its children in order with running prefix s = fl(s + child): the first child whose new prefix exceeds u,
  u = fl(u - s) with s the prefix before it; none: the last non-zero child, same subtraction; all children 0: attempt fails.
  A leaf of 0 or a slot that is not valid fails the attempt; after MAX_DRAW_ATTEMPTS the row yields -1.

Weights of one part's drawn rows: w_b = (p_min / p_b)^beta, p_min = the smallest non-zero leaf among that part's rows -
Schaul's (N P(b))^-beta / max w, where N and the root cancel.  A row of priority 0 (an explicit index) gets w = 0.

Critic loss of a batch with weights w (serl_critic_loss_weighted): sum_{e,b} w_b (Q[e,b] - y_b)^2 / (E B), and the TD error
written back is delta_b = sum_e |Q[e,b] - y_b| / E.

Only tests/ may import this.
"""
from __future__ import annotations

import numpy as np

from .replay import MAX_DRAW_ATTEMPTS, U32, philox4x32

FANOUT = 32
F32 = np.float32


def check_args(alpha, beta, eps):
    """The rings' argument rules: ValueError when one is out of range."""
    if alpha is not None and not (np.isfinite(alpha) and alpha >= 0):
        raise ValueError(f"priority_alpha={alpha!r}: must be a finite float >= 0 (or None for uniform draws)")
    if not (np.isfinite(beta) and 0 <= beta <= 1):
        raise ValueError(f"priority_beta={beta!r}: must be in [0, 1]")
    if not (np.isfinite(eps) and eps > 0):
        raise ValueError(f"priority_eps={eps!r}: must be a finite float > 0")


def layout(capacity: int):
    """(offsets, counts) of the tree's levels, leaves first."""
    off, cnt, o, n = [], [], 0, int(capacity)
    while True:
        off.append(o)
        cnt.append(n)
        if n == 1:
            return off, cnt
        o += n
        n = (n + FANOUT - 1) // FANOUT


def nodes(capacity: int) -> int:
    off, _ = layout(capacity)
    return off[-1] + 1


def build(leaves) -> np.ndarray:
    """The whole tree (float32) over `leaves`."""
    leaves = np.asarray(leaves, F32)
    off, cnt = layout(leaves.shape[0])
    t = np.zeros(off[-1] + 1, F32)
    t[:cnt[0]] = leaves
    for l in range(1, len(off)):
        ch = np.zeros(cnt[l] * FANOUT, F32)
        ch[:cnt[l - 1]] = t[off[l - 1]:off[l - 1] + cnt[l - 1]]
        ch = ch.reshape(cnt[l], FANOUT)
        s = np.zeros(cnt[l], F32)
        for c in range(FANOUT):                      # ascending order, float32 rounding at every add
            s = s + ch[:, c]
        t[off[l]:off[l] + cnt[l]] = s
    return t


def last_wins(slots) -> dict:
    """slot -> index of its last entry in `slots`."""
    return {int(s): k for k, s in enumerate(np.asarray(slots).reshape(-1))}


def priorities(td, alpha: float, eps: float) -> np.ndarray:
    """float64 p = (|td| + eps)^alpha."""
    return (np.abs(np.asarray(td, np.float64)) + eps) ** alpha


def set_leaves(leaves, m: float, slots, *, td=None, valid=None, ring_valid=None, alpha: float = 1.0, eps: float = 0.0):
    """(new leaves as float64, new m): one priority write.  td given: p = (|td| + eps)^alpha (0 where ring_valid is False;
    non-finite td entries skipped) and m grows to the written maximum; else (a ring flush) p = valid ? m : 0."""
    out = np.asarray(leaves, np.float64).copy()
    written = []
    slots = np.asarray(slots).reshape(-1)
    keep = np.ones(slots.size, bool) if td is None else np.isfinite(np.asarray(td, np.float64).reshape(-1))
    for s, k in last_wins(slots[keep]).items():
        k = int(np.flatnonzero(keep)[k])
        if td is not None:
            p = 0.0 if ring_valid is not None and not ring_valid[s] else float(priorities(np.asarray(td).reshape(-1)[k], alpha, eps))
        else:
            p = m if valid[k] else 0.0
        out[s] = p
        written.append(p)
    if td is not None and written:
        m = max(m, max(written))
    return out, m


def draw(tree, capacity: int, seed: int, step: int, batch: int, lane_offset: int = 0, valid=None) -> np.ndarray:
    """Drawn slots (int32, -1 where every attempt failed) of one part of `batch` rows; `valid` defaults to every slot."""
    tree = np.asarray(tree, F32)
    valid = np.ones(capacity, bool) if valid is None else np.asarray(valid, bool)
    off, cnt = layout(capacity)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    b = np.arange(batch, dtype=np.int64)
    lanes = (b + lane_offset).astype(U32)
    root = tree[off[-1]]
    out = np.full(batch, -1, np.int32)
    pending = np.ones(batch, bool)
    for a in range(MAX_DRAW_ATTEMPTS):
        if not pending.any():
            break
        x = philox4x32((lanes, U32(a), U32(step & 0xFFFFFFFF), U32((step >> 32) & 0xFFFFFFFF)), key)[0]
        u = ((b.astype(F32) + x.astype(F32) * F32(2.0 ** -32)) / F32(batch)) * root
        j = np.zeros(batch, np.int64)
        fail = np.zeros(batch, bool)
        for l in range(len(off) - 1, 0, -1):
            n_ch = cnt[l - 1]
            s = np.zeros(batch, F32)
            pick, s_pick = np.full(batch, -1, np.int64), np.zeros(batch, F32)
            nz, s_nz = np.full(batch, -1, np.int64), np.zeros(batch, F32)
            for c in range(FANOUT):
                ci = FANOUT * j + c
                inb = ci < n_ch
                v = np.where(inb, tree[off[l - 1] + np.minimum(ci, n_ch - 1)], F32(0))
                s2 = s + v
                live = inb & (pick < 0)
                hit = live & (s2 > u)
                pick, s_pick = np.where(hit, ci, pick), np.where(hit, s, s_pick)
                go = live & ~hit
                upd = go & (v != 0)
                nz, s_nz = np.where(upd, ci, nz), np.where(upd, s, s_nz)
                s = np.where(go, s2, s)
            clamp = pick < 0
            fail |= clamp & (nz < 0)
            pick, s_pick = np.where(clamp, nz, pick), np.where(clamp, s_nz, s_pick)
            u = u - s_pick
            j = np.where(fail, 0, pick)
        ok = pending & ~fail & (tree[j] > 0) & valid[j]
        out[ok] = j[ok]
        pending &= ~ok
    return out


def weights(p, beta: float) -> np.ndarray:
    """float64 importance weights of one part's drawn leaves p."""
    p = np.asarray(p, np.float64)
    w = np.zeros_like(p)
    nz = p > 0
    if nz.any():
        w[nz] = (p[nz].min() / p[nz]) ** beta
    return w


def critic_loss(q, y, w):
    """float64 (loss, dQ / grad_scale, delta) of the weighted critic loss; q (E, B), y (B), w (B)."""
    q, y, w = (np.asarray(a, np.float64) for a in (q, y, w))
    E, B = q.shape
    d = q - y[None, :]
    return (w[None, :] * d * d).sum() / (E * B), 2 * w[None, :] * d / (E * B), np.abs(d).mean(axis=0)
