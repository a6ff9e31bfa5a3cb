"""CPU: proportional prioritized replay as oracle/per.py states it - draw frequencies, zero leaves, stratified uniform draws at
alpha = 0, weights, last-wins writes - the C host mirror of the draw against the oracle, and the rings' argument rules."""
import numpy as np
import pytest
from scipy import stats

from oracle import per as P


def _tree(leaves):
    return P.build(np.asarray(leaves, np.float32))


def test_layout_and_build():
    for cap, counts in ((1, [1]), (31, [31, 1]), (32, [32, 1]), (33, [33, 2, 1]), (1000, [1000, 32, 1]),
                        ((1 << 20) - 1, [(1 << 20) - 1, 32768, 1024, 32, 1]), (10 ** 6, [10 ** 6, 31250, 977, 31, 1])):
        off, cnt = P.layout(cap)
        assert cnt == counts and off[0] == 0 and all(off[l] == off[l - 1] + cnt[l - 1] for l in range(1, len(off)))
    leaves = np.random.default_rng(0).random(1000).astype(np.float32)
    t = _tree(leaves)
    off, cnt = P.layout(1000)
    s = np.float32(0)
    for c in range(32):                                       # node 0 of level 1: children 0..31 added in order from 0
        s = np.float32(s + leaves[c])
    assert t[off[1]] == s
    s = np.float32(0)
    for c in range(992, 1000):                                # the last, partial node: its 8 children only
        s = np.float32(s + leaves[c])
    assert t[off[1] + 31] == s
    assert abs(float(t[-1]) - float(leaves.astype(np.float64).sum())) < 1e-3


def test_draw_frequencies_match_priorities():
    rng = np.random.default_rng(1)
    cap = 1000
    p = (rng.random(cap) ** 3).astype(np.float32)
    p[rng.random(cap) < 0.2] = 0                             # invalid slots
    t = _tree(p)
    B, steps = 4096, 245                                     # ~1e6 draws
    counts = np.zeros(cap, np.int64)
    for step in range(steps):
        idx = P.draw(t, cap, seed=77, step=step, batch=B)
        assert (idx >= 0).all()
        counts += np.bincount(idx, minlength=cap)
    assert counts[p == 0].sum() == 0                         # zero leaves are never drawn
    nz = p > 0
    expect = p[nz].astype(np.float64) / p[nz].astype(np.float64).sum() * counts.sum()
    keep = expect >= 5
    obs = np.append(counts[nz][keep], counts[nz][~keep].sum())
    exp = np.append(expect[keep], expect[~keep].sum())
    assert stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue > 1e-3


def test_alpha_zero_is_stratified_uniform():
    cap = 64
    valid = np.ones(cap, bool)
    valid[[3, 10, 40]] = False
    leaves, m = P.set_leaves(np.zeros(cap), 1.0, np.arange(cap), td=np.random.default_rng(2).normal(size=cap), alpha=0.0, eps=1e-6)
    leaves[~valid] = 0
    assert m == 1.0 and set(np.unique(leaves)) == {0.0, 1.0}
    t = _tree(leaves)
    B = int(valid.sum())
    idx = P.draw(t, cap, seed=5, step=0, batch=B)
    assert sorted(idx.tolist()) == np.flatnonzero(valid).tolist()   # one row per stratum: every valid slot exactly once


def test_all_zero_tree_fails_every_row():
    assert (P.draw(np.zeros(P.nodes(40), np.float32), 40, seed=1, step=0, batch=8) == -1).all()


def test_weights_formula():
    p = np.array([0.5, 2.0, 1.0, 0.25], np.float32)
    for beta in (0.0, 0.4, 1.0):
        w = P.weights(p, beta)
        n_prob = len(p) * p.astype(np.float64) / p.sum()       # Schaul: (N P)^-beta / max w
        ref = n_prob ** -beta / (n_prob ** -beta).max()
        np.testing.assert_allclose(w, ref, rtol=1e-12)
        assert w.max() == 1.0


def test_weights_zero_leaf_and_writes_to_invalid_or_nonfinite():
    np.testing.assert_array_equal(P.weights([0.0, 2.0, 1.0], 1.0), [0.0, 0.5, 1.0])
    leaves, m = P.set_leaves(np.full(4, 0.5), 1.0, [0, 1, 2, 1], td=[3.0, 5.0, np.nan, np.inf], ring_valid=[True, False, True, True],
                             alpha=1.0, eps=0.0)
    assert leaves.tolist() == [3.0, 0.0, 0.5, 0.5] and m == 3.0   # slot 1 is invalid -> 0 (its inf entry skipped); NaN skipped


def test_duplicate_slots_last_wins():
    leaves, m = P.set_leaves(np.zeros(8), 1.0, [3, 5, 3, 3, 5], td=[1.0, 2.0, 3.0, 0.5, 4.0], alpha=1.0, eps=0.0)
    assert leaves[3] == 0.5 and leaves[5] == 4.0 and m == 4.0
    leaves, m = P.set_leaves(leaves, 4.0, [5, 6, 5], valid=[True, True, False])
    assert leaves[5] == 0.0 and leaves[6] == 4.0 and m == 4.0


def test_host_mirror_matches_oracle():
    import __graft_entry__ as G
    G.build()
    from serl_b200 import _lib as L
    rng = np.random.default_rng(3)
    for cap in (1, 31, 33, 1000, 40000):
        p = rng.random(cap).astype(np.float32)
        p[rng.random(cap) < 0.3] = 0
        if cap == 1:
            p[0] = 0.7
        t = _tree(p)
        for B, step, lane in ((1, 0, 0), (256, 3, 0), (300, (1 << 33) + 1, 9)):
            out = np.zeros(B, np.int32)
            valid = (rng.random(cap) < 0.9).astype(np.uint8)      # a non-zero leaf of a slot that is not valid costs an attempt
            valid[0] = 1
            L.call("serl_host_draw_prio", t.ctypes.data, valid.ctypes.data, cap, (7 << 32) | 11, step, lane, B, out.ctypes.data)
            np.testing.assert_array_equal(out, P.draw(t, cap, (7 << 32) | 11, step, B, lane_offset=lane, valid=valid.astype(bool)))
            assert valid[out[out >= 0]].all()


class _Box:
    def __init__(self, n):
        self.shape = (n,)


@pytest.mark.parametrize("kw", [dict(priority_alpha=-0.5), dict(priority_alpha=float("nan")), dict(priority_alpha=0.6, priority_beta=1.5),
                                dict(priority_alpha=0.6, priority_beta=-0.1), dict(priority_alpha=0.6, priority_eps=0.0),
                                dict(priority_alpha=0.6, priority_eps=float("inf")), dict(priority_alpha=True), dict(priority_alpha="0.6")])
def test_argument_validation(kw):
    from serl_b200.data.data_store import MemoryEfficientReplayBufferDataStore, ReplayBufferDataStore
    from serl_b200.data.replay_buffer import ReplayBuffer, check_priority_args
    with pytest.raises(ValueError):                           # before any device allocation
        ReplayBuffer(_Box(3), _Box(2), 16, **kw)
    with pytest.raises(ValueError):
        ReplayBufferDataStore(_Box(3), _Box(2), 16, **kw)
    with pytest.raises(ValueError):
        MemoryEfficientReplayBufferDataStore(None, _Box(2), 16, **kw)
    args = (kw.get("priority_alpha"), kw.get("priority_beta", 0.4), kw.get("priority_eps", 1e-6))
    with pytest.raises(ValueError):
        check_priority_args(*args)
    if not isinstance(args[0], (bool, str)):
        with pytest.raises(ValueError):
            P.check_args(*args)


def test_argument_validation_accepts():
    from serl_b200.data.replay_buffer import check_priority_args
    for args in ((None, 0.4, 1e-6), (0.0, 1.0, 1e-6), (0.6, 0.0, 1e-3)):
        check_priority_args(*args)
        P.check_args(*args)


def test_descent_tie_goes_to_the_next_child():
    """A prefix equal to u does not exceed it: with leaves (u, 1 - u) and root 1, row 0 of a one-row draw lands on slot 1
    (the oracle and the C code the device runs, through its host mirror)."""
    import __graft_entry__ as G
    G.build()
    from oracle.replay import philox4x32
    from serl_b200 import _lib as L
    seed = 5
    for step in range(100):
        x = philox4x32((np.uint32(0), np.uint32(0), np.uint32(step), np.uint32(0)), (seed, 0))[0]
        u = np.float32(np.float32(x) * np.float32(2.0 ** -32))
        if u >= 0.5 and float(np.float32(1) - u) == 1.0 - float(u):
            break
    t = _tree([u, np.float32(1) - u])
    assert t[-1] == np.float32(1)
    assert P.draw(t, 2, seed, step, 1).tolist() == [1]
    out = np.zeros(1, np.int32)
    valid = np.ones(2, np.uint8)
    L.call("serl_host_draw_prio", t.ctypes.data, valid.ctypes.data, 2, seed, step, 0, 1, out.ctypes.data)
    assert out.tolist() == [1]
