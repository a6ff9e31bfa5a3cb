"""GPU: prioritized replay rings against oracle/per.py.

* the sum tree after priority writes with duplicate slots, at capacities 1 .. 10^6: leaves within 1e-6 of float64
  (|td| + eps)^alpha, the last entry of a duplicated slot winning, and every interior node bitwise the oracle's rebuild;
* the importance weights within 1e-6 of float64;
* draws through every sampler kernel path (frame, banded, bytewise, state-only) with n_step 1 and 3: indices bit-exact against
  the oracle's draw over the device tree, each row's leaf, and the gathered fields and crops bit-exact;
* the tree after inserts (episode ends, a ring wrap, the frame-dedup ring's mid-episode wrap) and after a save / load;
* the refusals: a prioritized handle to a consumer that ignores its weights, and data-parallel stores.
"""
import numpy as np
import pytest
import torch

import test_replay_sampler_paths_gpu as SP

pytestmark = pytest.mark.gpu


def _host(t):
    return t.detach().cpu().numpy()


def _check_tree(tree, cap):
    """Interior nodes bitwise the oracle's rebuild from the device's own leaves; returns the leaves."""
    from oracle import per as P
    t = _host(tree)
    np.testing.assert_array_equal(t.view(np.uint32), P.build(t[:cap]).view(np.uint32))
    return t[:cap]


# ---- priority writes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [1, 31, 33, 1000, (1 << 20) - 1, 10 ** 6])
def test_priority_set_tree_bitwise(cap):
    from oracle import per as P
    from serl_b200 import ops
    rng = np.random.default_rng(cap)
    tree = torch.zeros(P.nodes(cap), dtype=torch.float32, device="cuda")
    mx = torch.ones(1, dtype=torch.float32, device="cuda")
    t = ops.priority_tree(tree, mx, cap)
    want, m = np.zeros(cap), 1.0
    alpha, eps = 0.6, 1e-6
    for n in (1, 300, 4096):
        slots = rng.integers(0, cap, n).astype(np.int32)
        td = rng.standard_normal(n).astype(np.float32) * 3
        if n > 1:                                  # duplicates: an early entry far from the last one
            slots[: n // 4] = slots[-(n // 4):]
            td[: n // 4] = 1e4
        ops.priority_set(t, torch.from_numpy(slots).cuda(), n, td=torch.from_numpy(td).cuda(), alpha=alpha, eps=eps)
        want, m = P.set_leaves(want, m, slots, td=td.astype(np.float64), alpha=alpha, eps=eps)
        leaves = _check_tree(tree, cap)
        np.testing.assert_allclose(leaves, want, rtol=1e-6, atol=0)
        assert abs(float(mx.item()) - m) <= 1e-6 * m
    valid = rng.random(min(cap, 4096)) < 0.5                 # a flush: m for valid slots, 0 for the rest
    slots = rng.permutation(cap)[: valid.size].astype(np.int32)
    ops.priority_set(t, torch.from_numpy(slots).cuda(), slots.size, valid=torch.from_numpy(valid.astype(np.uint8)).cuda())
    leaves = _check_tree(tree, cap)
    m_dev = np.float32(mx.item())
    np.testing.assert_array_equal(leaves[slots], np.where(valid, m_dev, np.float32(0)))


@pytest.mark.parametrize("n", [1, 2, 257, 4096])
def test_priority_weights_float64(n):
    from oracle import per as P
    from serl_b200 import ops
    p = (np.random.default_rng(n).random(n) * 10 + 1e-3).astype(np.float32)
    w = torch.empty(n, dtype=torch.float32, device="cuda")
    for beta in (0.0, 0.4, 1.0):
        ops.priority_weights(torch.from_numpy(p).cuda(), n, torch.full((1,), beta, device="cuda"), w)
        np.testing.assert_allclose(_host(w), P.weights(p, beta), rtol=1e-6, atol=0)


# ---- draws -----------------------------------------------------------------------------------------------------------------
def _prio_ring(ncam, T, H, W, C, cap, seed):
    """A full prioritized ring in HBM (seeded random frames, fields and validity, as tests/test_replay_sampler_paths_gpu.py
    builds its uniform rings) with its oracle twin, and random priorities on its valid slots."""
    from helpers import Box, DictSpace
    from oracle.replay import OracleFrameRing
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
    from serl_b200.data.replay_buffer import ReplayBuffer
    cams = tuple(f"cam{j}" for j in range(ncam))
    if ncam:
        space = DictSpace({**{c: Box((T, H, W, C), np.uint8) for c in cams}, "state": Box((T, SP.S_DIM))})
        dev = MemoryEfficientReplayBuffer(space, Box((SP.A_DIM,)), cap, pixel_keys=cams, seed=seed + 1000, priority_alpha=0.7)
    else:
        dev = ReplayBuffer(Box((SP.S_DIM,)), Box((SP.A_DIM,)), cap, seed=seed + 1000, priority_alpha=0.7)
    ora = OracleFrameRing(cap, cams, (H, W, C), T, SP.S_DIM, SP.A_DIM)
    rng = np.random.default_rng(seed)
    for c in cams:
        ora.frames[c] = rng.integers(0, 256, (cap, H, W, C), dtype=np.uint8)
        dev.frames[c].copy_(torch.from_numpy(ora.frames[c]))
    ora.state = rng.standard_normal((cap, T, SP.S_DIM)).astype(np.float32)
    ora.next_state = rng.standard_normal((cap, T, SP.S_DIM)).astype(np.float32)
    ora.actions = rng.uniform(-1, 1, (cap, SP.A_DIM)).astype(np.float32)
    ora.rewards = rng.standard_normal(cap).astype(np.float32)
    ora.masks = rng.random(cap).astype(np.float32)
    ora.dones = rng.random(cap) < 0.2
    ora.valid = rng.random(cap) < 0.75
    ora.size, ora.cursor = cap, 0
    dev.state.copy_(torch.from_numpy(ora.state.reshape(cap, -1)))
    dev.next_state.copy_(torch.from_numpy(ora.next_state.reshape(cap, -1)))
    for name in ("actions", "rewards", "masks"):
        getattr(dev, name).copy_(torch.from_numpy(getattr(ora, name)))
    dev.dones.copy_(torch.from_numpy(ora.dones.astype(np.uint8)))
    dev.valid.copy_(torch.from_numpy(ora.valid.astype(np.uint8)))
    dev._valid_host[:] = ora.valid
    dev._size = cap
    dev.size_dev.fill_(cap)
    slots = np.flatnonzero(ora.valid).astype(np.int32)
    dev.update_priorities(slots, rng.standard_normal(slots.size) * 2)
    torch.cuda.synchronize()
    return dev, ora


def _launch_prio(dev, *, batch, B_total, off, step, n_step):
    from serl_b200 import _lib as L
    cams, (H, W, Cc), T = dev.cams, dev.frame_shape, dev.T
    u8 = lambda *s: torch.full(s, SP.SENTINEL, dtype=torch.uint8, device="cuda")
    nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device="cuda")
    i32 = lambda *s: u8(*s[:-1], 4 * s[-1]).view(torch.int32)          # 0xA5 bytes, as the uniform sampler test prefills
    pix = {(c, w): u8(B_total, T, H, W, Cc) for c in cams for w in ("obs", "next")}
    bufs = dict(obs_state=nan(B_total, T * dev.S), next_state=nan(B_total, T * dev.S), actions=nan(B_total, dev.A),
                rewards=nan(B_total), masks=nan(B_total), dones=u8(B_total), idx=i32(B_total), off_obs=i32(B_total * T, 2),
                off_next=i32(B_total * T, 2), status=torch.zeros(1, dtype=torch.int32, device="cuda"))
    out = L.BatchOut()
    for j, c in enumerate(cams):
        out.obs_pix[j], out.next_pix[j] = pix[(c, "obs")].data_ptr(), pix[(c, "next")].data_ptr()
    for name, t in bufs.items():
        setattr(out, name, t.data_ptr())
    k_obs, k_next = SP._keys(step)
    key_t = torch.from_numpy(np.stack([k_obs, k_next]).astype(np.uint32).reshape(-1).view(np.int32)).cuda()
    prio, m_out, j_out = nan(B_total), i32(B_total), i32(B_total)
    part = dict(ring=dev, seed=dev._seed, step=step, batch=batch, indx=None, n_step=n_step, discount=0.9 if n_step > 1 else None)
    dev.launch_sample(part, out, crop_total=B_total * T, out_row_offset=off, key_obs=key_t.data_ptr(), key_next=key_t.data_ptr() + 8,
                      record_event=False, prio_out=prio, nstep_out=(m_out, j_out) if n_step > 1 else None)
    res = {k: _host(v) for k, v in bufs.items()}
    res["pix"] = {k: _host(v) for k, v in pix.items()}
    res["prio"], res["m"], res["j"] = _host(prio), _host(m_out), _host(j_out)
    return res, (k_obs, k_next)


_PATHS = [pytest.param(2, 2, 128, 128, 3, id="frame-128x128x3-T2-2cam"), pytest.param(1, 1, 256, 128, 3, id="banded-256x128x3"),
          pytest.param(1, 9, 32, 32, 3, id="banded-32x32x3-T9"), pytest.param(1, 1, 84, 84, 3, id="bytewise-84x84x3"),
          pytest.param(0, 1, 1, 1, 1, id="state-only")]


@pytest.mark.parametrize("n_step", [1, 3])
@pytest.mark.parametrize("ncam,T,H,W,C", _PATHS)
def test_prioritized_draw_matches_oracle(ncam, T, H, W, C, n_step):
    from oracle import jax_prng as J
    from oracle import nstep as N
    from oracle import per as P
    cap, B, off, B_total, step = 48, 40, 3, 45, 5
    dev, ora = _prio_ring(ncam, T, H, W, C, cap, seed=H + W + T)
    tree = _host(dev.tree)
    res, (k_obs, k_next) = _launch_prio(dev, batch=B, B_total=B_total, off=off, step=step, n_step=n_step)
    idx = P.draw(tree, cap, dev._seed, step, B)
    assert (idx >= 0).all() and ora.valid[idx].all() and res["status"][0] == 0
    rows = off + np.arange(B)
    np.testing.assert_array_equal(res["idx"][rows], idx)
    np.testing.assert_array_equal(res["prio"][rows].view(np.uint32), tree[idx].view(np.uint32))
    assert np.isnan(res["prio"][np.setdiff1d(np.arange(B_total), rows)]).all()
    n = B_total * ora.T
    if n_step == 1 and ncam:
        SP._check(ora, res, off=off, batch=B, idx=idx, off_obs=J.crop_offsets(k_obs, n), off_next=J.crop_offsets(k_next, n))
        return
    np.testing.assert_array_equal(res["obs_state"][rows], ora.state[idx].reshape(B, -1))
    np.testing.assert_array_equal(res["actions"][rows], ora.actions[idx])
    m, j = N.window(idx, n_step, capacity=cap, head=0, dones=ora.dones, valid=ora.valid)
    sc = N.scalars(idx, m, capacity=cap, rewards=ora.rewards, masks=ora.masks, dones=ora.dones, discount=0.9)
    if n_step > 1:
        np.testing.assert_array_equal(res["m"][rows], m)
        np.testing.assert_array_equal(res["j"][rows], j)
    np.testing.assert_array_equal(res["rewards"][rows].view(np.uint32), sc["rewards32"].view(np.uint32))
    np.testing.assert_array_equal(res["masks"][rows].view(np.uint32), sc["masks32"].view(np.uint32))
    np.testing.assert_array_equal(res["dones"][rows], sc["dones"].astype(np.uint8))
    np.testing.assert_array_equal(res["next_state"][rows], ora.next_state[j].reshape(B, -1))
    if ncam:
        from oracle.replay import random_shift
        c = ora.image_keys[0]
        g = (rows[:, None] * T + np.arange(T)).reshape(-1)
        want = random_shift(ora.gather_packed(idx)["observations"][c][:, :-1].reshape(-1, H, W, C), J.crop_offsets(k_obs, n)[g], SP.PAD)
        np.testing.assert_array_equal(res["pix"][(c, "obs")][rows].reshape(-1, H, W, C), want)
        want = random_shift(ora.gather_packed(j)["observations"][c][:, 1:].reshape(-1, H, W, C), J.crop_offsets(k_next, n)[g], SP.PAD)
        np.testing.assert_array_equal(res["pix"][(c, "next")][rows].reshape(-1, H, W, C), want)


def test_gather_dict_weights_and_explicit_indices():
    from oracle import per as P
    dev, ora = _prio_ring(1, 1, 84, 84, 3, 48, seed=3)
    dev.priority_beta = 0.8
    h = dev.sample(32)
    d = h.to_dict()
    tree = _host(dev.tree)
    idx = P.draw(tree, 48, dev._seed, h.parts[0]["step"], 32)
    np.testing.assert_array_equal(_host(d["_indices"]), idx)
    np.testing.assert_allclose(_host(d["_weights"]), P.weights(tree[idx], 0.8), rtol=1e-6, atol=0)
    fixed = np.flatnonzero(ora.valid)[:5]
    d = dev.sample(5, indx=fixed).to_dict()                   # indx= skips the draw; the weights are those rows'
    np.testing.assert_array_equal(_host(d["_indices"]), fixed)
    np.testing.assert_allclose(_host(d["_weights"]), P.weights(tree[fixed], 0.8), rtol=1e-6, atol=0)


# ---- the tree follows the ring ---------------------------------------------------------------------------------------------
def test_tree_after_inserts_wraps_and_updates(tmp_path):
    from helpers import Box, DictSpace
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
    T, cap = 2, 23
    space = DictSpace({"pixels": Box((T, 16, 16, 3), np.uint8), "state": Box((T, 4))})
    ring = MemoryEfficientReplayBuffer(space, Box((2,)), cap, seed=1, priority_alpha=0.5, priority_beta=0.3)
    rng = np.random.default_rng(0)

    def insert(done):
        obs = {"pixels": rng.integers(0, 256, (T, 16, 16, 3), dtype=np.uint8), "state": rng.standard_normal((T, 4)).astype(np.float32)}
        ring.insert(dict(observations=obs, next_observations=obs, actions=np.zeros(2, np.float32), rewards=0.0, masks=1.0, dones=done))

    m, mid_wraps = 1.0, 0
    for k in range(70):                                       # episodes of 7 and an unfinished one: wraps end and mid-episode
        mid_wraps += ring._insert_index == 0 and len(ring) == cap and not ring._first
        insert(done=(k % 7 == 6) and k < 60)
        if k % 9 == 4:
            ring.flush()
            valid = _host(ring.valid).astype(bool)
            slots = np.flatnonzero(valid)[:6]
            ring.update_priorities(np.concatenate([slots, slots[:2]]), rng.standard_normal(slots.size + min(2, slots.size)) * 4)
            torch.cuda.synchronize()
            m = float(ring.max_priority_dev.item())
        ring.flush()
        leaves = _check_tree(ring.tree, cap)
        valid = _host(ring.valid).astype(bool)
        assert (leaves[~valid] == 0).all(), "a slot made invalid kept its priority"
        assert (leaves[valid] > 0).all()
    assert m > 1.0 and mid_wraps > 0
    last = _host(ring.tree)
    path = tmp_path / "ring.npz"
    ring.save(path)
    again = MemoryEfficientReplayBuffer(space, Box((2,)), cap, seed=9, priority_alpha=0.5)
    again.load(path)
    np.testing.assert_array_equal(_host(again.tree).view(np.uint32), last.view(np.uint32))
    assert again.priority_beta == pytest.approx(0.3) and float(again.max_priority_dev.item()) == np.float32(m)
    uniform = MemoryEfficientReplayBuffer(space, Box((2,)), cap, seed=9)
    with pytest.raises(ValueError, match="priority_alpha"):
        uniform.load(path)
    with pytest.raises(ValueError, match="priority_eps"):
        MemoryEfficientReplayBuffer(space, Box((2,)), cap, priority_alpha=0.5, priority_eps=1e-3).load(path)
    uniform.save(tmp_path / "u.npz")
    with pytest.raises(ValueError, match="priority_alpha"):
        again.load(tmp_path / "u.npz")


# ---- refusals --------------------------------------------------------------------------------------------------------------
def test_refusals():
    from helpers import Box
    from serl_b200 import _lib as L
    from serl_b200.data.data_parallel import DataParallelDataStore
    from serl_b200.data.replay_buffer import ReplayBuffer, refuse_prioritized
    from serl_b200.utils.train_utils import concat_batches
    ring = ReplayBuffer(Box((3,)), Box((2,)), 16, priority_alpha=0.6)
    plain = ReplayBuffer(Box((3,)), Box((2,)), 16)
    for r in (ring, plain):
        for _ in range(6):
            r.insert(dict(observations=np.ones(3, np.float32), next_observations=np.ones(3, np.float32), actions=np.zeros(2, np.float32),
                          rewards=1.0, masks=1.0, dones=False))
    mixed = concat_batches(plain.sample(4), ring.sample(4), axis=0)
    refuse_prioritized(plain.sample(4), "x")
    with pytest.raises(NotImplementedError, match="prioritized"):
        refuse_prioritized(mixed, "SACAgent.update")
    with pytest.raises(NotImplementedError, match="prioritized"):       # a consumer that does not take the rows' priorities
        ring.launch_sample(mixed.parts[1], L.BatchOut(), crop_total=8, out_row_offset=4)
    with pytest.raises(NotImplementedError, match="data-parallel"):
        DataParallelDataStore(ring)
    with pytest.raises(ValueError, match="draws uniformly"):
        plain.update_priorities([0], [1.0])
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
    from helpers import DictSpace
    with pytest.raises(NotImplementedError, match="shard"):
        MemoryEfficientReplayBuffer(DictSpace({"pixels": Box((1, 16, 16, 3), np.uint8)}), Box((2,)), 16, priority_alpha=0.6,
                                    frame_shard=(0, 2))


@pytest.mark.parametrize("cap", [1100, 40000])                   # 3- and 5-level trees
def test_prioritized_draw_deep_tree(cap):
    from oracle import per as P
    dev, ora = _prio_ring(0, 1, 1, 1, 1, cap, seed=cap)
    B, off = 300, 0
    res, _ = _launch_prio(dev, batch=B, B_total=B, off=off, step=9, n_step=1)
    tree = _host(dev.tree)
    idx = P.draw(tree, cap, dev._seed, 9, B, valid=ora.valid)
    assert (idx >= 0).all()
    np.testing.assert_array_equal(res["idx"], idx)
    np.testing.assert_array_equal(res["prio"].view(np.uint32), tree[idx].view(np.uint32))
    np.testing.assert_array_equal(res["rewards"].view(np.uint32), ora.rewards[idx].view(np.uint32))


def test_invalid_slots_are_never_drawn_or_reprioritized():
    """A learner may write a TD error back to a slot that an insert has made invalid since the draw: the leaf stays 0.  And a
    non-zero leaf on a slot that is not valid (written through the raw C entry point) costs the draw an attempt."""
    from oracle import per as P
    from serl_b200 import ops
    cap = 48
    dev, ora = _prio_ring(1, 1, 84, 84, 3, cap, seed=11)
    bad = np.flatnonzero(ora.valid)[:6]
    dev.valid[torch.from_numpy(bad).long().cuda()] = 0          # made invalid behind the learner's back (leaves still > 0)
    ora.valid[bad] = False
    dev.update_priorities(bad[:3], [5.0, 6.0, 7.0])              # through the ring: the validity check writes 0
    torch.cuda.synchronize()
    leaves = _check_tree(dev.tree, cap)
    assert (leaves[bad[:3]] == 0).all() and (leaves[bad[3:]] > 0).all()
    res, (k_obs, k_next) = _launch_prio(dev, batch=40, B_total=40, off=0, step=2, n_step=1)
    idx = P.draw(_host(dev.tree), cap, dev._seed, 2, 40, valid=ora.valid)
    ok = idx >= 0                                # a stratum whose mass sits on invalid slots fails its row, and says so
    np.testing.assert_array_equal(res["idx"][ok], idx[ok])
    assert ora.valid[idx[ok]].all() and ok.sum() > 20 and (res["status"][0] != 0) == (not ok.all())
    td = torch.tensor([1.0, float("nan"), float("inf")], device="cuda")     # non-finite TD errors leave their leaves alone
    slots = torch.from_numpy(np.flatnonzero(ora.valid)[:3].astype(np.int32)).cuda()
    before = _host(dev.tree)
    ops.priority_set(dev.priority_tree(), slots, 3, td=td, alpha=0.7, eps=1e-6)
    after = _check_tree(dev.tree, cap)
    s = _host(slots)
    assert after[s[0]] != before[s[0]] and after[s[1]] == before[s[1]] and after[s[2]] == before[s[2]]
    w = torch.empty(3, device="cuda")                            # an explicit index on a zero leaf weighs 0, the others stay finite
    ops.priority_weights(torch.tensor([0.0, 2.0, 1.0], device="cuda"), 3, torch.full((1,), 1.0, device="cuda"), w)
    np.testing.assert_array_equal(_host(w), [0.0, 0.5, 1.0])
