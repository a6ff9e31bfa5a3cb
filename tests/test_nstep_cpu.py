"""CPU: the n-step oracle (oracle/nstep.py) against a per-row loop written from the definition, and the host side of the
n-step option (argument checks, handle bookkeeping, refusals).  Kernel launches are replaced by a recorder."""
import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

GAMMA = 0.9


# ---- brute force: one row at a time, straight from the definition -------------------------------------------------------
def _brute(ring, i, n, discount, head):
    cap = ring.capacity
    newest = (head - 1) % cap

    def written(k):                   # slot i+k is at or behind the newest slot, counting forward from i
        return k <= (newest - i) % cap

    m = 1
    while m < n and written(m) and ring.valid[(i + m) % cap] and not ring.dones[(i + m - 1) % cap]:
        m += 1
    j = (i + m - 1) % cap
    R = sum(float(ring.rewards[(i + k) % cap]) * discount ** k for k in range(m))
    return m, j, R, discount ** (m - 1) * float(ring.masks[j]), bool(ring.dones[j])


def _check_against_brute(ring, idx, n, discount=GAMMA, head=None):
    from oracle.nstep import nstep_batch
    head = ring.cursor if head is None else head
    got = nstep_batch(ring, idx, n, discount, head)
    for r, i in enumerate(idx):
        m, j, R, mask, done = _brute(ring, int(i), n, discount, head)
        assert (got["m"][r], got["next_idx"][r], got["dones"][r]) == (m, j, done), (i, n)
        np.testing.assert_allclose(got["rewards"][r], R, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(got["masks"][r], mask, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(got["rewards32"][r], R, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(got["masks32"][r], mask, rtol=1e-6, atol=1e-6)
        np.testing.assert_array_equal(got["next_observations"]["state"][r], ring.next_state[j])
        packed = ring.gather_packed(np.array([j]))["observations"]
        for c in ring.image_keys:
            np.testing.assert_array_equal(got["next_observations"][c][r], packed[c][0, 1:])
            np.testing.assert_array_equal(got["observations"][c][r], ring.gather_packed(np.array([i]))["observations"][c][0, :-1])
    return got


def _hand_ring(cap, T=1, cams=()):
    from oracle.replay import OracleFrameRing
    ring = OracleFrameRing(cap, cams, (4, 4, 3), T, 2, 1)
    rng = np.random.default_rng(cap)
    ring.rewards = rng.standard_normal(cap).astype(np.float32)
    ring.masks = np.ones(cap, np.float32)
    ring.next_state = rng.standard_normal((cap, T, 2)).astype(np.float32)
    for c in cams:
        ring.frames[c] = rng.integers(0, 256, (cap, 4, 4, 3), dtype=np.uint8)
    ring.valid[:] = True
    return ring


def test_done_inside_at_end_and_at_the_drawn_slot():
    ring = _hand_ring(20)
    ring.cursor, ring.size = 0, 20                       # full ring, head at 0: slot 19 is the newest
    ring.dones[[3, 8, 12]] = True
    ring.masks[[3, 8]] = 0.0                             # terminations; 12 is a truncation (mask 1)
    got = _check_against_brute(ring, [1, 6, 8, 10, 12, 13], 3)
    assert list(got["m"]) == [3, 3, 1, 3, 1, 3]          # 1: done at the window's last slot 3; 6: done at 8 = last; 8, 12: at i
    assert got["masks"][0] == 0.0 and got["masks"][3] == pytest.approx(GAMMA ** 2)   # truncation at 12 still bootstraps
    got = _check_against_brute(ring, [2, 7, 11], 5)
    assert list(got["m"]) == [2, 2, 2]                   # a done mid-window stops it


def test_window_reaches_the_newest_slot_before_and_after_the_wrap():
    ring = _hand_ring(16)
    ring.cursor, ring.size = 9, 9                        # not wrapped: newest slot 8
    got = _check_against_brute(ring, [5, 6, 7, 8], 4)
    assert list(got["m"]) == [4, 3, 2, 1]
    ring.cursor, ring.size = 3, 16                       # wrapped: newest slot 2, windows cross slot 15 -> 0
    got = _check_against_brute(ring, [13, 14, 15, 0, 2], 5)
    assert list(got["m"]) == [5, 5, 4, 3, 1]
    assert list(got["next_idx"]) == [1, 2, 2, 2, 2]


def test_full_ring_overwritten_past_the_drawn_slot():
    ring = _hand_ring(12)
    ring.cursor, ring.size = 5, 12                       # slots 5.. are the oldest; slot 4 the newest
    got = _check_against_brute(ring, [5, 10, 11, 2, 3, 4], 3)
    assert list(got["m"]) == [3, 3, 3, 3, 2, 1]
    assert list(got["next_idx"]) == [7, 0, 1, 4, 4, 4]


def test_invalid_copies_of_a_mid_episode_wrap_end_the_window():
    ring = _hand_ring(10, T=2, cams=("a",))
    ring.cursor, ring.size = 5, 10
    ring.valid[[0, 1]] = False                           # the frame-dedup ring's re-inserted copies of slots 8, 9
    got = _check_against_brute(ring, [7, 8, 9, 2], 4)
    assert list(got["m"]) == [3, 2, 1, 3]


@pytest.mark.parametrize("T", [1, 2])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 16])
def test_oracle_matches_brute_force_on_inserted_rings(T, n):
    """Rings filled through the frame-dedup insert (episode fillers, wrap re-insert), at several fill levels."""
    from oracle.replay import OracleFrameRing
    cams = ("a", "b")
    rng = np.random.default_rng(10 * T + n)
    ring = OracleFrameRing(23, cams, (8, 8, 3), T, 7, 4)
    for s, tr in enumerate(random_transitions(rng, 70, cams, 8, T, mean_ep=5)):
        tr = dict(tr, rewards=np.float32(rng.standard_normal()))
        ring.insert(tr)
        if s % 9 == 8 and ring.size > T:
            idx = np.flatnonzero(ring.valid[:ring.size])
            got = _check_against_brute(ring, idx, n)
            if n == 1:
                np.testing.assert_array_equal(got["m"], 1)
                np.testing.assert_array_equal(got["rewards32"], ring.rewards[idx])
                np.testing.assert_array_equal(got["masks32"], ring.masks[idx])


def test_fp32_order_is_the_documented_one():
    from oracle.nstep import scalars
    r = np.array([1e8, 1.0, 1.0, 3.0], np.float32)
    got = scalars(np.array([0]), np.array([4]), capacity=4, rewards=r, masks=np.ones(4, np.float32), dones=np.zeros(4, bool),
                  discount=0.5)
    g, R = np.float32(1), r[0]
    for k in range(1, 4):
        g = np.float32(g * np.float32(0.5))
        R = np.float32(R + np.float32(g * r[k]))
    assert got["rewards32"][0] == R and got["masks32"][0] == np.float32(0.125)


# ---- host side of the option -------------------------------------------------------------------------------------------
@pytest.fixture()
def dry(monkeypatch):
    from serl_b200 import _lib as L
    calls = []
    real_call = L.call

    def fake_call(name, *args):
        if name.startswith("serl_host_"):
            return real_call(name, *args)
        calls.append((name, args))
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    monkeypatch.setattr(L, "call", fake_call)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(L, "new_event", lambda: Ev())
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: len(calls))
    return calls


def _rings(cams=("front",), hw=16):
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(cams, hw), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams),
                            device="cpu", seed=1)
    demo = make_replay_buffer(fake_env(cams, hw), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams),
                              device="cpu", seed=2)
    trs = random_transitions(np.random.default_rng(0), 30, cams, hw)
    for tr in trs:
        rb.insert(tr)
        demo.insert(tr)
    return rb, demo, trs


@pytest.mark.parametrize("bad", [0, 17, -1, 2.5, True, "3"])
def test_n_step_range(dry, bad):
    rb, _, _ = _rings()
    with pytest.raises(ValueError, match="n_step"):
        rb.sample(4, n_step=bad, discount=0.9)


def test_n_step_needs_a_discount(dry):
    rb, _, _ = _rings()
    with pytest.raises(ValueError, match="discount"):
        rb.sample(4, n_step=3)
    with pytest.raises(ValueError, match="discount"):
        next(rb.get_iterator(sample_args={"batch_size": 4, "n_step": 2}))
    h = rb.sample(4, n_step=1, discount=0.9)             # n = 1 needs none and records none
    assert h.n_step == (1, None) and rb.sample(4).n_step == (1, None)
    h = next(rb.get_iterator(sample_args={"batch_size": 4, "n_step": 3, "discount": 0.99}))
    assert h.n_step == (3, 0.99) and h.parts[0]["n_step"] == 3 and h.parts[0]["discount"] == 0.99


def test_concat_of_mixed_handles_raises(dry):
    from serl_b200.utils.train_utils import concat_batches
    rb, demo, _ = _rings()
    a = rb.sample(4, n_step=3, discount=0.99)
    assert concat_batches(a, demo.sample(4, n_step=3, discount=0.99), axis=0).n_step == (3, 0.99)
    for other in (demo.sample(4), demo.sample(4, n_step=2, discount=0.99), demo.sample(4, n_step=3, discount=0.9)):
        with pytest.raises(ValueError, match="n-step"):
            concat_batches(a, other, axis=0)


def test_launches_pick_the_entry_point_and_head_follows_inserts(dry):
    from serl_b200 import _lib as L
    rb, _, trs = _rings()
    rb.flush()
    assert int(rb.head_dev[0]) == rb._insert_index > 0
    out = L.BatchOut()
    del dry[:]
    rb.launch_sample(rb.sample(4).parts[0], out, crop_total=4, out_row_offset=0)
    rb.launch_sample(rb.sample(4, n_step=3, discount=0.99).parts[0], out, crop_total=4, out_row_offset=0)
    names = [c[0] for c in dry if c[0].startswith("serl_replay_sample")]
    assert names == ["serl_replay_sample_crop", "serl_replay_sample_crop_nstep"]
    ns = [c[1][2] for c in dry if c[0] == "serl_replay_sample_crop_nstep"][0]._obj
    assert (ns.n, ns.head_dev) == (3, rb.head_dev.data_ptr()) and ns.discount == pytest.approx(0.99)
    rb.insert(trs[0])
    rb.sample(4)                                          # sample flushes: head_dev is the new insert index
    assert int(rb.head_dev[0]) == rb._insert_index


def test_agent_checks_discount_and_refuses_backup_entropy(dry):
    from serl_b200.agents.continuous.sac import SACAgent
    from serl_b200.data.replay_buffer import ReplayBuffer
    from helpers import Box
    rng = np.random.default_rng(0)
    obs, act = rng.standard_normal(6).astype(np.float32), np.zeros(2, np.float32)
    rb = ReplayBuffer(Box((6,)), Box((2,)), 32, device="cpu", seed=0)
    for s in range(20):
        rb.insert(dict(observations=obs, next_observations=obs, actions=act, rewards=1.0, masks=1.0, dones=s % 7 == 6))
    agent = SACAgent.create_states(0, obs, act, discount=0.99, device="cpu")
    with pytest.raises(ValueError, match="discount"):
        agent.update(rb.sample(8, n_step=3, discount=0.9))
    agent.update(rb.sample(8, n_step=3, discount=0.99))
    assert any(c[0] == "serl_replay_sample_crop_nstep" for c in dry)
    ent = SACAgent.create_states(0, obs, act, discount=0.99, backup_entropy=True, device="cpu")
    with pytest.raises(NotImplementedError, match="backup_entropy"):
        ent.update(rb.sample(8, n_step=3, discount=0.99))
    ent.update(rb.sample(8))                              # one-step batches keep working


def test_vice_bc_and_classifier_refuse_n_step_batches(dry):
    """The guards run before anything else in these methods, so a stand-in `self` is enough to reach them."""
    from serl_b200.agents.continuous.bc import BCAgent
    from serl_b200.agents.continuous.vice import VICEAgent
    from serl_b200.networks.reward_classifier import RewardClassifier
    rb, _, _ = _rings()
    h = rb.sample(4, n_step=2, discount=0.96)
    for call in (lambda: VICEAgent.update_critics(object(), h), lambda: VICEAgent.update_high_utd(object(), h, utd_ratio=1),
                 lambda: VICEAgent.update_vice(object(), h), lambda: BCAgent.update(object(), h),
                 lambda: RewardClassifier.train_step(object(), h, None)):
        with pytest.raises(NotImplementedError, match="n-step"):
            call()
