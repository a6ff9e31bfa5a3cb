"""GPU: saving and loading HBM replay rings (`save` / `load`, serl_b200/data/replay_io.py format) - bitwise round trips
against the uninterrupted ring and oracle/replay.py, draws that continue, integrity, the ring lock, bounded pinned staging,
and the pcb_insert learner's pause-and-save branch resumed in a fresh process state."""
import os
import pickle
import threading
import time
import types

import numpy as np
import pytest
import torch

from helpers import Box, fake_env, random_transitions, to_numpy_tree

pytestmark = pytest.mark.gpu

HOST_FIELDS = ("_size", "_insert_index", "_seed", "_draw_step", "_dev_step_mirror")


def _frame_ring(cams, cap, hw, T, seed=11):
    from serl_b200.utils.launcher import make_replay_buffer
    return make_replay_buffer(fake_env(cams, hw, T), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams),
                              seed=seed)


def _state_ring(cap, seed=11, S=7, A=4):
    from serl_b200.utils.launcher import make_replay_buffer
    env = types.SimpleNamespace(observation_space=Box((S,)), action_space=Box((A,)))
    return make_replay_buffer(env, capacity=cap, type="replay_buffer", seed=seed)


def _state_transitions(rng, n, S=7, A=4):
    return [dict(observations=rng.standard_normal(S).astype(np.float32), next_observations=rng.standard_normal(S).astype(np.float32),
                 actions=rng.uniform(-1, 1, A).astype(np.float32), rewards=np.float32(rng.random()), masks=np.float32(1.0),
                 dones=bool(rng.random() < 0.1)) for _ in range(n)]


def _snapshot(ring) -> dict:
    """Every device array (whole capacity) and every host bookkeeping field of a ring."""
    ring.flush()
    torch.cuda.synchronize()
    snap = {name: t.cpu().numpy().copy() for name, t in ring._io_arrays()}
    snap.update(size_dev=int(ring.size_dev.item()), step_dev=int(ring.step_dev.item()), _valid_host=ring._valid_host.copy())
    snap.update({k: getattr(ring, k) for k in (*HOST_FIELDS, *ring._IO_EMPTY)})
    return snap


def _assert_same(a: dict, b: dict):
    assert a.keys() == b.keys()
    for k in a:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]), err_msg=k)


def _assert_matches_oracle(ring, ora, cams):
    ring.flush()
    m = ora.size
    assert len(ring) == m and ring._insert_index == ora.cursor and ring._first == ora.episode_start
    np.testing.assert_array_equal(ring.valid.cpu().numpy()[:m].astype(bool), ora.valid[:m])
    for c in cams:
        np.testing.assert_array_equal(ring.frames[c].cpu().numpy()[:m], ora.frames[c][:m])
    np.testing.assert_array_equal(ring.state.cpu().numpy()[:m], ora.state.reshape(ora.capacity, -1)[:m])
    np.testing.assert_array_equal(ring.actions.cpu().numpy()[:m], ora.actions[:m])
    np.testing.assert_array_equal(ring.rewards.cpu().numpy()[:m], ora.rewards[:m])


def _mid_episode(trs, mid):
    tr = trs[-1]
    if mid:                                           # the last transition saved does not end its episode: _first is False
        tr["dones"], tr["masks"] = False, np.float32(1.0)
    else:
        tr["dones"], tr["masks"] = True, np.float32(0.0)
    return trs


# ---- 1. bitwise round trip ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cams,T,hw,cap,n,mid", [
    (("front",), 1, 128, 50, 30, False),              # partially filled
    (("front",), 1, 16, 40, 95, True),                # full after wrap-around, mid-episode
    (("front", "wrist"), 1, 128, 45, 100, True),
    (("front", "wrist"), 1, 16, 60, 41, True),
    (("a",), 2, 16, 37, 20, True),
    (("a",), 2, 16, 37, 90, False),
    (("a", "b"), 2, 12, 33, 80, True),
])
def test_frame_ring_round_trip_bitwise(tmp_path, cams, T, hw, cap, n, mid):
    from oracle.replay import OracleFrameRing
    rng = np.random.default_rng(n)
    trs = random_transitions(rng, n + cap, cams, hw, T, mean_ep=9)
    head, tail = _mid_episode(trs[:n], mid), trs[n:]
    ring, ora = _frame_ring(cams, cap, hw, T), OracleFrameRing(cap, cams, (hw, hw, 3), T, 7, 4)
    for tr in head:
        ring.insert(tr)
        ora.insert(tr)
    ring.sample(4, pack_obs_and_next_obs=True)         # a draw before the save: _draw_step 1
    ring.step_dev.fill_(17)                            # as left by CUDA-graph replays
    ring._dev_step_mirror = 17
    before = _snapshot(ring)
    assert before["_first"] is (not mid)
    assert before["_size"] == cap if n >= cap else before["_size"] < cap
    path = tmp_path / "ring.npz"
    size = ring.save(path)
    assert size == os.path.getsize(path)
    _assert_same(_snapshot(ring), before)              # saving changes nothing
    loaded = _frame_ring(cams, cap, hw, T, seed=999)
    for tr in random_transitions(np.random.default_rng(1), 7, cams, hw, T):    # a ring that was used before the load
        loaded.insert(tr)
    assert loaded.load(path) is loaded
    _assert_same(_snapshot(loaded), before)
    for tr in tail:                                    # both continue identically, and like the oracle
        ring.insert(tr)
        loaded.insert(tr)
        ora.insert(tr)
    _assert_same(_snapshot(loaded), _snapshot(ring))
    _assert_matches_oracle(loaded, ora, cams)


@pytest.mark.parametrize("n", [0, 25, 130])
def test_state_ring_round_trip_bitwise(tmp_path, n):
    from serl_b200.data.data_store import ReplayBufferDataStore
    cap = 64
    trs = _state_transitions(np.random.default_rng(n), n + 70)
    ring = _state_ring(cap)
    assert isinstance(ring, ReplayBufferDataStore)
    for tr in trs[:n]:
        ring.insert(tr)
    before = _snapshot(ring)
    ring.save(tmp_path / "state.npz")
    loaded = _state_ring(cap, seed=3).load(tmp_path / "state.npz")
    _assert_same(_snapshot(loaded), before)
    for tr in trs[n:]:
        ring.insert(tr)
        loaded.insert(tr)
    _assert_same(_snapshot(loaded), _snapshot(ring))
    last = trs[-1]                                     # the plain ring: slot = insert order modulo capacity
    np.testing.assert_array_equal(loaded.state.cpu().numpy()[(len(trs) - 1) % cap], last["observations"])


def test_np_load_reads_a_ring_file(tmp_path):
    cams = ("front", "wrist")
    ring = _frame_ring(cams, 30, 16, 1)
    for tr in random_transitions(np.random.default_rng(0), 20, cams, 16):
        ring.insert(tr)
    ring.save(tmp_path / "r.npz")
    with np.load(tmp_path / "r.npz") as z:
        assert z["frames/front"].shape == (len(ring), 16, 16, 3) and z["frames/front"].dtype == np.uint8
        np.testing.assert_array_equal(z["frames/wrist"], ring.frames["wrist"][:len(ring)].cpu().numpy())
        np.testing.assert_array_equal(z["valid"], ring.valid[:len(ring)].cpu().numpy())


# ---- 2. draws continue ------------------------------------------------------------------------------------------------
def _draw(ring, h, keys):
    """Indices, gathered fields and DrQ crops of a handle's part, with the crop keys `keys` (uint32[4]: obs, next)."""
    from serl_b200 import _lib as L
    part, (H, W, Cc) = h.parts[0], ring.frame_shape
    B, T = part["batch"], ring.T
    e = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")
    obs = {c: e(B, T, H, W, Cc, dt=torch.uint8) for c in ring.cams}
    nxt = {c: e(B, T, H, W, Cc, dt=torch.uint8) for c in ring.cams}
    bufs = dict(st=e(B, T * ring.S), nst=e(B, T * ring.S), ac=e(B, ring.A), rw=e(B), mk=e(B), dn=e(B, dt=torch.uint8),
                idx=e(B, dt=torch.int32), oo=e(B * T, 2, dt=torch.int32), on=e(B * T, 2, dt=torch.int32), status=e(1, dt=torch.int32))
    out = L.BatchOut()
    for j, c in enumerate(ring.cams):
        out.obs_pix[j], out.next_pix[j] = obs[c].data_ptr(), nxt[c].data_ptr()
    out.obs_state, out.next_state, out.actions = bufs["st"].data_ptr(), bufs["nst"].data_ptr(), bufs["ac"].data_ptr()
    out.rewards, out.masks, out.dones = bufs["rw"].data_ptr(), bufs["mk"].data_ptr(), bufs["dn"].data_ptr()
    out.idx, out.off_obs, out.off_next, out.status = (bufs["idx"].data_ptr(), bufs["oo"].data_ptr(), bufs["on"].data_ptr(),
                                                      bufs["status"].data_ptr())
    k = torch.from_numpy(np.asarray(keys, np.uint32).view(np.int32)).cuda()
    ring.launch_sample(part, out, crop_total=B * T, out_row_offset=0, key_obs=k.data_ptr(), key_next=k.data_ptr() + 8)
    torch.cuda.synchronize()
    assert int(bufs["status"].item()) == 0
    res = {f"obs/{c}": obs[c].cpu().numpy() for c in ring.cams}
    res.update({f"next/{c}": nxt[c].cpu().numpy() for c in ring.cams})
    res.update({k: v.cpu().numpy() for k, v in bufs.items()})
    res.update({f"dict/{k}": v for k, v in _flat(to_numpy_tree(h.to_dict())).items()})
    return res


def _flat(d, pre=""):
    out = {}
    for k, v in d.items():
        out.update(_flat(v, f"{pre}{k}/") if isinstance(v, dict) else {pre + k: v})
    return out


@pytest.mark.parametrize("cams,T", [(("front",), 1), (("front", "wrist"), 1), (("a",), 2)])
def test_draws_continue_after_load(tmp_path, cams, T):
    cap, hw, B, K = 70, 128 if T == 1 else 16, 32, 4
    ring = _frame_ring(cams, cap, hw, T, seed=123)
    for tr in random_transitions(np.random.default_rng(2), 160, cams, hw, T, mean_ep=9):
        ring.insert(tr)
    for _ in range(3):
        ring.sample(B, pack_obs_and_next_obs=True)
    ring.save(tmp_path / "r.npz")
    loaded = _frame_ring(cams, cap, hw, T, seed=5).load(tmp_path / "r.npz")
    rng = np.random.default_rng(9)
    for _ in range(K):
        keys = rng.integers(0, 2 ** 32, 4, dtype=np.uint64).astype(np.uint32)
        a = _draw(ring, ring.sample(B, pack_obs_and_next_obs=True), keys)
        b = _draw(loaded, loaded.sample(B, pack_obs_and_next_obs=True), keys)
        _assert_same(a, b)
        assert len(np.unique(a["idx"])) > 1 and not (a["oo"] == 4).all()     # real draws, real shifts


# ---- 3. integrity -----------------------------------------------------------------------------------------------------
def _assert_empty(ring):
    torch.cuda.synchronize()
    assert len(ring) == 0 and ring._insert_index == 0 and ring._first
    assert int(ring.size_dev.item()) == 0 and not ring.valid.any().item() and not ring._valid_host.any()


def _filled(cams=("front", "wrist"), cap=60, n=90, seed=0):
    ring = _frame_ring(cams, cap, 128, 1)
    for tr in random_transitions(np.random.default_rng(seed), n, cams):
        ring.insert(tr)
    return ring


@pytest.mark.parametrize("damage", ["flip", "truncate", "capacity", "cams"])
def test_damaged_or_mismatched_file_raises_and_leaves_the_ring_empty(tmp_path, damage):
    import zipfile
    ring = _filled()
    path = tmp_path / "r.npz"
    ring.save(path)
    target, match = _filled(seed=4), "frames/wrist"
    if damage == "flip":
        raw = bytearray(path.read_bytes())
        with zipfile.ZipFile(path) as zf:
            info = zf.getinfo("frames/wrist.npy")
        raw[info.header_offset + 200 + info.file_size // 2] ^= 1
        path.write_bytes(bytes(raw))
    elif damage == "truncate":
        path.write_bytes(path.read_bytes()[:os.path.getsize(path) - 1000])
        match = "not a complete zip archive"
    elif damage == "capacity":
        target, match = _frame_ring(("front", "wrist"), 61, 128, 1), "capacity"
    else:
        target, match = _frame_ring(("front", "side"), 60, 128, 1), "cams"
    with pytest.raises(ValueError, match=match):
        target.load(path)
    _assert_empty(target)
    target.insert(random_transitions(np.random.default_rng(1), 1, target.cams)[0])     # still a working ring
    assert len(target) == 2


def test_failed_save_leaves_the_previous_file(tmp_path, monkeypatch):
    from serl_b200.data import replay_buffer as RB
    ring = _filled()
    path = tmp_path / "r.npz"
    ring.save(path)
    before = path.read_bytes()
    for tr in random_transitions(np.random.default_rng(3), 5, ring.cams):
        ring.insert(tr)
    os.mkdir(str(path) + ".tmp")                      # the temporary cannot be created: an unwritable location
    with pytest.raises(OSError):
        ring.save(path)
    assert path.read_bytes() == before
    os.rmdir(str(path) + ".tmp")
    real = RB._CudaStager.d2h

    def failing(self, k, src, lo, hi):
        if lo > 0:
            raise RuntimeError("copy failed")
        return real(self, k, src, lo, hi)

    monkeypatch.setattr(RB._CudaStager, "d2h", failing)
    with pytest.raises(RuntimeError, match="copy failed"):
        ring.save(path, chunk_bytes=1 << 20)          # fails part-way through the frames
    assert path.read_bytes() == before and not os.path.exists(str(path) + ".tmp")
    with pytest.raises(OSError):
        ring.save(tmp_path / "no_such_dir" / "r.npz")


# ---- 4. concurrency ---------------------------------------------------------------------------------------------------
def test_insert_during_save_waits_for_the_snapshot(tmp_path, monkeypatch):
    from oracle.replay import OracleFrameRing
    from serl_b200.data import replay_io as RIO
    cams, cap = ("front", "wrist"), 60
    trs = random_transitions(np.random.default_rng(8), 71, cams)
    ring, ora = _frame_ring(cams, cap, 128, 1), OracleFrameRing(cap, cams, (128, 128, 3), 1, 7, 4)
    for tr in trs[:70]:
        ring.insert(tr)
        ora.insert(tr)
    before = _snapshot(ring)
    real, seen = RIO.write_ring_file, {}

    def writing(*a, **kw):                            # runs with the ring's lock held
        t = threading.Thread(target=ring.insert, args=(trs[70],))
        t.start()
        time.sleep(0.5)
        seen.update(alive=t.is_alive(), size=ring._size, cursor=ring._insert_index)
        seen["thread"] = t
        return real(*a, **kw)

    monkeypatch.setattr(RIO, "write_ring_file", writing)
    ring.save(tmp_path / "r.npz")
    seen["thread"].join(timeout=60)
    assert seen["alive"] and (seen["size"], seen["cursor"]) == (before["_size"], before["_insert_index"])
    monkeypatch.setattr(RIO, "write_ring_file", real)
    loaded = _frame_ring(cams, cap, 128, 1).load(tmp_path / "r.npz")
    _assert_same(_snapshot(loaded), before)            # the file is the pre-insert snapshot
    ora.insert(trs[70])
    _assert_matches_oracle(ring, ora, cams)            # and the insert landed afterwards


# ---- 5. bounded pinned staging ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [1 << 20, None])
def test_save_and_load_pin_two_chunks(tmp_path, monkeypatch, chunk):
    from serl_b200 import _lib as L
    from serl_b200.data import replay_io as RIO
    cams, hw = ("front", "wrist"), 128
    bound = 2 * (chunk or RIO.CHUNK_BYTES)
    slot_bytes = len(cams) * hw * hw * 3
    cap = 10 * (chunk or RIO.CHUNK_BYTES) // slot_bytes + 50
    ring = _frame_ring(cams, cap, hw, 1)
    g = torch.Generator(device="cuda").manual_seed(0)
    for c in cams:                                    # synthetic fill straight in HBM
        ring.frames[c].copy_(torch.randint(0, 256, ring.frames[c].shape, generator=g, device="cuda", dtype=torch.uint8))
    ring.state.normal_(generator=g)
    ring.valid.fill_(1)
    ring._valid_host[:] = True
    ring._size, ring._insert_index = cap, 0
    ring.size_dev.fill_(cap)
    pinned = []
    real_pin = L.pin
    monkeypatch.setattr(L, "pin", lambda t: pinned.append(t.numel() * t.element_size()) or real_pin(t))
    ring.save(tmp_path / "big.npz", chunk_bytes=chunk)
    assert os.path.getsize(tmp_path / "big.npz") >= 10 * bound // 2
    assert sum(pinned) <= bound and ring.io_pinned_bytes == bound
    loaded = _frame_ring(cams, cap, hw, 1)
    pinned.clear()
    loaded.load(tmp_path / "big.npz", chunk_bytes=chunk)
    assert sum(pinned) <= bound
    for c in cams:
        assert torch.equal(loaded.frames[c], ring.frames[c])
    assert torch.equal(loaded.state, ring.state)


# ---- 6. learner resume (examples/async_pcb_insert_drq/async_drq_randomized.py: the pause-and-save branch) ---------------
CAMS, CAP, BATCH = ("front", "wrist"), 48, 8


def _build(precision, agent_seed, trs, ring_seeds=(21, 22)):
    from serl_launcher.utils.launcher import make_drq_agent, make_replay_buffer
    env = fake_env(CAMS)
    agent = make_drq_agent(seed=agent_seed, sample_obs=trs[0]["observations"], sample_action=trs[0]["actions"],
                           image_keys=list(CAMS), encoder_type="resnet-pretrained", precision=precision)
    replay_buffer = make_replay_buffer(env, capacity=CAP, type="memory_efficient_replay_buffer", image_keys=list(CAMS), seed=ring_seeds[0])
    demo_buffer = make_replay_buffer(env, capacity=CAP, type="memory_efficient_replay_buffer", image_keys=list(CAMS), seed=ring_seeds[1])
    return agent, replay_buffer, demo_buffer


def _loop(agent, replay_buffer, demo_buffer, actor_stream, steps, log, critic_actor_ratio=4):
    """The learner loop's body (as in test_learner_loop_conformance.py), with the actor's inserts between iterations."""
    from serl_launcher.utils.train_utils import concat_batches
    single_buffer_batch_size = BATCH // 2
    demo_iterator = demo_buffer.get_iterator(sample_args={"batch_size": single_buffer_batch_size, "pack_obs_and_next_obs": True})
    replay_iterator = replay_buffer.get_iterator(sample_args={"batch_size": single_buffer_batch_size, "pack_obs_and_next_obs": True})
    for step in range(steps):
        for tr in next(actor_stream):
            replay_buffer.insert(tr)
        for critic_step in range(critic_actor_ratio - 1):
            batch = concat_batches(next(replay_iterator), next(demo_iterator), axis=0)
            agent, critics_info = agent.update_critics(batch)
            log.append(to_numpy_tree(critics_info))
        batch = concat_batches(next(replay_iterator), next(demo_iterator), axis=0)
        agent, update_info = agent.update_high_utd(batch, utd_ratio=1)
        log.append(to_numpy_tree(update_info))
    return agent


def _actor(trs, start, per_step=5):
    i = start
    while True:
        yield trs[i:i + per_step]
        i += per_step


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_learner_resume_matches_an_uninterrupted_run(tmp_path, monkeypatch, precision):
    from serl_b200.utils import checkpoints
    monkeypatch.chdir(tmp_path)                        # the script saves into its working directory
    N, M, PER = 4, 4, 5
    trs = random_transitions(np.random.default_rng(0), 40 + (N + M) * PER, CAMS, mean_ep=7)
    demo_path = tmp_path / "demo.pkl"
    with open(demo_path, "wb") as f:
        pickle.dump(trs[:25], f)

    def fresh(agent_seed):
        agent, replay_buffer, demo_buffer = _build(precision, agent_seed, trs)
        with open(demo_path, "rb") as f:
            for traj in pickle.load(f):
                demo_buffer.insert(traj)
        for tr in trs[25:40]:
            replay_buffer.insert(tr)
        return agent, replay_buffer, demo_buffer

    # uninterrupted: N + M iterations
    log_a = []
    agent_a, rb_a, db_a = fresh(42)
    agent_a = _loop(agent_a, rb_a, db_a, _actor(trs, 40), N + M, log_a)
    # interrupted after N: the pause-and-save branch, then a fresh learner restores both halves and runs M more
    log_b = []
    agent, replay_buffer, demo_buffer = fresh(42)
    agent = _loop(agent, replay_buffer, demo_buffer, _actor(trs, 40), N, log_b)
    update_steps = N
    checkpoints.save_checkpoint(str(tmp_path / "ckpt"), agent.state, step=update_steps, keep=100)
    replay_buffer.save("replay_buffer_learner.npz")
    demo_buffer.save("demo_buffer_learner.npz")
    del agent, replay_buffer, demo_buffer
    agent_b, rb_b, db_b = _build(precision, 7, trs, ring_seeds=(None, None))     # the script's rings: seeds from entropy
    agent_b = agent_b.replace(state=checkpoints.restore_checkpoint(str(tmp_path / "ckpt"), agent_b.state))
    rb_b.load("replay_buffer_learner.npz")
    db_b.load("demo_buffer_learner.npz")
    agent_b = _loop(agent_b, rb_b, db_b, _actor(trs, 40 + N * PER), M, log_b)
    agent_a.check_status()
    agent_b.check_status()

    # ring contents and draws: bitwise on every build
    for a, b in ((rb_a, rb_b), (db_a, db_b)):
        _assert_same(_snapshot(b), _snapshot(a))
        _assert_same(_flat(to_numpy_tree(b.sample(16, pack_obs_and_next_obs=True).to_dict())),
                     _flat(to_numpy_tree(a.sample(16, pack_obs_and_next_obs=True).to_dict())))
    assert len(log_a) == len(log_b)
    fa, fb = [_flat(x) for x in log_a], [_flat(x) for x in log_b]
    same = [x.keys() == y.keys() and all(np.array_equal(x[k], y[k]) for k in x) for x, y in zip(fa, fb)]
    bitwise_first_leg, bitwise_logs = all(same[:4 * N]), all(same)      # the first N iterations ran the same way in both runs
    sa, sb = agent_a._store, agent_b._store
    mask = torch.ones_like(sa.params, dtype=torch.bool)
    mask[sa.info_off:sa.info_off + 16] = False                         # the info gap holds no parameters
    main = mask.clone()
    main[sa.n_main:] = False                                           # params / target have no aux part
    state_equal = {name: torch.equal(getattr(sa, name)[m], getattr(sb, name)[m])
                   for name, m in (("params", main), ("target", main), ("m", mask), ("v", mask))}
    state_equal["counts"] = torch.equal(sa.counts, sb.counts) and agent_a.state.step == agent_b.state.step
    state_equal["rng"] = np.array_equal(np.asarray(agent_a.state.rng), np.asarray(agent_b.state.rng))
    print(f"[{precision}] resumed run bitwise equal to the uninterrupted one: losses/infos {bitwise_logs} (first {N} iterations, "
          f"before any restore: {bitwise_first_leg}), state {state_equal}")
    if precision == "fp32":
        assert bitwise_logs and all(state_equal.values()), state_equal
    else:
        for x, y in zip(fa, fb):
            for k in x:
                if k.endswith("_loss"):
                    assert abs(float(x[k]) - float(y[k])) <= 1e-2 * max(abs(float(x[k])), 1.0), (k, x[k], y[k])
