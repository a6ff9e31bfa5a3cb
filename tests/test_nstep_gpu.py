"""GPU: n-step replay targets (serl_replay_sample_crop_nstep) against oracle/nstep.py, and the critic step on n-step batches.

* Kernel vs oracle, at the frame shapes that select each sampler kernel, n in {1, 2, 3, 5}, one and two cameras, state and
  pixel-only rings, and RLPD halves of one output batch: indices, window lengths, next-observation slots, dones, frames, crops
  and state rows bit for bit; rewards and masks bit for bit against the oracle's fp32 restatement in the kernel's documented
  order (and within 1e-6 of its float64 values).  n = 1 equals serl_replay_sample_crop bit for bit.
* Graph replay: a captured sampler launch sees transitions inserted (episode ends included) between replays.
* The critic step: `update_critics` on an n-step batch vs oracle/drq.py fed the oracle's n-step batch; the pipelined path vs
  the serial one, and `update_high_utd(utd_ratio=4)` on an n-step handle vs the same call on the oracle's batch, with the
  pretrained ResNet-10 and the "small" encoder.
"""
import numpy as np
import pytest
import torch

from helpers import Box, fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, to_numpy_tree
from test_replay_sampler_paths_gpu import A_DIM, PAD, S_DIM, SENTINEL, _all_offsets, _keys, _ring

pytestmark = pytest.mark.gpu
GAMMA = 0.97


def _outputs(dev, B_total):
    cams, (H, W, Cc), T = dev.cams, dev.frame_shape, dev.T

    def sent(*shape, dt=torch.uint8):
        t = torch.empty(*shape, dtype=dt, device="cuda")
        t.view(torch.uint8).fill_(SENTINEL)
        return t

    nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device="cuda")
    bufs = dict(obs_state=nan(B_total, max(T * dev.S, 1)), next_state=nan(B_total, max(T * dev.S, 1)), actions=nan(B_total, dev.A),
                rewards=nan(B_total), masks=nan(B_total), dones=sent(B_total), idx=sent(B_total, dt=torch.int32),
                off_obs=sent(B_total * T, 2, dt=torch.int32), off_next=sent(B_total * T, 2, dt=torch.int32),
                status=torch.zeros(1, dtype=torch.int32, device="cuda"), m=sent(B_total, dt=torch.int32),
                next_idx=sent(B_total, dt=torch.int32))
    pix = {(c, w): sent(B_total, T, H, W, Cc) for c in cams for w in ("obs", "next")}
    return bufs, pix


def _bind(bufs, pix, cams):
    from serl_b200 import _lib as L
    out = L.BatchOut()
    for j, c in enumerate(cams):
        out.obs_pix[j], out.next_pix[j] = pix[(c, "obs")].data_ptr(), pix[(c, "next")].data_ptr()
    for name in ("obs_state", "next_state", "actions", "rewards", "masks", "dones", "idx", "off_obs", "off_next", "status"):
        setattr(out, name, bufs[name].data_ptr())
    return out


def _launch(launches, B_total, keys, expl=None):
    """launches: [(ring, part, out_row_offset)] into ONE set of B_total-row outputs.  Returns numpy outputs."""
    dev0 = launches[0][0]
    bufs, pix = _outputs(dev0, B_total)
    out = _bind(bufs, pix, dev0.cams)
    k = torch.from_numpy(np.stack(keys).astype(np.uint32).reshape(-1).view(np.int32)).cuda()
    expl_t = None if expl is None else tuple(torch.as_tensor(e, dtype=torch.int32).cuda() for e in expl)
    for ring, part, off in launches:
        ring.launch_sample(part, out, crop_total=B_total * ring.T, out_row_offset=off, key_obs=k.data_ptr(), key_next=k.data_ptr() + 8,
                           explicit_off=expl_t, record_event=False, nstep_out=(bufs["m"], bufs["next_idx"]))
    torch.cuda.synchronize()
    res = {n: v.cpu().numpy() for n, v in bufs.items()}
    res["pix"] = {n: v.cpu().numpy() for n, v in pix.items()}
    return res


def _check(ora, res, rows, idx, n, off_obs, off_next):
    from oracle.nstep import nstep_batch
    from oracle.replay import random_shift
    T = ora.T
    want = nstep_batch(ora, idx, n, GAMMA)
    bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)
    np.testing.assert_array_equal(res["idx"][rows], idx)
    assert res["status"][0] == 0
    if n > 1:
        np.testing.assert_array_equal(res["m"][rows], want["m"])
        np.testing.assert_array_equal(res["next_idx"][rows], want["next_idx"])
    else:
        assert (res["m"].view(np.uint8) == SENTINEL).all()          # the n = 1 path is the one-step kernel
    np.testing.assert_array_equal(res["dones"][rows], want["dones"].astype(np.uint8))
    np.testing.assert_array_equal(bits(res["rewards"][rows]), bits(want["rewards32"]))
    np.testing.assert_array_equal(bits(res["masks"][rows]), bits(want["masks32"]))
    np.testing.assert_allclose(res["rewards"][rows], want["rewards"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(res["masks"][rows], want["masks"], rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(bits(res["actions"][rows]), bits(want["actions"]))
    if ora.state.shape[-1]:
        np.testing.assert_array_equal(bits(res["obs_state"][rows]), bits(want["observations"]["state"].reshape(len(rows), -1)))
        np.testing.assert_array_equal(bits(res["next_state"][rows]), bits(want["next_observations"]["state"].reshape(len(rows), -1)))
    g = (rows[:, None] * T + np.arange(T)[None, :]).reshape(-1)
    for c in ora.image_keys:
        H, W, Cc = ora.frames[c].shape[1:]
        np.testing.assert_array_equal(res["off_obs"][g], off_obs[g])
        np.testing.assert_array_equal(res["off_next"][g], off_next[g])
        for which, offs, key in (("obs", off_obs, "observations"), ("next", off_next, "next_observations")):
            exp = random_shift(want[key][c].reshape(-1, H, W, Cc), offs[g], PAD)
            np.testing.assert_array_equal(res["pix"][(c, which)][rows].reshape(-1, H, W, Cc), exp, err_msg=f"{c} {which}")
    return want


def _set_head(dev, ora, head):
    ora.cursor = head
    dev.head_dev.fill_(head)
    dev._insert_index = dev._head_mirror = head


# (cameras, T, H, W, C): the frame kernel (one and two cameras, a frame stack), the banded kernel, the bytewise kernel
SHAPES = [pytest.param(1, 1, 128, 128, 3, id="frame-128-1cam"), pytest.param(2, 1, 128, 128, 3, id="frame-128-2cam"),
          pytest.param(2, 2, 64, 64, 3, id="frame-64-T2"), pytest.param(1, 1, 256, 128, 3, id="banded-256x128"),
          pytest.param(1, 1, 84, 84, 3, id="byte-84")]


@pytest.mark.parametrize("n", [1, 2, 3, 5])
@pytest.mark.parametrize("ncam,T,H,W,C", SHAPES)
def test_nstep_kernel_matches_oracle(ncam, T, H, W, C, n):
    from oracle import jax_prng as P
    from oracle.replay import draw_indices
    cap, B = 97, 40
    dev, ora = _ring(ncam, T, H, W, C, cap, seed=n)
    for head, step in ((cap // 3, 2), (0, 5)):                       # mid-ring newest slot, and a ring that just wrapped
        _set_head(dev, ora, head)
        k_obs, k_next = _keys(head)
        part = dict(ring=dev, seed=dev._seed, step=step, batch=B, indx=None, n_step=n, discount=GAMMA if n > 1 else None)
        res = _launch([(dev, part, 0)], B, (k_obs, k_next))
        idx = draw_indices(dev._seed, step, B, ora.size, ora.valid)
        _check(ora, res, np.arange(B), idx, n, P.crop_offsets(k_obs, B * T), P.crop_offsets(k_next, B * T))
        # every (cy, cx) pair
        expl = (_all_offsets(B * T, 10, 1), _all_offsets(B * T, 7, 3))
        res = _launch([(dev, part, 0)], B, (k_obs, k_next), expl)
        _check(ora, res, np.arange(B), idx, n, *expl)


def _nstep_launch_direct(dev, part, B, keys, expl):
    """serl_replay_sample_crop_nstep called directly, n = part's n_step (also for n = 1)."""
    import ctypes as C
    from serl_b200 import _lib as L
    bufs, pix = _outputs(dev, B)
    out = _bind(bufs, pix, dev.cams)
    k = torch.from_numpy(np.stack(keys).astype(np.uint32).reshape(-1).view(np.int32)).cuda()
    e = tuple(torch.as_tensor(x, dtype=torch.int32).cuda() for x in expl)
    rq = L.SampleRequest()
    rq.seed, rq.step, rq.batch, rq.size_dev = part["seed"], part["step"], B, dev.size_dev.data_ptr()
    rq.key_obs, rq.key_next, rq.explicit_off_obs, rq.explicit_off_next = k.data_ptr(), k.data_ptr() + 8, e[0].data_ptr(), e[1].data_ptr()
    rq.crop_total, rq.padding = B * dev.T, PAD
    ns = L.NStepDesc()
    ns.n, ns.discount, ns.head_dev, ns.m_out, ns.next_idx_out = part["n_step"], GAMMA, dev.head_dev.data_ptr(), bufs["m"].data_ptr(), bufs["next_idx"].data_ptr()
    v = dev.view()
    L.call("serl_replay_sample_crop_nstep", C.byref(v), C.byref(rq), C.byref(ns), C.byref(out), L.stream_ptr())
    torch.cuda.synchronize()
    return {n: t.cpu().numpy() for n, t in bufs.items()}, {n: t.cpu().numpy() for n, t in pix.items()}


@pytest.mark.parametrize("ncam,T,H,W,C", [SHAPES[1], SHAPES[2], SHAPES[3], SHAPES[4]])
def test_nstep_entry_point_with_n1_equals_the_one_step_kernel(ncam, T, H, W, C):
    """The n-step kernels at n = 1 (called directly: the rings route n = 1 to serl_replay_sample_crop) write what it writes."""
    dev, ora = _ring(ncam, T, H, W, C, 61, seed=3)
    _set_head(dev, ora, 17)
    B = 24
    expl = (_all_offsets(B * T, 10, 1), _all_offsets(B * T, 7, 3))
    part = dict(ring=dev, seed=dev._seed, step=4, batch=B, indx=None, n_step=1, discount=None)
    res, pix = _nstep_launch_direct(dev, part, B, _keys(1), expl)
    one = _launch([(dev, part, 0)], B, _keys(1), expl)
    for name in ("obs_state", "next_state", "actions", "rewards", "masks", "dones", "idx", "off_obs", "off_next"):
        np.testing.assert_array_equal(res[name].view(np.uint8), one[name].view(np.uint8), err_msg=name)
    for k in pix:
        np.testing.assert_array_equal(pix[k], one["pix"][k])
    np.testing.assert_array_equal(res["m"], 1)
    np.testing.assert_array_equal(res["next_idx"], res["idx"])


def _state_ring(cap, seed):
    from oracle.replay import OracleFrameRing
    from serl_b200.data.replay_buffer import ReplayBuffer
    dev = ReplayBuffer(Box((S_DIM,)), Box((A_DIM,)), cap, seed=seed + 100)
    ora = OracleFrameRing(cap, (), (1, 1, 1), 1, S_DIM, A_DIM)
    rng = np.random.default_rng(seed)
    ora.state = rng.standard_normal((cap, 1, S_DIM)).astype(np.float32)
    ora.next_state = rng.standard_normal((cap, 1, S_DIM)).astype(np.float32)
    ora.actions = rng.uniform(-1, 1, (cap, A_DIM)).astype(np.float32)
    ora.rewards = rng.standard_normal(cap).astype(np.float32)
    ora.masks = (rng.random(cap) < 0.8).astype(np.float32)
    ora.dones = rng.random(cap) < 0.15
    ora.valid[:] = True
    ora.size = cap
    dev.state.copy_(torch.from_numpy(ora.state.reshape(cap, -1)))
    dev.next_state.copy_(torch.from_numpy(ora.next_state.reshape(cap, -1)))
    for name in ("actions", "rewards", "masks"):
        getattr(dev, name).copy_(torch.from_numpy(getattr(ora, name)))
    dev.dones.copy_(torch.from_numpy(ora.dones.astype(np.uint8)))
    dev.valid.fill_(1)
    dev._valid_host[:] = True
    dev._size = cap
    dev.size_dev.fill_(cap)
    return dev, ora


@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_state_ring_and_rlpd_halves(n):
    """A state-only ring (make_sac_agent's), and two pixel rings filling the two halves of one RLPD batch."""
    from oracle.replay import draw_indices
    dev, ora = _state_ring(70, n)
    _set_head(dev, ora, 31)
    B = 50
    part = dict(ring=dev, seed=dev._seed, step=1, batch=B, indx=None, n_step=n, discount=GAMMA if n > 1 else None)
    res = _launch([(dev, part, 0)], B, _keys(0))
    _check(ora, res, np.arange(B), draw_indices(dev._seed, 1, B, ora.size, ora.valid), n, None, None)

    (d1, o1), (d2, o2) = _ring(2, 1, 128, 128, 3, 80, seed=11), _ring(2, 1, 128, 128, 3, 50, seed=12)
    _set_head(d1, o1, 44)
    _set_head(d2, o2, 3)
    half = 16
    expl = (_all_offsets(2 * half, 10, 1), _all_offsets(2 * half, 7, 3))
    p1 = dict(ring=d1, seed=d1._seed, step=6, batch=half, indx=None, n_step=n, discount=GAMMA if n > 1 else None)
    p2 = dict(p1, ring=d2, seed=d2._seed, step=9)
    res = _launch([(d1, p1, 0), (d2, p2, half)], 2 * half, _keys(2), expl)
    _check(o1, res, np.arange(half), draw_indices(d1._seed, 6, half, o1.size, o1.valid), n, *expl)
    _check(o2, res, half + np.arange(half), draw_indices(d2._seed, 9, half, o2.size, o2.valid), n, *expl)


def test_graph_replay_sees_inserts_made_after_capture():
    """A sampler launch captured in a CUDA graph reads the draw counter, the fill level and the insert index on the device:
    after each round of inserts (with an episode end among them) the replay equals an eager draw at the same step."""
    from serl_b200 import ops
    from serl_b200.utils.launcher import make_replay_buffer
    cams, B, n = ("a", "b"), 32, 3
    rb = make_replay_buffer(fake_env(cams, 32), capacity=90, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=5)
    trs = random_transitions(np.random.default_rng(2), 200, cams, 32, mean_ep=6)
    for tr in trs[:40]:
        rb.insert(tr)
    handle = rb.sample(B, n_step=n, discount=GAMMA)
    part = handle.parts[0]
    bufs, pix = _outputs(rb, B)
    out = _bind(bufs, pix, cams)
    key = torch.from_numpy(np.stack(_keys(4)).astype(np.uint32).reshape(-1).view(np.int32)).cuda()

    def body():
        rb.launch_sample(part, out, crop_total=B, out_row_offset=0, key_obs=key.data_ptr(), key_next=key.data_ptr() + 8,
                         step_dev=rb.step_dev, record_event=False, nstep_out=(bufs["m"], bufs["next_idx"]))
        ops.counter_add(rb.step_dev, 1)

    rb.step_dev.fill_(part["step"])
    body()                                                              # eager warm-up
    rb.step_dev.fill_(part["step"])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    pos, step, seen_done = 40, part["step"], False
    for rnd in range(6):
        for tr in trs[pos:pos + 23]:
            rb.insert(tr)
            seen_done |= bool(tr["dones"])
        pos += 23
        rb.flush()
        g.replay()
        torch.cuda.synchronize()
        got = {k: v.clone() for k, v in bufs.items()}
        got_pix = {k: v.clone() for k, v in pix.items()}
        eager = dict(part, step=step)
        res = _launch([(rb, eager, 0)], B, _keys(4))
        for name in ("idx", "m", "next_idx", "rewards", "masks", "dones", "obs_state", "next_state", "actions", "off_obs", "off_next"):
            np.testing.assert_array_equal(got[name].cpu().numpy().view(np.uint8), res[name].view(np.uint8), err_msg=f"round {rnd} {name}")
        for k in pix:
            np.testing.assert_array_equal(got_pix[k].cpu().numpy(), res["pix"][k], err_msg=f"round {rnd} {k}")
        assert int(rb.head_dev[0]) == rb._insert_index
        step += 1
    assert seen_done and len(rb) == 90                                   # episode ends and a wrap happened between replays


# ---- the critic step --------------------------------------------------------------------------------------------------------
def _drq_setup(cams, precision, encoder="resnet-pretrained", seed=42, cap=200, n_fill=260, agent=True):
    from oracle.replay import OracleFrameRing
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    rb = make_replay_buffer(fake_env(cams), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
    ora = OracleFrameRing(cap, cams, (128, 128, 3), 1, 7, 4)
    rng = np.random.default_rng(seed)
    trs = random_transitions(rng, n_fill, cams, mean_ep=8)
    for tr in trs:
        tr = dict(tr, rewards=np.float32(rng.standard_normal()))
        rb.insert(tr)
        ora.insert(tr)
    if not agent:
        return None, rb, ora
    agent = make_drq_agent(seed, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type=encoder, precision=precision)
    return agent, rb, ora


def _oracle_host_batch(ora, rb, step, B, n, discount):
    """The oracle's n-step batch of the handle drawn at `step`, in the layout oracle/drq.py takes (un-augmented, unpacked)."""
    from oracle.nstep import nstep_batch
    from oracle.replay import draw_indices
    idx = draw_indices(rb._seed, step, B, ora.size, ora.valid)
    nb = dict(nstep_batch(ora, idx, n, discount), idx=idx)
    return {"observations": nb["observations"], "next_observations": nb["next_observations"], "actions": nb["actions"],
            "rewards": nb["rewards32"], "masks": nb["masks32"], "dones": nb["dones"]}, nb


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("fp16", 1e-2)])
def test_update_critics_on_nstep_batches_matches_oracle(precision, tol):
    from oracle import drq as O
    from test_agent_gpu import G_TOL, _perturb
    cams, B, n = ("front", "wrist"), 16, 3
    agent, rb, ora = _drq_setup(cams, precision)
    _perturb(agent)
    ocfg = oracle_cfg_from_agent(agent)
    discount = agent.config["discount"]
    it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True, "n_step": n, "discount": discount})
    short = 0
    for step in range(3):                                              # eager, capture + replay, replay
        ostate = oracle_state_from_agent(agent)
        batch = next(it)
        host, nb = _oracle_host_batch(ora, rb, batch.parts[0]["step"], B, n, discount)
        short += int((nb["m"] < n).sum())
        agent, info = agent.update_critics(batch)
        oinfo = O.update_critics(ostate, ocfg, host)
        eng = agent._engines[B]
        np.testing.assert_array_equal(eng.idx.cpu().numpy(), nb["idx"])
        for cam in cams:
            pix = eng.pix[cam].cpu().numpy()
            np.testing.assert_array_equal(pix[:B], oinfo["_aug"]["observations"][cam][:, 0])
            np.testing.assert_array_equal(pix[B:], oinfo["_aug"]["next_observations"][cam][:, 0])
        np.testing.assert_array_equal(eng.rewards.cpu().numpy().view(np.uint32), host["rewards"].view(np.uint32))
        np.testing.assert_array_equal(eng.masks.cpu().numpy().view(np.uint32), host["masks"].view(np.uint32))
        for k in ("critic_loss", "predicted_qs", "target_qs"):
            np.testing.assert_allclose(float(info["critic"][k]), oinfo["critic"][k], rtol=tol, atol=tol * 0.1)
        if step == 0 and precision == "fp32":
            st = agent._store
            for leaf in st.spec:
                if leaf.group == 0:
                    ref = oinfo["_grads"]["critic"][leaf.path].numpy()
                    got = st.view(st.grad, leaf.path).cpu().numpy()
                    assert np.abs(got - ref).max() <= G_TOL * max(np.abs(ref).max(), 1e-8), leaf.path
    assert short > 0                                                   # some windows were cut by an episode end
    agent.check_status()


@pytest.mark.parametrize("encoder", ["resnet-pretrained", "small"])
def test_pipeline_and_high_utd_on_nstep_batches(encoder):
    from serl_b200.utils.train_utils import concat_batches
    cams, B, n, tol = ("front", "wrist"), 32, 3, 2e-5
    a_pipe, rb1, ora = _drq_setup(cams, "fp32", encoder)
    a_ser, rb2, _ = _drq_setup(cams, "fp32", encoder)
    _, demo1, _ = _drq_setup(cams, "fp32", encoder, seed=5, cap=120, n_fill=150, agent=False)
    _, demo2, _ = _drq_setup(cams, "fp32", encoder, seed=5, cap=120, n_fill=150, agent=False)
    a_pipe.pipeline_critic_steps = True
    sa = {"batch_size": B // 2, "pack_obs_and_next_obs": True, "n_step": n, "discount": a_pipe.config["discount"]}
    its = [r.get_iterator(sample_args=sa) for r in (rb1, demo1, rb2, demo2)]
    for step in range(6):
        a_pipe, i1 = a_pipe.update_critics(concat_batches(next(its[0]), next(its[1]), axis=0))
        a_ser, i2 = a_ser.update_critics(concat_batches(next(its[2]), next(its[3]), axis=0))
        e1, e2 = a_pipe._last_engine, a_ser._engines[B]
        for name in ("idx", "rewards", "masks", "actions"):
            assert torch.equal(getattr(e1, name), getattr(e2, name)), (step, name)
        for cam in cams:
            assert torch.equal(e1.pix[cam], e2.pix[cam]), (step, cam)
        l1, l2 = float(i1["critic"]["critic_loss"]), float(i2["critic"]["critic_loss"])
        assert abs(l1 - l2) <= tol * max(abs(l2), 1e-6), (step, l1, l2)
        p1, p2 = a_pipe._store.params, a_ser._store.params
        assert float((p1 - p2).abs().max()) <= tol * float(p2.abs().max()), step

    # update_high_utd(utd_ratio=4) on an n-step handle == the same call on the oracle's n-step batch as a dict
    h_agent, rb, ora = _drq_setup(cams, "fp32", encoder)
    d_agent, _, _ = _drq_setup(cams, "fp32", encoder)
    discount = h_agent.config["discount"]
    for _ in range(2):
        handle = rb.sample(B, pack_obs_and_next_obs=True, n_step=n, discount=discount)
        host, _ = _oracle_host_batch(ora, rb, handle.parts[0]["step"], B, n, discount)
        h_agent, ih = h_agent.update_high_utd(handle, utd_ratio=4)
        d_agent, id_ = d_agent.update_high_utd(to_numpy_tree(host), utd_ratio=4)
        np.testing.assert_array_equal(h_agent.state.rng, d_agent.state.rng)
        for k in ("critic_loss", "predicted_qs", "target_qs"):
            np.testing.assert_allclose(float(ih["critic"][k]), float(id_["critic"][k]), rtol=tol, atol=1e-7)
        p1, p2 = h_agent._store.params, d_agent._store.params
        assert float((p1 - p2).abs().max()) <= tol * float(p2.abs().max())
    h_agent.check_status()
