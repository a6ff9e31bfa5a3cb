"""GPU: HBM replay ring + sampler kernel vs the oracle (bit-exact integers / bytes), through the C-ABI."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

pytestmark = pytest.mark.gpu


def _mk(cams, cap, hw, T=1, S=7, A=4, seed=11):
    from oracle.replay import OracleFrameRing
    from serl_b200.utils.launcher import make_replay_buffer
    env = fake_env(cams, hw, T, S, A)
    dev = make_replay_buffer(env, capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=seed)
    ora = OracleFrameRing(cap, cams, (hw, hw, 3), T, S, A)
    return dev, ora


def _fill(dev, ora, n, cams, hw, T=1, S=7, A=4, seed=0):
    rng = np.random.default_rng(seed)
    for tr in random_transitions(rng, n, cams, hw, T, S, A, mean_ep=9):
        dev.insert(tr)
        ora.insert(tr)
    dev.flush()


@pytest.mark.parametrize("cams,cap,hw,T,n", [(("front",), 97, 128, 1, 260), (("front", "wrist"), 61, 128, 1, 150),
                                              (("a",), 53, 8, 2, 200), (("a", "b"), 40, 12, 1, 41),
                                              (("a",), 37, 10, 1, 90)])            # 300-byte frames: the scatter's bytewise copy
def test_ring_storage_matches_oracle(cams, cap, hw, T, n):
    dev, ora = _mk(cams, cap, hw, T)
    _fill(dev, ora, n, cams, hw, T)
    assert len(dev) == ora.size and dev._insert_index == ora.cursor
    m = ora.size
    np.testing.assert_array_equal(dev.valid.cpu().numpy()[:m].astype(bool), ora.valid[:m])
    np.testing.assert_array_equal(dev._valid_host[:m], ora.valid[:m])
    for c in cams:
        np.testing.assert_array_equal(dev.frames[c].cpu().numpy()[:m], ora.frames[c][:m])
    np.testing.assert_array_equal(dev.state.cpu().numpy()[:m], ora.state.reshape(cap, -1)[:m])
    np.testing.assert_array_equal(dev.next_state.cpu().numpy()[:m], ora.next_state.reshape(cap, -1)[:m])
    np.testing.assert_array_equal(dev.actions.cpu().numpy()[:m], ora.actions[:m])
    np.testing.assert_array_equal(dev.rewards.cpu().numpy()[:m], ora.rewards[:m])
    np.testing.assert_array_equal(dev.masks.cpu().numpy()[:m], ora.masks[:m])
    np.testing.assert_array_equal(dev.dones.cpu().numpy()[:m].astype(bool), ora.dones[:m])
    assert int(dev.size_dev.item()) == m


@pytest.mark.parametrize("cams,cap,hw,T", [(("front",), 97, 128, 1), (("front", "wrist"), 61, 128, 1), (("a",), 53, 8, 2)])
def test_sample_indices_and_gather_bit_exact(cams, cap, hw, T):
    from oracle.replay import draw_indices
    dev, ora = _mk(cams, cap, hw, T, seed=77)
    _fill(dev, ora, 3 * cap, cams, hw, T)
    for step in range(3):
        h = dev.sample(64, pack_obs_and_next_obs=True)
        d = h.to_dict()
        idx = draw_indices(77, step, 64, ora.size, ora.valid)
        np.testing.assert_array_equal(d["_indices"].cpu().numpy(), idx)
        ref = ora.gather_packed(idx)
        for c in cams:
            np.testing.assert_array_equal(d["observations"][c].cpu().numpy(), ref["observations"][c])
            assert c not in d["next_observations"]
        np.testing.assert_array_equal(d["observations"]["state"].cpu().numpy(), ref["observations"]["state"])
        np.testing.assert_array_equal(d["next_observations"]["state"].cpu().numpy(), ref["next_observations"]["state"])
        for k in ("actions", "rewards", "masks"):
            np.testing.assert_array_equal(d[k].cpu().numpy(), ref[k])
        np.testing.assert_array_equal(d["dones"].cpu().numpy(), ref["dones"])


def test_valid_slot_zero_gathers_the_reference_window_in_bounds():
    """A valid slot idx < T (episode filler on the last slot, first transition on slot 0): the sampler must read the window the
    reference reads (slots capacity-2, capacity-1: numpy's negative window index) - and nothing in front of the frame buffer
    (compute-sanitizer caught the round-1 kernel reading slot -1)."""
    cams, cap, hw = ("front",), 10, 128
    dev, ora = _mk(cams, cap, hw, seed=5)
    rng = np.random.default_rng(3)
    for n in (8, 3):
        for i, tr in enumerate(random_transitions(rng, n, cams, hw, mean_ep=10 ** 9)):
            tr["dones"] = bool(i == n - 1)
            tr["masks"] = np.float32(1.0)
            dev.insert(tr)
            ora.insert(tr)
    dev.flush()
    assert ora.valid[0] and bool(dev.valid[0].item())
    idx = np.array([0, 1, 2, cap - 2, 0, 0], np.int32)
    part = dict(ring=dev, seed=5, step=0, batch=len(idx), indx=torch.as_tensor(idx).cuda())
    d = dev._gather_dict(part, True)
    ref = ora.gather_packed(idx.astype(np.int64))
    np.testing.assert_array_equal(d["observations"]["front"].cpu().numpy(), ref["observations"]["front"])
    np.testing.assert_array_equal(d["observations"]["front"].cpu().numpy()[0], ora.frames["front"][[cap - 2, cap - 1]])
    np.testing.assert_array_equal(d["observations"]["state"].cpu().numpy(), ref["observations"]["state"])


def _crop_call(dev, part, B, key_obs, key_next, T=1, expl=None):
    from serl_b200 import _lib as L
    cams, (H, W, Cc) = dev.cams, dev.frame_shape
    e = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")
    obs = {c: e(B, T, H, W, Cc, dt=torch.uint8) for c in cams}
    nxt = {c: e(B, T, H, W, Cc, dt=torch.uint8) for c in cams}
    out = L.BatchOut()
    for j, c in enumerate(cams):
        out.obs_pix[j], out.next_pix[j] = obs[c].data_ptr(), nxt[c].data_ptr()
    bufs = dict(st=e(B, T * dev.S), nst=e(B, T * dev.S), ac=e(B, dev.A), rw=e(B), mk=e(B), dn=e(B, dt=torch.uint8),
                idx=e(B, dt=torch.int32), oo=e(B * T, 2, dt=torch.int32), on=e(B * T, 2, dt=torch.int32), status=e(1, dt=torch.int32))
    out.obs_state, out.next_state, out.actions = bufs["st"].data_ptr(), bufs["nst"].data_ptr(), bufs["ac"].data_ptr()
    out.rewards, out.masks, out.dones = bufs["rw"].data_ptr(), bufs["mk"].data_ptr(), bufs["dn"].data_ptr()
    out.idx, out.off_obs, out.off_next, out.status = (bufs["idx"].data_ptr(), bufs["oo"].data_ptr(), bufs["on"].data_ptr(),
                                                      bufs["status"].data_ptr())
    keys = torch.from_numpy(np.concatenate([key_obs, key_next]).astype(np.uint32).view(np.int32)).view(torch.uint32).cuda()
    dev.launch_sample(part, out, crop_total=B * T, out_row_offset=0, key_obs=keys.data_ptr(), key_next=keys.data_ptr() + 8,
                      explicit_off=expl)
    torch.cuda.synchronize()
    assert int(bufs["status"].item()) == 0
    return obs, nxt, bufs


@pytest.mark.parametrize("cams,hw,T", [(("front",), 128, 1), (("front", "wrist"), 128, 1), (("a",), 8, 2), (("a",), 20, 1),
                                       (("a", "b", "c"), 128, 2)])
def test_drq_shift_bit_exact_and_keyed_like_jax(cams, hw, T):
    from oracle import jax_prng as P
    from oracle.replay import draw_indices, random_shift
    cap, B = 80, 48
    dev, ora = _mk(cams, cap, hw, T, seed=5)
    _fill(dev, ora, 200, cams, hw, T)
    k_obs, k_next = P.prng_key(123), P.prng_key(456)
    part = dict(ring=dev, seed=5, step=9, batch=B, indx=None)
    obs, nxt, bufs = _crop_call(dev, part, B, k_obs, k_next, T)
    idx = draw_indices(5, 9, B, ora.size, ora.valid)
    np.testing.assert_array_equal(bufs["idx"].cpu().numpy(), idx)
    off_o, off_n = P.crop_offsets(k_obs, B * T), P.crop_offsets(k_next, B * T)
    np.testing.assert_array_equal(bufs["oo"].cpu().numpy(), off_o)
    np.testing.assert_array_equal(bufs["on"].cpu().numpy(), off_n)
    assert not (off_o == off_n).all()
    packed = ora.gather_packed(idx)["observations"]
    for c in cams:                                     # same offsets for every camera of a sample (drq.py:245-252)
        fo = packed[c][:, :-1].reshape(B * T, hw, hw, 3)
        fn = packed[c][:, 1:].reshape(B * T, hw, hw, 3)
        np.testing.assert_array_equal(obs[c].cpu().numpy().reshape(B * T, hw, hw, 3), random_shift(fo, off_o))
        np.testing.assert_array_equal(nxt[c].cpu().numpy().reshape(B * T, hw, hw, 3), random_shift(fn, off_n))


def test_shift_edge_offsets_clamp():
    from oracle.replay import draw_indices, random_shift
    cams, hw, B = ("front",), 128, 9
    dev, ora = _mk(cams, 50, hw, 1, seed=3)
    _fill(dev, ora, 120, cams, hw, 1)
    offs = np.array([[0, 0], [8, 8], [0, 8], [8, 0], [4, 4], [1, 7], [7, 1], [4, 0], [0, 4]], dtype=np.int32)
    expl = (torch.as_tensor(offs).cuda(), torch.as_tensor(offs[::-1].copy()).cuda())
    part = dict(ring=dev, seed=3, step=0, batch=B, indx=None)
    key = np.zeros(2, np.uint32)
    obs, nxt, bufs = _crop_call(dev, part, B, key, key, 1, expl)
    idx = draw_indices(3, 0, B, ora.size, ora.valid)
    packed = ora.gather_packed(idx)["observations"]["front"]
    np.testing.assert_array_equal(obs["front"].cpu().numpy()[:, 0], random_shift(packed[:, 0], offs))
    np.testing.assert_array_equal(nxt["front"].cpu().numpy()[:, 0], random_shift(packed[:, 1], offs[::-1]))


def test_full_size_properties_100k():
    """BASELINE config 2 size (replay 100k x 1 cam in HBM, B=256): size-independent properties."""
    from serl_b200.utils.launcher import make_replay_buffer
    cams, hw, cap, B = ("front",), 128, 100_000, 256
    dev = make_replay_buffer(fake_env(cams, hw), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=1)
    # synthetic fill directly in HBM: frame of slot s is filled with byte (s % 251); episodes of 100 -> 1 filler per 101 slots
    slots = torch.arange(cap, device="cuda")
    dev.frames["front"].copy_((slots % 251).to(torch.uint8)[:, None, None, None].expand(cap, hw, hw, 3))
    valid = (slots % 101) != 0
    dev.valid.copy_(valid.to(torch.uint8))
    dev._valid_host[:] = valid.cpu().numpy()
    dev.state.copy_(slots[:, None].float().expand(cap, dev.S))
    dev._size = cap
    dev.size_dev.fill_(cap)
    seen = []
    for _ in range(4):
        d = dev.sample(B, pack_obs_and_next_obs=True).to_dict()
        idx = d["_indices"].cpu().numpy()
        seen.append(idx)
        assert (idx % 101 != 0).all() and idx.min() >= 1 and idx.max() < cap
        pix = d["observations"]["front"].cpu().numpy()
        assert (pix[:, 0] == ((idx - 1) % 251)[:, None, None, None]).all()       # obs frame = slot idx-1
        assert (pix[:, 1] == (idx % 251)[:, None, None, None]).all()             # next frame = slot idx
        assert (d["observations"]["state"].cpu().numpy()[:, 0, 0] == idx).all()
    assert len(np.unique(np.concatenate(seen))) > 0.98 * 4 * B                   # fresh draws every step
