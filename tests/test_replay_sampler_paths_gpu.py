"""GPU: every replay-sampler kernel against the oracle, bit for bit, at the frame geometries that select it.

`serl_replay_sample_crop` (serl_b200/csrc/sampler.cu) draws the indices, gathers the frame windows and applies the DrQ shift in
one launch, and its host dispatcher picks one of three kernels from the frame geometry:

  sample_frames_kernel               rows of 16-byte multiples, T <= 8, <= 8 bands of 32 rows whose buffers fit in 96 KiB
  sample_gather_crop_kernel<true>    rows of 16-byte multiples the frame kernel cannot hold, while one 32-row band fits in
                                     the device's opt-in shared memory
  sample_gather_crop_kernel<false>   every other row width, and rows too wide for one band in shared memory

Every case builds a ring directly in HBM (seeded random frames and fields, random validity) with the same arrays in an
`OracleFrameRing`, prefills the outputs with sentinels (0xA5 bytes, NaN floats), and checks the indices against
`draw_indices`, the crop offsets against `crop_offsets` (or the explicit offsets passed in), every camera's obs and next pixels
against `random_shift(gather_packed(idx))`, the small fields bitwise, and that rows outside the launch keep their sentinels.
The kernel that ran is read from torch.profiler, so a dispatcher change cannot move a case to another path unnoticed.
"""
import math
import re
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FRAME = "sample_frames_kernel"
BANDED, BYTE = "sample_gather_crop_kernel<true>", "sample_gather_crop_kernel<false>"
PAD, SPAN = 4, 9                                      # DrQ padding 4: offsets (cy, cx) in [0, 9)
S_DIM, A_DIM = 5, 3
SENTINEL = 0xA5

# all 81 (cy, cx) pairs; frame g of a launch gets pair (a*g + b) % 81, so any 81 consecutive frames take every pair once
_PAIRS = np.array([(cy, cx) for cy in range(SPAN) for cx in range(SPAN)], np.int32)


def _all_offsets(n_frames, a, b):
    return _PAIRS[(np.arange(n_frames) * a + b) % len(_PAIRS)]


# ---- ring ------------------------------------------------------------------------------------------------------------------
def _ring(ncam, T, H, W, C, cap, seed=0, valid=None):
    """A full MemoryEfficientReplayBuffer of shape (T, H, W, C) filled in HBM, and an OracleFrameRing holding the same arrays."""
    from helpers import Box, DictSpace
    from oracle.replay import OracleFrameRing
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
    cams = tuple(f"cam{j}" for j in range(ncam))
    space = DictSpace({**{c: Box((T, H, W, C), np.uint8) for c in cams}, "state": Box((T, S_DIM))})
    dev = MemoryEfficientReplayBuffer(space, Box((A_DIM,)), cap, pixel_keys=cams, seed=seed + 1000)
    ora = OracleFrameRing(cap, cams, (H, W, C), T, S_DIM, A_DIM)
    rng = np.random.default_rng(seed)
    for c in cams:
        ora.frames[c] = rng.integers(0, 256, (cap, H, W, C), dtype=np.uint8)
    ora.state = rng.standard_normal((cap, T, S_DIM)).astype(np.float32)
    ora.next_state = rng.standard_normal((cap, T, S_DIM)).astype(np.float32)
    ora.actions = rng.uniform(-1, 1, (cap, A_DIM)).astype(np.float32)
    ora.rewards = rng.standard_normal(cap).astype(np.float32)
    ora.masks = rng.random(cap).astype(np.float32)
    ora.dones = rng.random(cap) < 0.2
    ora.valid = (rng.random(cap) < 0.75) if valid is None else np.asarray(valid, bool)
    ora.size, ora.cursor = cap, 0
    for c in cams:
        dev.frames[c].copy_(torch.from_numpy(ora.frames[c]))
    dev.state.copy_(torch.from_numpy(ora.state.reshape(cap, -1)))
    dev.next_state.copy_(torch.from_numpy(ora.next_state.reshape(cap, -1)))
    for name in ("actions", "rewards", "masks"):
        getattr(dev, name).copy_(torch.from_numpy(getattr(ora, name)))
    dev.dones.copy_(torch.from_numpy(ora.dones.astype(np.uint8)))
    dev.valid.copy_(torch.from_numpy(ora.valid.astype(np.uint8)))
    dev._valid_host[:] = ora.valid
    dev._size = cap
    dev.size_dev.fill_(cap)
    torch.cuda.synchronize()
    return dev, ora


# ---- one sampling launch ---------------------------------------------------------------------------------------------------
_KERNEL_RE = re.compile(r"sample_frames_kernel|sample_gather_crop_kernel(?:<(true|false)>|ILb([01])E)")


def _sampler_kernels(prof):
    """Names of the sampler kernels a torch.profiler session recorded, one entry per launch (demangled or not)."""
    out = []
    for e in prof.events():
        m = _KERNEL_RE.search(e.name)
        if not m:
            continue
        if m.group(0).startswith("sample_gather_crop_kernel"):
            out.append(BANDED if (m.group(1) == "true" or m.group(2) == "1") else BYTE)
        else:
            out.append(m.group(0))
    return out


def _launch(dev, *, batch, B_total, off, step=0, keys=None, expl=None, indx=None):
    """One serl_replay_sample_crop call writing rows [off, off + batch) of B_total-row outputs prefilled with sentinels.
    Returns the outputs as numpy arrays and the sampler kernels it launched."""
    from serl_b200 import _lib as L
    cams, (H, W, Cc), T = dev.cams, dev.frame_shape, dev.T

    def sent(*shape, dt=torch.uint8):
        t = torch.empty(*shape, dtype=dt, device="cuda")
        t.view(torch.uint8).fill_(SENTINEL)
        return t

    def nan(*shape):
        return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")

    pix = {(c, w): sent(B_total, T, H, W, Cc) for c in cams for w in ("obs", "next")}
    bufs = dict(obs_state=nan(B_total, T * dev.S), next_state=nan(B_total, T * dev.S), actions=nan(B_total, dev.A),
                rewards=nan(B_total), masks=nan(B_total), dones=sent(B_total), idx=sent(B_total, dt=torch.int32),
                off_obs=sent(B_total * T, 2, dt=torch.int32), off_next=sent(B_total * T, 2, dt=torch.int32),
                status=torch.zeros(1, dtype=torch.int32, device="cuda"))
    out = L.BatchOut()
    for j, c in enumerate(cams):
        out.obs_pix[j], out.next_pix[j] = pix[(c, "obs")].data_ptr(), pix[(c, "next")].data_ptr()
    for name, t in bufs.items():
        setattr(out, name, t.data_ptr())
    k = np.zeros((2, 2), np.uint32) if keys is None else np.stack(keys).astype(np.uint32)
    key_t = torch.from_numpy(k.reshape(-1).view(np.int32)).cuda()
    expl_t = None if expl is None else tuple(torch.as_tensor(e, dtype=torch.int32).cuda() for e in expl)
    part = dict(ring=dev, seed=dev._seed, step=step, batch=batch,
                indx=None if indx is None else torch.as_tensor(np.asarray(indx), dtype=torch.int32).cuda())
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    # the profiler drops device records that fall outside its capture window as the host clock sees it, so the launch keeps
    # a margin from both ends of the window (without one, some launches went unrecorded)
    with torch.profiler.profile(activities=acts) as prof:
        time.sleep(0.02)
        dev.launch_sample(part, out, crop_total=B_total * T, out_row_offset=off, key_obs=key_t.data_ptr(),
                          key_next=key_t.data_ptr() + 8, explicit_off=expl_t, record_event=False)
        torch.cuda.synchronize()
        time.sleep(0.02)
    res = {k: v.cpu().numpy() for k, v in bufs.items()}
    res["pix"] = {k: v.cpu().numpy() for k, v in pix.items()}
    res["device_events"] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    return res, _sampler_kernels(prof)


def _check(ora, res, *, off, batch, idx, off_obs, off_next):
    """Compare one launch's outputs with the oracle.  idx: (batch,) oracle slots, -1 where the draw fails; off_obs/off_next:
    (crop_total, 2) offsets of every frame of the batch.  Rows outside the launch and failed rows must keep their sentinels."""
    from oracle.replay import random_shift
    T = ora.T
    B_total = res["rewards"].shape[0]
    ok = idx >= 0
    rows = off + np.flatnonzero(ok)                         # output rows the launch must have written
    untouched = np.setdiff1d(np.arange(B_total), rows)      # everything else keeps its sentinel
    outside = np.setdiff1d(np.arange(B_total), off + np.arange(batch))
    i_ok = idx[ok].astype(np.int64)
    assert (res["status"][0] != 0) == (not ok.all()), ("status", int(res["status"][0]))
    np.testing.assert_array_equal(res["idx"][rows], idx[ok])
    bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)
    np.testing.assert_array_equal(bits(res["obs_state"][rows]), bits(ora.state[i_ok].reshape(len(rows), -1)))
    np.testing.assert_array_equal(bits(res["next_state"][rows]), bits(ora.next_state[i_ok].reshape(len(rows), -1)))
    for name in ("actions", "rewards", "masks"):
        np.testing.assert_array_equal(bits(res[name][rows]), bits(getattr(ora, name)[i_ok]), err_msg=name)
    np.testing.assert_array_equal(res["dones"][rows], ora.dones[i_ok].astype(np.uint8))
    for name in ("obs_state", "next_state", "actions", "rewards", "masks"):
        assert np.isnan(res[name][untouched]).all(), f"{name}: a row outside the launch or with a failed draw was written"
    assert (res["dones"][untouched] == SENTINEL).all() and (res["idx"][untouched].view(np.uint8) == SENTINEL).all()
    # offsets: every frame of a written row; frames of rows outside the launch keep the sentinel
    g = (rows[:, None] * T + np.arange(T)[None, :]).reshape(-1)
    np.testing.assert_array_equal(res["off_obs"][g], off_obs[g])
    np.testing.assert_array_equal(res["off_next"][g], off_next[g])
    g_out = (outside[:, None] * T + np.arange(T)[None, :]).reshape(-1)
    assert (res["off_obs"][g_out].view(np.uint8) == SENTINEL).all() and (res["off_next"][g_out].view(np.uint8) == SENTINEL).all()
    packed = ora.gather_packed(i_ok)["observations"]
    H, W, Cc = ora.frames[ora.image_keys[0]].shape[1:]
    for c in ora.image_keys:
        for which, frames, offs in (("obs", packed[c][:, :-1], off_obs), ("next", packed[c][:, 1:], off_next)):
            got = res["pix"][(c, which)]
            want = random_shift(frames.reshape(-1, H, W, Cc), offs[g], PAD)
            np.testing.assert_array_equal(got[rows].reshape(-1, H, W, Cc), want, err_msg=f"{c} {which}")
            assert (got[untouched] == SENTINEL).all(), f"{c} {which}: a row outside the launch or with a failed draw was written"


def _keys(seed):
    from oracle import jax_prng as P
    return P.prng_key(seed), P.prng_key(seed + 7919)


def _run_keyed(dev, ora, *, batch, B_total, off, step, kernel, seed=0, indx=None):
    """Keyed crop offsets (the threefry chain on the device), drawn or explicit indices."""
    from oracle import jax_prng as P
    from oracle.replay import draw_indices
    k_obs, k_next = _keys(seed)
    res, ran = _launch(dev, batch=batch, B_total=B_total, off=off, step=step, keys=(k_obs, k_next), indx=indx)
    assert ran == [kernel], (ran, res["device_events"])
    n = B_total * ora.T
    idx = np.asarray(indx, np.int32) if indx is not None else draw_indices(dev._seed, step, batch, ora.size, ora.valid)
    _check(ora, res, off=off, batch=batch, idx=idx, off_obs=P.crop_offsets(k_obs, n), off_next=P.crop_offsets(k_next, n))
    return res


def _run_explicit(dev, ora, *, batch, B_total, off, step, kernel, indx=None):
    """Explicit offsets cycling through all 81 (cy, cx) pairs (every clamp and byte shift), drawn or explicit indices."""
    from oracle.replay import draw_indices
    n = B_total * ora.T
    expl = (_all_offsets(n, 10, 1), _all_offsets(n, 7, 3))
    res, ran = _launch(dev, batch=batch, B_total=B_total, off=off, step=step, keys=_keys(5), expl=expl, indx=indx)
    assert ran == [kernel], (ran, res["device_events"])
    idx = np.asarray(indx, np.int32) if indx is not None else draw_indices(dev._seed, step, batch, ora.size, ora.valid)
    _check(ora, res, off=off, batch=batch, idx=idx, off_obs=expl[0], off_next=expl[1])
    return res


# ---- geometry table --------------------------------------------------------------------------------------------------------
# (cameras, T, H, W, C, kernel).  Frame kernel: W*C % 16 == 0, T <= 8 and ceil(H/32) * (32*W*C + 32) <= 96 KiB.  Banded kernel:
# the rest of the 16-byte rows while 32*W*C + 32 (+ static shared memory) fits the 227 KiB opt-in limit.  Byte kernel: the rest.
GEOMETRIES = [
    pytest.param(1, 1, 128, 128, 3, FRAME, id="128x128x3"),
    pytest.param(2, 1, 128, 128, 3, FRAME, id="128x128x3-2cam"),
    pytest.param(2, 2, 128, 128, 3, FRAME, id="128x128x3-T2-2cam"),
    pytest.param(1, 3, 128, 128, 3, FRAME, id="128x128x3-T3"),
    pytest.param(1, 8, 128, 128, 3, FRAME, id="128x128x3-T8"),                # largest stack the frame kernel takes
    pytest.param(1, 1, 112, 112, 3, FRAME, id="112x112x3-partial-band"),      # last band 16 rows
    pytest.param(1, 1, 64, 176, 3, FRAME, id="64x176x3-33-chunks"),           # second pass of the 31-chunk row loop
    pytest.param(1, 1, 128, 128, 1, FRAME, id="128x128x1"),
    pytest.param(1, 1, 96, 96, 4, FRAME, id="96x96x4"),
    pytest.param(3, 1, 128, 128, 3, FRAME, id="128x128x3-3cam"),
    pytest.param(4, 1, 128, 128, 3, FRAME, id="128x128x3-4cam"),
    pytest.param(1, 1, 224, 128, 3, FRAME, id="224x128x3-7-bands"),           # 86,240 B: fits
    pytest.param(1, 1, 256, 128, 3, BANDED, id="256x128x3-8-bands"),          # 98,560 B: 256 B over the frame kernel's 96 KiB
    pytest.param(1, 1, 256, 256, 3, BANDED, id="256x256x3"),
    pytest.param(1, 9, 32, 32, 3, BANDED, id="32x32x3-T9"),                   # stack deeper than the frame kernel's 8
    pytest.param(1, 1, 48, 512, 3, BANDED, id="48x512x3-band-over-48KiB"),    # 49,184 B per band: needs the opt-in
    pytest.param(1, 1, 84, 84, 3, BYTE, id="84x84x3"),                        # 252-byte rows
    pytest.param(1, 1, 127, 127, 1, BYTE, id="127x127x1"),
    pytest.param(1, 1, 40, 2432, 3, BYTE, id="40x2432x3-band-over-optin"),    # 7,296-byte rows: a band needs 233,504 B
]


@pytest.mark.parametrize("ncam,T,H,W,C,kernel", GEOMETRIES)
def test_sampler_kernel_matches_oracle(ncam, T, H, W, C, kernel):
    """Keyed draws and offsets over a whole batch, then all 81 offset pairs at out_row_offset 3 inside a wider batch."""
    dev, ora = _ring(ncam, T, H, W, C, cap=48, seed=H * 7 + W + T)
    B = max(math.ceil(len(_PAIRS) / T), 9)
    _run_keyed(dev, ora, batch=B, B_total=B, off=0, step=3, kernel=kernel)
    _run_explicit(dev, ora, batch=B, B_total=B + 5, off=3, step=4, kernel=kernel)


# one geometry per kernel, at frame stacks 2 and 3
_STACKED = [(1, 128, 128, 3, FRAME), (1, 256, 128, 3, BANDED), (1, 84, 84, 3, BYTE)]


@pytest.mark.parametrize("ncam,H,W,C,kernel", _STACKED, ids=["frame", "banded", "byte"])
@pytest.mark.parametrize("T", [1, 2, 3])
def test_valid_slot_below_frame_stack_takes_numpys_negative_window(ncam, H, W, C, kernel, T):
    """A valid slot idx < T indexes numpy's sliding window at idx - T < 0, i.e. the LAST windows of the ring (as the reference
    does); the kernels must gather those slots, and nothing before the start of the frame buffer."""
    cap = 40
    dev, ora = _ring(ncam, T, H, W, C, cap=cap, seed=T)
    indx = np.array([0, 1, T - 1, T, cap - 1, 17, 0, T - 1], np.int32)
    _run_explicit(dev, ora, batch=len(indx), B_total=len(indx) + 3, off=1, step=0, kernel=kernel, indx=indx)
    _run_keyed(dev, ora, batch=len(indx), B_total=len(indx), off=0, step=0, kernel=kernel, seed=9, indx=indx)


@pytest.mark.parametrize("ncam,T,H,W,C,kernel", [(1, 1, 128, 128, 3, FRAME), (1, 9, 32, 32, 3, BANDED), (1, 1, 84, 84, 3, BYTE)],
                         ids=["frame", "banded", "byte"])
def test_failed_draws_set_status_and_leave_their_rows_alone(ncam, T, H, W, C, kernel):
    """One valid slot in 1,000: most lanes exhaust their 64 draws.  status must be 1, those rows must keep their sentinels,
    and the rows that found the slot must match the oracle."""
    from oracle.replay import draw_indices
    cap, batch = 1000, 64
    valid = np.zeros(cap, bool)
    valid[611] = True
    dev, ora = _ring(ncam, T, H, W, C, cap=cap, seed=1, valid=valid)
    idx = draw_indices(dev._seed, 2, batch, cap, valid)
    assert (idx < 0).any() and (idx >= 0).any()
    res = _run_keyed(dev, ora, batch=batch, B_total=batch + 4, off=2, step=2, kernel=kernel, seed=1)
    assert int(res["status"][0]) == 1
