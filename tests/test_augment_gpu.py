"""GPU: serl_b200.vision.data_augmentations against oracle/augment.py.

Crops, flips and solarize are compared bit for bit; colour jitter and blur to 2e-6 absolute of the float64 oracle on [0, 1]
images, with every random decision, drawn parameter and jitter order equal to the oracle's.  Every output is written into a
NaN- (or sentinel-) filled buffer with a guard band on both sides, and every function is checked for repeatability, CUDA-graph
capture and replay, and batched == per-image calls.  The crop is also pinned to the replay sampler's crops for the same key."""
import numpy as np
import pytest
import torch

from oracle import augment as A
from oracle import jax_prng as P

pytestmark = pytest.mark.gpu

GUARD = 256                     # elements of guard band on each side of an output
SENTINEL = 0xAB
TOL = 2e-6


def _key_rows(seed, n):
    return P.split(P.prng_key(seed), n) if n else np.zeros((0, 2), np.uint32)


def _dev_keys(k):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(k, np.uint32)).view(np.int32)).cuda()


class Guarded:
    """An output tensor inside a buffer prefilled with NaN (float) or SENTINEL bytes, GUARD elements of margin on each side."""

    def __init__(self, shape, dtype):
        n = int(np.prod(shape))
        self.buf = torch.empty(GUARD + n + GUARD, dtype=dtype, device="cuda")
        self.buf.view(torch.uint8).fill_(SENTINEL)
        if dtype.is_floating_point:
            self.buf.fill_(float("nan"))
        self.out = self.buf[GUARD:GUARD + n].view(shape)

    def check_guards(self):
        torch.cuda.synchronize()
        for g in (self.buf[:GUARD], self.buf[-GUARD:]):
            if g.dtype.is_floating_point:
                assert torch.isnan(g).all(), "a write landed in the guard band"
            else:
                assert (g.view(torch.uint8) == SENTINEL).all(), "a write landed in the guard band"


def _run(fn, x, keys, draws=None, **kw):
    """One launch of private launcher `fn` of the module into a guarded buffer; returns the output (guards checked) as numpy."""
    from serl_b200.vision import data_augmentations as DA
    g = Guarded(tuple(x.shape), x.dtype)
    args = (x, keys) if draws is None else (x, keys, draws)
    getattr(DA, fn)(*args, out=g.out, **kw)
    g.check_guards()
    return g.out.cpu().numpy()


def _images(seed, shape, dtype=torch.float32):
    rng = np.random.default_rng(seed)
    if dtype == torch.uint8:
        return torch.from_numpy(rng.integers(0, 256, shape, dtype=np.uint8)).cuda()
    return torch.from_numpy(rng.random(shape).astype(np.float32)).to(dtype).cuda()


# ---- crop -----------------------------------------------------------------------------------------------------------------------
def _check_crop(x, key, padding, nb):
    got = _run("_batched_crop", x, _dev_keys(key), padding=padding, num_batch_dims=nb)
    host = x.cpu()
    want = A.batched_random_crop(host.view(torch.uint8).numpy() if x.dtype == torch.uint8 else host.numpy(), key, padding, nb)
    np.testing.assert_array_equal(got.view(np.uint8), np.ascontiguousarray(want).view(np.uint8))


@pytest.mark.parametrize("n", [1, 3, 256, 1000])
def test_batched_crop_batch_sizes(n):
    _check_crop(_images(n, (n, 128, 128, 3), torch.uint8), P.prng_key(n), 4, 1)


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
@pytest.mark.parametrize("padding", [0, 1, 4, 8])
@pytest.mark.parametrize("C", [3, 4])
@pytest.mark.parametrize("hw", [(128, 128), (64, 96), (127, 129)])
def test_batched_crop_shapes_bit_exact(hw, C, padding, dtype):
    _check_crop(_images(C + padding, (3, *hw, C), dtype), P.prng_key(100 + padding), padding, 1)


@pytest.mark.parametrize("T", [1, 3])
def test_batched_crop_two_batch_dims(T):
    _check_crop(_images(T, (5, T, 64, 96, 3), torch.uint8), P.prng_key(T), 4, 2)


@pytest.mark.parametrize("dtype,C", [(torch.float16, 3), (torch.float64, 3), (torch.float32, 1), (torch.int64, 2)])
def test_crop_other_element_sizes(dtype, C):
    _check_crop(_images(7, (4, 31, 33, C), torch.float32).mul(100).to(dtype), P.prng_key(9), 3, 1)


def test_crop_unaligned_buffer():
    """A contiguous view one byte into its storage: the byte-unit kernel instead of the 16-byte one."""
    base = torch.zeros(1 + 3 * 128 * 128 * 3, dtype=torch.uint8, device="cuda")
    x = base[1:].view(3, 128, 128, 3)
    x.copy_(_images(1, (3, 128, 128, 3), torch.uint8))
    _check_crop(x, P.prng_key(2), 4, 1)


@pytest.mark.parametrize("lead", [(), (6,), (2, 3)])
def test_random_crop_per_image_keys(lead):
    x = _images(3, (*lead, 40, 52, 3), torch.uint8)
    keys = _key_rows(5, int(np.prod(lead))).reshape(*lead, 2)
    got = _run("_crop", x, _dev_keys(keys), padding=4)
    flat, kf = x.cpu().numpy().reshape(-1, 40, 52, 3), keys.reshape(-1, 2)
    want = np.stack([A.random_crop(f, k, 4) for f, k in zip(flat, kf)]).reshape(x.shape)
    np.testing.assert_array_equal(got, want)


def test_batched_crop_equals_the_replay_samplers_crops():
    """For the same frames and key, batched_random_crop(frames, key, padding=4, num_batch_dims=2) is the sampler's DrQ crop of
    every camera, bit for bit."""
    from helpers import Box, DictSpace
    from oracle.replay import OracleFrameRing
    from serl_b200 import _lib as L
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer
    from serl_b200.vision.data_augmentations import batched_random_crop
    cams, T, H, W, C, cap, B, S, Ad = ("front", "wrist"), 2, 128, 128, 3, 40, 16, 5, 3
    dev = MemoryEfficientReplayBuffer(DictSpace({**{c: Box((T, H, W, C), np.uint8) for c in cams}, "state": Box((T, S))}), Box((Ad,)),
                                      cap, pixel_keys=cams, seed=1)
    ora = OracleFrameRing(cap, cams, (H, W, C), T, S, Ad)
    rng = np.random.default_rng(0)
    for c in cams:
        ora.frames[c] = rng.integers(0, 256, (cap, H, W, C), dtype=np.uint8)
        dev.frames[c].copy_(torch.from_numpy(ora.frames[c]))
    ora.state = ora.next_state = np.zeros((cap, T, S), np.float32)
    ora.actions, ora.rewards, ora.masks = np.zeros((cap, Ad), np.float32), np.zeros(cap, np.float32), np.ones(cap, np.float32)
    ora.dones, ora.valid, ora.size = np.zeros(cap, bool), np.ones(cap, bool), cap
    dev.valid.fill_(1)
    dev._valid_host[:] = True
    dev._size = cap
    dev.size_dev.fill_(cap)
    idx = rng.integers(T, cap, B).astype(np.int32)
    key = P.prng_key(77)
    pix = {c: torch.zeros(B, T, H, W, C, dtype=torch.uint8, device="cuda") for c in cams}
    scratch = {c: torch.zeros(B, T, H, W, C, dtype=torch.uint8, device="cuda") for c in cams}
    f32 = lambda *s: torch.zeros(*s, dtype=torch.float32, device="cuda")
    bufs = dict(obs_state=f32(B, T * S), next_state=f32(B, T * S), actions=f32(B, Ad), rewards=f32(B), masks=f32(B),
                dones=torch.zeros(B, dtype=torch.uint8, device="cuda"), idx=torch.zeros(B, dtype=torch.int32, device="cuda"),
                off_obs=torch.zeros(B * T, 2, dtype=torch.int32, device="cuda"),
                off_next=torch.zeros(B * T, 2, dtype=torch.int32, device="cuda"),
                status=torch.zeros(1, dtype=torch.int32, device="cuda"))
    out = L.BatchOut()
    for j, c in enumerate(cams):
        out.obs_pix[j], out.next_pix[j] = pix[c].data_ptr(), scratch[c].data_ptr()
    for name, t in bufs.items():
        setattr(out, name, t.data_ptr())
    key_t = _dev_keys(np.stack([key, P.prng_key(78)]).reshape(-1))
    part = dict(ring=dev, seed=dev._seed, step=0, batch=B, indx=torch.from_numpy(idx).cuda())
    dev.launch_sample(part, out, crop_total=B * T, out_row_offset=0, key_obs=key_t.data_ptr(), key_next=key_t.data_ptr() + 8,
                      record_event=False)
    torch.cuda.synchronize()
    assert int(bufs["status"][0]) == 0
    packed = ora.gather_packed(idx)["observations"]
    for c in cams:
        frames = torch.from_numpy(np.ascontiguousarray(packed[c][:, :-1])).cuda()       # (B, T, H, W, C), uncropped
        got = batched_random_crop(frames, key, padding=4, num_batch_dims=2)
        assert torch.equal(got, pix[c]), c


# ---- colour ---------------------------------------------------------------------------------------------------------------------
FULL = dict(brightness=0.4, contrast=0.4, saturation=0.4, hue=0.1, to_grayscale_prob=0.2, color_jitter_prob=0.8, apply_prob=0.9,
            shuffle=True)


def _check_color(x, keys, kw, tol=TOL):
    """Every image of x (n, H, W, 3) against the oracle: draws exactly, values to tol.  Returns the oracle draws."""
    n = x.shape[0]
    draws = torch.full((n, 12), float("nan"), device="cuda")
    got = _run("_color", x, _dev_keys(keys), draws, **kw)
    dr = draws.cpu().numpy()
    host = x.cpu().numpy().astype(np.float64)
    out = []
    for i in range(n):
        want, d = A.color_transform(host[i], keys[i], **kw)
        assert (bool(dr[i, 0]), bool(dr[i, 1]), bool(dr[i, 2])) == (d["apply"], d["jitter"], d["gray"]), i
        np.testing.assert_array_equal(dr[i, 3:7].astype(int), d["order"])
        np.testing.assert_array_equal(dr[i, 7:11], d["params"])            # exact (a zero strength draws +-0)
        err = np.abs(got[i] - want).max()
        assert err <= tol, (i, err, A.color_ops(d, kw["brightness"], kw["contrast"], kw["saturation"], kw["hue"]))
        out.append(d)
    return out


@pytest.mark.parametrize("shuffle", [True, False])
def test_color_transform_against_the_oracle(shuffle):
    n = 64
    ds = _check_color(_images(1, (n, 32, 40, 3)), _key_rows(3, n), {**FULL, "shuffle": shuffle})
    orders = {tuple(d["order"]) for d in ds}
    assert (len(orders) > 4) == shuffle
    assert {d["apply"] for d in ds} == {True, False} and {d["gray"] for d in ds} == {True, False}


def test_color_transform_benchmark_shape():
    _check_color(_images(2, (8, 128, 128, 3)), _key_rows(8, 8), {**FULL, "apply_prob": 1.0, "color_jitter_prob": 1.0})


@pytest.mark.parametrize("op", ["brightness", "contrast", "saturation", "hue"])
def test_each_colour_op_on_its_own(op):
    kw = dict(brightness=0.0, contrast=0.0, saturation=0.0, hue=0.0, to_grayscale_prob=0.0, color_jitter_prob=1.0, apply_prob=1.0,
              shuffle=True)
    kw[op] = 0.5
    for d in _check_color(_images(4, (16, 24, 24, 3)), _key_rows(4, 16), kw):
        assert d["apply"] and d["jitter"] and not d["gray"]


def test_color_hard_cases():
    """Constant images (contrast's mean equals every pixel), grey pixels (range 0), hues either side of the wrap at 1.0 and pixels
    at 0 and 1."""
    n, H, W = 12, 16, 16
    rng = np.random.default_rng(6)
    x = rng.random((n, H, W, 3)).astype(np.float32)
    x[0] = 0.25
    x[1] = rng.random(3).astype(np.float32)                              # constant per channel
    x[2] = np.repeat(rng.random((H, W, 1)), 3, axis=-1)                  # grey everywhere
    eps = rng.random((n, H, W)) * 0.02
    x[3:6, ..., 0], x[3:6, ..., 1], x[3:6, ..., 2] = 0.9, 0.3, 0.3 + eps[3:6]    # hue just below 1 (b > g, r max)
    x[6:8, ..., 0], x[6:8, ..., 2], x[6:8, ..., 1] = 0.9, 0.3, 0.3 + eps[6:8]    # hue just above 0
    x[8] = (rng.random((H, W, 3)) > 0.5)                                  # 0 and 1 only
    for kw in ({**FULL, "apply_prob": 1.0, "color_jitter_prob": 1.0, "to_grayscale_prob": 0.5},
               dict(brightness=0.0, contrast=0.0, saturation=0.0, hue=0.5, to_grayscale_prob=0.0, color_jitter_prob=1.0, apply_prob=1.0,
                    shuffle=False),
               dict(brightness=0.0, contrast=0.8, saturation=0.0, hue=0.0, to_grayscale_prob=0.0, color_jitter_prob=1.0, apply_prob=1.0,
                    shuffle=False)):
        _check_color(torch.from_numpy(x).cuda(), _key_rows(11, n), kw)


def test_color_probability_zero_and_one():
    x = _images(5, (32, 16, 16, 3))
    keys = _key_rows(12, 32)
    got = _run("_color", x, _dev_keys(keys), **{**FULL, "apply_prob": 0.0})
    np.testing.assert_array_equal(got, x.cpu().numpy())                  # nothing applied, and the final clip is exact on [0, 1]
    ds = _check_color(x, keys, {**FULL, "apply_prob": 1.0, "color_jitter_prob": 1.0, "to_grayscale_prob": 1.0})
    assert all(d["apply"] and d["jitter"] and d["gray"] for d in ds)


# ---- blur, flip, solarize -----------------------------------------------------------------------------------------------------------
def _check_blur(x, keys, **kw):
    n = x.shape[0]
    draws = torch.full((n, 2), float("nan"), device="cuda")
    got = _run("_blur", x, _dev_keys(keys), draws, **{**dict(blur_divider=10.0, sigma_min=0.1, sigma_max=2.0, apply_prob=1.0), **kw})
    dr = draws.cpu().numpy()
    host = x.cpu().numpy()
    ds = []
    for i in range(n):
        want, d = A.gaussian_blur(host[i], keys[i], **kw)
        assert bool(dr[i, 0]) == d["apply"] and dr[i, 1] == d["sigma"], (i, dr[i], d)
        if d["apply"]:
            assert np.abs(got[i] - want).max() <= TOL, (i, np.abs(got[i] - want).max())
        else:
            np.testing.assert_array_equal(got[i], host[i])
        ds.append(d)
    return ds


@pytest.mark.parametrize("shape", [(4, 128, 128, 3), (3, 64, 96, 3), (3, 127, 129, 4), (2, 40, 300, 1)])
def test_gaussian_blur_against_the_oracle(shape):
    _check_blur(_images(shape[1], shape), _key_rows(shape[2], shape[0]))


@pytest.mark.parametrize("divider,sigma", [(2.0, (0.5, 8.0)), (40.0, (0.1, 2.0)), (200.0, (0.1, 2.0))])
def test_gaussian_blur_radii(divider, sigma):
    """Radius 32, 1 and 0 (a single tap: the identity up to rounding)."""
    _check_blur(_images(2, (3, 128, 64, 3)), _key_rows(2, 3), blur_divider=divider, sigma_min=sigma[0], sigma_max=sigma[1])


def test_gaussian_blur_probabilities():
    ds = _check_blur(_images(3, (16, 32, 32, 3)), _key_rows(3, 16), apply_prob=0.5)
    assert {d["apply"] for d in ds} == {True, False}
    ds = _check_blur(_images(3, (4, 32, 32, 3)), _key_rows(4, 4), apply_prob=0.0)
    assert not any(d["apply"] for d in ds)


@pytest.mark.parametrize("shape", [(64, 32, 48, 3), (8, 17, 33, 1), (4, 128, 128, 3)])
def test_random_flip_bit_exact(shape):
    x = _images(4, shape)
    keys = _key_rows(5, shape[0])
    got = _run("_flip", x, _dev_keys(keys))
    host = x.cpu().numpy()
    want = np.stack([A.random_flip(host[i], keys[i]) for i in range(shape[0])])
    np.testing.assert_array_equal(got, want)
    if shape[0] >= 64:
        assert len({A.flip_decision(k) for k in keys}) == 2


@pytest.mark.parametrize("apply_prob", [0.0, 0.5, 1.0])
def test_solarize_bit_exact(apply_prob):
    n = 48
    x = _images(6, (n, 24, 20, 3))
    keys = _key_rows(7, n)
    got = _run("_solarize", x, _dev_keys(keys), threshold=0.4, apply_prob=apply_prob)
    host = x.cpu().numpy()
    want = np.stack([A.solarize(host[i], keys[i], threshold=0.4, apply_prob=apply_prob) for i in range(n)])
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    flags = {A.solarize_decision(k, apply_prob) for k in keys}
    assert flags == {0.0: {False}, 0.5: {True, False}, 1.0: {True}}[apply_prob]


# ---- every function: single calls, repeatability, CUDA graphs -------------------------------------------------------------------
def _public_calls():
    from serl_b200.vision import data_augmentations as DA
    return {
        "crop": (lambda x, k: DA.random_crop(x, k, padding=4), torch.uint8),
        "color": (lambda x, k: DA.color_transform(x, k, **FULL), torch.float32),
        "blur": (lambda x, k: DA.gaussian_blur(x, k, apply_prob=0.7), torch.float32),
        "flip": (lambda x, k: DA.random_flip(x, k), torch.float32),
        "solarize": (lambda x, k: DA.solarize(x, k, threshold=0.5, apply_prob=0.6), torch.float32),
    }


@pytest.mark.parametrize("fn", ["crop", "color", "blur", "flip", "solarize"])
def test_batched_call_equals_single_calls_and_repeats_bitwise(fn):
    call, dtype = _public_calls()[fn]
    n = 6
    x = _images(8, (2, 3, 48, 40, 3), dtype)
    keys = _key_rows(9, n).reshape(2, 3, 2)
    kt = _dev_keys(keys)
    a, b = call(x, kt), call(x, kt)
    assert a.shape == x.shape and a.dtype == x.dtype and a.is_cuda
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    for i in range(2):
        for j in range(3):
            single = call(x[i, j].cpu().numpy(), keys[i, j])                  # host image and host key: the reference call
            assert torch.equal(single.view(torch.uint8), a[i, j].view(torch.uint8)), (i, j)


def test_batched_random_crop_single_image_and_host_inputs():
    from serl_b200.vision.data_augmentations import batched_random_crop
    x = _images(10, (5, 36, 44, 3), torch.uint8)
    key = P.prng_key(3)
    dev = batched_random_crop(x, _dev_keys(key), padding=4)
    host = batched_random_crop(x.cpu().numpy(), key, padding=4)
    assert torch.equal(dev, host)
    one = batched_random_crop(x[0], key, padding=4, num_batch_dims=0)
    np.testing.assert_array_equal(one.cpu().numpy(), A.random_crop(x[0].cpu().numpy(), P.split(key, 1)[0], 4))


@pytest.mark.parametrize("fn", ["crop", "batched_crop", "color", "blur", "flip", "solarize"])
def test_cuda_graph_replay_equals_eager(fn):
    from serl_b200.vision import data_augmentations as DA
    calls = dict(_public_calls())
    calls["batched_crop"] = (lambda x, k: DA.batched_random_crop(x, k[0, 0], padding=4, num_batch_dims=2), torch.uint8)
    call, dtype = calls[fn]
    x = _images(11, (4, 3, 64, 64, 3), dtype)
    keys = _dev_keys(_key_rows(13, 12).reshape(4, 3, 2))
    eager = call(x, keys)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call(x, keys)                                                          # warm-up off the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = call(x, keys)
    fresh = _images(12, tuple(x.shape), dtype)
    x.copy_(fresh)
    keys.copy_(_dev_keys(_key_rows(14, 12).reshape(4, 3, 2)))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.uint8), call(x, keys).view(torch.uint8))   # the replay read the new inputs
    x.copy_(_images(11, tuple(x.shape), dtype))
    keys.copy_(_dev_keys(_key_rows(13, 12).reshape(4, 3, 2)))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.uint8), eager.view(torch.uint8))
