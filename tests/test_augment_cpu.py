"""CPU: the augmentation oracle (oracle/augment.py) on cases worked out by hand, and the host logic of
serl_b200.vision.data_augmentations on the dry-launch recorder: one launch per call, and every malformed input refused before
anything is launched."""
import struct

import numpy as np
import pytest
import torch

from oracle import augment as A
from oracle import jax_prng as P


# ---- oracle self-checks ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rgb,hsv", [
    ((1, 0, 0), (0, 1, 1)), ((0, 1, 0), (1 / 3, 1, 1)), ((0, 0, 1), (2 / 3, 1, 1)),
    ((1, 1, 0), (1 / 6, 1, 1)),            # r == g == vv: the red branch
    ((0, 1, 1), (1 / 2, 1, 1)),            # g == b == vv: the green branch
    ((1, 0, 1), (5 / 6, 1, 1)),            # r == b == vv: red branch, negative hue wrapped by + 1
    ((0.5, 0.5, 0.5), (0, 0, 0.5)), ((0, 0, 0), (0, 0, 0)), ((1, 1, 1), (0, 0, 1)),   # greys: range 0
    ((0.8, 0.4, 0.2), (1 / 18, 0.75, 0.8)),
])
def test_rgb_to_hsv_primaries_greys_and_ties(rgb, hsv):
    got = A.rgb_to_hsv(*[np.float64(c) for c in rgb])
    np.testing.assert_allclose([float(g) for g in got], hsv, atol=1e-15)


def test_hsv_round_trips():
    rng = np.random.default_rng(0)
    rgb = [rng.random(4096) for _ in range(3)]
    rgb[1][:64] = rgb[0][:64]                                 # ties
    rgb[2][64:128] = rgb[1][64:128] = rgb[0][64:128]          # greys
    back = A.hsv_to_rgb(*A.rgb_to_hsv(*rgb))
    for c in range(3):
        np.testing.assert_allclose(back[c], rgb[c], atol=1e-12)
    h = rng.random(4096)
    s, v = rng.random(4096), rng.random(4096)
    h2, s2, v2 = A.rgb_to_hsv(*A.hsv_to_rgb(h, s, v))
    np.testing.assert_allclose(v2, v, atol=1e-12)
    np.testing.assert_allclose(s2, s, atol=1e-12)
    np.testing.assert_allclose(np.minimum(abs(h2 - h), 1 - abs(h2 - h)), 0, atol=1e-9)   # hue modulo 1


def test_crop_with_padding_zero_is_the_identity():
    img = np.random.default_rng(1).integers(0, 256, (2, 5, 7, 3), dtype=np.uint8)
    np.testing.assert_array_equal(A.batched_random_crop(img, P.prng_key(3), 0), img)


def _key_with_offsets(padding, want):
    for seed in range(10000):
        k = P.prng_key(seed)
        if tuple(A.crop_offsets(k, padding)) == want:
            return k
    raise AssertionError(want)


@pytest.mark.parametrize("corner", [(0, 0), (0, 4), (4, 0), (4, 4)])
def test_crop_edge_padding_at_the_four_corners(corner):
    """Offsets (0 | 2p, 0 | 2p) put the replicated edge in a p x p corner: that block is the nearest corner pixel, the rest the
    image shifted by p."""
    p, H, W = 2, 6, 9
    img = np.random.default_rng(2).integers(0, 256, (H, W, 3), dtype=np.uint8)
    out = A.random_crop(img, _key_with_offsets(p, corner), p)
    ys = slice(0, p) if corner[0] == 0 else slice(H - p, H)
    xs = slice(0, p) if corner[1] == 0 else slice(W - p, W)
    src = (0 if corner[0] == 0 else H - 1, 0 if corner[1] == 0 else W - 1)
    assert (out[ys, xs] == img[src]).all()
    dy, dx = corner[0] - p, corner[1] - p
    inner = out[max(0, -dy):H - max(0, dy), max(0, -dx):W - max(0, dx)]
    np.testing.assert_array_equal(inner, img[max(0, dy):H + min(0, dy), max(0, dx):W + min(0, dx)])


def test_crop_agrees_with_the_replay_oracle_shift():
    from oracle.replay import random_shift
    img = np.random.default_rng(4).integers(0, 256, (5, 8, 10, 3), dtype=np.uint8)
    key = P.prng_key(11)
    np.testing.assert_array_equal(A.batched_random_crop(img, key, 4), random_shift(img, P.crop_offsets(key, 5), 4))


def test_uniform_bit_construction_by_hand():
    key = P.prng_key(0)
    bits = int(P.threefry2x32(key, np.zeros(1, np.uint32), np.zeros(1, np.uint32))[0][0])   # random_bits(key, ()): counter pair (0, 0)
    f = struct.unpack("<f", struct.pack("<I", (bits >> 9) | 0x3F800000))[0] - 1.0           # exact: 23 mantissa bits
    assert A.uniform(key) == np.float32(f)
    assert A.uniform(key) == np.float32(0.41845703)        # jax.random.uniform(PRNGKey(0)) as jax's documentation prints it
    lo, hi = np.float32(1 - 0.3), np.float32(1 + 0.3)
    want = max(lo, np.float32(np.float32(np.float32(f) * np.float32(hi - lo)) + lo))
    assert A.uniform(key, 1 - 0.3, 1 + 0.3) == want
    assert A.uniform(key, -0.5, 0.5) == np.float32(np.float32(f) - np.float32(0.5))


def test_four_element_permutation_takes_one_sort_round():
    import vice_oracle
    assert A.shuffle_rounds(4) == 1
    key = P.prng_key(7)
    _, sub = P.split(key)
    np.testing.assert_array_equal(A.permutation(key, 4), np.argsort(P.random_bits(sub, (4,)), kind="stable"))
    for n in (4, 10, 1000):
        np.testing.assert_array_equal(A.permutation(P.prng_key(n), n), vice_oracle.permutation(P.prng_key(n), n))


def test_color_transform_oracle_steps():
    """With every strength 0 but one, the oracle applies that op alone, after drawing apply and jitter."""
    img = np.random.default_rng(5).random((4, 6, 3))
    kw = dict(brightness=0.3, contrast=0.0, saturation=0.0, hue=0.0, to_grayscale_prob=0.0, color_jitter_prob=1.0,
              apply_prob=1.0, shuffle=False)
    out, d = A.color_transform(img, P.prng_key(1), **kw)
    assert d["apply"] and d["jitter"] and not d["gray"]
    np.testing.assert_allclose(out, np.clip(img + float(d["params"][0]), 0, 1), atol=0)
    out0, _ = A.color_transform(img, P.prng_key(1), **{**kw, "apply_prob": 0.0})
    np.testing.assert_array_equal(out0, img)


# ---- host logic on the dry-launch recorder ---------------------------------------------------------------------------------------
@pytest.fixture()
def dry(monkeypatch):
    from serl_b200 import _lib as L
    from serl_b200.vision import data_augmentations as DA
    calls = []
    monkeypatch.setattr(L, "call", lambda name, *args: calls.append(name) or 0)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(DA, "_device", lambda: torch.device("cpu"))
    return calls


COLOR = dict(brightness=0.4, contrast=0.4, saturation=0.4, hue=0.1, to_grayscale_prob=0.2, color_jitter_prob=0.8, apply_prob=1.0,
             shuffle=True)


def _calls():
    from serl_b200.vision import data_augmentations as DA
    f32 = lambda *s: torch.rand(*s)
    k = lambda *lead: np.zeros((*lead, 2), np.uint32)
    return {
        "crop": (lambda: DA.random_crop(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), k(2), padding=4), "serl_aug_crop"),
        "batched_crop": (lambda: DA.batched_random_crop(torch.zeros(2, 3, 8, 8, 3, dtype=torch.uint8), k(), padding=4,
                                                        num_batch_dims=2), "serl_aug_crop"),
        "color": (lambda: DA.color_transform(f32(2, 8, 8, 3), k(2), **COLOR), "serl_aug_color"),
        "flip": (lambda: DA.random_flip(f32(8, 8, 3), k()), "serl_aug_flip"),
        "blur": (lambda: DA.gaussian_blur(f32(4, 16, 16, 3), k(4)), "serl_aug_blur"),
        "solarize": (lambda: DA.solarize(f32(3, 8, 8, 1), k(3), threshold=0.5, apply_prob=0.5), "serl_aug_solarize"),
    }


@pytest.mark.parametrize("fn", ["crop", "batched_crop", "color", "flip", "blur", "solarize"])
def test_each_function_records_one_launch(dry, fn):
    call, name = _calls()[fn]
    out = call()
    assert dry == [name]
    assert isinstance(out, torch.Tensor)


def _bad_inputs():
    from serl_b200.vision import data_augmentations as DA
    f32, u8 = torch.rand(2, 8, 8, 3), torch.zeros(2, 8, 8, 3, dtype=torch.uint8)
    k2 = np.zeros((2, 2), np.uint32)
    return {
        "key_shape_crop": lambda: DA.random_crop(u8, np.zeros((3, 2), np.uint32), padding=1),
        "key_single_for_batch": lambda: DA.random_flip(f32, np.zeros(2, np.uint32)),
        "key_shape_batched_crop": lambda: DA.batched_random_crop(u8, k2, padding=1),
        "key_float": lambda: DA.solarize(f32, np.zeros((2, 2), np.float32), threshold=0.5, apply_prob=1.0),
        "key_int64_tensor": lambda: DA.random_flip(f32, torch.zeros(2, 2, dtype=torch.int64)),
        "color_c4": lambda: DA.color_transform(torch.rand(2, 8, 8, 4), k2, **COLOR),
        "color_u8": lambda: DA.color_transform(u8, k2, **COLOR),
        "blur_f64": lambda: DA.gaussian_blur(f32.double(), k2),
        "flip_u8": lambda: DA.random_flip(u8, k2),
        "solarize_f16": lambda: DA.solarize(f32.half(), k2, threshold=0.5, apply_prob=1.0),
        "negative_padding": lambda: DA.random_crop(u8, k2, padding=-1),
        "batched_negative_padding": lambda: DA.batched_random_crop(u8, np.zeros(2, np.uint32), padding=-2),
        "fractional_padding": lambda: DA.random_crop(u8, k2, padding=1.5),
        "batch_dims": lambda: DA.batched_random_crop(u8, np.zeros(2, np.uint32), padding=1, num_batch_dims=2),
        "non_contiguous_image": lambda: DA.random_flip(torch.rand(2, 8, 8, 6)[..., ::2], k2),
        "non_contiguous_crop": lambda: DA.random_crop(torch.zeros(8, 2, 8, 3, dtype=torch.uint8).transpose(0, 1), k2, padding=1),
        "non_contiguous_key": lambda: DA.random_flip(f32, torch.zeros(2, 4, dtype=torch.int32)[:, ::2]),
        "blur_radius": lambda: DA.gaussian_blur(torch.rand(1, 200, 4, 1), np.zeros((1, 2), np.uint32), blur_divider=1.0),
        "blur_divider": lambda: DA.gaussian_blur(f32, k2, blur_divider=0.0),
        "not_an_image": lambda: DA.solarize(torch.rand(8, 8), np.zeros(2, np.uint32), threshold=0.5, apply_prob=1.0),
    }


@pytest.mark.parametrize("case", ["key_shape_crop", "key_single_for_batch", "key_shape_batched_crop", "key_float", "key_int64_tensor",
                                  "color_c4", "color_u8", "blur_f64", "flip_u8", "solarize_f16", "negative_padding",
                                  "batched_negative_padding", "fractional_padding", "batch_dims", "non_contiguous_image",
                                  "non_contiguous_crop", "non_contiguous_key", "blur_radius", "blur_divider", "not_an_image"])
def test_bad_inputs_are_refused_before_any_launch(dry, case):
    bad = _bad_inputs()
    assert case in bad
    with pytest.raises((ValueError, TypeError)):
        bad[case]()
    assert dry == []


def test_empty_batch_launches_nothing(dry):
    from serl_b200.vision import data_augmentations as DA
    out = DA.random_crop(torch.zeros(0, 8, 8, 3, dtype=torch.uint8), np.zeros((0, 2), np.uint32), padding=4)
    assert out.shape == (0, 8, 8, 3) and dry == []


def test_reference_import_path_resolves_to_the_device_module():
    from serl_launcher.vision.data_augmentations import batched_random_crop, color_transform, gaussian_blur, random_flip, solarize
    from serl_b200.vision import data_augmentations as DA
    assert (batched_random_crop, color_transform, gaussian_blur, random_flip, solarize) == (
        DA.batched_random_crop, DA.color_transform, DA.gaussian_blur, DA.random_flip, DA.solarize)


def test_torch_helpers_match_the_oracle():
    from serl_b200.vision import data_augmentations as DA
    rgb = [np.random.default_rng(c).random(512) for c in range(3)]
    rgb[1][:32] = rgb[0][:32]
    got = DA.rgb_to_hsv(*[torch.from_numpy(c) for c in rgb])
    for g, w in zip(got, A.rgb_to_hsv(*rgb)):
        np.testing.assert_allclose(g.numpy(), w, atol=1e-12)
    h, s, v = (torch.from_numpy(x) for x in A.rgb_to_hsv(*rgb))
    h2, s2, v2 = DA.adjust_hue(*DA.adjust_saturation(h, s, v, 0.5), 0.7)
    for g, w in zip(DA.hsv_to_rgb(h2, s2, v2), A.hsv_to_rgb((h.numpy() + 0.7) % 1.0, np.clip(s.numpy() * 0.5, 0, 1), v.numpy())):
        np.testing.assert_allclose(g.numpy(), w, atol=1e-12)
    img = torch.rand(5, 6)
    np.testing.assert_allclose(DA.adjust_contrast(img, 1.5).numpy(), (1.5 * (img - img.mean()) + img.mean()).numpy(), atol=1e-6)
    assert all(torch.equal(a, b + 0.25) for a, b in zip(DA.adjust_brightness((img, img), 0.25), (img, img)))
