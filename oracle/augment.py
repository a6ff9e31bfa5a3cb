"""ORACLE (test infrastructure, not product): NumPy restatement of vision/data_augmentations.py on oracle/jax_prng.py.

Random draws and decisions are restated bit for bit in float32 as jax builds them: uniform(key, (), float32, lo, hi) =
max(lo, f * (hi - lo) + lo) with f = bitcast(bits >> 9 | 0x3f800000) - 1 and every operation rounded to float32 on its own, and
the bounds and probabilities rounded to float32 first (jax's weak typing).  Pixel values are float64 (crops, flips and solarize,
which only move or mirror values, keep the input dtype).  Reference call sites (relative to serl_launcher/serl_launcher):

  random_crop / batched_random_crop   vision/data_augmentations.py:7-36
  _maybe_apply                        :39-42      uniform(rng) <= apply_prob
  gaussian blur                       :62-105, :312-333 (called as (image, rng), the docstring's intent)
  rgb_to_hsv / hsv_to_rgb / adjust_*  :108-208
  color_transform                     :224-302
  random_flip                         :305-309
  solarize                            :336-340
"""
from __future__ import annotations

import numpy as np

from oracle import jax_prng as P

F32 = np.float32
GRAY_WEIGHTS = np.array([0.2989, 0.5870, 0.1140], np.float32).astype(np.float64)   # jnp.array of Python floats: float32


def uniform(key, minval=0.0, maxval=1.0) -> np.float32:
    """jax.random.uniform(key, (), float32, minval, maxval)."""
    lo, hi = F32(minval), F32(maxval)
    f = F32(P.uniform01(key, ()))
    return np.maximum(lo, F32(F32(f * F32(hi - lo)) + lo))


def permutation(key, n):
    """jax.random.permutation(key, arange(n)) (jax's _shuffle): ceil(3 ln n / ln(2^32 - 1)) rounds of key, sub = split(key) and
    a stable sort of the entries by random_bits(sub, (n,))."""
    x = np.arange(n)
    key = np.asarray(key, np.uint32)
    for _ in range(shuffle_rounds(n)):
        key, sub = P.split(key)
        x = x[np.argsort(P.random_bits(sub, (n,)), kind="stable")]
    return x


def shuffle_rounds(n) -> int:
    return int(np.ceil(3 * np.log(max(1, n)) / np.log(np.iinfo(np.uint32).max)))


# ---- crops ---------------------------------------------------------------------------------------------------------------------
def crop_offsets(key, padding):
    return P.randint(key, (2,), 0, 2 * padding + 1)


def random_crop(img, key, padding):
    """(H, W, C) image of any dtype: edge pad, then the window at (cy, cx)."""
    cy, cx = crop_offsets(key, padding)
    H, W = img.shape[:2]
    padded = np.pad(img, ((padding, padding), (padding, padding), (0, 0)), mode="edge")
    return padded[cy:cy + H, cx:cx + W]


def batched_random_crop(img, key, padding, num_batch_dims=1):
    flat = img.reshape(-1, *img.shape[num_batch_dims:])
    keys = P.split(key, flat.shape[0])
    return np.stack([random_crop(f, k, padding) for f, k in zip(flat, keys)]).reshape(img.shape)


# ---- colour ---------------------------------------------------------------------------------------------------------------------
def rgb_to_hsv(r, g, b):
    vv = np.maximum(np.maximum(r, g), b)
    range_ = vv - np.minimum(np.minimum(r, g), b)
    with np.errstate(divide="ignore", invalid="ignore"):
        sat = np.where(vv > 0, range_ / vv, 0.0)
        norm = np.where(range_ != 0, 1.0 / (6.0 * range_), 1e9)
    hr = norm * (g - b)
    hg = norm * (b - r) + 2.0 / 6.0
    hb = norm * (r - g) + 4.0 / 6.0
    hue = np.where(r == vv, hr, np.where(g == vv, hg, hb))
    hue = hue * (range_ > 0)
    hue = hue + (hue < 0)
    return hue, sat, vv


def hsv_to_rgb(h, s, v):
    c = s * v
    m = v - c
    dh = (h % 1.0) * 6.0
    x = c * (1 - np.abs(dh % 2.0 - 1))
    hcat = np.floor(dh).astype(np.int32)
    rr = np.where((hcat == 0) | (hcat == 5), c, np.where((hcat == 1) | (hcat == 4), x, 0)) + m
    gg = np.where((hcat == 1) | (hcat == 2), c, np.where((hcat == 0) | (hcat == 3), x, 0)) + m
    bb = np.where((hcat == 3) | (hcat == 4), c, np.where((hcat == 2) | (hcat == 5), x, 0)) + m
    return rr, gg, bb


def color_draws(key, *, brightness, contrast, saturation, hue, to_grayscale_prob, color_jitter_prob, apply_prob, shuffle):
    """color_transform's random decisions: apply / jitter / grayscale, the jitter order and the four drawn parameters (drawn
    whatever the strengths; the reference draws an op's parameter only when it runs, from the same key)."""
    apply_rng, transform_rng = P.split(np.asarray(key, np.uint32))
    perm_rng, b_rng, c_rng, s_rng, h_rng, cj_rng, gs_rng = P.split(transform_rng, 7)
    return dict(
        apply=bool(uniform(apply_rng) <= F32(apply_prob)),
        jitter=bool(uniform(cj_rng) <= F32(color_jitter_prob)),
        gray=bool(uniform(gs_rng) <= F32(to_grayscale_prob)),
        order=permutation(perm_rng, 4) if shuffle else np.arange(4),
        params=np.array([uniform(b_rng, -brightness, brightness), uniform(c_rng, 1 - contrast, 1 + contrast),
                         uniform(s_rng, 1 - saturation, 1 + saturation), uniform(h_rng, -hue, hue)], np.float32))


def color_ops(d, brightness, contrast, saturation, hue):
    """The ops color_transform applies, in order: [(op, parameter)], op 0..3 = brightness, contrast, saturation, hue."""
    if not (d["apply"] and d["jitter"]):
        return []
    strengths = (brightness, contrast, saturation, hue)
    return [(int(op), float(d["params"][op])) for op in d["order"] if strengths[op] > 0]


def color_transform(image, key, **kw):
    """(float64 image, draws) of color_transform on one (H, W, 3) image."""
    d = color_draws(key, **kw)
    rgb = [np.asarray(image, np.float64)[..., c] for c in range(3)]
    for op, p in color_ops(d, kw["brightness"], kw["contrast"], kw["saturation"], kw["hue"]):
        if op == 0:
            rgb = [x + p for x in rgb]
        elif op == 1:
            rgb = [p * (x - x.mean()) + x.mean() for x in rgb]
        else:
            h, s, v = rgb_to_hsv(*rgb)
            if op == 2:
                s = np.clip(s * p, 0.0, 1.0)
            else:
                h = (h + p) % 1.0
            rgb = list(hsv_to_rgb(h, s, v))
        rgb = [np.clip(x, 0.0, 1.0) for x in rgb]
    out = np.stack(rgb, axis=-1)
    if d["apply"] and d["gray"]:
        out = np.repeat((out @ GRAY_WEIGHTS)[..., None], 3, axis=-1)
    return np.clip(out, 0.0, 1.0), d


# ---- blur, flip, solarize ---------------------------------------------------------------------------------------------------------
def blur_draws(key, sigma_min=0.1, sigma_max=2.0, apply_prob=1.0):
    apply_rng, transform_rng = P.split(np.asarray(key, np.uint32))
    (sigma_rng,) = P.split(transform_rng, 1)
    return dict(apply=bool(uniform(apply_rng) <= F32(apply_prob)), sigma=uniform(sigma_rng, sigma_min, sigma_max))


def blur_radius(H, blur_divider):
    return int(H / blur_divider / 2)


def gaussian_blur(image, key, *, blur_divider=10.0, sigma_min=0.1, sigma_max=2.0, apply_prob=1.0):
    """(float64 image, draws) of gaussian_blur(image, key) on one (H, W, C) image."""
    d = blur_draws(key, sigma_min, sigma_max, apply_prob)
    img = np.asarray(image, np.float64)
    if not d["apply"]:
        return img, d
    H, W = img.shape[:2]
    r = blur_radius(H, blur_divider)
    x = np.arange(-r, r + 1, dtype=np.float64)
    sigma = np.float64(d["sigma"])
    w = np.exp(-(x ** 2) / (2.0 * sigma ** 2))
    w /= w.sum()
    pad = np.pad(img, ((0, 0), (r, r), (0, 0)))
    horiz = sum(w[k] * pad[:, k:k + W] for k in range(2 * r + 1))
    pad = np.pad(horiz, ((r, r), (0, 0), (0, 0)))
    return sum(w[k] * pad[k:k + H] for k in range(2 * r + 1)), d


def flip_decision(key) -> bool:
    _, flip_rng = P.split(np.asarray(key, np.uint32))
    return bool(uniform(flip_rng) <= F32(0.5))


def random_flip(image, key):
    return image[:, ::-1] if flip_decision(key) else image


def solarize_decision(key, apply_prob) -> bool:
    return bool(uniform(np.asarray(key, np.uint32)) <= F32(apply_prob))


def solarize(image, key, *, threshold, apply_prob):
    """float32 in, float32 out: 1 - x is exact in float32 as in jax."""
    image = np.asarray(image, np.float32)
    if not solarize_decision(key, apply_prob):
        return image
    return np.where(image < F32(threshold), image, (F32(1.0) - image).astype(np.float32))
