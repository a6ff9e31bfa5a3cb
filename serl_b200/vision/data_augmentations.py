"""vision/data_augmentations.py of the reference on the GPU: random crops, colour jitter, flips, Gaussian blur and solarize.

Each function takes the reference's arguments and returns a device tensor of the input's shape and dtype.  Images may be CUDA
tensors (contiguous) or host arrays, which are copied to the current device once.  Keys are JAX-style uint32[2] keys (numpy
arrays or uint32 / int32 tensors); pass them as device tensors to capture a call in a CUDA graph.  Every draw, decision and key
split happens on the device (serl_b200/csrc/augment.cu), one launch per call, with nothing read back to the host.

Batching: called with one (H, W, C) image and one (2,) key, a function is the reference call.  Called with leading batch
dimensions and keys of the same leading shape (rng.shape == image.shape[:-3] + (2,)), it is jax.vmap of the reference function
over images and keys, in one pass.  batched_random_crop keeps its own semantics: split(rng, n)[i] crops image i of the n images
its num_batch_dims leading axes hold.

Where the reference cannot be read literally (DESIGN.md §4, "Randomness"):
  * gaussian_blur calls `blur_fn(rng, image)` into a function of `(image, rng, ...)`, i.e. it passes the key as the image; this
    module implements the docstring's intent, gaussian_blur(image, rng).
  * The five-argument `lax.cond(pred, true_operand, true_fun, false_operand, false_fun)` is `true_fun(true_operand)` when pred
    holds, else `false_fun(false_operand)`.
  * A batch of keys means jax.vmap, as above; a batch of images with one key is refused.

rgb_to_hsv, hsv_to_rgb and the adjust_* helpers are the reference's elementwise formulas in torch (no learner path calls them).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from serl_b200 import _lib as L
from serl_b200 import ops

__all__ = ["random_crop", "batched_random_crop", "color_transform", "random_flip", "gaussian_blur", "solarize", "rgb_to_hsv",
           "hsv_to_rgb", "adjust_brightness", "adjust_contrast", "adjust_saturation", "adjust_hue"]


def _device() -> torch.device:
    """Where host arrays are copied: the current CUDA device."""
    return torch.device("cuda", torch.cuda.current_device())


def _image(img, fn: str) -> torch.Tensor:
    if isinstance(img, torch.Tensor):
        if not img.is_contiguous():
            raise ValueError(f"{fn}: the image tensor must be contiguous")
        dev = img.device if img.device.type == "cuda" else _device()
        x = img if img.device == dev else img.to(dev)
    else:
        x = torch.from_numpy(np.ascontiguousarray(np.asarray(img))).to(_device())
    L.require_cuda(x.device)
    if x.dim() < 3:
        raise ValueError(f"{fn}: expected (..., H, W, C) images, got shape {tuple(x.shape)}")
    return x


def _float_image(img, fn: str) -> torch.Tensor:
    x = _image(img, fn)
    if x.dtype != torch.float32:
        raise TypeError(f"{fn}: takes float32 images, got {x.dtype}")
    return x


def _keys(rng, lead, device, fn: str) -> torch.Tensor:
    """rng as a contiguous int32 view of uint32 key words on `device`, checked to have shape lead + (2,)."""
    if isinstance(rng, torch.Tensor):
        if rng.dtype not in (torch.uint32, torch.int32):
            raise TypeError(f"{fn}: keys are uint32 pairs, got {rng.dtype}")
        if not rng.is_contiguous():
            raise ValueError(f"{fn}: the key tensor must be contiguous")
        k = rng.view(torch.int32)
    else:
        a = np.asarray(rng)
        if a.dtype.kind not in "ui":
            raise TypeError(f"{fn}: keys are uint32 pairs, got {a.dtype}")
        k = torch.from_numpy(np.ascontiguousarray(a.astype(np.uint32)).view(np.int32))
    want = tuple(lead) + (2,)
    if tuple(k.shape) != want:
        raise ValueError(f"{fn}: expected keys of shape {want} for images of leading shape {tuple(lead)}, got {tuple(k.shape)}")
    return k if k.device == device else k.to(device)


def _per_image(x: torch.Tensor, rng, fn: str):
    """(n, H, W, C, keys) of images (..., H, W, C) with one key per image."""
    lead = tuple(x.shape[:-3])
    H, W, C_ = x.shape[-3:]
    return math.prod(lead), H, W, C_, _keys(rng, lead, x.device, fn)


def _padding(padding, fn: str) -> int:
    if int(padding) != padding or padding < 0:
        raise ValueError(f"{fn}: padding must be an integer >= 0, got {padding}")
    return int(padding)


def _output(x: torch.Tensor, out):
    """A fresh result tensor, or the caller's (the tests hand in guarded, NaN-filled buffers)."""
    if out is None:
        return torch.empty_like(x)
    if out.shape != x.shape or out.dtype != x.dtype or out.device != x.device or not out.is_contiguous():
        raise ValueError("the output must be a contiguous tensor of the input's shape, dtype and device")
    return out


def _on(device):
    return torch.cuda.device(device) if device.type == "cuda" else _NoDevice()


class _NoDevice:
    def __enter__(self): return self
    def __exit__(self, *a): return False


# ---- crops ------------------------------------------------------------------------------------------------------------------------
def random_crop(img, rng, *, padding):
    """Edge-pad each image by `padding` and take the (H, W) window at randint(key, (2,), 0, 2 padding + 1); any dtype."""
    return _crop(img, rng, padding)


def _crop(img, rng, padding, out=None):
    x = _image(img, "random_crop")
    p = _padding(padding, "random_crop")
    n, H, W, C_, keys = _per_image(x, rng, "random_crop")
    out = _output(x, out)
    if n:
        with _on(x.device):
            ops.aug_crop(x, out, keys, 0, n, H, W, C_, p)
    return out


def batched_random_crop(img, rng, *, padding, num_batch_dims: int = 1):
    """random_crop of each of the n images the num_batch_dims leading axes hold, image i with split(rng, n)[i]; any dtype."""
    return _batched_crop(img, rng, padding, num_batch_dims)


def _batched_crop(img, rng, padding, num_batch_dims, out=None):
    x = _image(img, "batched_random_crop")
    p = _padding(padding, "batched_random_crop")
    nb = int(num_batch_dims)
    if nb < 0 or x.dim() != nb + 3:
        raise ValueError(f"batched_random_crop: {nb} batch dims leave {tuple(x.shape[max(nb, 0):])}, not (H, W, C)")
    keys = _keys(rng, (), x.device, "batched_random_crop")
    n = math.prod(x.shape[:nb])
    H, W, C_ = x.shape[nb:]
    out = _output(x, out)
    if n:
        with _on(x.device):
            ops.aug_crop(x, out, keys, n, n, H, W, C_, p)
    return out


# ---- colour, blur, flip, solarize --------------------------------------------------------------------------------------------------
def _color(image, rng, draws=None, out=None, *, brightness, contrast, saturation, hue, to_grayscale_prob, color_jitter_prob,
           apply_prob, shuffle):
    x = _float_image(image, "color_transform")
    if x.shape[-1] != 3:
        raise ValueError(f"color_transform: needs 3 channels, got {x.shape[-1]}")
    n, H, W, _, keys = _per_image(x, rng, "color_transform")
    f = np.float32
    lo = [f(-brightness), f(1 - contrast), f(1 - saturation), f(-hue)]
    hi = [f(brightness), f(1 + contrast), f(1 + saturation), f(hue)]
    enabled = sum(1 << k for k, s in enumerate((brightness, contrast, saturation, hue)) if s > 0)
    out = _output(x, out)
    if n:
        with _on(x.device):
            ops.aug_color(x, out, keys, draws, n, H, W, lo, hi, enabled, bool(shuffle), apply_prob, color_jitter_prob,
                          to_grayscale_prob)
    return out


def color_transform(image, rng, *, brightness, contrast, saturation, hue, to_grayscale_prob, color_jitter_prob, apply_prob,
                    shuffle):
    """Colour jitter of float32 RGB images: with apply and jitter drawn, brightness / contrast / saturation / hue (each whose
    strength is > 0) in the drawn order, each followed by a clip to [0, 1]; grayscale with apply and its own draw; a final clip."""
    return _color(image, rng, brightness=brightness, contrast=contrast, saturation=saturation, hue=hue,
                  to_grayscale_prob=to_grayscale_prob, color_jitter_prob=color_jitter_prob, apply_prob=apply_prob, shuffle=shuffle)


def _blur(image, rng, draws=None, out=None, *, blur_divider, sigma_min, sigma_max, apply_prob):
    x = _float_image(image, "gaussian_blur")
    n, H, W, C_, keys = _per_image(x, rng, "gaussian_blur")
    if not blur_divider > 0:
        raise ValueError(f"gaussian_blur: blur_divider must be > 0, got {blur_divider}")
    radius = int(H / blur_divider / 2)
    if radius > L.BLUR_MAX_RADIUS:
        raise ValueError(f"gaussian_blur: a kernel of radius {radius} (H {H} / blur_divider {blur_divider} / 2) exceeds "
                         f"{L.BLUR_MAX_RADIUS}")
    out = _output(x, out)
    if n:
        with _on(x.device):
            ops.aug_blur(x, out, keys, draws, n, H, W, C_, radius, sigma_min, sigma_max, apply_prob)
    return out


def gaussian_blur(image, rng, *, blur_divider=10.0, sigma_min=0.1, sigma_max=2.0, apply_prob=1.0):
    """With probability apply_prob, a Gaussian blur of float32 images: sigma ~ U(sigma_min, sigma_max), radius
    int(H / blur_divider / 2), normalised taps along W then H with zero padding (SAME)."""
    return _blur(image, rng, blur_divider=blur_divider, sigma_min=sigma_min, sigma_max=sigma_max, apply_prob=apply_prob)


def random_flip(image, rng):
    """Flip float32 images along W when uniform(split(rng)[1]) <= 0.5."""
    return _flip(image, rng)


def _flip(image, rng, out=None):
    x = _float_image(image, "random_flip")
    n, H, W, C_, keys = _per_image(x, rng, "random_flip")
    out = _output(x, out)
    if n:
        with _on(x.device):
            ops.aug_flip(x, out, keys, n, H, W, C_)
    return out


def solarize(image, rng, *, threshold, apply_prob):
    """With probability apply_prob, where(x < threshold, x, 1 - x) on float32 images."""
    return _solarize(image, rng, threshold, apply_prob)


def _solarize(image, rng, threshold, apply_prob, out=None):
    x = _float_image(image, "solarize")
    n, H, W, C_, keys = _per_image(x, rng, "solarize")
    out = _output(x, out)
    if n:
        with _on(x.device):
            ops.aug_solarize(x, out, keys, n, H, W, C_, threshold, apply_prob)
    return out


# ---- elementwise helpers (torch) ----------------------------------------------------------------------------------------------------
def _tree_map(fn, x):
    return type(x)(fn(e) for e in x) if isinstance(x, (tuple, list)) else fn(x)


def rgb_to_hsv(r, g, b):
    """The TF rgb_to_hsv kernel: (h, s, v) with h in [0, 1)."""
    vv = torch.maximum(torch.maximum(r, g), b)
    range_ = vv - torch.minimum(torch.minimum(r, g), b)
    sat = torch.where(vv > 0, range_ / vv, torch.zeros_like(vv))
    norm = torch.where(range_ != 0, 1.0 / (6.0 * range_), torch.full_like(range_, 1e9))
    hr = norm * (g - b)
    hg = norm * (b - r) + 2.0 / 6.0
    hb = norm * (r - g) + 4.0 / 6.0
    hue = torch.where(r == vv, hr, torch.where(g == vv, hg, hb))
    hue = hue * (range_ > 0)
    hue = hue + (hue < 0)
    return hue, sat, vv


def hsv_to_rgb(h, s, v):
    """The TF hsv_to_rgb kernel: (r, g, b)."""
    c = s * v
    m = v - c
    dh = torch.remainder(h, 1.0) * 6.0
    x = c * (1 - torch.abs(torch.remainder(dh, 2.0) - 1))
    hcat = torch.floor(dh).to(torch.int32)
    zero = torch.zeros_like(c)
    rr = torch.where((hcat == 0) | (hcat == 5), c, torch.where((hcat == 1) | (hcat == 4), x, zero)) + m
    gg = torch.where((hcat == 1) | (hcat == 2), c, torch.where((hcat == 0) | (hcat == 3), x, zero)) + m
    bb = torch.where((hcat == 3) | (hcat == 4), c, torch.where((hcat == 2) | (hcat == 5), x, zero)) + m
    return rr, gg, bb


def adjust_brightness(rgb_tuple, delta):
    return _tree_map(lambda x: x + delta, rgb_tuple)


def adjust_contrast(image, factor):
    def channel(x):
        mean = x.mean(dim=(-2, -1), keepdim=True)
        return factor * (x - mean) + mean
    return _tree_map(channel, image)


def adjust_saturation(h, s, v, factor):
    return h, torch.clamp(s * factor, 0.0, 1.0), v


def adjust_hue(h, s, v, delta):
    return torch.remainder(h + delta, 1.0), s, v
