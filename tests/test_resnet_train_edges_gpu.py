"""GPU: the trainable ResNet-10's kernels (csrc/resnet_train.cu, and the fp32 GroupNorm / max-pool forwards they pair with)
against float64 torch at shapes the ResNet-10 layers of a 128x128 image never take, but the C ABI accepts.

  convs       serl_rconv_fwd / _dgrad / _wgrad through the C ABI (kh != kw is only reachable there), on the CUDA cores (tc = 0)
              and the tensor cores (tc = 1): non-square maps and kernels (5x3, 1x7); Ci and Co off multiples of 32 (taps change
              inside a 32-wide k-block) and of 64 (a partial N tile); Cw < Ci; stride 2 with pads (1, 1), whose parity classes
              differ from ResNet's (0, 1); stride 3, with a 2x2 kernel so some parity classes have no taps (accumulate leaves
              dx there untouched); several M tiles; wgrad over K < 32 pixels and where rounding k_split up to 32 leaves fewer
              splits than wgrad_splits asked for.  Against F.pad + F.conv2d autograd in float64, within 2e-5 of the output's
              max (3xTF32 and fp32 FMA are both fp32-class), and two launches bitwise equal.  Unsupported shapes raise and
              launch nothing.
  GroupNorm   serl_groupnorm_bwd_nhwc and the forward at G in {1, 2, 4, 8}, C/G in {4, ..., 512} and 4x4 / 16x16 maps (a group
              of <= 512 and > 512 channel quads), plain, relu and relu + residual.  The widths where 512 % (C/G/4) != 0 (12,
              24, 48, 320) once made the backward's threads change channel quad as they walked the group.
  max-pool    the 3x3/2 SAME forward and backward on 64x64, 63x63, 64x63, 63x64, 2x2 and 1x1 maps with tied and all-zero
              windows (backward also at C % 4 != 0): per-axis SAME pads, the first-max rule.  Maps whose H and W differ in
              parity once took one low pad for both axes.
  stem prep   serl_rconv_stem_prep bitwise against the same fp32 expression, past its grid cap of 132 * 16 * 256 pixels."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import drq
from resnet_encoder_oracle import max_pool_first_max

pytestmark = pytest.mark.gpu
CONV_TOL = 2e-5
TK, TM, TN, WGRAD_CTAS = 32, 128, 64, 2 * 132

#       N, H, W, Ci, Cw, Co, kh, kw, stride, pad_lo, pad_hi
CONVS = {
    "5x3-ci12-co36": (2, 12, 10, 12, 12, 36, 5, 3, 1, 2, 2),
    "1x7-co68": (2, 9, 14, 16, 16, 68, 1, 7, 1, 0, 3),
    "3x3-c100": (1, 7, 11, 100, 100, 100, 3, 3, 1, 1, 1),
    "cw9-of-ci16": (2, 10, 6, 16, 9, 36, 3, 3, 1, 1, 1),
    "s2-pads11-3mtiles": (3, 20, 18, 36, 36, 100, 3, 3, 2, 1, 1),
    "s2-pads11-5x5": (2, 10, 14, 20, 20, 44, 5, 5, 2, 1, 1),
    "s3-2x2": (2, 9, 12, 8, 8, 40, 2, 2, 3, 0, 0),
    "s3-5x5-pads22": (1, 12, 9, 12, 12, 24, 5, 5, 3, 2, 2),
    "wgrad-k24": (1, 4, 6, 8, 8, 12, 3, 3, 1, 1, 1),
    "wgrad-k2050-13-of-16-splits": (2, 25, 41, 8, 8, 16, 1, 1, 1, 0, 0),
}


def _err(got, ref):
    ref = ref.detach().double()
    return float((got.double() - ref).abs().max() / max(float(ref.abs().max()), 1e-12))


def _call(name, *args):
    from serl_b200 import _lib as L
    L.call(name, *args)


def _conv64(x, w, stride, lo, hi):
    """NHWC x, (kh, kw, Ci, Co) w; the same (lo, hi) zero pad on both axes, as the C ABI takes it."""
    xin = F.pad(x.permute(0, 3, 1, 2), (lo, hi, lo, hi))
    return F.conv2d(xin, w.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)


def _wgrad_splits(N, Ho, Wo, Ci, Co, kh, kw):
    """The split count serl_rconv_wgrad asks for (rconv::wgrad_splits)."""
    tiles = -(-kh * kw * Ci // TM) * -(-Co // TN)
    return max(1, min(WGRAD_CTAS // tiles, N * Ho * Wo // (4 * TK)))


@pytest.mark.parametrize("tc", [0, 1], ids=["cuda-cores", "tensor-cores"])
@pytest.mark.parametrize("case", list(CONVS))
def test_rconv_edges_match_float64(case, tc):
    from serl_b200 import _lib as L
    N, H, W, Ci, Cw, Co, kh, kw, s, lo, hi = CONVS[case]
    st = L.stream_ptr()
    g = torch.Generator(device="cuda").manual_seed(list(CONVS).index(case))
    x = torch.randn(N, H, W, Ci, device="cuda", generator=g)
    w = torch.randn(kh, kw, Cw, Co, device="cuda", generator=g) / (kh * kw * Cw) ** 0.5
    x64, w64 = x[..., :Cw].double().requires_grad_(), w.double().requires_grad_()
    ref = _conv64(x64, w64, s, lo, hi)
    _, Ho, Wo, _ = ref.shape
    ys = [torch.empty(N, Ho, Wo, Co, device="cuda") for _ in range(2)]
    for y in ys:
        _call("serl_rconv_fwd", x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, W, Ci, Cw, Co, kh, kw, s, lo, hi, tc, st)
    errs = {"fwd": _err(ys[0], ref)}
    assert torch.equal(ys[0], ys[1]), "fwd: two launches differ"
    dz = torch.randn(N, Ho, Wo, Co, device="cuda", generator=g)
    (ref * dz.double()).sum().backward()

    import ctypes as C
    nws = C.c_longlong(0)
    _call("serl_rconv_wgrad_workspace", N, H, W, Ci, Co, kh, kw, s, lo, hi, C.byref(nws))
    z = nws.value // (kh * kw * Ci * Co)                      # the splits the kernel runs
    asked = _wgrad_splits(N, Ho, Wo, Ci, Co, kh, kw)
    if case == "wgrad-k24":
        assert N * Ho * Wo < TK and z == 1
    if case == "wgrad-k2050-13-of-16-splits":
        assert (asked, z) == (16, 13), (asked, z)
    ws = torch.empty(nws.value, device="cuda")
    dws = [torch.empty_like(w) for _ in range(2)]
    for dw in dws:
        _call("serl_rconv_wgrad", x.data_ptr(), dz.data_ptr(), dw.data_ptr(), ws.data_ptr(), ws.numel() * 4, N, H, W, Ci, Cw, Co, kh, kw,
              s, lo, hi, tc, st)
    errs["wgrad"] = _err(dws[0], w64.grad)
    assert torch.equal(dws[0], dws[1]), "wgrad: two launches differ"

    if Cw == Ci:                                               # the input gradient takes the full-width kernel
        dxs = [torch.empty_like(x) for _ in range(2)]
        for dx in dxs:
            _call("serl_rconv_dgrad", dz.data_ptr(), w.data_ptr(), dx.data_ptr(), N, H, W, Ci, Co, kh, kw, s, lo, hi, 0, tc, st)
        errs["dgrad"] = _err(dxs[0], x64.grad)
        assert torch.equal(dxs[0], dxs[1]), "dgrad: two launches differ"
        base = torch.randn(x.shape, device="cuda", generator=g)
        acc = base.clone()
        _call("serl_rconv_dgrad", dz.data_ptr(), w.data_ptr(), acc.data_ptr(), N, H, W, Ci, Co, kh, kw, s, lo, hi, 1, tc, st)
        errs["dgrad accumulate"] = _err(acc - base, x64.grad)
        if case == "s3-2x2":                                   # rows / columns 2 mod 3: parity classes without a tap
            untouched = (x64.grad == 0).all(-1).cpu()
            assert untouched[:, 2::3].all() and untouched[:, :, 2::3].all()
            assert torch.equal(acc[:, 2::3], base[:, 2::3]) and torch.equal(acc[:, :, 2::3], base[:, :, 2::3])
            assert torch.equal(dxs[0][:, 2::3], torch.zeros_like(dxs[0][:, 2::3]))
    torch.cuda.synchronize()
    print(f"[{case} tc={tc}] wgrad splits {z} (asked {asked}); " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v < CONV_TOL for v in errs.values()), errs


#            what, entry point, N, H, W, Ci, Cw, Co, kh, kw, stride, pad_lo, pad_hi
REFUSED = [("Ci % 4 != 0", "fwd", 1, 8, 8, 6, 6, 16, 3, 3, 1, 1, 1),
           ("Ci % 4 != 0", "wgrad", 1, 8, 8, 6, 6, 16, 3, 3, 1, 1, 1),
           ("Cw > Ci", "fwd", 1, 8, 8, 8, 12, 16, 3, 3, 1, 1, 1),
           ("Cw > Ci", "wgrad", 1, 8, 8, 8, 12, 16, 3, 3, 1, 1, 1),
           ("pad_lo >= kh", "fwd", 1, 8, 8, 8, 8, 16, 3, 3, 1, 3, 1),
           ("pad_lo >= kw", "dgrad", 1, 8, 8, 8, 8, 16, 3, 1, 1, 1, 1),
           ("pad_lo >= kw", "wgrad", 1, 8, 8, 8, 8, 16, 5, 2, 1, 2, 2),
           ("H % stride != 0", "dgrad", 1, 9, 8, 8, 8, 16, 3, 3, 2, 1, 1),
           ("W % stride != 0", "dgrad", 1, 9, 10, 8, 8, 16, 3, 3, 3, 1, 1)]


@pytest.mark.parametrize("refused", REFUSED, ids=[f"{r[1]}: {r[0]}" for r in REFUSED])
def test_rconv_refuses_unsupported_shapes(refused):
    from serl_b200 import _lib as L
    _, mode, N, H, W, Ci, Cw, Co, kh, kw, s, lo, hi = refused
    st = L.stream_ptr()
    big = torch.zeros(1 << 20, device="cuda")
    p = big.data_ptr()
    n0 = L.launch_count()
    with pytest.raises(L.SerlError, match="unsupported shape"):
        if mode == "fwd":
            _call("serl_rconv_fwd", p, p, p, N, H, W, Ci, Cw, Co, kh, kw, s, lo, hi, 1, st)
        elif mode == "dgrad":
            _call("serl_rconv_dgrad", p, p, p, N, H, W, Ci, Co, kh, kw, s, lo, hi, 0, 1, st)
        else:
            _call("serl_rconv_wgrad", p, p, p, p, big.numel() * 4, N, H, W, Ci, Cw, Co, kh, kw, s, lo, hi, 1, st)
    assert L.launch_count() == n0
    torch.cuda.synchronize()
    assert not big.any()


GN_WIDTHS = (4, 12, 24, 48, 64, 320, 512)          # C / G; 512 % (C/G/4) != 0 at 12, 24, 48 and 320


@pytest.mark.parametrize("mode", ["plain", "relu", "relu+residual"])
@pytest.mark.parametrize("cg", GN_WIDTHS)
def test_groupnorm_widths_match_float64(cg, mode):
    from serl_b200 import ops
    relu, res_on = mode != "plain", mode == "relu+residual"
    g = torch.Generator(device="cuda").manual_seed(1000 * cg + len(mode))
    N, worst = 2, {}
    for G in (1, 2, 4, 8):
        C = G * cg
        for H in (4, 16):
            x = torch.randn(N, H, H, C, device="cuda", generator=g) * 2 + 0.5
            sc = 1 + 0.3 * torch.randn(C, device="cuda", generator=g)
            bi = 0.2 * torch.randn(C, device="cuda", generator=g)
            res = torch.randn(x.shape, device="cuda", generator=g) if res_on else None
            y = torch.empty_like(x)
            ops.groupnorm_nhwc(x, y, sc, bi, res, G, 1e-5, relu)
            x64, s64, b64 = x.double().requires_grad_(), sc.double().requires_grad_(), bi.double().requires_grad_()
            r64 = res.double().requires_grad_() if res_on else None
            ref = drq.group_norm_nhwc(x64, s64, b64, groups=G)
            if res_on:
                ref = ref + r64
            fwd = ref.relu() if relu else ref
            e = {"fwd": _err(y, fwd)}
            dy = torch.randn(x.shape, device="cuda", generator=g)
            if relu:                                # the kernel's mask is the fp32 forward's output: gate the reference the same way
                ref = ref * (y > 0).double()
            (ref * dy.double()).sum().backward()
            ws = torch.empty(ops.groupnorm_bwd_workspace(N, C, G), device="cuda")
            outs = []
            for _ in range(2):
                o = (torch.full_like(x, float("nan")), torch.full_like(x, float("nan")) if res_on else None, torch.empty_like(sc),
                     torch.empty_like(bi))
                ops.groupnorm_bwd_nhwc(x.data_ptr(), y.data_ptr(), dy.data_ptr(), sc.data_ptr(), o[0].data_ptr(),
                                       o[1].data_ptr() if res_on else None, o[2].data_ptr(), o[3].data_ptr(), ws, N, H * H, C, G, 1e-5, relu)
                outs.append(o)
            dx, dres, ds, db = outs[0]
            e.update(dx=_err(dx, x64.grad), dscale=_err(ds, s64.grad), dbias=_err(db, b64.grad))
            if res_on:
                e["dres"] = _err(dres, r64.grad)
            for a, b in zip(outs[0], outs[1]):
                assert a is None or torch.equal(a, b), (G, H, "two launches differ")
            for k, v in e.items():
                worst[k] = max(worst.get(k, 0.0), v)
            assert all(v < 2e-4 for v in e.values()), (G, H, e)       # (a NaN, i.e. an entry never written, fails too)
    print(f"[C/G={cg} {mode}] " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


@pytest.mark.parametrize("hw", [(64, 64), (63, 63), (64, 63), (63, 64), (2, 2), (1, 1)], ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_maxpool_sizes_match_first_max(hw):
    """Values on a coarse grid (many ties) with a block of all-zero windows: the forward bitwise equal to the float64 SAME pool,
    the backward's gradient on each window's first maximal element."""
    from serl_b200 import _lib as L
    from serl_b200 import ops
    H, W = hw
    N = 2
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    for C in (8, 6):
        g = torch.Generator(device="cuda").manual_seed(H * 100 + W + C)
        x = torch.randint(0, 4, (N, H, W, C), device="cuda", generator=g).float() * 0.5
        x[:, :5, :5] = 0
        x64 = x.double().requires_grad_()
        ref = max_pool_first_max(x64)
        assert ref.shape == (N, Ho, Wo, C)
        if C % 4 == 0:                                  # the forward takes float4 channel groups
            y = torch.full((N, Ho, Wo, C), float("nan"), device="cuda")
            L.call("serl_maxpool3x3s2_nhwc_f32", x.data_ptr(), y.data_ptr(), N, H, W, C, L.stream_ptr())
            assert torch.equal(y.double(), ref.detach()), (hw, C, int((y.double() != ref.detach()).sum()))
        dy = torch.randn(N, Ho, Wo, C, device="cuda", generator=g)
        (ref * dy.double()).sum().backward()
        dxs = [torch.full_like(x, float("nan")) for _ in range(2)]
        for dx in dxs:
            ops.maxpool3x3s2_bwd_nhwc(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), N, H, W, C)
        assert _err(dxs[0], x64.grad) < 1e-6, (hw, C, _err(dxs[0], x64.grad))
        assert ((dxs[0] != 0) == (x64.grad != 0)).all(), (hw, C)
        assert torch.equal(dxs[0], dxs[1]), (hw, C)


def test_stem_prep_past_grid_cap_bitwise():
    from serl_b200 import ops
    N, H, W = 3, 480, 400                               # 576000 pixels > 132 * 16 * 256 = 540672: the grid strides
    assert N * H * W > 132 * 16 * 256
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device="cuda", generator=g)
    x[0, 0, 0] = torch.tensor([0, 255, 128], dtype=torch.uint8)
    y = torch.full((N, H, W, 4), float("nan"), device="cuda")
    ops.rconv_stem_prep(x.data_ptr(), y.data_ptr(), N, H, W)
    mean = torch.tensor(drq.IMAGENET_MEAN, dtype=torch.float32, device="cuda")
    std = torch.tensor(drq.IMAGENET_STD, dtype=torch.float32, device="cuda")
    ref = (x.float() / torch.full((), 255.0, device="cuda") - mean) / std     # a tensor divisor: torch divides, as the kernel
    assert torch.equal(y[..., :3], ref), int((y[..., :3] != ref).sum())
    assert torch.equal(y[..., 3], torch.zeros_like(y[..., 3]))
