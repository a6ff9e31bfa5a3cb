"""GPU: the fused stem (conv_init + GroupNorm sums + 3x3/2 max-pool) at the benchmark's camera-pass size, where every CTA
runs several images and its two consumer warpgroups alternate chunk by chunk, and at the extremes of the sign mask (every
GroupNorm scale positive, every one negative, mixed).  The pooled bits must equal conv -> finalize -> maxpool(relu(a x + b)),
and the statistics the float64 sums of that conv's raw output."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _gamma(kind, rng):
    g = rng.standard_normal(64) + 0.3
    if kind == "positive":
        g = np.abs(g) + 0.05
    elif kind == "negative":
        g = -np.abs(g) - 0.05
    return torch.as_tensor(g.astype(np.float32)).cuda()


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("N", [512, 515])
@pytest.mark.parametrize("signs", ["positive", "negative", "mixed"])
def test_stem_pool_bench_size_sign_masks(N, prec, signs):
    from oracle.drq import IMAGENET_MEAN, IMAGENET_STD, conv_nhwc
    from serl_b200 import _lib as L
    from serl_b200 import trunk_bf16 as T
    rng = np.random.default_rng(31)
    pix = torch.as_tensor(rng.integers(0, 256, (N, 128, 128, 3), dtype=np.uint8)).cuda()
    w = torch.as_tensor((rng.standard_normal((7, 7, 3, 64)) * np.sqrt(2.0 / 147)).astype(np.float32)).cuda()
    gamma = _gamma(signs, rng)
    beta = torch.as_tensor((0.2 * rng.standard_normal(64)).astype(np.float32)).cuda()
    wp = T.pack_stem_weight(w, DT[prec])
    plan = T._Plan(N, 128, "cuda", prec)
    s = L.stream_ptr()
    L.call("serl_trunk_stem_prep_h16", pix.data_ptr(), plan.xs.data_ptr(), N, 128, 128, plan.fmt, s)
    # separate path: raw conv -> finalize -> pool(relu(affine))
    st_ref = torch.zeros(N, 4, 2, device="cuda")
    y0 = torch.empty(N, 64, 64, 64, dtype=DT[prec], device="cuda")
    T._conv(plan, plan.xs, wp, y0, st_ref, N, plan.hs, plan.hs, 12, 64, 64, 64, 4, 1, 0, stem=True)
    aff = torch.empty(2, N, 64, device="cuda")
    a, b = T._finalize(st_ref, gamma, beta, aff, N, 64, 64 * 64)
    ref = torch.empty(N, 32, 32, 64, dtype=DT[prec], device="cuda")
    L.call("serl_maxpool_affine_h16", y0.data_ptr(), a.data_ptr(), b.data_ptr(), ref.data_ptr(), N, 64, 64, 64, plan.fmt, s)
    # fused path
    st = torch.zeros(N, 4, 2, device="cuda")
    pooled = torch.full((N, 32, 32, 64), float("nan"), dtype=DT[prec], device="cuda")
    side = torch.full((N, 4, 32, 64), float("nan"), dtype=DT[prec], device="cuda")
    d = L.StemPoolDesc()
    d.xs, d.w, d.pooled, d.side, d.stats, d.error = plan.xs.data_ptr(), wp.data_ptr(), pooled.data_ptr(), side.data_ptr(), st.data_ptr(), plan.error.data_ptr()
    d.neg_mask = sum(1 << c for c, g in enumerate(gamma.cpu().tolist()) if g < 0)
    d.N, d.fmt = N, plan.fmt
    L.call("serl_stem_conv_pool_tc_h16", C.byref(d), s)
    out = torch.empty(N, 32, 32, 64, dtype=DT[prec], device="cuda")
    L.call("serl_pool_finish_h16", pooled.data_ptr(), side.data_ptr(), a.data_ptr(), b.data_ptr(), out.data_ptr(), N, plan.fmt, s)
    torch.cuda.synchronize()
    assert int(plan.error.item()) == 0, f"pipeline barrier timeout (flags {int(plan.error.item())})"
    assert (d.neg_mask == 0) == (signs == "positive") and (d.neg_mask == (1 << 64) - 1) == (signs == "negative")
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
    # statistics: float64 sums of the raw conv output, the 7x7/2 conv restated in float64 on the 16-bit operands
    xn = (pix.double() / 255.0 - torch.tensor(IMAGENET_MEAN, device="cuda").double()) / torch.tensor(IMAGENET_STD, device="cuda").double()
    y64 = conv_nhwc(xn.float().to(DT[prec]).double(), w.to(DT[prec]).double(), 2, 3, 3)
    G = y64.reshape(N, 64 * 64, 4, 16)
    want = torch.stack([G.sum(dim=(1, 3)), (G * G).sum(dim=(1, 3))], -1).cpu().numpy()
    np.testing.assert_allclose(st.double().cpu().numpy(), want, rtol=1e-4, atol=1e-2)
