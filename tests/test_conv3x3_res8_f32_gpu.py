"""GPU: the 8x8x256 conv + GroupNorm written as fp32 (out_f32) vs float64 on the 16-bit operands.  The trunk writes fp32 only at
4x4, so this is the only check of the 8x8 kernel's fp32 store; it also covers the residual modes and relu off there."""
import numpy as np
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _gn64(y, gamma, beta, eps=1e-5):
    n, h, w, c = y.shape
    g = y.reshape(n, h * w, 4, c // 4)
    mean = g.mean(dim=(1, 3), keepdim=True)
    var = ((g * g).mean(dim=(1, 3), keepdim=True) - mean * mean).clamp_min(0)
    return ((g - mean) / torch.sqrt(var + eps)).reshape(n, h, w, c) * gamma + beta


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("N,mode,relu", [(5, "proj", True), (131, "identity", True), (7, "plain", False)])
def test_conv3x3_res_8x8_out_f32_matches_float64(N, mode, relu, prec):
    from oracle.drq import conv_nhwc
    from serl_b200 import trunk_bf16 as T
    HW, C = 8, 256
    rng = np.random.default_rng(8000 + N)
    dt = DT[prec]
    q = lambda v: torch.as_tensor(v).to(dt)
    x = q(np.abs(rng.standard_normal((N, HW, HW, C))).astype(np.float32))
    w = (rng.standard_normal((3, 3, C, C)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)
    gamma = (1 + 0.3 * rng.standard_normal(C)).astype(np.float32)
    beta = (0.2 * rng.standard_normal(C)).astype(np.float32)
    ref = _gn64(conv_nhwc(x.double(), q(w).double(), 1, 1, 1), torch.as_tensor(gamma).double(), torch.as_tensor(beta).double())
    cu = lambda t: torch.as_tensor(t).cuda().contiguous()
    kw = {}
    if mode == "identity":
        res = q(np.abs(rng.standard_normal((N, HW, HW, C))).astype(np.float32))
        ref = ref + res.double()
        kw = dict(res=cu(res))
    elif mode == "proj":
        raw = q((2 * rng.standard_normal((N, HW, HW, C)) + 0.5).astype(np.float32))
        rg = (1 + 0.3 * rng.standard_normal(C)).astype(np.float32)
        rb = (0.2 * rng.standard_normal(C)).astype(np.float32)
        ref = ref + _gn64(raw.double(), torch.as_tensor(rg).double(), torch.as_tensor(rb).double())
        G = raw.double().reshape(N, HW * HW, 4, C // 4)
        st = torch.stack([G.sum(dim=(1, 3)), (G * G).sum(dim=(1, 3))], dim=-1).float()
        kw = dict(res=cu(raw), res_stats=cu(st), res_gamma=cu(rg), res_beta=cu(rb))
    ref = ref.relu() if relu else ref
    plan = T._Plan(N, 128, "cuda", prec)
    yf = torch.full((N, HW, HW, C), float("nan"), dtype=torch.float32, device="cuda")
    T._conv_res(plan, cu(x), T.pack_conv_weight(cu(w), dt), None, cu(gamma), cu(beta), N, HW, C, relu=relu, out_f32=yf, **kw)
    torch.cuda.synchronize()
    assert int(plan.error.item()) == 0, f"pipeline barrier timeout (flags {int(plan.error.item())})"
    got = yf.cpu().numpy()
    assert np.isfinite(got).all()
    assert rel_err(got, ref.numpy()) < 2e-5
