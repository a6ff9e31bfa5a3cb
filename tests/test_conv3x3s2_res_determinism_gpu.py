"""GPU: the stride-2 block head (3x3/2 conv + GroupNorm + ReLU and the 1x1/2 projection + GroupNorm in one kernel) is
deterministic.  Every GroupNorm group of a work item lies inside one CTA and its sums are reduced in a fixed order (thread,
warp shuffles, warps in order), so two launches on the same input give bit-identical y and r, including the partial last item
of a multi-image head (N not a multiple of the images per item)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("Wo,Co,N", [(16, 128, 77), (8, 256, 123), (4, 512, 141)])
def test_conv3x3s2_res_two_launches_bitwise_equal(Wo, Co, N, prec):
    from serl_b200 import trunk_bf16 as T
    rng = np.random.default_rng(Wo + N)
    dt, Ci = DT[prec], Co // 2
    cu = lambda v: torch.as_tensor(v).cuda().contiguous()
    x = cu(np.abs(rng.standard_normal((N, 2 * Wo, 2 * Wo, Ci))).astype(np.float32)).to(dt)
    w = T.pack_conv_weight(cu((rng.standard_normal((3, 3, Ci, Co)) * np.sqrt(2.0 / (9 * Ci))).astype(np.float32)), dt)
    wp = T.pack_conv_weight(cu((rng.standard_normal((1, 1, Ci, Co)) * np.sqrt(2.0 / Ci)).astype(np.float32)), dt)
    g0, b0, gp, bp = [cu((s + 0.3 * rng.standard_normal(Co)).astype(np.float32)) for s in (1, 0, 1, 0)]
    plan = T._Plan(N, 128, "cuda", prec)
    outs = []
    for _ in range(2):
        y = torch.full((N, Wo, Wo, Co), float("nan"), dtype=dt, device="cuda")
        r = torch.full((N, Wo, Wo, Co), float("nan"), dtype=dt, device="cuda")
        T._conv_s2_res(plan, x, w, wp, y, r, g0, b0, gp, bp, N, Wo, Ci, Co)
        torch.cuda.synchronize()
        assert int(plan.error.item()) == 0, f"pipeline barrier timeout (flags {int(plan.error.item())})"
        assert torch.isfinite(y.float()).all() and torch.isfinite(r.float()).all()
        outs.append((y.view(torch.int16).cpu(), r.view(torch.int16).cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
