"""GPU: the 8x8x256 and 4x4x512 stride-1 3x3 conv + GroupNorm kernel is deterministic.  Each CTA item holds whole images x 128
channels, so every GroupNorm group is reduced inside one CTA in a fixed order (no float atomics): two launches on the same input
give bit-identical outputs, in every residual mode and with partial items (N not a multiple of the images per item).  With it
the whole default 16-bit trunk is bitwise repeatable."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("HW,C,N,mode", [
    (8, 256, 5, "plain"), (8, 256, 301, "identity"), (8, 256, 19, "proj"), (8, 256, 5, "proj_f32"),
    (4, 512, 19, "plain"), (4, 512, 5, "identity"), (4, 512, 301, "proj"), (4, 512, 19, "proj_f32")])
def test_conv3x3_res_deep_two_launches_bitwise_equal(HW, C, N, mode, prec):
    from serl_b200 import trunk_bf16 as T
    rng = np.random.default_rng(HW * 1000 + N)
    dt = DT[prec]
    cu = lambda v: torch.as_tensor(v).cuda().contiguous()
    x = cu(np.abs(rng.standard_normal((N, HW, HW, C))).astype(np.float32)).to(dt)
    w = T.pack_conv_weight(cu((rng.standard_normal((3, 3, C, C)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)), dt)
    gamma = cu((1 + 0.3 * rng.standard_normal(C)).astype(np.float32))
    beta = cu((0.2 * rng.standard_normal(C)).astype(np.float32))
    kw = {}
    if mode == "identity":
        kw = dict(res=cu(np.abs(rng.standard_normal((N, HW, HW, C))).astype(np.float32)).to(dt))
    elif mode.startswith("proj"):
        raw = cu((2 * rng.standard_normal((N, HW, HW, C)) + 0.5).astype(np.float32)).to(dt)
        G = raw.double().reshape(N, HW * HW, 4, C // 4)
        st = torch.stack([G.sum(dim=(1, 3)), (G * G).sum(dim=(1, 3))], dim=-1).float().contiguous()
        kw = dict(res=raw, res_stats=st, res_gamma=cu((1 + 0.3 * rng.standard_normal(C)).astype(np.float32)),
                  res_beta=cu((0.2 * rng.standard_normal(C)).astype(np.float32)))
    f32 = mode == "proj_f32"
    plan = T._Plan(N, 128, "cuda", prec)
    outs = []
    for _ in range(2):
        y = torch.full((N, HW, HW, C), float("nan"), dtype=torch.float32 if f32 else dt, device="cuda")
        T._conv_res(plan, x, w, None if f32 else y, gamma, beta, N, HW, C, relu=True, out_f32=y if f32 else None, **kw)
        torch.cuda.synchronize()
        assert int(plan.error.item()) == 0, f"pipeline barrier timeout (flags {int(plan.error.item())})"
        outs.append(y.view(torch.int32 if f32 else torch.int16).cpu())
    assert torch.isfinite(y.float()).all()
    assert torch.equal(outs[0], outs[1])


def test_trunk_forward_bitwise_repeatable():
    """Two passes of the default 16-bit trunk over the same 512 frames give bit-identical fp32 features."""
    from serl_b200.utils.launcher import make_drq_agent
    from helpers import random_transitions
    cams = ("cam0",)
    tr = random_transitions(np.random.default_rng(0), 1, cams)[0]
    agent = make_drq_agent(42, tr["observations"], tr["actions"], image_keys=cams, encoder_type="resnet-pretrained", precision="fp16")
    eng = agent._engine(256)
    g = torch.Generator(device="cuda").manual_seed(3)
    eng.pix["cam0"].copy_(torch.randint(0, 256, eng.pix["cam0"].shape, dtype=torch.uint8, device="cuda", generator=g))
    N = eng.pix["cam0"].shape[0]
    assert N == 512
    outs = []
    for _ in range(2):
        eng.feats["cam0"].fill_(float("nan"))
        eng.trunk_forward("cam0", eng.pix["cam0"], eng.feats["cam0"])
        torch.cuda.synchronize()
        outs.append(eng.feats["cam0"][:N].clone())
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
