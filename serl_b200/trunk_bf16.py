"""16-bit / tensor-core (wgmma) build of the frozen ResNet-10 trunk: orchestration + weight packing.

Same layer algebra as the fp32 build (trunk.TrunkRunner.forward; reference vision/resnet_v1.py:217-286),
re-associated so that GroupNorm never makes its own pass over HBM:
  every conv (tensor cores) writes its raw 16-bit output and accumulates the GroupNorm sums in its epilogue;
  the consumer of that output derives the per-(image, channel) affine from the sums in registers and applies it:
    stem:   the 3x3/2 max-pool runs inside the stem epilogue on sign-adjusted raw values, `pool_finish` applies relu(|a|x+b);
    Conv_0: `affine_relu` materialises relu(GN(y)) in place (one HBM-speed pass), so Conv_1's operands are plain async copies;
    Conv_1 / conv_proj: `block_combine` applies both affines, adds the residual and the ReLU.
The projection conv of a block runs on a side stream next to the Conv_0 -> Conv_1 chain.  Weights and scratch come from
trunk.py: `FrozenTrunk.packed` keeps the packing (`pack_trunk`) of each camera, a `TrunkRunner` the plans and side streams.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _lib as L
from .params import STAGES


def _s():
    return L.stream_ptr()


# Stride-1 3x3 convs go through serl_conv3x3s1_tc_h16 (on sm_90a the implicit-GEMM kernel serves it as well).
USE_SHIFTED_WINDOW = True
BASE_OFFSET_MODE = 0

# conv_init + GroupNorm + ReLU + max-pool: pool inside the stem epilogue (the 64x64x64 map never reaches HBM).
USE_FUSED_STEM_POOL = True

# GroupNorm affines derived inside the consumers from the conv epilogue sums (no serl_gn_finalize launches in the chain).
USE_FUSED_GN = True
GN_EPS = 1e-5

# Stride-1 3x3 convs with GroupNorm (+ residual) (+ ReLU) inside the conv kernel (conv3x3_res.cu): an image's fp32 accumulators
# stay in registers until its statistics are complete, so neither the raw conv output nor a normalisation pass touches HBM
# (no affine_relu after ResNetBlock_0/Conv_0, no block_combine after any Conv_1).  SERL_RES_CONV=0 selects the conv +
# GroupNorm-pass path.
USE_RES_CONV = os.environ.get("SERL_RES_CONV", "1") != "0"

# Head of ResNetBlock_1..3 (stride-2 3x3 conv + GN + ReLU AND the 1x1 stride-2 projection + GN) in one kernel
# (conv3x3s2_res_kernel): no separate projection conv, no affine_relu pass.  Needs USE_RES_CONV.  SERL_RES_S2=0 keeps round 1's kernels.
USE_RES_S2 = os.environ.get("SERL_RES_S2", "1") != "0"

FMT = {"bf16": (L.FMT_BF16, torch.bfloat16), "fp16": (L.FMT_FP16, torch.float16)}


def pack_conv_weight(w: torch.Tensor, dt=torch.bfloat16) -> torch.Tensor:
    """HWIO fp32 (kh,kw,Ci,Co) -> 16-bit [Co][kh*kw*Ci], K-major (K order = (kh, kw, ci), the im2col gather order)."""
    kh, kw, ci, co = w.shape
    return w.permute(3, 0, 1, 2).reshape(co, kh * kw * ci).to(dt).contiguous()


def pack_stem_weight(w: torch.Tensor, dt=torch.bfloat16) -> torch.Tensor:
    """conv_init (7,7,3,64) -> exact 4x4 space-to-depth kernel, 16-bit [64][4 rows x 64] (4 taps x (12 real + 4 zero) ch per row).
    ws[r', s', p, q, c, co] = w8[2r'+p, 2s'+q, c, co] with w8 = w zero-extended to 8x8."""
    co = w.shape[-1]
    w8 = torch.zeros(8, 8, 3, co, dtype=w.dtype, device=w.device)
    w8[:7, :7] = w
    ws = w8.view(4, 2, 4, 2, 3, co).permute(0, 2, 1, 3, 4, 5)            # (r', s', p, q, c, co)
    rows = ws.reshape(4, 4, 12, co)                                     # (r', s', (p*2+q)*3 + c, co)
    out = torch.zeros(co, 4, 4, 16, dtype=torch.float32, device=w.device)  # k within a row = s'*16 + (p*2+q)*3 + c; 4 zero channels per tap
    out[:, :, :, :12] = rows.permute(3, 0, 1, 2)
    return out.reshape(co, 256).to(dt).contiguous()


def pack_trunk(w, dt) -> dict:
    """One camera's fp32 HWIO leaves -> the kernels' 16-bit weights, and the stem's sign mask."""
    packed = {k: (pack_stem_weight(v, dt) if k == "conv_init/kernel" else pack_conv_weight(v, dt)) for k, v in w.items() if k.endswith("kernel")}
    # sign of the frozen norm_init scale per channel: which way relu(a*x+b) is monotone (fused stem max-pool)
    packed["_stem_neg_mask"] = sum(1 << c for c, g in enumerate(w["norm_init/scale"].detach().cpu().tolist()) if g < 0)
    return packed


class _Plan:
    """16-bit activation buffers of one camera's passes over up to N images.  `error` is the fault flag the kernels raise on a
    pipeline-barrier timeout: a trunk runner passes its own; a plan made alone (kernel tests) gets a fresh one."""

    def __init__(self, N, hw, dev, precision="bf16", error=None):
        self.fmt, self.dt = FMT[precision]
        bf = lambda *s: torch.empty(*s, dtype=self.dt, device=dev)
        s2 = hw // 2
        self.hs = s2 + 3
        self.xs = bf(N, self.hs, self.hs, 16)
        self.fused_pool = USE_FUSED_STEM_POOL and hw == 128
        if self.fused_pool:
            self.pooled, self.side = bf(N, 32, 32, 64), bf(N, 4, 32, 64)
        else:
            self.y0 = bf(N, s2, s2, 64)
        self.buf = [bf(N * (s2 // 2) * (s2 // 2) * 64) for _ in range(5)]
        self.stats = torch.zeros(16, N, 4, 2, dtype=torch.float32, device=dev)     # one slot per conv, zeroed by ONE memset per pass
        self.aff = torch.empty(3, 2, N, 512, dtype=torch.float32, device=dev)
        self.error = torch.zeros(1, dtype=torch.int32, device=dev) if error is None else error


def _conv(plan, x, w, y, stats, N, Hi, Wi, Ci, Ho, Wo, Co, k, stride, pad_lo, in_ab=None, stem=False):
    d = L.ConvTcDesc()
    d.x, d.w, d.y, d.stats = x.data_ptr(), w.data_ptr(), y.data_ptr(), stats.data_ptr()
    if in_ab is not None:
        d.in_a, d.in_b = in_ab[0].data_ptr(), in_ab[1].data_ptr()
    d.error = plan.error.data_ptr()
    d.N, d.Hi, d.Wi, d.Ci, d.Ho, d.Wo, d.Co, d.kh, d.kw, d.stride, d.pad_lo, d.stem, d.fmt = N, Hi, Wi, Ci, Ho, Wo, Co, k, k, stride, pad_lo, int(stem), plan.fmt
    if USE_SHIFTED_WINDOW and k == 3 and stride == 1 and pad_lo == 1 and in_ab is None and not stem and Wi <= 32 and Ci % 64 == 0:
        L.call("serl_conv3x3s1_tc_h16", C.byref(d), BASE_OFFSET_MODE, _s())
    else:
        L.call("serl_conv2d_tc_h16", C.byref(d), _s())


def _conv_res(plan, x, w, y, gamma, beta, N, HW_, C_, *, res=None, res_stats=None, res_gamma=None, res_beta=None, relu=True, out_f32=None):
    """y = [relu](GN(conv3x3(x)) [+ res | + GN_res(res)]) in one launch (serl_conv3x3_res_h16)."""
    d = L.Conv3x3ResDesc()
    d.x, d.w = x.data_ptr(), w.data_ptr()
    d.y = None if y is None else y.data_ptr()
    d.out_f32 = None if out_f32 is None else out_f32.data_ptr()
    d.res = None if res is None else res.data_ptr()
    d.gamma, d.beta = gamma.data_ptr(), beta.data_ptr()
    if res_stats is not None:
        d.res_stats, d.res_gamma, d.res_beta = res_stats.data_ptr(), res_gamma.data_ptr(), res_beta.data_ptr()
    d.error = plan.error.data_ptr()
    d.N, d.H, d.W, d.Ci, d.Co, d.relu, d.fmt, d.eps = N, HW_, HW_, C_, C_, int(relu), plan.fmt, GN_EPS
    L.call("serl_conv3x3_res_h16", C.byref(d), _s())


def _conv_s2_res(plan, x, w, w_proj, y, r, gamma, beta, gamma_p, beta_p, N, Wo, Ci, Co):
    """y = relu(GN(conv3x3 s2 (x))), r = GN(conv1x1 s2 (x)) in one launch (serl_conv3x3s2_res_h16)."""
    d = L.Conv3x3S2ResDesc()
    d.x, d.w, d.w_proj, d.y, d.r = x.data_ptr(), w.data_ptr(), w_proj.data_ptr(), y.data_ptr(), r.data_ptr()
    d.gamma, d.beta, d.gamma_proj, d.beta_proj = gamma.data_ptr(), beta.data_ptr(), gamma_p.data_ptr(), beta_p.data_ptr()
    d.error = plan.error.data_ptr()
    d.N, d.Wo, d.Ci, d.Co, d.fmt, d.eps = N, Wo, Ci, Co, plan.fmt, GN_EPS
    L.call("serl_conv3x3s2_res_h16", C.byref(d), _s())


def _finalize(stats, gamma, beta, ab, N, Cc, HW):
    a, b = ab[0].view(-1)[:N * Cc].view(N, Cc), ab[1].view(-1)[:N * Cc].view(N, Cc)
    L.call("serl_gn_finalize", stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), a.data_ptr(), b.data_ptr(), N, Cc, HW, 1e-5, _s())
    return a, b


def forward(p: _Plan, w, wp, side, pix: torch.Tensor, feats: torch.Tensor):
    """pix (N,hw,hw,3) uint8 -> feats[:N] (N,4,4,512) fp32 on the plan's buffers; w: fp32 leaves, wp: their packing (pack_trunk),
    side: the side stream of the projection convs, or None to run them in stream order."""
    N, hw = pix.shape[0], pix.shape[1]
    s = hw // 2
    L.call("serl_trunk_stem_prep_h16", pix.data_ptr(), p.xs.data_ptr(), N, hw, hw, p.fmt, _s())
    p.stats.zero_()
    st = iter(p.stats)
    st0 = next(st)
    if p.fused_pool:
        d = L.StemPoolDesc()
        d.xs, d.w, d.pooled, d.side = p.xs.data_ptr(), wp["conv_init/kernel"].data_ptr(), p.pooled.data_ptr(), p.side.data_ptr()
        d.stats, d.error, d.neg_mask, d.N, d.fmt = st0.data_ptr(), p.error.data_ptr(), wp["_stem_neg_mask"], N, p.fmt
        L.call("serl_stem_conv_pool_tc_h16", C.byref(d), _s())
    else:
        _conv(p, p.xs, wp["conv_init/kernel"], p.y0, st0, N, p.hs, p.hs, 12, s, s, 64, 4, 1, 0, stem=True)
    g0, be0 = w["norm_init/scale"], w["norm_init/bias"]
    if not (USE_FUSED_GN and p.fused_pool):
        a0, b0 = _finalize(st0, g0, be0, p.aff[0], N, 64, s * s)
    s //= 2
    x = p.buf[0][:N * s * s * 64].view(N, s, s, 64)
    if p.fused_pool and USE_FUSED_GN:
        L.call("serl_pool_finish_gn_h16", p.pooled.data_ptr(), p.side.data_ptr(), st0.data_ptr(), g0.data_ptr(), be0.data_ptr(), x.data_ptr(),
               N, GN_EPS, p.fmt, _s())
    elif p.fused_pool:
        L.call("serl_pool_finish_h16", p.pooled.data_ptr(), p.side.data_ptr(), a0.data_ptr(), b0.data_ptr(), x.data_ptr(), N, p.fmt, _s())
    else:
        L.call("serl_maxpool_affine_h16", p.y0.data_ptr(), a0.data_ptr(), b0.data_ptr(), x.data_ptr(), N, 2 * s, 2 * s, 64, p.fmt, _s())
    free, cur, cin = [1, 2, 3, 4], 0, 64
    for i, (f, stride) in enumerate(STAGES):
        b = f"ResNetBlock_{i}"
        so = s // stride
        iy, iy2, ir, io = free
        view = lambda j: p.buf[j][:N * so * so * f].view(N, so, so, f)
        yA, yB, yP, out = view(iy), view(iy2), view(ir), view(io)
        sA, sB, sP = next(st), next(st), next(st)
        lo = 1 if stride == 1 else 0                                   # XLA SAME on even sizes: pad low 0 / high 1
        gA, bA = w[f"{b}/MyGroupNorm_0/scale"], w[f"{b}/MyGroupNorm_0/bias"]
        gB, bB = w[f"{b}/MyGroupNorm_1/scale"], w[f"{b}/MyGroupNorm_1/bias"]
        proj = stride != 1 or cin != f
        last = i == len(STAGES) - 1
        res_ok = USE_RES_CONV and USE_FUSED_GN and {32: 64, 16: 128, 8: 256, 4: 512}.get(so) == f
        if res_ok and USE_RES_S2 and proj and stride == 2 and f == 2 * cin:
            gP, bP = w[f"{b}/norm_proj/scale"], w[f"{b}/norm_proj/bias"]
            _conv_s2_res(p, x, wp[f"{b}/Conv_0/kernel"], wp[f"{b}/conv_proj/kernel"], yA, yP, gA, bA, gP, bP, N, so, cin, f)
            _conv_res(p, yA, wp[f"{b}/Conv_1/kernel"], None if last else out, gB, bB, N, so, f, res=yP, relu=True, out_f32=feats if last else None)
            free, cur = [cur, iy, iy2, ir], io
            x, s, cin = out, so, f
            continue
        if proj:
            gP, bP = w[f"{b}/norm_proj/scale"], w[f"{b}/norm_proj/bias"]
            if side is not None:
                side.fork()
                with side:
                    _conv(p, x, wp[f"{b}/conv_proj/kernel"], yP, sP, N, s, s, cin, so, so, f, 1, stride, 0)
        if res_ok and stride == 1 and cin == f:
            # ResNetBlock_0: both convs are stride-1 3x3: conv -> GN -> ReLU in one kernel (activated output, no affine_relu pass)
            _conv_res(p, x, wp[f"{b}/Conv_0/kernel"], yA, gA, bA, N, so, f, relu=True)
        else:
            _conv(p, x, wp[f"{b}/Conv_0/kernel"], yA, sA, N, s, s, cin, so, so, f, 3, stride, lo)
            # materialise relu(GN(yA)) in place (one HBM-speed pass); the conv operands are then plain async copies
            if USE_FUSED_GN:
                L.call("serl_affine_relu_gn_h16", yA.data_ptr(), sA.data_ptr(), gA.data_ptr(), bA.data_ptr(), N, so * so, f, GN_EPS, p.fmt, _s())
            else:
                abA = _finalize(sA, gA, bA, p.aff[0], N, f, so * so)
                L.call("serl_affine_relu_h16", yA.data_ptr(), abA[0].data_ptr(), abA[1].data_ptr(), N, so * so, f, p.fmt, _s())
        if res_ok:
            # Conv_1 -> GN -> (+ residual: block input, or GN(projection) applied on the fly) -> ReLU in one kernel: no block_combine
            if proj and side is None:
                _conv(p, x, wp[f"{b}/conv_proj/kernel"], yP, sP, N, s, s, cin, so, so, f, 1, stride, 0)
            elif proj:
                side.join()
            _conv_res(p, yA, wp[f"{b}/Conv_1/kernel"], None if last else out, gB, bB, N, so, f, res=yP if proj else x,
                      res_stats=sP if proj else None, res_gamma=gP if proj else None, res_beta=bP if proj else None, relu=True,
                      out_f32=feats if last else None)
            free, cur = [cur, iy, iy2, ir], io
            x, s, cin = out, so, f
            continue
        _conv(p, yA, wp[f"{b}/Conv_1/kernel"], yB, sB, N, so, so, f, so, so, f, 3, 1, 1)
        if proj and side is None:
            _conv(p, x, wp[f"{b}/conv_proj/kernel"], yP, sP, N, s, s, cin, so, so, f, 1, stride, 0)
        elif proj:
            side.join()
        o16, o32 = (None if last else out.data_ptr()), (feats.data_ptr() if last else None)
        if USE_FUSED_GN:
            L.call("serl_block_combine_gn_h16", yB.data_ptr(), sB.data_ptr(), gB.data_ptr(), bB.data_ptr(), yP.data_ptr() if proj else x.data_ptr(),
                   sP.data_ptr() if proj else None, gP.data_ptr() if proj else None, bP.data_ptr() if proj else None, o16, o32,
                   N, so * so, f, GN_EPS, p.fmt, _s())
        else:
            abB = _finalize(sB, gB, bB, p.aff[1], N, f, so * so)
            if proj:
                abP = _finalize(sP, gP, bP, p.aff[2], N, f, so * so)
                res, ar, br = yP, abP[0].data_ptr(), abP[1].data_ptr()
            else:
                res, ar, br = x, None, None
            L.call("serl_block_combine_h16", yB.data_ptr(), abB[0].data_ptr(), abB[1].data_ptr(), res.data_ptr(), ar, br, o16, o32,
                   N, so * so, f, p.fmt, _s())
        free, cur = [cur, iy, iy2, ir], io
        x, s, cin = out, so, f
    return feats
