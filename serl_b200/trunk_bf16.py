"""16-bit / tensor-core (wgmma) build of the frozen ResNet-10 trunk on 128x128 frames: orchestration + weight packing.

Same layer algebra as the fp32 build (trunk.TrunkRunner.forward; reference vision/resnet_v1.py:217-286),
re-associated so that GroupNorm never makes its own pass over HBM.  One camera pass is eleven launches:
  stem:   `stem_prep` (uint8 -> normalised 16-bit space-to-depth image), `stem_conv_pool` (conv_init with the 3x3/2 max-pool in
          its epilogue, on sign-adjusted raw values, plus the GroupNorm sums), `pool_finish_gn` (relu(|a|x+b) from those sums);
  ResNetBlock_0: two `conv3x3_res` (conv -> GroupNorm -> [+ identity] -> ReLU, the fp32 accumulators normalised in registers);
  ResNetBlock_1..3: `conv3x3s2_res` (the stride-2 3x3 conv with GroupNorm + ReLU AND the 1x1 stride-2 projection with its
          GroupNorm, from one read of the block input), then `conv3x3_res` adding the projected residual; the last one writes
          the fp32 features.
Weights and scratch come from trunk.py: `FrozenTrunk.packed` keeps the packing (`pack_trunk`) of each camera, a `TrunkRunner`
the plans.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L
from .params import STAGES


def _s():
    return L.stream_ptr()


GN_EPS = 1e-5

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
    """16-bit activation buffers of one camera's passes over up to N 128x128 frames.  `error` is the fault flag the kernels raise
    on a pipeline-barrier timeout: a trunk runner passes its own; a plan made alone (kernel tests) gets a fresh one."""

    def __init__(self, N, hw, dev, precision="bf16", error=None):
        if hw != 128:
            raise NotImplementedError(f"the 16-bit trunk takes 128x128 frames, got {hw}x{hw}")
        self.N, (self.fmt, self.dt) = N, FMT[precision]
        bf = lambda *s: torch.empty(*s, dtype=self.dt, device=dev)
        self.hs = 67
        self.xs = bf(N, self.hs, self.hs, 16)                          # stem input: 64x64 space-to-depth image, padded 3 / 3
        self.pooled, self.side = bf(N, 32, 32, 64), bf(N, 4, 32, 64)   # the stem's max-pool, before pool_finish joins the halves
        self.buf = [bf(N * 32 * 32 * 64) for _ in range(3)]            # block activations (the largest is 32x32x64)
        self.stats = torch.zeros(N, 4, 2, dtype=torch.float32, device=dev)   # the stem's GroupNorm sums, zeroed every pass
        self.error = torch.zeros(1, dtype=torch.int32, device=dev) if error is None else error


def _conv(plan, x, w, y, stats, N, Hi, Wi, Ci, Ho, Wo, Co, k, stride, pad_lo, stem=False):
    """The unfused stem conv (serl_conv2d_tc_h16, stem=True): raw 16-bit output + GroupNorm sums.  Not on the product path: with
    _finalize and serl_maxpool_affine_h16 it is the reference the fused stem is tested against bit for bit."""
    d = L.ConvTcDesc()
    d.x, d.w, d.y, d.stats = x.data_ptr(), w.data_ptr(), y.data_ptr(), stats.data_ptr()
    d.error = plan.error.data_ptr()
    d.N, d.Hi, d.Wi, d.Ci, d.Ho, d.Wo, d.Co, d.kh, d.kw, d.stride, d.pad_lo, d.stem, d.fmt = N, Hi, Wi, Ci, Ho, Wo, Co, k, k, stride, pad_lo, int(stem), plan.fmt
    L.call("serl_conv2d_tc_h16", C.byref(d), _s())


def _finalize(stats, gamma, beta, ab, N, Cc, HW):
    """(N,4,2) GroupNorm sums -> the per-(image, channel) affine (a, b) in ab (serl_gn_finalize), for the stem reference above."""
    a, b = ab[0].view(-1)[:N * Cc].view(N, Cc), ab[1].view(-1)[:N * Cc].view(N, Cc)
    L.call("serl_gn_finalize", stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), a.data_ptr(), b.data_ptr(), N, Cc, HW, GN_EPS, _s())
    return a, b


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


def forward(p: _Plan, w, wp, pix: torch.Tensor, feats: torch.Tensor):
    """pix (N,128,128,3) uint8 -> feats[:N] (N,4,4,512) fp32 on the plan's buffers; w: fp32 leaves, wp: their packing (pack_trunk).
    A pass of more images than the plan holds is refused before any launch: its kernels would write past every plan buffer."""
    N = pix.shape[0]
    if not 1 <= N <= p.N:
        raise ValueError(f"trunk pass of {N} images on a plan for 1..{p.N}")
    L.call("serl_trunk_stem_prep_h16", pix.data_ptr(), p.xs.data_ptr(), N, 128, 128, p.fmt, _s())
    p.stats.zero_()
    d = L.StemPoolDesc()
    d.xs, d.w, d.pooled, d.side = p.xs.data_ptr(), wp["conv_init/kernel"].data_ptr(), p.pooled.data_ptr(), p.side.data_ptr()
    d.stats, d.error, d.neg_mask, d.N, d.fmt = p.stats.data_ptr(), p.error.data_ptr(), wp["_stem_neg_mask"], N, p.fmt
    L.call("serl_stem_conv_pool_tc_h16", C.byref(d), _s())
    x, h, r = p.buf                      # x: a block's output (the next block's input), h: its Conv_0 output, r: its residual
    L.call("serl_pool_finish_gn_h16", p.pooled.data_ptr(), p.side.data_ptr(), p.stats.data_ptr(), w["norm_init/scale"].data_ptr(),
           w["norm_init/bias"].data_ptr(), r.data_ptr(), N, GN_EPS, p.fmt, _s())
    gn = lambda b, n: (w[f"{b}/{n}/scale"], w[f"{b}/{n}/bias"])
    # ResNetBlock_0: two stride-1 convs at 32x32x64, the identity residual is the pooled stem output
    _conv_res(p, r, wp["ResNetBlock_0/Conv_0/kernel"], h, *gn("ResNetBlock_0", "MyGroupNorm_0"), N, 32, 64)
    _conv_res(p, h, wp["ResNetBlock_0/Conv_1/kernel"], x, *gn("ResNetBlock_0", "MyGroupNorm_1"), N, 32, 64, res=r)
    s, cin = 32, 64
    for i, (f, stride) in enumerate(STAGES[1:], 1):
        # ResNetBlock_1..3: stride-2 head (Conv_0 + projection), then Conv_1 with the projected residual
        b, s, last = f"ResNetBlock_{i}", s // stride, i == len(STAGES) - 1
        _conv_s2_res(p, x, wp[f"{b}/Conv_0/kernel"], wp[f"{b}/conv_proj/kernel"], h, r, *gn(b, "MyGroupNorm_0"), *gn(b, "norm_proj"),
                     N, s, cin, f)
        _conv_res(p, h, wp[f"{b}/Conv_1/kernel"], None if last else x, *gn(b, "MyGroupNorm_1"), N, s, f, res=r,
                  out_f32=feats if last else None)
        cin = f
    return feats
