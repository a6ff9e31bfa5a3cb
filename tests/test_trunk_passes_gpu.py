"""GPU: the 16-bit frozen trunk launch by launch against float64, at every pass size where its kernels change regime, on fp16 and
bf16, with guard bands around every buffer.

A. The eleven launches of trunk_bf16.forward are chained by hand, each on buffers of its own.  Every launch is compared with a
   float64 restatement computed on its own 16-bit inputs (the previous launch's output, the residual, the weights rounded to
   16 bits), so each keeps the per-kernel bar instead of an accumulated one.
B. Pass sizes: fixed sizes that straddle the images of an item (2 per stem cluster pair, 4 at 8x8, 8 in the 4x4 head, 16 at
   4x4), and for every persistent kernel the n where its work fills the resident grid exactly and by one more, in one and two
   waves.  The resident units come at run time from serl_trunk_resident_units, the occupancy queries the entry points size
   their grids with.
C. Guard bands: every buffer holds n + 16 images and the launch is told N = n.  Tail inputs are NaN (255 for the uint8 frames);
   the valid outputs must be finite and bitwise equal to the same launch on a zero tail, and every output (the GroupNorm sums
   and the fp32 features included) must keep its NaN prefill from image n on.  An overrun lands in the test's own allocation.
D. Through FrozenTrunk runners: two cameras with different weights, interleaved passes, bitwise equal to the hand chain and
   within the whole-trunk bar of each camera's own float64 oracle; a small pass after a full one on the same runner.
E. Batch composition: every GroupNorm reduction is per image, so an image's features do not depend on the other images of a
   pass or on its position in it, bit for bit.
"""
from types import SimpleNamespace

import ctypes as C
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
OUT_TOL = {"bf16": 6e-3, "fp16": 8e-4}          # output rounding of the fp32 accumulators: 2^-9 / 2^-12 (+ margin)
F32_TOL = 2e-5                                  # the fp32 features: no output rounding
TRUNK_TOL = {"fp16": 5e-3, "bf16": 3e-2}        # whole trunk vs the float64 oracle (test_trunk_bf16_gpu.py's feature bars)
GUARD = 16
GN_EPS = 1e-5
f32 = torch.float32
BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}


def _s():
    from serl_b200 import _lib as L
    return L.stream_ptr()


def _leaves(seed):
    """fp32 trunk leaves with every GroupNorm affine perturbed away from its init, about one scale in six negative; norm_init
    has a zero scale and both signs (the fused stem pools sign-adjusted raw values)."""
    from serl_b200.params import init_trunk
    rng = np.random.default_rng(seed)
    w = {}
    for k, v in init_trunk(rng).items():
        if k.endswith("scale"):
            v = v * (1 + 0.3 * rng.standard_normal(v.shape)) * np.where(rng.random(v.shape) < 0.15, -1.0, 1.0)
            if k == "norm_init/scale":
                v[0], v[1], v[2] = 0.0, -abs(v[1]), abs(v[2])
        elif k.endswith("bias"):
            v = 0.2 * rng.standard_normal(v.shape)
        w[k] = torch.as_tensor(np.asarray(v, np.float32)).cuda().contiguous()
    return w


def _frames(n, seed):
    return torch.as_tensor(np.random.default_rng(seed).integers(0, 256, (n, 128, 128, 3), dtype=np.uint8)).cuda()


# ---------------------------------------------------------------------------------------------------------------------------
# the hand chain: trunk_bf16.forward's launches, one buffer set each
# ---------------------------------------------------------------------------------------------------------------------------
class _Chain:
    # (step, inputs, outputs) in launch order; a block's head writes its Conv_0 output h and its projected residual r
    STEPS = [("stem_prep", ("pix",), ("xs",)),
             ("stem_conv_pool", ("xs",), ("pooled", "side", "stats")),
             ("pool_finish_gn", ("pooled", "side", "stats"), ("a0",)),
             ("b0_conv0", ("a0",), ("b0h",)),
             ("b0_conv1", ("b0h", "a0"), ("b0x",)),
             ("b1_head", ("b0x",), ("b1h", "b1r")),
             ("b1_conv1", ("b1h", "b1r"), ("b1x",)),
             ("b2_head", ("b1x",), ("b2h", "b2r")),
             ("b2_conv1", ("b2h", "b2r"), ("b2x",)),
             ("b3_head", ("b2x",), ("b3h", "b3r")),
             ("b3_conv1", ("b3h", "b3r"), ("feats",))]
    # block i: (input width, output width, channels in, channels out)
    BLOCKS = {1: (32, 16, 64, 128), 2: (16, 8, 128, 256), 3: (8, 4, 256, 512)}

    def __init__(self, w, prec, n, wp=None):
        from serl_b200 import trunk_bf16 as T
        self.w, self.prec, self.n = w, prec, n
        self.fmt, self.dt = T.FMT[prec]
        self.wp = T.pack_trunk(w, self.dt) if wp is None else wp
        self.plan = SimpleNamespace(fmt=self.fmt, error=torch.zeros(1, dtype=torch.int32, device="cuda"))

    def _out(self, *shape, dt=None):
        return torch.full((self.n + GUARD, *shape), float("nan"), dtype=dt or self.dt, device="cuda")

    def _gn(self, b, g):
        pre = f"{b}/{g}" if b else g
        return self.w[f"{pre}/scale"], self.w[f"{pre}/bias"]

    def launch(self, step, ins):
        """Runs one launch on `ins` (buffers of n + GUARD images) into fresh NaN-prefilled outputs; returns them by name."""
        from serl_b200 import _lib as L
        from serl_b200 import trunk_bf16 as T
        n, wp, p = self.n, self.wp, self.plan
        if step == "stem_prep":
            xs = self._out(67, 67, 16)
            L.call("serl_trunk_stem_prep_h16", ins["pix"].data_ptr(), xs.data_ptr(), n, 128, 128, self.fmt, _s())
            return {"xs": xs}
        if step == "stem_conv_pool":
            pooled, side, stats = self._out(32, 32, 64), self._out(4, 32, 64), self._out(4, 2, dt=f32)
            stats[:n] = 0                                            # the sums accumulate: forward zeroes them every pass
            d = L.StemPoolDesc()
            d.xs, d.w, d.pooled, d.side = ins["xs"].data_ptr(), wp["conv_init/kernel"].data_ptr(), pooled.data_ptr(), side.data_ptr()
            d.stats, d.error, d.neg_mask, d.N, d.fmt = stats.data_ptr(), p.error.data_ptr(), wp["_stem_neg_mask"], n, self.fmt
            L.call("serl_stem_conv_pool_tc_h16", C.byref(d), _s())
            return {"pooled": pooled, "side": side, "stats": stats}
        if step == "pool_finish_gn":
            a0 = self._out(32, 32, 64)
            L.call("serl_pool_finish_gn_h16", ins["pooled"].data_ptr(), ins["side"].data_ptr(), ins["stats"].data_ptr(),
                   self.w["norm_init/scale"].data_ptr(), self.w["norm_init/bias"].data_ptr(), a0.data_ptr(), n, GN_EPS, self.fmt, _s())
            return {"a0": a0}
        if step == "b0_conv0":
            y = self._out(32, 32, 64)
            T._conv_res(p, ins["a0"], wp["ResNetBlock_0/Conv_0/kernel"], y, *self._gn("ResNetBlock_0", "MyGroupNorm_0"), n, 32, 64)
            return {"b0h": y}
        if step == "b0_conv1":
            y = self._out(32, 32, 64)
            T._conv_res(p, ins["b0h"], wp["ResNetBlock_0/Conv_1/kernel"], y, *self._gn("ResNetBlock_0", "MyGroupNorm_1"), n, 32, 64,
                        res=ins["a0"])
            return {"b0x": y}
        i = int(step[1])
        b, (_, wo, ci, co) = f"ResNetBlock_{i}", self.BLOCKS[i]
        if step.endswith("head"):
            h, r = self._out(wo, wo, co), self._out(wo, wo, co)
            T._conv_s2_res(p, ins[f"b{i - 1}x"], wp[f"{b}/Conv_0/kernel"], wp[f"{b}/conv_proj/kernel"], h, r, *self._gn(b, "MyGroupNorm_0"),
                           *self._gn(b, "norm_proj"), n, wo, ci, co)
            return {f"b{i}h": h, f"b{i}r": r}
        last = i == 3
        y = self._out(wo, wo, co, dt=f32 if last else None)
        T._conv_res(p, ins[f"b{i}h"], wp[f"{b}/Conv_1/kernel"], None if last else y, *self._gn(b, "MyGroupNorm_1"), n, wo, co,
                    res=ins[f"b{i}r"], out_f32=y if last else None)
        return {"feats" if last else f"b{i}x": y}

    def tail(self, t, nan_tail):
        """A copy of t whose images n.. are NaN (255 for frames) or zero."""
        c = t.clone()
        c[self.n:] = (255 if c.dtype == torch.uint8 else float("nan")) if nan_tail else 0
        return c

    def run(self, pix):
        """The whole chain on pix (n + GUARD frames) with NaN tails: {step: (inputs, outputs)}."""
        acts, rec = {"pix": pix}, {}
        for step, ins, _ in self.STEPS:
            i = {k: self.tail(acts[k], True) for k in ins}
            o = self.launch(step, i)
            rec[step] = (i, o)
            acts.update(o)
        return rec


# ---------------------------------------------------------------------------------------------------------------------------
# float64 restatements on the kernels' own 16-bit inputs (on the GPU: the CPU oracle is too slow at N = 1000)
# ---------------------------------------------------------------------------------------------------------------------------
def _rel(got, ref):
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-12))


def _w64(ch, k):
    return ch.w[k].to(ch.dt).double()


def _gn64(ch, x, b, g):
    from oracle.drq import group_norm_nhwc
    s, t = ch._gn(b, g)
    return group_norm_nhwc(x, s.double(), t.double(), 4, GN_EPS)


def _xs_to_image(xs):
    """(n, 67, 67, 16) space-to-depth stem input -> the (n, 128, 128, 3) image it holds: xs[n, a, b, (2p + q) 3 + c] is pixel
    (2a + p - 3, 2b + q - 3) (stem_prep_kernel)."""
    n = xs.shape[0]
    full = xs[..., :12].reshape(n, 67, 67, 2, 2, 3).permute(0, 1, 3, 2, 4, 5).reshape(n, 134, 134, 3)
    return full[:, 3:131, 3:131]


def _prep64(pix):
    from oracle.drq import IMAGENET_MEAN, IMAGENET_STD
    mean, std = (torch.tensor(v, dtype=torch.float64, device="cuda") for v in (IMAGENET_MEAN, IMAGENET_STD))
    x = (pix.double() / 255.0 - mean) / std
    n = x.shape[0]
    full = torch.zeros(n, 134, 134, 3, dtype=torch.float64, device="cuda")
    full[:, 3:131, 3:131] = x
    xs = torch.zeros(n, 67, 67, 16, dtype=torch.float64, device="cuda")
    xs[..., :12] = full.reshape(n, 67, 2, 67, 2, 3).permute(0, 1, 3, 2, 4, 5).reshape(n, 67, 67, 12)
    return xs


def _ulps(got, want64, dt):
    """Distance in units in the last place between the 16-bit got and want64 rounded to dt (same sign required)."""
    w = want64.to(dt)
    gb, wb = got.view(torch.int16).int(), w.view(torch.int16).int()
    same_sign = ((gb < 0) == (wb < 0)) | (w == 0) | (got == 0)
    return torch.where(same_sign, ((gb & 0x7FFF) - (wb & 0x7FFF)).abs(), torch.full_like(gb, 1 << 16)).max().item()


def _check_launch(ch, step, ins, outs, errs):
    """Compares one launch's valid outputs with float64 on its own inputs; records the error by step."""
    from oracle.drq import conv_nhwc, max_pool_3x3_s2_same
    n, tol = ch.n, OUT_TOL[ch.prec]
    v = lambda t: t[:n]
    if step == "stem_prep":
        u = _ulps(v(outs["xs"]), _prep64(v(ins["pix"])), ch.dt)
        errs[step] = u
        assert u <= 1, f"stem_prep is {u} ulp from the float64 normalisation"
        return
    if step == "stem_conv_pool":                             # its sums here; its pooled maxima through pool_finish_gn next
        y64 = conv_nhwc(_xs_to_image(v(ins["xs"])).double(), _w64(ch, "conv_init/kernel"), 2, 3, 3)
        G = y64.reshape(n, 64 * 64, 4, 16)
        want = torch.stack([G.sum(dim=(1, 3)), (G * G).sum(dim=(1, 3))], -1)
        got = v(outs["stats"]).double()
        errs[step] = float(((got - want).abs() / (1e-2 + 1e-4 * want.abs())).max())
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-2)
        ch._stem64 = y64
        return
    if step == "pool_finish_gn":                             # the fused stem and its finish: conv, GroupNorm, ReLU, max-pool
        ref = max_pool_3x3_s2_same(_gn64(ch, ch._stem64, None, "norm_init").relu())
        del ch._stem64
        got, key = v(outs["a0"]), step
    elif step.startswith("b0"):
        x = v(ins["a0"] if step == "b0_conv0" else ins["b0h"]).double()
        k = "ResNetBlock_0/Conv_0/kernel" if step == "b0_conv0" else "ResNetBlock_0/Conv_1/kernel"
        ref = _gn64(ch, conv_nhwc(x, _w64(ch, k), 1, 1, 1), "ResNetBlock_0", "MyGroupNorm_0" if step == "b0_conv0" else "MyGroupNorm_1")
        if step == "b0_conv1":
            ref = ref + v(ins["a0"]).double()
        got, key = v(outs[next(iter(outs))]), step
        ref = ref.relu()
    elif step.endswith("head"):
        i = int(step[1])
        b, x = f"ResNetBlock_{i}", v(ins[f"b{i - 1}x"]).double()
        ref_h = _gn64(ch, conv_nhwc(x, _w64(ch, f"{b}/Conv_0/kernel"), 2, 0, 1), b, "MyGroupNorm_0").relu()
        ref_r = _gn64(ch, conv_nhwc(x, _w64(ch, f"{b}/conv_proj/kernel"), 2, 0, 0), b, "norm_proj")
        for name, ref in ((f"b{i}h", ref_h), (f"b{i}r", ref_r)):
            got = v(outs[name])
            assert torch.isfinite(got).all(), f"{step}: non-finite {name}"
            errs[f"{step}:{name[-1]}"] = e = _rel(got, ref)
            assert e < tol, f"{step} {name}: rel err {e:.3e} (bar {tol:.0e})"
        return
    else:
        i = int(step[1])
        b = f"ResNetBlock_{i}"
        conv = conv_nhwc(v(ins[f"b{i}h"]).double(), _w64(ch, f"{b}/Conv_1/kernel"), 1, 1, 1)
        ref = (_gn64(ch, conv, b, "MyGroupNorm_1") + v(ins[f"b{i}r"]).double()).relu()
        got, key = v(outs[next(iter(outs))]), step
        if i == 3:
            tol = F32_TOL
    assert torch.isfinite(got).all(), f"{step}: non-finite output"
    errs[key] = e = _rel(got, ref)
    assert e < tol, f"{step}: rel err {e:.3e} (bar {tol:.0e})"


# ---------------------------------------------------------------------------------------------------------------------------
# pass sizes: fixed, and the wave boundaries of every persistent kernel
# ---------------------------------------------------------------------------------------------------------------------------
# per persistent launch: (the launch's serl_trunk_resident_units id, images per item, channel slices), as its host entry point
# splits the work: a work unit is an image (images per item None: the stem and the 32x32 convs run one 4-CTA cluster per image,
# the 16x16 conv a CTA pair) or an item of that many images x one channel slice (one CTA each).  Every launch takes
# ceil(work / resident) rounds on the fewest units that still need that many.
PERSISTENT = {
    "stem_conv_pool": ("TRUNK_STEM", None, None),
    "b0_conv0": ("TRUNK_RES32", None, None),
    "b0_conv1": ("TRUNK_RES32", None, None),
    "b1_head": ("TRUNK_HEAD16", 1, 2),
    "b1_conv1": ("TRUNK_RES16", None, None),
    "b2_head": ("TRUNK_HEAD8", 4, 4),
    "b2_conv1": ("TRUNK_RES8", 4, 4),
    "b3_head": ("TRUNK_HEAD4", 8, 4),
    "b3_conv1": ("TRUNK_RES4", 16, 4),
}
# the launches whose wave boundaries a case targets (the 16x16 head and conv, and both 8x8 launches, share their n)
WAVE_GROUPS = {"stem": ("stem_conv_pool",), "32x32": ("b0_conv0", "b0_conv1"), "16x16": ("b1_head", "b1_conv1"),
               "8x8": ("b2_head", "b2_conv1"), "4x4-head": ("b3_head",), "4x4-conv": ("b3_conv1",)}
FIXED = [1, 2, 3, 4, 5, 15, 16, 17, 512, 515, 1024]
WAVES = [f"{g}:{k}w{'+1' if plus else ''}" for g in WAVE_GROUPS for k in (1, 2) for plus in (False, True)]


def _resident(prec):
    """Work units resident at once per persistent launch, from the occupancy queries the entry points size their grids with."""
    from serl_b200 import _lib as L
    lib = L.load()
    sms = int(lib.serl_device_sm_count(torch.cuda.current_device()))
    fmt = {"fp16": L.FMT_FP16, "bf16": L.FMT_BF16}[prec]
    out = {step: int(lib.serl_trunk_resident_units(getattr(L, launch), fmt)) for step, (launch, _, _) in PERSISTENT.items()}
    for step, units in out.items():
        assert units > 0, (step, L.load().serl_last_error())
        if PERSISTENT[step][1] is not None:
            assert units % sms == 0, (step, units, sms)      # whole CTAs per SM
        else:
            assert units <= sms, (step, units, sms)          # images of several CTAs each
    print(f"[{prec}] {sms} SMs; work units resident at once: {out}")
    return out


def _work(step, n):
    _, imgs, nsl = PERSISTENT[step]
    return n if imgs is None else -(-n // imgs) * nsl


def _wave_n(case, units):
    """The pass size of a wave case: the largest n whose work fills `waves` waves of the group's first launch, then one more
    image (one more unit of work)."""
    group, k = case.split(":")
    plus, waves = k.endswith("+1"), int(k[0])
    step = WAVE_GROUPS[group][0]
    _, imgs, nsl = PERSISTENT[step]
    n = waves * units[step] if imgs is None else imgs * (waves * units[step] // nsl)
    return n + plus, waves + plus


# ---------------------------------------------------------------------------------------------------------------------------
# A + B + C
# ---------------------------------------------------------------------------------------------------------------------------
def _launch_by_launch(prec, n, seed):
    w = _leaves(seed)
    ch = _Chain(w, prec, n)
    rec = ch.run(_frames(n + GUARD, seed))
    torch.cuda.synchronize()
    assert int(ch.plan.error.item()) == 0, "pipeline barrier timeout"
    errs = {}
    for step, _, _ in _Chain.STEPS:
        ins, outs = rec[step]
        for name, o in outs.items():                        # nothing written from image n on
            nan = torch.full_like(o[n:], float("nan"))
            assert torch.equal(o[n:].view(BITS[o.dtype]), nan.view(BITS[o.dtype])), f"{step} wrote {name} past image {n}"
        zero = ch.launch(step, {k: ch.tail(t, False) for k, t in ins.items()})   # the same launch on a zero tail
        for name, o in outs.items():
            assert torch.equal(o[:n].view(BITS[o.dtype]), zero[name][:n].view(BITS[o.dtype])), \
                f"{step}: {name} depends on the images past n"
        _check_launch(ch, step, ins, outs, errs)
    torch.cuda.synchronize()
    assert int(ch.plan.error.item()) == 0, "pipeline barrier timeout"
    print(f"[{prec} n={n}] " + "  ".join(f"{k} {v:.3e}" if isinstance(v, float) else f"{k} {v}ulp" for k, v in errs.items()))
    return ch, rec


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("n", FIXED)
def test_each_launch_matches_float64_with_guard_bands(prec, n):
    _launch_by_launch(prec, n, seed=n)


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("case", WAVES)
def test_each_launch_matches_float64_at_wave_boundaries(prec, case):
    units = _resident(prec)
    n, rounds = _wave_n(case, units)
    rounds_at = lambda step, work: -(-work // units[step])
    for step in WAVE_GROUPS[case.split(":")[0]]:             # the case is the wave boundary it claims to be
        work, unit = _work(step, n), PERSISTENT[step][2] or 1
        assert rounds_at(step, work) == rounds, (step, n, rounds)
        if case.endswith("+1"):                               # one unit of work less fits one wave fewer
            assert rounds_at(step, work - unit) == rounds - 1, (step, n)
        else:                                                 # one unit of work more needs one wave more
            assert rounds_at(step, work + unit) == rounds + 1, (step, n)
    _launch_by_launch(prec, n, seed=n + 7)


# ---------------------------------------------------------------------------------------------------------------------------
# D: through FrozenTrunk runners
# ---------------------------------------------------------------------------------------------------------------------------
def _hand_feats(w, prec, pix, wp=None):
    n = pix.shape[0]
    ch = _Chain(w, prec, n, wp)
    padded = torch.cat([pix, torch.zeros(GUARD, 128, 128, 3, dtype=torch.uint8, device="cuda")])
    return ch.run(padded)["b3_conv1"][1]["feats"][:n]


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_two_camera_runner_equals_the_hand_chain_and_each_cameras_oracle(prec):
    from oracle import drq as O
    from serl_b200.trunk import FrozenTrunk
    N = 11
    w = {"cam0": _leaves(1), "cam1": _leaves(2)}
    trunk = FrozenTrunk(w, prec)
    runner = trunk.runner(N, "cuda")
    pix = {"cam0": _frames(N, 10), "cam1": _frames(N, 11)}
    got = []
    for cam in ("cam0", "cam1", "cam0"):
        feats = torch.full((N, 4, 4, 512), float("nan"), device="cuda")
        runner.forward(cam, pix[cam], feats)
        torch.cuda.synchronize()
        assert int(runner.error.item()) == 0
        got.append((cam, feats))
    trunk.check_error()
    bits = lambda t: t.view(torch.int32)
    assert torch.equal(bits(got[0][1]), bits(got[2][1]))
    for cam in ("cam0", "cam1"):
        hand = _hand_feats(w[cam], prec, pix[cam])
        feats = dict(got[:2])[cam]
        assert torch.equal(bits(feats), bits(hand)), f"{cam}: the runner's features differ from the hand chain's"
        params = {f"{O.ENC}/encoder_{cam}/pretrained_encoder/{k}": v.cpu() for k, v in w[cam].items()}
        ref = O.trunk_forward(params, cam, pix[cam].cpu(), torch.float64).cuda()
        errs = [_rel(feats[i], ref[i]) for i in range(N)]
        print(f"[{prec}] {cam}: whole-trunk feature rel err per image, worst {max(errs):.3e}")
        assert max(errs) < TRUNK_TOL[prec], (cam, errs)


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_a_small_pass_after_a_full_one_equals_a_fresh_runner(prec):
    from serl_b200.trunk import FrozenTrunk
    w = {"cam": _leaves(3)}
    trunk = FrozenTrunk(w, prec)
    big, small = trunk.runner(512, "cuda"), trunk.runner(5, "cuda")
    feats = torch.full((512, 4, 4, 512), float("nan"), device="cuda")
    big.forward("cam", _frames(512, 20), feats)
    torch.cuda.synchronize()
    assert int(big.error.item()) == 0 and torch.isfinite(feats).all()
    before = feats.clone()
    pix5 = _frames(5, 21)
    big.forward("cam", pix5, feats)
    fresh = torch.full((5, 4, 4, 512), float("nan"), device="cuda")
    small.forward("cam", pix5, fresh)
    torch.cuda.synchronize()
    trunk.check_error()
    bits = lambda t: t.view(torch.int32)
    assert torch.equal(bits(feats[:5]), bits(fresh))
    assert not torch.equal(bits(feats[:5]), bits(before[:5]))
    assert torch.equal(bits(feats[5:]), bits(before[5:])), "a pass of 5 wrote features past image 5"


# ---------------------------------------------------------------------------------------------------------------------------
# E: batch composition
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_features_do_not_depend_on_the_rest_of_the_pass(prec):
    from serl_b200.trunk import FrozenTrunk
    n = 24
    trunk = FrozenTrunk({"cam": _leaves(4)}, prec)
    runner, one = trunk.runner(n, "cuda"), trunk.runner(1, "cuda")
    bits = lambda t: t.view(torch.int32)

    def enc(r, pix):
        f = torch.full((pix.shape[0], 4, 4, 512), float("nan"), device="cuda")
        r.forward("cam", pix, f)
        return f

    pix = _frames(n, 30)
    base = enc(runner, pix)
    perm = torch.as_tensor(np.random.default_rng(31).permutation(n)).cuda()
    assert torch.equal(bits(enc(runner, pix[perm])), bits(base[perm])), "features do not permute with their images"
    x = _frames(1, 32)
    alone = enc(one, x)
    small = enc(runner, x)                                   # one image on a runner of 24
    assert torch.equal(bits(small), bits(alone))
    others = _frames(n, 33)
    for pos in (0, 3, 17, n - 1):
        p = others.clone()
        p[pos] = x[0]
        f = enc(runner, p)
        assert torch.equal(bits(f[pos]), bits(alone[0])), f"image at position {pos} of {n} differs from the same image alone"
    torch.cuda.synchronize()
    trunk.check_error()


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("n", [1, 5, 133])
def test_8x8_fp32_store_stays_inside_its_images(prec, n):
    """The 8x8 conv's fp32 output (out_f32), which the trunk does not take (it writes fp32 at 4x4 only), under the same guard
    bands: its store is the one the kernel guards separately from the 16-bit one."""
    from oracle.drq import conv_nhwc
    from serl_b200 import trunk_bf16 as T
    ch = _Chain(_leaves(n), prec, n)
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.rand((n + GUARD, 8, 8, 256), generator=g, device="cuda").to(ch.dt)
    r = torch.randn((n + GUARD, 8, 8, 256), generator=g, device="cuda").to(ch.dt)
    b, wk = "ResNetBlock_2", "ResNetBlock_2/Conv_1/kernel"

    def run(nan_tail):
        y = ch._out(8, 8, 256, dt=f32)
        T._conv_res(ch.plan, ch.tail(x, nan_tail), ch.wp[wk], None, *ch._gn(b, "MyGroupNorm_1"), n, 8, 256, res=ch.tail(r, nan_tail),
                    out_f32=y)
        return y

    y, y0 = run(True), run(False)
    torch.cuda.synchronize()
    assert int(ch.plan.error.item()) == 0
    nan = torch.full_like(y[n:], float("nan"))
    assert torch.equal(y[n:].view(torch.int32), nan.view(torch.int32)), f"the fp32 store wrote past image {n}"
    assert torch.equal(y[:n].view(torch.int32), y0[:n].view(torch.int32))
    assert torch.isfinite(y[:n]).all()
    ref = (_gn64(ch, conv_nhwc(x[:n].double(), _w64(ch, wk), 1, 1, 1), b, "MyGroupNorm_1") + r[:n].double()).relu()
    assert _rel(y[:n], ref) < F32_TOL
