"""GPU: the dropout Q-function heads' masked kernels (serl_tgemm_tf32_masked, csrc/tgemm.cu; serl_layernorm_tanh_bwd_multi_masked,
csrc/heads_fused.cu) op by op against a float64 restatement of Dense -> Dropout -> LayerNorm (eps 1e-6, fast variance) -> tanh,
with the value head or the tanh-Gaussian policy head where the epilogue has one.

Every launch carries two problems with DIFFERENT masks, as the critic's online / target launch does with critic_subsample_size:
without it the two masks are equal and a kernel reading problem 0's mask for both would pass.  Rates reach 0.9, because
LayerNorm hides a wrong 1/(1 - rate) in h and Q (LN(c z) = LN(z) up to eps): it shows in rstd (compared element by element here)
and in the backward's dz, by a factor of 1/(1 - rate).  The bias is nonzero, since Dropout applies to acc + bias.  Planted mask
rows: fully dropped (h = tanh(ln_bias), xhat = 0, rstd = 1/sqrt(eps)), a single kept unit, fully kept.  Outputs are prefilled
with NaN and the rows at or past M must stay so.  Measured errors: DESIGN.md §5."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 5e-5                    # max |err| / max |ref| (rstd: element-wise relative); 3xTF32 GEMM + fp32 epilogue, float64 reference
EPS = 1e-6
RATES = (0.01, 0.1, 0.5, 0.9)
PAD = 3                       # NaN rows after each member's M rows
#          epilogue, Z members sharing the mask, head_n, deterministic
EPIS = {"ln-z1": ("LN_TANH", 1, 0, False), "ln-z2": ("LN_TANH", 2, 0, False), "ln-z10": ("LN_TANH", 10, 0, False),
        "head": ("LN_TANH_HEAD", 2, 1, False), "policy-det": ("LN_TANH_POLICY", 1, 4, True), "policy-noise": ("LN_TANH_POLICY", 1, 4, False)}
MS = (1, 127, 128, 129, 257, 1024, 5120)


def cu(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def rel_err(a, b):
    return float(np.max(np.abs(np.asarray(a, np.float64) - b)) / (np.max(np.abs(b)) + 1e-30))


def _mask(rng, rows, rate, plant):
    """(rows, 256) keep mask with planted rows: plant = [(row, "dropped" | "single" | "kept"), ...]."""
    m = (rng.random((rows, 256)) >= rate).astype(np.uint8)
    for r, kind in plant:
        m[r] = 1 if kind == "kept" else 0
        if kind == "single":
            m[r, 77] = 1
    return m


def _plants(M, i):
    """Problem i's planted rows: the first, middle and last row, each problem giving them the three kinds in another order (at
    M = 1 problem 0's row is fully dropped and problem 1's keeps a single unit)."""
    rows = sorted({0, M // 2, M - 1})
    kinds = ("dropped", "single", "kept")
    return [(r, kinds[(j + i) % 3]) for j, r in enumerate(rows)]


def _ln_tanh(z, sc, lb):
    """float64 LayerNorm (fast variance) + tanh; returns h, xhat, rstd."""
    mean = z.mean(-1, keepdims=True)
    var = np.maximum((z * z).mean(-1, keepdims=True) - mean * mean, 0.0)
    rstd = 1.0 / np.sqrt(var + EPS)
    xh = (z - mean) * rstd
    return np.tanh(xh * sc + lb), xh, rstd[..., 0]


def _policy_ref(h, wm, bm, wl, bl, noise, deterministic, std_min=1e-5, std_max=5.0):
    mu, ls = h @ wm + bm, h @ wl + bl
    sd = np.clip(np.exp(ls), std_min, std_max)
    u = mu if deterministic else mu + sd * noise
    zn = (u - mu) / sd
    lp = (-0.5 * zn * zn - np.log(sd) - 0.5 * np.log(2 * np.pi) - 2 * (np.log(2) - u - np.logaddexp(0, -2 * u))).sum(-1)
    return dict(mu=mu, ls=ls, act=np.tanh(u), logp=lp, u=u, std=sd)


class _Problem:
    """One problem of a masked LayerNorm-epilogue launch: fp32 operands on the device, NaN-prefilled outputs with PAD rows per
    member, and the float64 reference of the masked layer."""

    def __init__(self, rng, M, K, Z, epi, head_n, deterministic, mask, rate):
        self.M, self.Z, self.epi, self.A = M, Z, epi, head_n
        x = rng.standard_normal((M, K)).astype(np.float32)
        w = (rng.standard_normal((Z, K, 256)) / np.sqrt(K)).astype(np.float32)
        b = (0.5 + 0.3 * rng.standard_normal((Z, 256))).astype(np.float32)           # nonzero: dropout applies to acc + bias
        sc = (1 + 0.2 * rng.standard_normal((Z, 256))).astype(np.float32)
        lb = (0.2 * rng.standard_normal((Z, 256))).astype(np.float32)
        z = x.astype(np.float64) @ w.astype(np.float64) + b[:, None, :]
        for r in np.flatnonzero(mask.sum(1) == 1):
            # a single kept unit v makes xhat = v / sqrt(v^2 / 257 + eps) (scaled), whose slope reaches 1/sqrt(eps) as v -> 0 and
            # would amplify the GEMM's rounding of v: keep the column where every member's |z| is largest
            mask[r] = 0
            mask[r, np.argmax(np.abs(z[:, r]).min(0))] = 1
        self.host = dict(x=x, w=w, b=b, sc=sc, lb=lb, mask=mask)
        Mp = M + PAD
        nan = lambda *sh: torch.full(sh, float("nan"), device="cuda")
        self.out = dict(h=nan(Z, Mp, 256), xhat=nan(Z, Mp, 256), rstd=nan(Z, Mp))
        self.dev = dict(x=cu(x), w=cu(w), b=cu(b), sc=cu(sc), lb=cu(lb), mask=cu(mask))
        z = np.where(mask.astype(bool)[None], z / (1.0 - rate), 0.0)
        h, xh, rs = _ln_tanh(z, sc[:, None, :].astype(np.float64), lb[:, None, :].astype(np.float64))
        self.ref = dict(h=h, xhat=xh, rstd=rs)
        kw = {}
        if epi == "LN_TANH_HEAD":
            hw = (rng.standard_normal((Z, 256, head_n)) / 16).astype(np.float32)
            hb = rng.standard_normal((Z, head_n)).astype(np.float32)
            self.dev.update(hw=cu(hw), hb=cu(hb))
            self.out["q"] = nan(Z, Mp, head_n)
            self.ref["q"] = h @ hw.astype(np.float64) + hb[:, None, :]
            kw = dict(head_w=self.dev["hw"].data_ptr(), head_b=self.dev["hb"].data_ptr(), sHeadWz=256 * head_n, sHeadBz=head_n,
                      head_out=self.out["q"].data_ptr(), sHeadOutZ=Mp * head_n, ld_head=head_n)
        elif epi == "LN_TANH_POLICY":
            A = head_n
            wm, wl = [(rng.standard_normal((256, A)) / 16).astype(np.float32) for _ in range(2)]
            bm, bl = [(0.3 * rng.standard_normal(A)).astype(np.float32) for _ in range(2)]
            noise = rng.standard_normal((M, A)).astype(np.float32)
            self.dev.update(wm=cu(wm), wl=cu(wl), bm=cu(bm), bl=cu(bl), noise=cu(noise))
            for k in ("mu", "ls", "act", "u", "std"):
                self.out[k] = nan(Mp, A)
            self.out["logp"] = nan(Mp)
            f64 = lambda a: a.astype(np.float64)
            self.ref.update(_policy_ref(h[0], f64(wm), f64(bm), f64(wl), f64(bl), f64(noise), deterministic))
            kw = dict(head_w=self.dev["wm"].data_ptr(), head_b=self.dev["bm"].data_ptr(), head_out=self.out["mu"].data_ptr(),
                      head_w2=self.dev["wl"].data_ptr(), head_b2=self.dev["bl"].data_ptr(), head_out2=self.out["ls"].data_ptr(),
                      noise=self.dev["noise"].data_ptr(), act=self.out["act"].data_ptr(), ld_act=A, logp=self.out["logp"].data_ptr(),
                      u_out=self.out["u"].data_ptr(), std_out=self.out["std"].data_ptr())
        self.kw, self.K = kw, K

    def problem(self):
        from serl_b200 import ops
        d, o, M, Mp = self.dev, self.out, self.M, self.M + PAD
        return ops.tgemm_problem(d["x"].data_ptr(), d["w"].data_ptr(), sAm=self.K, sAk=1, sBk=256, sBn=1, Z=self.Z, sAz=0, sBz=self.K * 256,
                                 C_=o["h"].data_ptr(), sCz=Mp * 256, ldc=256, bias=d["b"].data_ptr(), sBiasZ=256, ln_scale=d["sc"].data_ptr(),
                                 ln_bias=d["lb"].data_ptr(), sLnZ=256, xhat=o["xhat"].data_ptr(), rstd=o["rstd"].data_ptr(), sXhatZ=Mp * 256,
                                 sRstdZ=Mp, **self.kw)

    def got(self):
        """The outputs' M live rows (per member where there are members) as float64 numpy, after checking the pad rows are NaN."""
        out = {}
        for k, t in self.out.items():
            a = t.cpu().numpy().astype(np.float64)
            if k in ("h", "xhat", "rstd", "q"):
                assert np.isnan(a[:, self.M:]).all(), f"{k}: rows at or past M were written"
                out[k] = a[:, :self.M]
            else:
                assert np.isnan(a[self.M:]).all(), f"{k}: rows at or past M were written"
                out[k] = a[:self.M]
        return out


def _launch(probs, M, K, epi, head_n, deterministic, inv_keep, masks):
    from serl_b200 import _lib as L
    from serl_b200 import ops
    ops.tgemm(None, [p.problem() for p in probs], M, 256, K, epilogue=getattr(L, f"TGEMM_{epi}"), head_n=head_n,
              deterministic=deterministic, masks=masks, inv_keep=inv_keep)


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("case", list(EPIS))
def test_masked_tgemm_epilogues_match_float64(case, M):
    epi, Z, head_n, det = EPIS[case]
    K = 260                                                 # eight whole 32-wide k-blocks and a 4-wide tail
    worst = {}
    for ri, rate in enumerate(RATES):
        rng = np.random.default_rng(1000 * M + ri)
        probs = [_Problem(rng, M, K, Z, epi, head_n, det, _mask(rng, M, rate, _plants(M, i)), rate) for i in range(2)]
        assert not np.array_equal(probs[0].host["mask"], probs[1].host["mask"])
        _launch(probs, M, K, epi, head_n, det, np.float32(1.0 / (1.0 - rate)), [p.dev["mask"] for p in probs])
        for i, p in enumerate(probs):
            got = p.got()
            for k, ref in p.ref.items():
                g = got[k]
                assert np.isfinite(g).all(), (rate, i, k)
                e = float(np.max(np.abs(g - ref) / ref)) if k == "rstd" else rel_err(g, ref)
                worst[k] = max(worst.get(k, 0.0), e)
                assert e < TOL, f"rate {rate} problem {i} {k}: {e:.2e}"
            mk = p.host["mask"].astype(bool)
            for r in np.flatnonzero(~mk.any(1)):            # fully dropped rows: z' = 0
                assert (got["xhat"][:, r] == 0).all(), (rate, i, r)
                np.testing.assert_allclose(got["rstd"][:, r], 1 / np.sqrt(EPS), rtol=1e-6)
                np.testing.assert_allclose(got["h"][:, r], np.tanh(p.host["lb"].astype(np.float64)), rtol=0, atol=1e-6)
    print(f"[{case} M={M}] " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


@pytest.mark.parametrize("case", list(EPIS))
def test_masked_tgemm_all_ones_is_bitwise_unmasked_and_reruns_are_bitwise(case):
    """An all-ones mask with inv_keep = 1 runs the unmasked kernel's arithmetic; two launches of the same masked problem agree."""
    epi, Z, head_n, det = EPIS[case]
    M, K = 257, 260
    rng = np.random.default_rng(7)
    ones = np.ones((M, 256), np.uint8)
    probs = [_Problem(np.random.default_rng(9 + i), M, K, Z, epi, head_n, det, ones, 0.0) for i in range(2)]
    _launch(probs, M, K, epi, head_n, det, 1.0, None)
    plain = [{k: t.clone() for k, t in p.out.items()} for p in probs]
    _launch(probs, M, K, epi, head_n, det, 1.0, [p.dev["mask"] for p in probs])
    for p, ref in zip(probs, plain):
        for k, t in p.out.items():
            assert torch.equal(t.nan_to_num(), ref[k].nan_to_num()), k          # (the NaN pad rows are untouched by both)
    masks = [cu(_mask(rng, M, 0.5, _plants(M, i))) for i in range(2)]
    runs = []
    for _ in range(2):
        _launch(probs, M, K, epi, head_n, det, 2.0, masks)
        runs.append([{k: t.clone() for k, t in p.out.items()} for p in probs])
    for a, b in zip(*runs):
        for k in a:
            assert torch.equal(a[k].nan_to_num(), b[k].nan_to_num()), k


# ---- LayerNorm + tanh backward through the forward's Dropout mask --------------------------------------------------------------
def _bwd_problem(rng, E, B, rate, source, plant):
    """Float64 forward of the masked layer over R = E B rows (row r reads mask row r % B), its fp32 saves, an upstream gradient and
    float64 autograd's dz (w.r.t. acc + bias, ahead of the Dropout) and dy (w.r.t. the LayerNorm output)."""
    R, D = E * B, 256
    # the (B, 256) mask is the head of an (R, 256) buffer whose other rows hold other bits: rows past B must wrap, not read on
    buf = (rng.random((R, D)) >= rate).astype(np.uint8)
    buf[:B] = _mask(rng, B, rate, plant)
    mask = buf[:B]
    z = torch.tensor(rng.standard_normal((R, D)) + 0.4, dtype=torch.float64, requires_grad=True)
    sc = torch.tensor(1 + 0.2 * rng.standard_normal((E, D)))
    lb = torch.tensor(0.2 * rng.standard_normal((E, D)))
    keep = torch.as_tensor(np.tile(mask, (E, 1)).astype(bool))
    zd = torch.where(keep, z / (1.0 - rate), torch.zeros_like(z))
    mean = zd.mean(-1, keepdim=True)
    var = torch.clamp((zd * zd).mean(-1, keepdim=True) - mean * mean, min=0.0)
    rstd = 1.0 / torch.sqrt(var + EPS)
    xh = (zd - mean) * rstd
    y = xh * sc.repeat_interleave(B, 0) + lb.repeat_interleave(B, 0)
    y.retain_grad()
    h = torch.tanh(y)
    p = dict(t=h.detach().numpy().astype(np.float32), xh=xh.detach().numpy().astype(np.float32),
             rstd=rstd.detach().numpy()[:, 0].astype(np.float32), sc=sc.numpy().astype(np.float32), buf=buf)
    if source == "dq":
        p["dq"] = rng.standard_normal(R).astype(np.float32)
        p["hw"] = rng.standard_normal(D).astype(np.float32)
        dt = np.outer(p["dq"].astype(np.float64), p["hw"].astype(np.float64))
    else:
        p["parts"] = rng.standard_normal((3, R, D)).astype(np.float32)
        p["dt2"] = rng.standard_normal((R, D)).astype(np.float32)
        dt = p["parts"].astype(np.float64).sum(0) + p["dt2"]
    (h * torch.as_tensor(dt)).sum().backward()
    p["ref_dz"], p["ref_dy"] = z.grad.numpy(), y.grad.numpy()
    return p


def _bwd_args(T, p, E, B, dz, dy):
    R, D = E * B, 256
    base = dict(t=T["t"].data_ptr(), ld_t=D, xhat=T["xh"].data_ptr(), rstd=T["rstd"].data_ptr(), scale=T["sc"].data_ptr(), rows_per_group=B,
                group_stride=D, R=R, D=D, dz=dz.data_ptr(), dy=dy.data_ptr())
    if "dq" in p:
        return dict(base, dq=T["dq"].data_ptr(), head_w=T["hw"].data_ptr(), head_w_stride=0)
    return dict(base, dt=T["parts"].data_ptr(), ld_dt=D, dt_parts=3, dt_part_stride=R * D, dt2=T["dt2"].data_ptr(), ld_dt2=D)


@pytest.mark.parametrize("E", (2, 10))
@pytest.mark.parametrize("B", (1, 127, 129, 257, 5120))
def test_masked_ln_tanh_bwd_multi_matches_float64_autograd(B, E):
    from serl_b200 import ops
    R = E * B
    worst = {}
    for ri, rate in enumerate(RATES):
        rng = np.random.default_rng(100 * B + 10 * E + ri)
        ps = [_bwd_problem(rng, E, B, rate, src, _plants(B, i)) for i, src in enumerate(("dq", "dt"))]
        Ts = [{k: cu(v) for k, v in p.items() if not k.startswith("ref")} for p in ps]
        outs = [(torch.full((R, 256), float("nan"), device="cuda"), torch.full((R, 256), float("nan"), device="cuda")) for _ in ps]
        ops.ln_tanh_bwd_multi([_bwd_args(T, p, E, B, dz, dy) for T, p, (dz, dy) in zip(Ts, ps, outs)],
                              masks=[T["buf"] for T in Ts], mask_rows=B, inv_keep=np.float32(1.0 / (1.0 - rate)))
        for i, (p, (dz, dy)) in enumerate(zip(ps, outs)):
            gz, gy = dz.cpu().numpy(), dy.cpu().numpy()
            # dz row by row against the size of the terms the kernel sums over the row, |rstd dy scale| inv_keep: a row with a
            # single kept unit is scale-invariant, so its exact dz is ~0, what is left after those terms cancel
            kept = np.tile(p["buf"][:B], (E, 1)).astype(bool)
            terms = np.abs(p["rstd"][:, None] * p["ref_dy"] * np.repeat(p["sc"], B, 0)).max(1) / (1.0 - rate)
            live = kept.any(1)                                                # (rows with no kept unit: dz == 0 below)
            errs = dict(dz=float((np.abs(gz - p["ref_dz"]).max(1)[live] / terms[live]).max()) if live.any() else 0.0,
                        dy=rel_err(gy, p["ref_dy"]))
            for k, e in errs.items():
                worst[k] = max(worst.get(k, 0.0), e)
                assert e < TOL, f"rate {rate} problem {i} {k}: {e:.2e}"
            assert np.isfinite(gz).all() and np.isfinite(gy).all(), (rate, i)
            assert (gz[~kept] == 0).all(), (rate, i)                          # exactly zero through a dropped unit
            assert kept.all() or np.count_nonzero(gy[~kept]) > 0              # dy is not masked
    print(f"[B={B} E={E}] " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


def test_masked_ln_tanh_bwd_multi_all_ones_is_bitwise_unmasked():
    from serl_b200 import ops
    E, B = 2, 129
    rng = np.random.default_rng(3)
    ps = [_bwd_problem(rng, E, B, 0.0, src, _plants(B, i)) for i, src in enumerate(("dq", "dt"))]
    Ts = [{k: cu(v) for k, v in p.items() if not k.startswith("ref")} for p in ps]
    ones = cu(np.ones((B, 256), np.uint8))
    res = []
    for masks in (None, [ones, ones]):
        outs = [(torch.zeros(E * B, 256, device="cuda"), torch.zeros(E * B, 256, device="cuda")) for _ in ps]
        ops.ln_tanh_bwd_multi([_bwd_args(T, p, E, B, dz, dy) for T, p, (dz, dy) in zip(Ts, ps, outs)], masks=masks, mask_rows=B, inv_keep=1.0)
        res.append(outs)
    for (a, b), (c, d) in zip(*res):
        assert torch.equal(a, c) and torch.equal(b, d)


# ---- host refusals: SerlError, and nothing written ----------------------------------------------------------------------------
def test_masked_entry_points_refuse_bad_masks_and_leave_outputs_untouched():
    from serl_b200 import _lib as L
    from serl_b200 import ops
    M, K = 130, 260
    rng = np.random.default_rng(4)
    probs = [_Problem(rng, M, K, 2, "LN_TANH_HEAD", 1, False, _mask(rng, M, 0.5, _plants(M, i)), 0.5) for i in range(2)]
    good = [p.dev["mask"] for p in probs]
    raw = torch.zeros(M * 256 + 16, dtype=torch.uint8, device="cuda")
    store_out = torch.full((M, 256), float("nan"), device="cuda")
    store = ops.tgemm_problem(probs[0].dev["x"].data_ptr(), probs[0].dev["w"].data_ptr(), sAm=K, sAk=1, sBk=256, sBn=1, C_=store_out.data_ptr(), ldc=256)
    bad = [("a mask on the STORE epilogue", lambda: ops.tgemm(None, [store], M, 256, K, masks=good[:1], inv_keep=2.0)),
           ("a mask 1 byte off 16-byte alignment", lambda: _launch(probs, M, K, "LN_TANH_HEAD", 1, False, 2.0, [good[0], raw[1:]])),
           ("a null mask", lambda: _launch(probs, M, K, "LN_TANH_HEAD", 1, False, 2.0, [good[0], None])),
           ("inv_keep = 0", lambda: _launch(probs, M, K, "LN_TANH_HEAD", 1, False, 0.0, good)),
           ("inv_keep < 0", lambda: _launch(probs, M, K, "LN_TANH_HEAD", 1, False, -2.0, good)),
           ("inv_keep NaN", lambda: _launch(probs, M, K, "LN_TANH_HEAD", 1, False, float("nan"), good))]
    E, B = 2, 33
    bp = _bwd_problem(rng, E, B, 0.5, "dq", _plants(B, 0))
    T = {k: cu(v) for k, v in bp.items() if not k.startswith("ref")}
    dz, dy = torch.full((E * B, 256), float("nan"), device="cuda"), torch.full((E * B, 256), float("nan"), device="cuda")
    args = [_bwd_args(T, bp, E, B, dz, dy)]
    bad += [("backward: a null mask", lambda: ops.ln_tanh_bwd_multi(args, masks=[None], mask_rows=B, inv_keep=2.0)),
            ("backward: inv_keep = 0", lambda: ops.ln_tanh_bwd_multi(args, masks=[T["buf"]], mask_rows=B, inv_keep=0.0)),
            ("backward: inv_keep < 0", lambda: ops.ln_tanh_bwd_multi(args, masks=[T["buf"]], mask_rows=B, inv_keep=-1.0)),
            ("backward: inv_keep NaN", lambda: ops.ln_tanh_bwd_multi(args, masks=[T["buf"]], mask_rows=B, inv_keep=float("nan"))),
            ("backward: mask_rows = 0", lambda: ops.ln_tanh_bwd_multi(args, masks=[T["buf"]], mask_rows=0, inv_keep=2.0)),
            ("backward: mask_rows < 0", lambda: ops.ln_tanh_bwd_multi(args, masks=[T["buf"]], mask_rows=-B, inv_keep=2.0))]
    for what, call in bad:
        with pytest.raises(L.SerlError):
            call()
        torch.cuda.synchronize()
        outs = [store_out, dz, dy] + [t for p in probs for t in p.out.values()]
        assert all(bool(torch.isnan(t).all()) for t in outs), f"{what}: an output was written"
