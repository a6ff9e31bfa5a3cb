"""GPU: every serl_vice_* entry point of csrc/vice.cu op by op (through the C-ABI), each against a float64 restatement of the same
operation on the same fp32 inputs.

Draws and masks are restated with oracle/jax_prng.py and tests/vice_oracle.py and must match bit for bit; the LayerNorm +
activation kernels against tests/vice_oracle.py's ln_act and its forward-mode tangent, their backward against float64 autograd
of sum(ybar y + ydotbar ydot) through that tangent.  The shapes reach what update_vice at batch 8 does not: two sort rounds
(N >= 1626) and a key whose first round has tied sort keys, more rows than one 256-thread CTA reduces in one pass, partial
8-row LayerNorm blocks, three cameras, row masks that differ from row to row.  Outputs carry SENTINEL tails and strided
operands NaN gaps, so a read or write outside an operand's rows shows up.  Bars and measured errors: DESIGN.md §5."""
import numpy as np
import pytest
import torch

import vice_oracle as V
from oracle import jax_prng as P

pytestmark = pytest.mark.gpu
TOL = 2e-6                  # forward values and reductions, of the output's max
# LayerNorm forward outputs, of each row's own max: the fast variance E[x^2] - E[x]^2 loses digits on rows whose mean is a few
# times their spread, and the scale-30 columns carry that rounding into the output (measured 3.9e-6 on an H100)
LN_FWD_TOL = 1e-5
LN_BWD_TOL = 5e-5           # LayerNorm backward outputs
SENTINEL = -1234.5
TAIL = 64
KEEP = 0.9
TIE_KEY = (0, 17220)        # first sort round at N = 2048 has a tie (tests/test_vice_ops_cpu.py)


def L():
    from serl_b200 import _lib
    return _lib


def cu(x, dt=torch.float32):
    return torch.as_tensor(np.asarray(x)).to("cuda", dt).contiguous()


def f64(x):
    return torch.as_tensor(np.asarray(x)).double()


def host(t):
    return t.cpu().numpy()


def _tail(n, fill=SENTINEL, dt=torch.float32):
    return torch.full((n + TAIL,), fill, dtype=dt, device="cuda")


def _call(name, *args):
    """C-ABI call on the current stream; tensors are passed as device pointers and stay alive until the call returns"""
    L().call(name, *[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args], L().stream_ptr())


def _keys(*ks):
    return cu(np.concatenate([np.asarray(k, np.uint32) for k in ks]).view(np.int32), torch.int32)


def _rel(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def _rowrel(got, ref):
    """worst |got - ref| of a row over that row's max (floored at 1e-3 of the whole output's max)"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    scale = np.maximum(np.abs(ref).max(1), 1e-3 * np.abs(ref).max())
    return float((np.abs(got - ref).max(1) / scale).max())


def _report(name, err, bar):
    print(f"VICE_OP_ERR {name} {err:.3e} bar {bar:.0e}")
    assert err <= bar, (name, err, bar)


# ---- serl_vice_draws -------------------------------------------------------------------------------------------------
def _cam_keys(seed, ncams):
    return [list(P.split(P.fold_in(P.prng_key(seed), j), 3)) for j in range(ncams)]


@pytest.mark.parametrize("ncams,N,tie", [(1, 2, None), (3, 16, None), (1, 512, None), (3, 1624, None), (1, 1626, None),
                                         (2, 2048, None), (1, 2048, TIE_KEY), (2, 2048, (0, 19942)), (3, 2048, (0, 27595))])
def test_draws_bit_exact(ncams, N, tie):
    from serl_b200.agents.continuous.vice import permutation_rounds
    ks = _cam_keys(N, ncams)
    if tie is not None:                                       # the tie key permutes the last camera
        ks[-1][1] = np.array(tie, np.uint32)
        bits = P.random_bits(P.split(ks[-1][1])[1], (N,))
        assert np.unique(bits).size < N, "the tie key has no tie in its first round"
    lam, perm, eps = _tail(ncams), _tail(ncams * N, -7, torch.int32), _tail(ncams * N // 2)
    _call("serl_vice_draws", _keys(*[k for c in ks for k in c]), ncams, N, permutation_rounds(N), lam.data_ptr(),
             perm.data_ptr(), eps.data_ptr())
    lh, ph, eh = host(lam), host(perm), host(eps)
    for j, (k0, k1, ke) in enumerate(ks):
        assert lh[j] == P.uniform01(k0, ()), j
        assert np.array_equal(ph[j * N:(j + 1) * N], V.permutation(k1, N)), j
        assert np.array_equal(eh[j * N // 2:(j + 1) * N // 2], P.uniform01(ke, (N // 2,))), j
    assert (lh[ncams:] == SENTINEL).all() and (ph[ncams * N:] == -7).all() and (eh[ncams * N // 2:] == SENTINEL).all()


@pytest.mark.parametrize("N", [15, 0, 2050])
def test_draws_rejects_bad_row_counts_before_launching(N):
    lam, perm, eps = _tail(1), _tail(4096, 0, torch.int32), _tail(2048)
    k = _keys(*_cam_keys(0, 1)[0])
    n0 = L().launch_count()
    with pytest.raises(L().SerlError):
        _call("serl_vice_draws", k.data_ptr(), 1, N, 2, lam.data_ptr(), perm.data_ptr(), eps.data_ptr())
    assert L().launch_count() == n0
    assert (host(perm) == 0).all()


# ---- serl_vice_mix ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncams,N,D,lam_kind", [(1, 2, 8192, "random"), (3, 2, 37, "zero"), (2, 2048, 37, "random"),
                                                (1, 2048, 8192, "one"), (3, 16, 8192, "random"), (2, 6, 37, "one")])
def test_mix_and_interpolates(ncams, N, D, lam_kind):
    rng = np.random.default_rng(N + D + ncams)
    H = N // 2
    in_stride, out_stride = N * D + 37, 3 * H * D + 53
    feats = np.full((ncams, in_stride), np.nan, np.float32)
    feats[:, :N * D] = rng.standard_normal((ncams, N * D)).astype(np.float32)
    lam = {"zero": np.zeros(ncams), "one": np.ones(ncams), "random": rng.random(ncams)}[lam_kind].astype(np.float32)
    perm = np.stack([rng.permutation(N) for _ in range(ncams)]).astype(np.int32)
    eps = rng.random((ncams, H)).astype(np.float32)
    eps[:, 0] = 0.0
    out = torch.full((ncams * out_stride + TAIL,), np.nan, device="cuda")
    _call("serl_vice_mix", cu(feats), in_stride, cu(lam), cu(perm, torch.int32), cu(eps),
             out.data_ptr(), out_stride, ncams, N, D)
    o = host(out)
    assert np.isnan(o[ncams * out_stride:]).all()
    worst = 0.0
    for j in range(ncams):
        oc = o[j * out_stride:(j + 1) * out_stride]
        assert np.isnan(oc[3 * H * D:]).all(), j                 # the gap behind row 3N/2 survives
        f = feats[j, :N * D].reshape(N, D).astype(np.float64)
        l, l1 = float(lam[j]), float(np.float32(1) - lam[j])
        a, b = l * f, l1 * f[perm[j]]
        mix = oc[:N * D].reshape(N, D).astype(np.float64)
        worst = max(worst, float((np.abs(mix - (a + b)) / (np.abs(a) + np.abs(b) + 1e-30)).max()))
        e = eps[j].astype(np.float64)[:, None]
        e1 = (np.float32(1) - eps[j]).astype(np.float64)[:, None]
        ia, ib = e * mix[:H], e1 * mix[H:]
        gp = oc[N * D:3 * H * D].reshape(H, D).astype(np.float64)
        worst = max(worst, float((np.abs(gp - (ia + ib)) / (np.abs(ia) + np.abs(ib) + 1e-30)).max()))
        if lam_kind != "random":                                 # lam 0 or 1: one operand exactly
            assert np.array_equal(mix, f if lam_kind == "one" else f[perm[j]])
    _report(f"mix[{ncams},{N},{D},{lam_kind}] (of |terms|)", worst, 2.0 ** -22)   # two roundings, FMA contraction


def test_mix_rejects_odd_rows():
    x = _tail(64)
    with pytest.raises(L().SerlError):
        _call("serl_vice_mix", x.data_ptr(), 64, x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), 64, 1, 3, 4)


# ---- serl_vice_bce ---------------------------------------------------------------------------------------------------
def _bce(x, y):
    return np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))


@pytest.mark.parametrize("N", [2, 16, 512, 2048])
@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
def test_bce_loss_and_dlogit(N, grad_scale):
    rng = np.random.default_rng(N)
    x = (3 * rng.standard_normal(N)).astype(np.float32)
    special = np.array([100, -100, 30, -30, 0, 0], np.float32)[:N]
    at = np.sort(rng.choice(N, special.size, replace=False))
    if N > 256:
        at[-1] = N - 1                                        # one special logit in the last 256-row pass
    x[at] = special
    lam = np.float32(0.37)
    perm = rng.permutation(N).astype(np.int32)
    dlogit, info = _tail(N), torch.full((4,), SENTINEL, device="cuda")
    _call("serl_vice_bce", cu(x), cu([lam]), cu(perm, torch.int32), grad_scale, dlogit.data_ptr(),
             info.data_ptr(), N)
    y = V.labels(N).astype(np.float64)
    xd, l = x.astype(np.float64), float(lam)
    sg = 1 / (1 + np.exp(-xd))
    ref_d = grad_scale * (l * (sg - y) + (1 - l) * (sg - y[perm])) / N
    ref_loss = grad_scale * (l * _bce(xd, y).mean() + (1 - l) * _bce(xd, y[perm]).mean())
    d, inf = host(dlogit), host(info)
    assert (d[N:] == SENTINEL).all() and (inf[1:] == SENTINEL).all()
    _report(f"bce dlogit[{N},{grad_scale}]", _rel(d[:N], ref_d), TOL)
    _report(f"bce loss[{N},{grad_scale}]", abs(float(inf[0]) - ref_loss) / abs(ref_loss), TOL)


# ---- serl_vice_ln_act_fwd / _bwd -------------------------------------------------------------------------------------
LAYOUTS = [(5, 32, 11), (0, 6, 2)]          # (R0, R, P): primal rows [R0, R), tangent rows [R, R + P) of partners [R - P, R)
CASES = [dict(mask=False, head=False, pre=False), dict(mask=True, head=True, pre=False), dict(mask=True, head=False, pre=True),
         dict(mask=False, head=True, pre=True)]


def _ln_inputs(D, R0, R, Pn, case, seed):
    rng = np.random.default_rng(seed)
    T = R + Pn
    z = (1.5 * rng.standard_normal((T, D)) + 0.2).astype(np.float32)
    z[R0] = 0.375                                              # constant rows: var 0, rstd = eps^-1/2 (one unpaired, one paired)
    z[R - 1] = 0.375
    z[R - 2] = (1e-4 * rng.standard_normal(D)).astype(np.float32)   # near-constant: var 1e-8 << eps
    scale = (1 + 0.3 * rng.standard_normal(D)).astype(np.float32)
    bias = (0.2 * rng.standard_normal(D)).astype(np.float32)
    scale[:4] = 30.0                                           # saturated tanh / large leaky slopes
    scale[4:8], bias[4:8] = 0.0, 0.0                           # activation input exactly 0 (leaky_relu: slope 1, jax's >=)
    mask = rng.random((T, D)) < KEEP if case["mask"] else None  # a different mask on every row, tangent rows included
    pb = (0.1 * rng.standard_normal(D)).astype(np.float32) if case["pre"] else None
    hw = (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32)
    hb = np.float32(0.3)
    dy = rng.standard_normal((T, D)).astype(np.float32)
    dlogit = rng.standard_normal(R).astype(np.float32) if case["mask"] else None   # head: a dlogit array, or dlogit_const
    return z, scale, bias, mask, pb, hw, hb, dy, dlogit


def _strided(x, ld, c0, fill, dt=torch.float32):
    buf = np.full((x.shape[0], ld), fill, np.asarray(x).dtype)
    buf[:, c0:c0 + x.shape[1]] = x
    return cu(buf, dt)


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: "R0_%d_R_%d_P_%d" % l)
@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(k for k, v in c.items() if v) or "plain")
@pytest.mark.parametrize("act", ["tanh", "leaky_relu"])
@pytest.mark.parametrize("D", [256, 512])
def test_ln_act_fwd_bwd(D, act, case, layout):
    lib = L()
    R0, R, Pn = layout
    T = R + Pn
    z, scale, bias, mask, pb, hw, hb, dy, dlogit = _ln_inputs(D, R0, R, Pn, case, seed=D + R + len(act))
    a_id = getattr(lib, "ACT_" + act.upper())
    head = case["head"]
    dlogit_const, tan_seed = np.float32(0.7), np.float32(1.3)
    ld_z, cz, ld_y, cy, ld_m, ld_dz = D + 24, 8, 2 * D + 8, D, D + 16, D + 4
    zin = z.copy()
    zin[:R0] = np.nan                                          # rows below R0 are never read
    zd = _strided(zin, ld_z, cz, np.nan)
    yd = torch.full((T, ld_y), SENTINEL, device="cuda")
    xhat, rstd, logit = _tail(T * D), _tail(T), _tail(T)
    md = _strided(mask.astype(np.uint8), ld_m, 0, 3, torch.uint8) if mask is not None else None
    sc, bi, hwd, hbd = cu(scale), cu(bias), cu(hw), cu(np.array([hb]))
    pbd = cu(pb) if pb is not None else None
    p = lambda t, off=0: None if t is None else t.data_ptr() + 4 * off
    zp, yp = p(zd, cz), p(yd, cy)
    st = lib.stream_ptr()
    for tangent in (0, 1):
        r0, r1 = (R0, R) if not tangent else (R, T)
        lib.call("serl_vice_ln_act_fwd", zp, ld_z, p(pbd), None if md is None else md.data_ptr(), ld_m, KEEP, sc.data_ptr(), bi.data_ptr(),
                 yp, ld_y, xhat.data_ptr(), rstd.data_ptr(), p(hwd) if head and not tangent else None,
                 p(hbd) if head and not tangent else None, logit.data_ptr() if head and not tangent else None, r0, r1,
                 Pn if tangent else 0, tangent, D, a_id, 1e-6, st)
    dz = torch.full((T, ld_dz), SENTINEL, device="cuda")
    dsr, dbr, dwr = _tail(T * D), _tail(T * D), _tail(T * D)
    dyd = None if head else _strided(dy, D + 12, 0, np.nan)
    dld = cu(dlogit) if head and dlogit is not None else None
    lib.call("serl_vice_ln_act_bwd", p(dyd), D + 12, p(dld),
             float(dlogit_const), p(hwd) if head else None, float(tan_seed), xhat.data_ptr(), rstd.data_ptr(), zp, ld_z,
             None if md is None else md.data_ptr(), ld_m, KEEP, sc.data_ptr(), bi.data_ptr(), yp, ld_y, dz.data_ptr(), ld_dz,
             dsr.data_ptr(), dbr.data_ptr(), dwr.data_ptr() if head else None, R0, R, Pn, D, a_id, st)

    # ---- float64 reference ----
    mP = None if mask is None else mask[R0:R]
    mT = None if mask is None else mask[R - Pn:R]              # a tangent row uses its partner's mask
    zP, zD = f64(z[R0:R]).requires_grad_(True), f64(z[R:T]).requires_grad_(True)
    S = f64(np.broadcast_to(scale, (R - R0, D))).clone().requires_grad_(True)   # one parameter row per primal row: per-row terms
    Bi = f64(np.broadcast_to(bias, (R - R0, D))).clone().requires_grad_(True)
    pbt = None if pb is None else f64(pb)
    y = V.ln_act(zP, S, Bi, act, mP, pbt)
    _, ydot = V.ln_act_jvp(zP[-Pn:], zD, S[-Pn:], Bi[-Pn:], act, mT, pbt)
    x = f64(z[R0:R]) + (0 if pbt is None else pbt)
    if mP is not None:
        x = torch.where(torch.as_tensor(mP), x / KEEP, torch.zeros_like(x))
    mean = x.mean(-1, keepdim=True)
    rs = torch.rsqrt(((x * x).mean(-1, keepdim=True) - mean * mean).clamp_min(0) + 1e-6)

    yh = host(yd)
    assert (yh[:R0] == SENTINEL).all() and (yh[:, :cy] == SENTINEL).all() and (yh[:, cy + D:] == SENTINEL).all()
    g = lambda t: t.detach().numpy()
    _report(f"ln_fwd y[{D},{act},{case},{layout}]", _rowrel(yh[R0:R, cy:cy + D], g(y)), LN_FWD_TOL)
    _report(f"ln_fwd ydot[{D},{act},{case},{layout}]", _rowrel(yh[R:T, cy:cy + D], g(ydot)), LN_FWD_TOL)
    xh, rh = host(xhat), host(rstd)
    _report(f"ln_fwd xhat[{D},{act},{case},{layout}]", _rowrel(xh[R0 * D:R * D].reshape(-1, D), g((x - mean) * rs)), LN_FWD_TOL)
    _report(f"ln_fwd rstd[{D},{act},{case},{layout}]", float(np.abs(rh[R0:R] / g(rs)[:, 0] - 1).max()), LN_FWD_TOL)
    assert (xh[:R0 * D] == SENTINEL).all() and (xh[R * D:] == SENTINEL).all() and (rh[:R0] == SENTINEL).all() and (rh[R:] == SENTINEL).all()
    # the tangent rows' masked input is written back to z, bit for bit
    zh = host(zd)
    want = z[R:T] if mask is None else np.where(mask[R - Pn:R], z[R:T] / np.float32(KEEP), np.float32(0))
    assert np.array_equal(zh[R:T, cz:cz + D], want)
    assert np.array_equal(zh[R0:R, cz:cz + D], z[R0:R])       # primal rows keep their input
    lh = host(logit)
    if head:
        _report(f"ln_fwd logit[{D},{act},{case},{layout}]", _rel(lh[R0:R], g(y @ f64(hw) + float(hb))), LN_FWD_TOL)
    assert (lh[:R0] == SENTINEL).all() and (lh[R:] == SENTINEL).all()

    # backward: cotangents of y (rows [R0, R)) and ydot (tangent rows)
    if head:
        a = f64(dlogit[R0:R]) if dlogit is not None else torch.full((R - R0,), float(dlogit_const), dtype=torch.float64)
        ybar, ydotbar = a[:, None] * f64(hw)[None, :], float(tan_seed) * f64(hw).expand(Pn, D)
    else:
        ybar, ydotbar = f64(dy[R0:R]), f64(dy[R:T])
    obj = (ybar * y).sum() + (ydotbar * ydot).sum()
    gz, gzd, gs, gb = (g(t) for t in torch.autograd.grad(obj, [zP, zD, S, Bi]))
    dzh = host(dz)
    assert (dzh[:R0] == SENTINEL).all() and (dzh[:, D:] == SENTINEL).all()
    tag = f"[{D},{act},{case},{layout}]"
    _report("ln_bwd dz " + tag, _rowrel(dzh[R0:R, :D], gz), LN_BWD_TOL)
    _report("ln_bwd dzdot " + tag, _rowrel(dzh[R:T, :D], gzd), LN_BWD_TOL)
    ds, db = host(dsr), host(dbr)
    for name, got, ref in (("dscale", ds, gs), ("dbias", db, gb)):
        assert (got[:R0 * D] == SENTINEL).all() and (got[R * D:] == SENTINEL).all(), name
        rows = got[R0 * D:R * D].reshape(-1, D)
        _report(f"ln_bwd {name}_rows " + tag, _rowrel(rows, ref), LN_BWD_TOL)
        _report(f"ln_bwd {name} colsum " + tag, _rel(rows.astype(np.float64).sum(0), ref.sum(0)), LN_BWD_TOL)
    dw = host(dwr)
    if head:
        ref = (a[:, None] * y).detach().clone()
        ref[-Pn:] += float(tan_seed) * ydot.detach()
        _report("ln_bwd dw_rows " + tag, _rowrel(dw[R0 * D:R * D].reshape(-1, D), g(ref)), LN_BWD_TOL)
    else:
        assert (dw == SENTINEL).all()


# ---- serl_vice_sle_input_grad ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 13, 1024])
def test_sle_input_grad(R):
    rng = np.random.default_rng(R)
    ld = 4096 + 68
    ds = np.full((R, ld), np.nan, np.float32)
    ds[:, :4096] = rng.standard_normal((R, 4096))
    k = rng.standard_normal((4, 4, 512, 8)).astype(np.float32)
    dx = _tail(R * 16 * 512)
    _call("serl_vice_sle_input_grad", cu(ds), ld, cu(k), dx.data_ptr(), R, 16, 512)
    d3, k3 = ds[:, :4096].reshape(R, 512, 8).astype(np.float64), k.reshape(16, 512, 8).astype(np.float64)
    ref = np.einsum("rcf,pcf->rpc", d3, k3)
    mag = np.einsum("rcf,pcf->rpc", np.abs(d3), np.abs(k3))
    got = host(dx)
    assert (got[R * 8192:] == SENTINEL).all()
    _report(f"sle_input_grad[{R}] (of sum |terms|)", float((np.abs(got[:R * 8192].reshape(R, 16, 512) - ref) / mag).max()), TOL)


def test_sle_input_grad_rejects_misaligned_operands():
    ds, k, dx = _tail(2 * 4096), _tail(16 * 512 * 8), _tail(2 * 8192)
    for ptr, ld in ((ds.data_ptr() + 4, 4096), (ds.data_ptr(), 4098)):
        with pytest.raises(L().SerlError):
            _call("serl_vice_sle_input_grad", ptr, ld, k.data_ptr(), dx.data_ptr(), 1, 16, 512)
    assert (host(dx) == SENTINEL).all()


# ---- serl_vice_mask_fill ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,n,fold,keep,broadcast", [(7, 13, 0, 0.9, 0), (512, 4096, 1, 0.9, 0), (9, 255, 3, 0.5, 0),
                                                        (6, 256, 2, 0.9, 1), (5, 7, 1, 0.5, 1), (1024, 4096, 0, 0.9, 1)])
def test_mask_fill_bit_exact(rows, n, fold, keep, broadcast):
    key = P.split(P.prng_key(rows * n))[1]
    out = _tail(rows * n, 7, torch.uint8)
    _call("serl_vice_mask_fill", _keys(key), fold, keep, out.data_ptr(), rows, n, broadcast)
    k = P.fold_in(key, fold)
    want = np.broadcast_to(P.bernoulli(k, keep, (n,)), (rows, n)) if broadcast else P.bernoulli(k, keep, (rows, n))
    got = host(out)
    assert np.array_equal(got[:rows * n].reshape(rows, n), want.astype(np.uint8))
    assert (got[rows * n:] == 7).all()


# ---- serl_vice_gp_rows / serl_vice_gp_finish -------------------------------------------------------------------------
@pytest.mark.parametrize("ncams,B,D", [(1, 1, 8192), (3, 1024, 8192), (2, 5, 300), (3, 7, 300)])
def test_gp_rows(ncams, B, D):
    rng = np.random.default_rng(B * D)
    gs, vs = B * D + 19, B * D + 41
    g = np.full((ncams, gs), np.nan, np.float32)
    rows = (rng.standard_normal((ncams, B, D)) * rng.uniform(0.1, 3.0, (ncams, B, 1)) / np.sqrt(D)).astype(np.float32)
    rows[0, 0] = 0.0                                          # |g| = sqrt(D 1e-6)
    if B > 1:                                                  # |g| within fp32 rounding of 1
        rows[-1, 1] *= np.float32(np.sqrt((1 - D * 1e-6) / np.sum(rows[-1, 1].astype(np.float64) ** 2)))
    g[:, :B * D] = rows.reshape(ncams, -1)
    v = torch.full((ncams * vs + TAIL,), SENTINEL, device="cuda")
    norms = _tail(ncams * B)
    coef = 10.0 * 2.0 / (ncams * B)
    _call("serl_vice_gp_rows", cu(g), gs, v.data_ptr(), vs, coef, norms.data_ptr(), ncams, B, D)
    r = rows.astype(np.float64)
    nrm = np.sqrt((r ** 2 + 1e-6).sum(-1))
    want = coef * ((nrm - 1) / nrm)[..., None] * r
    got_n, got_v = host(norms), host(v)
    _report(f"gp_rows norms[{ncams},{B},{D}]", float(np.abs(got_n[:ncams * B] / nrm.reshape(-1) - 1).max()), TOL)
    vv = np.stack([got_v[j * vs:j * vs + B * D] for j in range(ncams)]).reshape(ncams, B, D)
    _report(f"gp_rows v[{ncams},{B},{D}]", _rel(vv, want), TOL)
    assert (vv[0, 0] == 0).all()
    for j in range(ncams):
        assert (got_v[j * vs + B * D:(j + 1) * vs] == SENTINEL).all()
    assert (got_v[ncams * vs:] == SENTINEL).all() and (got_n[ncams * B:] == SENTINEL).all()


@pytest.mark.parametrize("M", [1, 255, 256, 257, 2048])
@pytest.mark.parametrize("info_scale", [1.0, 0.5])
def test_gp_finish(M, info_scale):
    rng = np.random.default_rng(M)
    n = rng.uniform(0.2, 2.5, M).astype(np.float32)
    n[-1] = 4.0                                               # the last norm weighs in: it sits in the pass past 256 for M > 256
    info = cu(np.array([0.37, SENTINEL, SENTINEL, SENTINEL, SENTINEL], np.float32))
    _call("serl_vice_gp_finish", cu(n), M, 10.0, info_scale, info.data_ptr())
    nd = n.astype(np.float64)
    m1, gp = info_scale * nd.mean(), info_scale * ((nd - 1) ** 2).mean()
    got = host(info)
    assert got[0] == np.float32(0.37) and got[4] == SENTINEL
    for name, gv, rv in (("mean_norm", got[1], m1), ("gp", got[2], gp), ("total", got[3], float(np.float32(0.37)) + 10 * gp)):
        _report(f"gp_finish {name}[{M},{info_scale}]", abs(float(gv) - rv) / abs(rv), TOL)


# ---- serl_vice_reward ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 255, 256, 257, 1024])
@pytest.mark.parametrize("threshold", [0, 1])
@pytest.mark.parametrize("with_mean", [True, False])
def test_reward(B, threshold, with_mean):
    rng = np.random.default_rng(B)
    x = (4 * rng.standard_normal(B)).astype(np.float32)
    x[np.abs(x) < 1e-3] = 0.5                                 # fp32 and float64 sigmoids agree on the side of 0.5 away from 0
    special = np.array([0, 1e-30, -1e-30, 100, -100, 0], np.float32)[:B]
    at = rng.choice(B, special.size, replace=False)
    if B > 256:
        at[0] = B - 1                                         # an exact 0 in the last 256-row pass
    x[at] = special
    rew, mean = _tail(B), (_tail(1) if with_mean else None)
    _call("serl_vice_reward", cu(x), rew.data_ptr(), None if mean is None else mean.data_ptr(), B, threshold)
    sg = 1 / (1 + np.exp(-x.astype(np.float64)))
    want = (sg >= 0.5).astype(np.float64) if threshold else sg
    got = host(rew)
    assert (got[B:] == SENTINEL).all()
    if threshold:
        assert np.array_equal(got[:B], want) and (got[:B][x == 0] == 1).all()
    else:
        _report(f"reward sigmoid[{B}]", _rel(got[:B], want), TOL)
    if with_mean:
        m = host(mean)
        assert (m[1:] == SENTINEL).all()
        _report(f"reward mean[{B},{threshold}]", abs(float(m[0]) - want.mean()) / max(want.mean(), 1e-30), TOL)
