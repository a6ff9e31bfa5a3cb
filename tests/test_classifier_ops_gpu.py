"""GPU: each entry point of csrc/classifier.cu against a float64 restatement on the same fp32 inputs, at the row counts where its
launch shape changes and on the rows where its arithmetic reaches an edge.  Every op is launched twice into outputs filled with
NaN (in place: twice from the same input), the two results must be bitwise equal, and the words after the last row must still
hold the sentinel.

  serl_layernorm_relu_head_fwd / _bwd   a warp per row, 8 rows per CTA: R in {1, 7, 8, 9, 130, 1024, 4096}, with and without
                                        the dropout mask; a constant row (var = 0, rstd = eps^-1/2), a row whose mean is four
                                        times its spread (the fast variance's cancellation), a row whose pre-activations are all
                                        negative (h = 0, logit = b, dz = 0) and, masked, a row whose mask drops everything.
  serl_bce_logits_loss                  one CTA of 256 threads: B in {1, 255, 256, 257, 1024, 4096}, so up to 16 rows per thread;
                                        logits of +-100, +-20, exactly 0 and -1e-9 (its fp32 sigmoid rounds to 0.5); grad_scale 2.5.
  serl_dropout_bwd_f32                  a grid capped at 1184 x 256 = 303,104 threads: n = 0, 1, 303,103, 303,104, 303,105 and
                                        2 x 256 x 4096 (two cameras at the reference's batch), bit-exact against the correctly
                                        rounded fp32 division.
Bars: LayerNorm forward outputs 1e-5 and backward outputs 5e-5 of each row's own max (the bars of tests/test_vice_ops_gpu.py
for the same LayerNorm statistics), the logit over its row's sum of |h w| + |b|; BCE loss and dlogit 2e-6; accuracy exact.
Measured errors: DESIGN.md §5."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D, KEEP, EPS = 256, 0.9, 1e-6
LN_FWD_TOL = 1e-5
LN_BWD_TOL = 5e-5
BCE_TOL = 2e-6
GUARD = 8                        # sentinel words after each output


def cu(x, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(x)).cuda()
    return t if dt is None else t.to(dt)


def _nan(n):
    return torch.full((n + GUARD,), float("nan"), device="cuda")


def _twice(launch, outs, sizes):
    """launch() twice into NaN-filled outputs: bitwise equal results, the guard words untouched; the outputs as float64."""
    res = []
    for _ in range(2):
        for o in outs:
            o.fill_(float("nan"))
        launch()
        res.append([o.clone() for o in outs])
    for a, b, n in zip(res[0], res[1], sizes):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two launches differ"
        assert torch.isnan(a[n:]).all(), "wrote past the last row"
    return [o[:n].cpu().numpy().astype(np.float64) for o, n in zip(res[1], sizes)]


def _row_err(got, ref):
    """max over rows of max|got - ref| / max|ref| within the row; a row whose reference is all zero must be exactly zero."""
    got, ref = np.atleast_2d(got), np.atleast_2d(ref)
    m, d = np.abs(ref).max(-1), np.abs(got - ref).max(-1)
    return float(np.where(m > 0, d / np.where(m > 0, m, 1.0), np.where(d == 0, 0.0, np.inf)).max())


# ---- LayerNorm + relu + Dense(1) head ------------------------------------------------------------------------------------
def _head_inputs(R, masked, seed):
    rng = np.random.default_rng(seed)
    z = (2 * rng.standard_normal((R, D)) + 0.3).astype(np.float32)
    mask = (rng.random((R, D)) < KEEP).astype(np.uint8)
    rows = {}
    for kind, r in (("constant", R - 1), ("offset", 0), ("dead", R // 2), ("dropped", 1)):
        if r < R and r not in rows.values():
            rows[kind] = r
    if "constant" in rows:
        z[rows["constant"]] = 1.5                        # exact sums: mean 1.5, var 0 (unmasked)
    if "offset" in rows:
        z[rows["offset"]] = 2 + 0.5 * rng.standard_normal(D)
    if "dead" in rows:                                   # xhat 1/sqrt(255) and -sqrt(255): every scale * xhat + bias < 0
        z[rows["dead"]] = 0
        z[rows["dead"], 17] = -40
        mask[rows["dead"], 17] = 1
    if masked and "dropped" in rows:
        mask[rows["dropped"]] = 0
    scale = (0.5 + 0.1 * rng.standard_normal(D)).astype(np.float32)
    bias = (-0.1 - 0.05 * np.abs(rng.standard_normal(D))).astype(np.float32)
    w = (0.1 * rng.standard_normal(D)).astype(np.float32)
    b = rng.standard_normal(1).astype(np.float32)
    dl = rng.standard_normal(R).astype(np.float32)
    return z, (mask if masked else None), scale, bias, w, b, dl, rows


@pytest.mark.parametrize("masked", [False, True], ids=["plain", "mask"])
@pytest.mark.parametrize("R", [1, 7, 8, 9, 130, 1024, 4096])
def test_ln_relu_head_fwd_bwd_rows(R, masked):
    from serl_b200 import ops
    z, mask, scale, bias, w, b, dl, rows = _head_inputs(R, masked, seed=R + masked)
    zd, sc, bi, wd, bd, dld = cu(z), cu(scale), cu(bias), cu(w), cu(b), cu(dl)
    md = cu(mask) if mask is not None else None
    mp = None if md is None else md.data_ptr()
    h, xh, rs, lo = _nan(R * D), _nan(R * D), _nan(R), _nan(R)
    h_, xh_, rs_, lo_ = _twice(lambda: ops.ln_relu_head_fwd(zd.data_ptr(), mp, KEEP, sc.data_ptr(), bi.data_ptr(), wd.data_ptr(), bd.data_ptr(),
                                                            h.data_ptr(), xh.data_ptr(), rs.data_ptr(), lo.data_ptr(), R),
                               [h, xh, rs, lo], [R * D, R * D, R, R])
    h_, xh_ = h_.reshape(R, D), xh_.reshape(R, D)
    dy, dz = _nan(R * D), _nan(R * D)
    dy_, dz_ = _twice(lambda: ops.ln_relu_head_bwd(dld.data_ptr(), wd.data_ptr(), h.data_ptr(), xh.data_ptr(), rs.data_ptr(), sc.data_ptr(),
                                                   mp, KEEP, dy.data_ptr(), dz.data_ptr(), R), [dy, dz], [R * D, R * D])
    dy_, dz_ = dy_.reshape(R, D), dz_.reshape(R, D)

    # float64: [dropout] -> LayerNorm (fast variance, eps 1e-6) -> relu -> Dense(1), and autograd of sum(dlogit * logit)
    f = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    zz = f(z).requires_grad_(True)
    x = zz if mask is None else torch.where(torch.as_tensor(mask).bool(), zz / KEEP, torch.zeros_like(zz))
    mean = x.mean(-1, keepdim=True)
    var = ((x * x).mean(-1, keepdim=True) - mean * mean).clamp_min(0)
    rstd = torch.rsqrt(var + EPS)
    xhat = (x - mean) * rstd
    y = xhat * f(scale) + f(bias)
    live = torch.as_tensor(h_ > 0)                      # the backward's relu takes the forward's h, as the kernel does
    yd = y.detach().numpy()
    assert ((h_ > 0) == (yd > 0))[np.abs(yd) > 1e-5].all(), "relu decisions differ away from 0"
    logit = torch.relu(y) @ f(w) + f(b)
    (gz,) = torch.autograd.grad(((torch.where(live, y, torch.zeros_like(y)) @ f(w)) * f(dl)).sum(), zz)
    hr = torch.relu(y).detach().numpy()
    terms = np.abs(hr) @ np.abs(w.astype(np.float64)) + abs(float(b[0]))
    errs = {"h": _row_err(h_, hr), "xhat": _row_err(xh_, xhat.detach().numpy()),
            "rstd": float((np.abs(rs_ - rstd.detach().numpy()[:, 0]) / rstd.detach().numpy()[:, 0]).max()),
            "logit": float((np.abs(lo_ - logit.detach().numpy()) / terms).max()),
            "dy": _row_err(dy_, np.where(h_ > 0, dl[:, None].astype(np.float64) * w.astype(np.float64)[None], 0.0)),
            "dz": _row_err(dz_, gz.numpy())}
    print(f"CLF_OPS_ERR ln_relu_head R={R} {'mask' if masked else 'plain'}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v <= (LN_BWD_TOL if k in ("dy", "dz") else LN_FWD_TOL), (k, v)
    if "constant" in rows and mask is None:
        r = rows["constant"]
        assert abs(rs_[r] - 1e3) <= 1e-3 and (xh_[r] == 0).all()     # rsqrtf(eps): within 2 ulp of eps^-1/2
    if "dead" in rows:
        r = rows["dead"]
        assert (h_[r] == 0).all() and lo_[r] == b[0] and (dy_[r] == 0).all() and (dz_[r] == 0).all()
    if mask is not None:
        assert (dz_[mask == 0] == 0).all()
        if "dropped" in rows:
            assert (dz_[rows["dropped"]] == 0).all()


# ---- sigmoid BCE + accuracy ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 255, 256, 257, 1024, 4096])
def test_bce_logits_loss_rows(B):
    from oracle import classifier as OC
    from serl_b200 import ops
    rng = np.random.default_rng(B)
    gs = 2.5
    xt = (3 * rng.standard_normal(B)).astype(np.float32)
    xe = (xt + 0.5 * rng.standard_normal(B)).astype(np.float32)
    for i, v in enumerate((100.0, -100.0, 20.0, -20.0, 0.0, -1e-9)[:B]):
        xt[(97 * i) % B] = xe[(97 * i) % B] = v
    y = (rng.random(B) < 0.5).astype(np.float32)
    xtd, xed, yd = cu(xt), cu(xe), cu(y)
    dl, info = _nan(B), _nan(2)
    dl_, info_ = _twice(lambda: ops.bce_logits_loss(xtd.data_ptr(), xed.data_ptr(), yd.data_ptr(), gs, dl.data_ptr(), info.data_ptr(), B),
                        [dl, info], [B, 2])
    x64, y64 = torch.as_tensor(xt, dtype=torch.float64), torch.as_tensor(y, dtype=torch.float64)
    loss = float(OC.bce(x64, y64).mean())
    dref = ((torch.sigmoid(x64) - y64) * gs / B).numpy()
    count = round(OC.accuracy(xe, y) * B)
    le = abs(info_[0] - loss) / max(abs(loss), 1.0)
    de = float(np.abs(dl_ - dref).max() / max(np.abs(dref).max(), 1e-30))   # B = 1: sigmoid(100) - 1 is 0 in both
    print(f"CLF_OPS_ERR bce B={B}: loss {le:.2e}, dlogit {de:.2e}, accuracy {count}/{B}")
    assert le <= BCE_TOL and de <= BCE_TOL, (le, de)
    assert np.float32(info_[1]) == np.float32(count) * (np.float32(1) / np.float32(B)), (info_[1], count)


# ---- dropout backward --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 303103, 303104, 303105, 2 * 256 * 4096])
def test_dropout_bwd_grid_stride(n):
    from serl_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, device="cuda", generator=g)
    m = (torch.rand(n + GUARD, device="cuda", generator=g) < KEEP).to(torch.uint8)
    keep = torch.tensor(KEEP, dtype=torch.float32).double()     # correctly rounded fp32 division, like the forward's x / keep
    ref = torch.where(m[:n].bool(), (x.double() / keep).float(), torch.zeros_like(x))
    outs = []
    for _ in range(2):
        dx = _nan(n)
        dx[:n] = x
        ops.dropout_bwd(dx.data_ptr(), m.data_ptr(), KEEP, n)
        assert torch.isnan(dx[n:]).all(), "wrote past n"
        outs.append(dx[:n].clone())
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    assert torch.equal(outs[0], ref)
