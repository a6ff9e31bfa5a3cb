"""GPU: the MLP layer, LayerNorm parameter-gradient, column-sum, policy std-head, loss and copy / fill kernels op by op (through
the C-ABI), each against a float64 torch restatement of the same operation on the same fp32 inputs.

Activations come from tests/arch_oracle.py, LayerNorm from oracle/drq.py and derivatives from float64 autograd.  The bars are
those of tests/test_ops_gpu.py (helpers.rel_err): 2e-5 for forward values and reductions, 5e-5 for LayerNorm backward outputs.
Strided operands are padded with NaN where a kernel reads and with SENTINEL where it writes, and dense outputs carry a SENTINEL
tail, so a read or write outside an operand's rows shows up."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from arch_oracle import ACTIVATIONS
from helpers import rel_err
from oracle.drq import layer_norm, tanh_normal_sample_logp

pytestmark = pytest.mark.gpu
TOL, LN_BWD_TOL = 2e-5, 5e-5
LN_EPS = 1e-6
ACTS = ("tanh", "relu", "swish", "leaky_relu", "gelu")
KINKED = ("relu", "leaky_relu")
SENTINEL = -1234.5
TAIL = 64
STD_MIN, STD_MAX = 1e-5, 5.0
# "exp" runs the launcher's entry points (serl_tanh_gaussian_fwd / serl_actor_loss), "exp_std" the same head through the _std ones
HEADS = ("exp", "exp_std", "softplus", "uniform")


def cu(x, dt=torch.float32):
    return torch.as_tensor(np.asarray(x)).to("cuda", dt).contiguous()


def f64(x):
    return torch.as_tensor(np.asarray(x)).double()


def host(t):
    return t.cpu().numpy()


def _addr(t):
    return None if t is None else t.data_ptr()


def _tail(n):
    """a device output of n floats followed by TAIL SENTINEL floats"""
    return torch.full((n + TAIL,), SENTINEL, device="cuda")


def _padded(x, ld, fill):
    """(R, D) host array -> (R, ld) device rows, columns D.. set to fill"""
    buf = np.full((x.shape[0], ld), fill, np.float32)
    buf[:, :x.shape[1]] = x
    return cu(buf)


def _act_id(act):
    from serl_b200 import _lib as L
    return getattr(L, "ACT_" + act.upper())


def _std_id(head):
    from serl_b200 import _lib as L
    return getattr(L, "STD_" + head.split("_")[0].upper())


# ---- serl_layernorm_act_fwd / _bwd --------------------------------------------------------------------------------------
def _layer_inputs(E, B, D, seed):
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((E * B, D)) * 2 + 0.3).astype(np.float32)
    sc = (1 + 0.2 * rng.standard_normal((E, D))).astype(np.float32)
    bi = (0.1 * rng.standard_normal((E, D))).astype(np.float32)
    dt = rng.standard_normal((E * B, D)).astype(np.float32)
    assert (dt != 0).all()
    return z, sc, bi, dt


def _run_layer(act, ln, z, sc, bi, dt, B, group_stride, lds=None):
    """serl_layernorm_act_fwd, then _bwd on the forward's own t (= out), xhat, rstd and pre (= z), as the engine calls them.
    lds = (ld_z, ld_out, ld_dt): row strides of z / pre, out / t and dt (D each by default).  Host arrays."""
    from serl_b200 import ops
    R, D = z.shape
    ld_z, ld_out, ld_dt = lds or (D, D, D)
    zd, dtd = _padded(z, ld_z, np.nan), _padded(dt, ld_dt, np.nan)
    scd, bid = (cu(sc), cu(bi)) if sc is not None else (None, None)
    out, out_inf = (torch.full((R, ld_out), SENTINEL, device="cuda") for _ in range(2))
    xhat, rstd, dz, dy = _tail(R * D), _tail(R), _tail(R * D), _tail(R * D)
    a = _act_id(act)
    ops.ln_act_fwd(zd.data_ptr(), ld_z, _addr(scd), _addr(bid), B, group_stride, out.data_ptr(), ld_out, xhat.data_ptr(), rstd.data_ptr(),
                   R, D, a, ln, LN_EPS)
    # inference (no statistics saved): the same output bits
    ops.ln_act_fwd(zd.data_ptr(), ld_z, _addr(scd), _addr(bid), B, group_stride, out_inf.data_ptr(), ld_out, None, None, R, D, a, ln, LN_EPS)
    ops.ln_act_bwd(dtd.data_ptr(), ld_dt, out.data_ptr(), ld_out, zd.data_ptr(), ld_z, xhat.data_ptr(), rstd.data_ptr(), _addr(scd), _addr(bid),
                   B, group_stride, dz.data_ptr(), dy.data_ptr(), R, D, a, ln)
    assert torch.equal(out, out_inf)
    o, xh, rs, dzh, dyh = host(out), host(xhat), host(rstd), host(dz), host(dy)
    got = dict(out=o[:, :D], out_pad=o[:, D:], xhat=xh[:R * D].reshape(R, D), rstd=rs[:R], dz=dzh[:R * D].reshape(R, D),
               dy=dyh[:R * D].reshape(R, D))
    np.testing.assert_array_equal(got["out_pad"], SENTINEL)
    for t, n in ((xh, R * D), (rs, R), (dzh, R * D), (dyh, R * D)):
        np.testing.assert_array_equal(t[n:], SENTINEL)
    if not ln:                          # without LayerNorm nothing but out and dz is written
        for t in (xh, rs, dyh):
            np.testing.assert_array_equal(t, SENTINEL)
    return got


def _act_ref(act, y, gate=None):
    """The activation in float64.  gate (relu / leaky_relu): which side of the kink each unit takes, here the kernel's own branch
    (a pre-activation within fp32 rounding of 0 may legitimately fall on the other side in float64)."""
    if gate is None or act not in KINKED:
        return ACTIVATIONS[act](y)
    one = torch.ones((), dtype=torch.float64)
    return y * torch.where(torch.as_tensor(gate), ACTIVATIONS[act](one), -ACTIVATIONS[act](-one))


def _layer_ref(act, ln, z, sc, bi, dt, B, gate=None):
    R, D = z.shape
    zt = f64(z).requires_grad_(True)
    y = zt
    if ln:
        sct, bit = f64(sc).requires_grad_(True), f64(bi).requires_grad_(True)
        y = layer_norm(zt.view(-1, B, D), sct[:, None, :], bit[:, None, :]).view(R, D)
        y.retain_grad()
    h = _act_ref(act, y, gate)
    h.backward(f64(dt))
    ref = dict(out=h.detach().numpy(), dz=zt.grad.numpy())
    if ln:
        zz = f64(z)
        ref["dy"] = y.grad.numpy()
        ref["xhat"] = layer_norm(zz, 1.0, 0.0).numpy()
        # flax's fast variance, as oracle.drq._norm_fast_var
        ref["rstd"] = torch.rsqrt(((zz * zz).mean(-1) - zz.mean(-1) ** 2).clamp_min(0) + LN_EPS).numpy()
    return ref


def _gates(act, got, dt, ln):
    """The branch each unit took: from the forward's output, and from the backward's dy = dt * act'(y) (dz without LayerNorm)."""
    d = got["dy"] if ln else got["dz"]
    if act == "relu":
        return got["out"] > 0, d != 0
    return got["out"] >= 0, d == dt


def _check_layer(act, ln, got, ref, rows=slice(None)):
    assert rel_err(got["out"][rows], ref["out"][rows]) < TOL
    if ln:
        assert rel_err(got["xhat"][rows], ref["xhat"][rows]) < TOL
        assert rel_err(got["rstd"][rows], ref["rstd"][rows]) < TOL
        assert rel_err(got["dy"][rows], ref["dy"][rows]) < LN_BWD_TOL
        assert rel_err(got["dz"][rows], ref["dz"][rows]) < LN_BWD_TOL
    else:
        assert rel_err(got["dz"][rows], ref["dz"][rows]) < TOL


@pytest.mark.parametrize("D", [64, 192, 1024])
@pytest.mark.parametrize("B", [13, 256])
@pytest.mark.parametrize("E", [1, 10])
@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("act", ACTS)
def test_layer_act_fwd_bwd(act, ln, E, B, D):
    """The engine's call shapes: the critic ensemble (E = 10: R = E*B rows, one scale / bias per member, group_stride = D) and
    the policy (E = 1, group_stride = 0).  B = 13: a CTA's 8 rows straddle two members."""
    z, sc, bi, dt = _layer_inputs(E, B, D, seed=E * 7 + B + D)
    got = _run_layer(act, ln, z, sc if ln else None, bi if ln else None, dt, B, D if E > 1 else 0)
    fwd_gate, bwd_gate = _gates(act, got, dt, ln)
    if act in KINKED:
        np.testing.assert_array_equal(fwd_gate, bwd_gate)
    _check_layer(act, ln, got, _layer_ref(act, ln, z, sc, bi, dt, B, gate=fwd_gate if ln else None))


@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("act", ACTS)
def test_layer_act_padded_strides(act, ln):
    """ld_z = ld_pre, ld_out = ld_t and ld_dt all wider than D (NaN / SENTINEL padding): nothing outside the rows is read or
    written."""
    E, B, D = 10, 13, 192
    z, sc, bi, dt = _layer_inputs(E, B, D, seed=11)
    got = _run_layer(act, ln, z, sc if ln else None, bi if ln else None, dt, B, D, lds=(D + 5, D + 3, D + 7))
    for k in ("out", "dz") + (("xhat", "rstd", "dy") if ln else ()):
        assert np.isfinite(got[k]).all(), k
    _check_layer(act, ln, got, _layer_ref(act, ln, z, sc, bi, dt, B, gate=_gates(act, got, dt, ln)[0] if ln else None))


# jax's derivatives at 0 (relu' = 0, leaky_relu' = 1: the kernel comments' convention)
ACT_GRAD_AT_0 = {"tanh": 1.0, "relu": 0.0, "swish": 0.5, "leaky_relu": 1.0, "gelu": 0.5}


@pytest.mark.parametrize("act", ACTS)
def test_layer_act_kinks_and_tails(act):
    """Without LayerNorm the kernel sees z itself: exact zeros, +-1e-30 and +-20 / +-100 tails.  dt = 1, so dz = act'(z)."""
    R, D = 4, 64
    z = (np.random.default_rng(5).standard_normal((R, D)) * 3).astype(np.float32)
    z[:, :8] = np.array([0.0, -0.0, 1e-30, -1e-30, 20.0, -20.0, 100.0, -100.0], np.float32)
    dt = np.ones((R, D), np.float32)
    got = _run_layer(act, False, z, None, None, dt, R, 0)
    assert np.isfinite(got["out"]).all() and np.isfinite(got["dz"]).all()       # e.g. swish(-100) = -0, not NaN
    np.testing.assert_array_equal(got["dz"][:, :2], ACT_GRAD_AT_0[act])
    at_tiny = {"relu": [1.0, 0.0], "leaky_relu": [1.0, 0.01]}.get(act, [ACT_GRAD_AT_0[act]] * 2)    # at +-1e-30
    np.testing.assert_allclose(got["dz"][:, 2:4], [at_tiny] * R, rtol=1e-6)
    if act in KINKED:
        np.testing.assert_array_equal(*_gates(act, got, dt, False))
    _check_layer(act, False, got, _layer_ref(act, False, z, None, None, dt, R))


@pytest.mark.parametrize("D", [64, 1024])
@pytest.mark.parametrize("act", ACTS)
def test_layer_norm_statistics_stress_rows(act, D):
    """A constant row of an exactly representable value (its fp32 sums are exact: var = 0, rstd = 1/sqrt(eps)) and a row whose
    mean sits ~4 sigma off 0 (E[x^2] - E[x]^2 cancels ~17:1; emulating the kernel's fp32 sums puts xhat within ~2e-6)."""
    rng = np.random.default_rng(6)
    z = np.stack([np.full(D, 0.5), 4.0 + rng.standard_normal(D)]).astype(np.float32)
    sc, bi = (1 + 0.2 * rng.standard_normal((1, D))).astype(np.float32), (0.1 * rng.standard_normal((1, D))).astype(np.float32)
    dt = rng.standard_normal((2, D)).astype(np.float32)
    got = _run_layer(act, True, z, sc, bi, dt, 2, 0)
    np.testing.assert_array_equal(got["xhat"][0], 0.0)
    np.testing.assert_allclose(got["rstd"][0], 1.0 / np.sqrt(np.float64(np.float32(LN_EPS))), rtol=2.5e-7)   # rsqrtf: 2 ulp
    ref = _layer_ref(act, True, z, sc, bi, dt, 2, gate=_gates(act, got, dt, True)[0])
    for r in range(2):                  # row by row: the constant row's dz is ~1/sqrt(eps) = 1000 times the other's
        _check_layer(act, True, got, ref, rows=r)


@pytest.mark.parametrize("act", KINKED)
def test_layer_kink_branch_agrees_between_fwd_and_bwd(act):
    """The backward recomputes y = xhat * scale + bias; the forward has y in a register.  With bias = -fp32(xhat * scale) on one
    row, its pre-activations sit within rounding of 0, and both passes must still take the same branch at every unit."""
    E, B, D, r0 = 10, 13, 192, 14       # row 14: member 1, in the CTA of rows 8..15 that straddles members 0 and 1
    z, sc, bi, dt = _layer_inputs(E, B, D, seed=12)
    first = _run_layer(act, True, z, sc, bi, dt, B, D)
    g0 = r0 // B
    bi = bi.copy()
    bi[g0] = -(first["xhat"][r0] * sc[g0])
    got = _run_layer(act, True, z, sc, bi, dt, B, D)
    np.testing.assert_array_equal(got["xhat"], first["xhat"])
    assert np.abs(got["out"][r0]).max() < 1e-5
    fwd_gate, bwd_gate = _gates(act, got, dt, True)
    np.testing.assert_array_equal(fwd_gate, bwd_gate)
    _check_layer(act, True, got, _layer_ref(act, True, z, sc, bi, dt, B, gate=fwd_gate))


# ---- serl_layernorm_param_grad, serl_colsum_f32 -------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 1024])
@pytest.mark.parametrize("B", [13, 256])
@pytest.mark.parametrize("E", [1, 10])
def test_layernorm_param_grad(E, B, D):
    from serl_b200 import ops
    rng = np.random.default_rng(E + B + D)
    dy, xhat = rng.standard_normal((2, E * B, D)).astype(np.float32)
    dyd, xd = cu(dy), cu(xhat)
    outs = []
    for _ in range(2):
        dsc, dbi = _tail(E * D), _tail(E * D)
        ops.ln_param_grad(dyd.data_ptr(), xd.data_ptr(), dsc.data_ptr(), dbi.data_ptr(), B, E * B, D)
        outs.append((host(dsc), host(dbi)))
    for k in range(2):                  # fixed summation order: bitwise repeatable
        np.testing.assert_array_equal(outs[0][k], outs[1][k])
        np.testing.assert_array_equal(outs[0][k][E * D:], SENTINEL)
    dyr, xr = f64(dy).view(E, B, D), f64(xhat).view(E, B, D)
    assert rel_err(outs[0][0][:E * D].reshape(E, D), (dyr * xr).sum(1).numpy()) < TOL
    assert rel_err(outs[0][1][:E * D].reshape(E, D), dyr.sum(1).numpy()) < TOL


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("groups,rows,D,ld", [
    (10, 13, 1, 1),             # per-member value-head bias
    (1, 2560, 1, 1),            # the pixel critic's shared value head
    (1, 256, 4, 4),             # log_stds / Dense_1 bias
    (10, 256, 1024, 1024),
    (1, 7, 64, 100),            # ld > D
])
def test_colsum(groups, rows, D, ld, accumulate):
    from serl_b200 import ops
    rng = np.random.default_rng(groups * rows + D)
    x = rng.standard_normal((groups * rows, D)).astype(np.float32)
    out0 = rng.standard_normal(groups * D).astype(np.float32)
    xd = _padded(x, ld, np.nan)
    outs = []
    for _ in range(2):
        out = _tail(groups * D)
        out[:groups * D] = cu(out0)
        ops.colsum(xd.data_ptr(), out.data_ptr(), groups, rows, D, ld, accumulate)
        outs.append(host(out))
    np.testing.assert_array_equal(outs[0], outs[1])                             # fixed summation order
    np.testing.assert_array_equal(outs[0][groups * D:], SENTINEL)
    ref = f64(x).view(groups, rows, D).sum(1).numpy().ravel() + (out0 if accumulate else 0.0)
    assert rel_err(outs[0][:groups * D], ref) < TOL


# ---- policy std heads: serl_tanh_gaussian_fwd[_std], serl_actor_loss[_std] ----------------------------------------------
def _raw_std(head, x):
    return F.softplus(x) if head == "softplus" else torch.exp(x)


def _std_ref(head, x, B, A):
    """actor_critic_nets.py's std heads: clip(exp(x) | softplus(x) | exp(log_stds) broadcast over the rows, std_min, std_max)"""
    return torch.clamp(_raw_std(head, x), STD_MIN, STD_MAX).expand(B, A)


def _head_input(head, rng, B, A):
    """The std head's output x: one (A,) leaf for "uniform", a (B, A) head output otherwise; entries below std_min and above
    std_max, and none within 1 % of a clip bound (exact ties are out of scope: DESIGN.md section 5)."""
    if head == "uniform":
        x = np.array([-14.0, 2.0, 0.3, -1.2, 1.1, -0.4, 0.7], np.float32)[:A]
    else:
        x = (rng.standard_normal((B, A)) * (3.0 if head == "softplus" else 1.5)).astype(np.float32)
        lo, hi = (-30.0, 10.0) if head == "softplus" else (-14.0, 2.0)
        x[0, 0] = x[B // 2, 3] = lo
        x[1, 1] = x[B - 1, A - 1] = hi
    raw = _raw_std(head, f64(x)).numpy()
    x[(np.abs(raw / STD_MIN - 1) < 0.01) | (np.abs(raw / STD_MAX - 1) < 0.01)] = 0.0
    raw = _raw_std(head, f64(x)).numpy()
    assert (raw < STD_MIN).any() and (raw > STD_MAX).any()
    return x


def _sample(head, mu, x, eps, act_addr, ld_act, logp, u, sd, B, A):
    """the forward the engine runs: act written at act_addr with row stride ld_act"""
    from serl_b200 import ops
    det = eps is None
    if head == "exp":
        ops.tanh_gaussian_fwd(mu, x, eps, STD_MIN, STD_MAX, act_addr, ld_act, logp, u, sd, B, A, deterministic=det)
    else:
        ops.tanh_gaussian_fwd_std(mu, x.data_ptr(), 0 if head == "uniform" else A, _std_id(head), eps, STD_MIN, STD_MAX, act_addr, ld_act,
                                  logp, u, sd, B, A, deterministic=det)


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("head", HEADS)
def test_tanh_gaussian_std_heads(head, deterministic):
    """B = 300 rows (three CTAs); act lands at column Fo of rows Fo + A wide, as in the critic's input."""
    from serl_b200 import ops
    rng = np.random.default_rng(HEADS.index(head))
    B, A, Fo = 300, 7, 40
    mu = rng.standard_normal((B, A)).astype(np.float32)
    x = _head_input(head, rng, B, A)
    eps = np.zeros((B, A), np.float32) if deterministic else rng.standard_normal((B, A)).astype(np.float32)
    act = torch.full((B, Fo + A), SENTINEL, device="cuda")
    logp, u, sd = _tail(B), _tail(B * A), _tail(B * A)
    _sample(head, cu(mu), cu(x), None if deterministic else cu(eps), ops.at(act, Fo), Fo + A, logp, u, sd, B, A)
    std = _std_ref(head, f64(x), B, A)
    a_ref, lp_ref = tanh_normal_sample_logp(f64(mu), std, f64(eps))
    got_a = host(act)
    np.testing.assert_array_equal(got_a[:, :Fo], SENTINEL)
    for t, n in ((logp, B), (u, B * A), (sd, B * A)):
        np.testing.assert_array_equal(host(t)[n:], SENTINEL)
    assert rel_err(got_a[:, Fo:], a_ref.numpy()) < TOL
    if deterministic:
        np.testing.assert_allclose(got_a[:, Fo:], np.tanh(mu.astype(np.float64)), rtol=0, atol=1e-6)
    np.testing.assert_allclose(host(sd)[:B * A].reshape(B, A), std.numpy(), rtol=1e-6)
    u_ref = (f64(mu) + std * f64(eps)).numpy()
    assert rel_err(host(u)[:B * A].reshape(B, A), u_ref) < TOL
    # z = (u - mu) / std recovers eps after u = mu + std * eps was rounded to fp32 (distrax does the same in JAX's float32):
    # that rounding (<= 2^-24 |u|) moves z by up to 2^-24 |u| / std and -z^2/2 by |z| times that, which is large on the std_min
    # clip (see test_ops_gpu.test_tanh_gaussian_and_losses) and for any small std.  Each row gets that term (x4) on top of the
    # usual bar (rows with std ~ 1 keep it: their term is ~1e-7); with eps = 0 nothing cancels.
    lp, lpr = host(logp)[:B], lp_ref.numpy()
    cancel = 2.0 ** -22 * (np.abs(eps) * np.abs(u_ref) / std.numpy()).sum(1)
    assert (np.abs(lp - lpr) <= TOL * np.abs(lpr).max() + cancel).all()


@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
@pytest.mark.parametrize("B", [64, 1100])
@pytest.mark.parametrize("head", HEADS)
def test_actor_loss_std_heads(head, B, grad_scale):
    """Gradients w.r.t. mu and the std head's output x against float64 autograd of
        L = grad_scale * (alpha / B) * sum_b logp_b + sum_{b,i} da[b,i] * a[b,i]
    (a, logp from mu, x and eps through the clipped std head; da stands in for the critic's input gradient), and the infos.
    One CTA of 1024 threads: B = 1100 loops.  da / act at the engine's strided addresses."""
    from serl_b200 import ops
    rng = np.random.default_rng(B + HEADS.index(head))
    E, A, Fo = 10, 7, 40
    mu = rng.standard_normal((B, A)).astype(np.float32)
    x = _head_input(head, rng, B, A)
    eps = rng.standard_normal((B, A)).astype(np.float32)
    q = (rng.standard_normal((E, B)) + 0.5).astype(np.float32)
    da = (rng.standard_normal((B, A)) / B).astype(np.float32)
    lam = np.array([-2.0], np.float32)
    mud, xd, epsd, lamd = cu(mu), cu(x), cu(eps), cu(lam)
    act = torch.full((B, Fo + A), SENTINEL, device="cuda")
    logp, u, sd = torch.empty(B, device="cuda"), torch.empty(B, A, device="cuda"), torch.empty(B, A, device="cuda")
    _sample(head, mud, xd, epsd, ops.at(act, Fo), Fo + A, logp, u, sd, B, A)
    dad = cu(np.concatenate([np.full((B, Fo), np.nan, np.float32), da], 1))
    dmu, dx, info = _tail(B * A), _tail(B * A), _tail(3)
    if head == "exp":
        ops.actor_loss(cu(q), logp, lamd.data_ptr(), ops.at(dad, Fo), Fo + A, ops.at(act, Fo), Fo + A, sd, xd, epsd, STD_MIN, STD_MAX,
                       grad_scale, dmu, dx, info.data_ptr(), E, B, A)
    else:
        ops.actor_loss_std(cu(q), logp, lamd.data_ptr(), ops.at(dad, Fo), Fo + A, ops.at(act, Fo), Fo + A, sd, xd.data_ptr(),
                           0 if head == "uniform" else A, _std_id(head), epsd, STD_MIN, STD_MAX, grad_scale, dmu, dx, info.data_ptr(), E, B, A)
    mut = f64(mu).requires_grad_(True)
    leaf = f64(x).requires_grad_(True)
    xt = leaf.expand(B, A) if head == "uniform" else leaf
    if head == "uniform":
        xt.retain_grad()                # per-row gradient of the broadcast leaf: what the kernel writes to dx
    a, lp = tanh_normal_sample_logp(mut, _std_ref(head, xt, B, A), f64(eps))
    alpha = F.softplus(f64(lam)[0])
    (grad_scale * (alpha / B) * lp.sum() + (f64(da) * a).sum()).backward()
    for t, n in ((dmu, B * A), (dx, B * A), (info, 3)):
        np.testing.assert_array_equal(host(t)[n:], SENTINEL)
    got_dx = host(dx)[:B * A].reshape(B, A)
    assert rel_err(host(dmu)[:B * A].reshape(B, A), mut.grad.numpy()) < TOL
    assert rel_err(got_dx, xt.grad.numpy()) < TOL
    raw = _raw_std(head, f64(x)).expand(B, A).numpy()
    assert (got_dx[(raw < STD_MIN) | (raw > STD_MAX)] == 0).all()            # a clipped std passes no gradient
    if head == "uniform":               # the log_stds gradient exactly as engine.policy_backward forms it
        g = _tail(A)
        ops.colsum(dx.data_ptr(), g.data_ptr(), 1, B, A, A)
        assert rel_err(host(g)[:A], leaf.grad.numpy()) < TOL
    lpk, qbar = f64(host(logp)), f64(q).mean(0)         # the infos are functions of the kernel's inputs q, logp, lagrange
    ref = grad_scale * torch.stack([-(qbar - alpha * lpk).mean(), alpha, -lpk.mean()])
    np.testing.assert_allclose(host(info)[:3], ref.numpy(), rtol=TOL)


# ---- serl_critic_loss -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sub,backup_entropy,grad_scale,B", [
    ((), False, 1.0, 1100),         # n_sub = 0: the minimum over the whole ensemble (critic_subsample_size=None)
    ((), True, 0.5, 256),
    ((4,), False, 0.5, 256),
    ((3, 3), True, 1.0, 1100),      # subsample with replacement: repeated indices
    ((7, 2), False, 0.5, 64),
])
def test_critic_loss_branches(sub, backup_entropy, grad_scale, B):
    from serl_b200 import ops
    E, gamma = 10, 0.96
    rng = np.random.default_rng(B + len(sub))
    q = (rng.standard_normal((E, B)) * 0.5 + 1.0).astype(np.float32)
    qn = (rng.standard_normal((E, B)) * 0.5 + 1.0).astype(np.float32)
    r, m = (rng.random(B) + 0.5).astype(np.float32), (rng.random(B) > 0.1).astype(np.float32)
    logp_n = (rng.standard_normal(B) - 3.0).astype(np.float32)
    lam = np.array([-1.0], np.float32)
    lamd, tq, dq, info = cu(lam), _tail(B), _tail(E * B), _tail(3)
    ops.critic_loss(cu(q), cu(qn), cu(np.array(sub or (0, 0), np.int32), torch.int32), len(sub), cu(r), cu(m), cu(logp_n), lamd.data_ptr(),
                    backup_entropy, gamma, grad_scale, tq, dq, info.data_ptr(), E, B)
    qn64 = f64(qn)
    y = f64(r) + gamma * f64(m) * (qn64[list(sub)] if sub else qn64).min(0).values
    if backup_entropy:
        y = y - F.softplus(f64(lam)[0]) * f64(logp_n)
    d = f64(q) - y
    for t, n in ((tq, B), (dq, E * B), (info, 3)):
        np.testing.assert_array_equal(host(t)[n:], SENTINEL)
    assert rel_err(host(tq)[:B], y.numpy()) < TOL
    assert rel_err(host(dq)[:E * B].reshape(E, B), (2 * d / (E * B) * grad_scale).numpy()) < TOL
    ref = grad_scale * torch.stack([(d * d).mean(), f64(q).mean(), y.mean()])
    np.testing.assert_allclose(host(info)[:3], ref.numpy(), rtol=TOL)


# ---- behaviour cloning and small helpers ----------------------------------------------------------------------------------
@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
def test_bc_loss(grad_scale):
    """-grad_scale * mean_b log N(a_b; mu_b, diag(clip(exp(log_std))^2)): dmu, dlog_std and {loss, mse} * grad_scale."""
    from serl_b200 import _lib as L
    rng = np.random.default_rng(8)
    B, A = 1100, 7
    mu = rng.standard_normal((B, A)).astype(np.float32)
    ls = _head_input("exp", rng, B, A)
    sd32 = np.clip(np.exp(ls.astype(np.float64)), STD_MIN, STD_MAX).astype(np.float32)
    act = (mu + sd32 * (0.8 * rng.standard_normal((B, A))).astype(np.float32)).astype(np.float32)
    mud, lsd, actd = cu(mu), cu(ls), cu(act)
    dmu, dls, info = _tail(B * A), _tail(B * A), _tail(2)
    L.call("serl_bc_loss", mud.data_ptr(), lsd.data_ptr(), actd.data_ptr(), STD_MIN, STD_MAX, grad_scale, dmu.data_ptr(),
           dls.data_ptr(), info.data_ptr(), B, A, L.stream_ptr())
    mut, lst = f64(mu).requires_grad_(True), f64(ls).requires_grad_(True)
    std = torch.clamp(torch.exp(lst), STD_MIN, STD_MAX)
    logp = torch.distributions.Normal(mut, std).log_prob(f64(act)).sum(-1)
    loss = -grad_scale * logp.mean()
    loss.backward()
    for t, n in ((dmu, B * A), (dls, B * A), (info, 2)):
        np.testing.assert_array_equal(host(t)[n:], SENTINEL)
    got_dmu = host(dmu)[:B * A].reshape(B, A)
    low = np.exp(ls.astype(np.float64)) < STD_MIN          # 1/std^2 = 1e10 there: compared apart so they do not set the scale
    for sel in (low, ~low):
        assert rel_err(got_dmu[sel], mut.grad.numpy()[sel]) < TOL
    assert rel_err(host(dls)[:B * A].reshape(B, A), lst.grad.numpy()) < TOL
    mse = grad_scale * ((f64(act) - f64(mu)) ** 2).sum(-1).mean()
    np.testing.assert_allclose(host(info)[:2], [loss.item(), mse.item()], rtol=TOL)


@pytest.mark.parametrize("n", [1, 1000, 65537])
def test_tanh_fwd_bwd(n):
    from serl_b200 import _lib as L
    rng = np.random.default_rng(n)
    z, dt = (rng.standard_normal(n) * 2).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    zd, dtd, out, dz = cu(z), cu(dt), _tail(n), _tail(n)
    L.call("serl_tanh_fwd", zd.data_ptr(), out.data_ptr(), n, L.stream_ptr())
    L.call("serl_tanh_bwd", dtd.data_ptr(), out.data_ptr(), dz.data_ptr(), n, L.stream_ptr())
    zt = f64(z).requires_grad_(True)
    t = torch.tanh(zt)
    t.backward(f64(dt))
    for g in (out, dz):
        np.testing.assert_array_equal(host(g)[n:], SENTINEL)
    assert rel_err(host(out)[:n], t.detach().numpy()) < TOL
    assert rel_err(host(dz)[:n], zt.grad.numpy()) < TOL


@pytest.mark.parametrize("R,D,ld_src,ld_dst,col", [(37, 7, 13, 47, 40), (2000, 300, 301, 333, 16)])
def test_copy2d_strided(R, D, ld_src, ld_dst, col):
    """e.g. the actions into the critic input at column F (rows F + A wide); 600k elements exceed one pass of the capped grid"""
    from serl_b200 import ops
    src = np.random.default_rng(R).standard_normal((R, D)).astype(np.float32)
    srcd, dst = _padded(src, ld_src, np.nan), torch.full((R, ld_dst), SENTINEL, device="cuda")
    ops.copy2d(srcd.data_ptr(), ld_src, ops.at(dst, col), ld_dst, R, D)
    got = host(dst)
    np.testing.assert_array_equal(got[:, col:col + D], src)
    np.testing.assert_array_equal(np.delete(got, np.s_[col:col + D], axis=1), SENTINEL)


@pytest.mark.parametrize("n", [1, 2560, 11000])
def test_fill(n):
    from serl_b200 import ops
    x, v = _tail(n), -0.5 / 2560
    ops.fill(x.data_ptr(), v, n)
    got = host(x)
    np.testing.assert_array_equal(got[:n], np.float32(v))
    np.testing.assert_array_equal(got[n:], SENTINEL)
