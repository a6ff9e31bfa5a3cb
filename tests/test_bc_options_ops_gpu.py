"""GPU: the kernels BC's options added, op by op through the C-ABI against float64 autograd on the same fp32 inputs, at the bars of
tests/test_mlp_policy_ops_gpu.py (2e-5 forward values and reductions, 5e-5 LayerNorm backward outputs):
serl_bc_loss_std for every std head with and without the tanh squash, serl_ln_act_dropout_fwd / _bwd for every (activation,
LayerNorm) pair, and serl_bc_loss bitwise equal to serl_bc_loss_std's <exp, no squash> instantiation."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from arch_oracle import ACTIVATIONS
from helpers import rel_err
from oracle.drq import layer_norm

pytestmark = pytest.mark.gpu
TOL, LN_BWD_TOL = 2e-5, 5e-5
LN_EPS = 1e-6
ACTS = ("tanh", "relu", "swish", "leaky_relu", "gelu")
HEADS = ("exp", "softplus", "uniform")
SENTINEL = -1234.5
TAIL = 64
STD_MIN, STD_MAX = 1e-5, 5.0


def cu(x, dt=torch.float32):
    return torch.as_tensor(np.asarray(x)).to("cuda", dt).contiguous()


def f64(x):
    return torch.as_tensor(np.asarray(x)).double()


def host(t):
    return t.cpu().numpy()


def _tail(n):
    return torch.full((n + TAIL,), SENTINEL, device="cuda")


def _raw_std(head, x):
    return F.softplus(x) if head == "softplus" else torch.exp(x)


def _head_input(head, rng, B, A):
    """The std head's output: (A,) for "uniform", (B, A) otherwise; entries on both sides of the clip, none within 1 % of a bound
    (clip ties: DESIGN.md section 5)."""
    if head == "uniform":
        x = np.array([-14.0, 2.0, 0.3, -1.2, 1.1, -0.4, 0.7], np.float32)[:A]
    else:
        x = (rng.standard_normal((B, A)) * (3.0 if head == "softplus" else 1.5)).astype(np.float32)
        lo, hi = (-30.0, 10.0) if head == "softplus" else (-14.0, 2.0)
        x[0, 0] = x[B // 2, 3] = lo
        x[1, 1] = x[B - 1, A - 1] = hi
    raw = _raw_std(head, f64(x)).numpy()
    x[(np.abs(raw / STD_MIN - 1) < 0.01) | (np.abs(raw / STD_MAX - 1) < 0.01)] = 0.0
    return x


def _bc_loss_std(L, head, squash, mud, xd, actd, grad_scale, B, A):
    dmu, dx, info = _tail(B * A), _tail(B * A), _tail(2)
    L.call("serl_bc_loss_std", mud.data_ptr(), xd.data_ptr(), 0 if head == "uniform" else A, getattr(L, "STD_" + head.upper()), int(squash),
           actd.data_ptr(), STD_MIN, STD_MAX, grad_scale, dmu.data_ptr(), dx.data_ptr(), info.data_ptr(), B, A, L.stream_ptr())
    return dmu, dx, info


@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
@pytest.mark.parametrize("B", [2, 1100])
@pytest.mark.parametrize("squash", [False, True])
@pytest.mark.parametrize("head", HEADS)
def test_bc_loss_std(head, squash, B, grad_scale):
    """-grad_scale * mean_b log pi(a_b) and grad_scale * mean_b sum (mode_b - a_b)^2 with their gradients w.r.t. mu and the std
    head's output (per row; "uniform": the column sum is the leaf's).  The squashed NLL is checked against torch's
    TransformedDistribution(Normal, TanhTransform).  One CTA of 1024 threads: B = 1100 loops."""
    from serl_b200 import _lib as L
    from serl_b200 import ops
    rng = np.random.default_rng(B + 10 * HEADS.index(head) + squash)
    A = 7
    mu = (rng.standard_normal((B, A)) * (0.5 if squash else 1.0)).astype(np.float32)
    x = _head_input(head, rng, B, A)
    sd32 = np.clip(_raw_std(head, f64(x)).numpy(), STD_MIN, STD_MAX)
    # squashed: u = atanhf(a) carries about an ulp of |u| <= 2, which (u - mu) / std^2 amplifies where the std is clipped to std_min;
    # a spread of at least 0.1 keeps u - mu well away from 0 there (DESIGN.md section 5)
    spread = np.maximum(sd32, 0.1) if squash else sd32
    u = mu + np.broadcast_to(spread, (B, A)) * 0.8 * rng.standard_normal((B, A))
    act = (np.tanh(np.clip(u, -2, 2)) if squash else u).astype(np.float32)
    dmu, dx, info = _bc_loss_std(L, head, squash, cu(mu), cu(x), cu(act), grad_scale, B, A)
    mut, leaf = f64(mu).requires_grad_(True), f64(x).requires_grad_(True)
    xt = leaf.expand(B, A) if head == "uniform" else leaf
    if head == "uniform":
        xt.retain_grad()
    std = torch.clamp(_raw_std(head, xt), STD_MIN, STD_MAX)
    base = torch.distributions.Normal(mut, std)
    dist = torch.distributions.TransformedDistribution(base, [torch.distributions.TanhTransform()]) if squash else base
    a64 = f64(act)
    logp = dist.log_prob(a64).sum(-1)
    loss = -grad_scale * logp.mean()
    loss.backward()
    for t, n in ((dmu, B * A), (dx, B * A), (info, 2)):
        np.testing.assert_array_equal(host(t)[n:], SENTINEL)
    got_dmu, got_dx = host(dmu)[:B * A].reshape(B, A), host(dx)[:B * A].reshape(B, A)
    low = np.broadcast_to(_raw_std(head, f64(x)).numpy(), (B, A)) < STD_MIN     # 1/std^2 = 1e10 there: compared apart
    for sel in (low, ~low):
        if sel.any():
            assert rel_err(got_dmu[sel], mut.grad.numpy()[sel]) < TOL
    assert rel_err(got_dx, xt.grad.numpy()) < TOL
    raw = np.broadcast_to(_raw_std(head, f64(x)).numpy(), (B, A))
    assert (got_dx[(raw < STD_MIN) | (raw > STD_MAX)] == 0).all()
    if head == "uniform":
        g = _tail(A)
        ops.colsum(dx.data_ptr(), g.data_ptr(), 1, B, A, A)
        assert rel_err(host(g)[:A], leaf.grad.numpy()) < TOL
    mode = torch.tanh(f64(mu)) if squash else f64(mu)
    mse = grad_scale * ((mode - a64) ** 2).sum(-1).mean()
    np.testing.assert_allclose(host(info)[:2], [loss.item(), mse.item()], rtol=TOL)


@pytest.mark.parametrize("B", [2, 1100])
def test_bc_loss_is_the_exp_instantiation(B):
    """serl_bc_loss (the launcher's entry point) and serl_bc_loss_std(exp, no squash) give the same bits."""
    from serl_b200 import _lib as L
    rng = np.random.default_rng(B)
    A = 7
    mu, ls = rng.standard_normal((B, A)).astype(np.float32), _head_input("exp", rng, B, A)
    act = (mu + rng.standard_normal((B, A))).astype(np.float32)
    mud, lsd, actd = cu(mu), cu(ls), cu(act)
    dmu, dls, info = _tail(B * A), _tail(B * A), _tail(2)
    L.call("serl_bc_loss", mud.data_ptr(), lsd.data_ptr(), actd.data_ptr(), STD_MIN, STD_MAX, 0.5, dmu.data_ptr(), dls.data_ptr(),
           info.data_ptr(), B, A, L.stream_ptr())
    for got, ref in zip(_bc_loss_std(L, "exp", False, mud, lsd, actd, 0.5, B, A), (dmu, dls, info)):
        assert torch.equal(got, ref)


# ---- serl_ln_act_dropout_fwd / _bwd ---------------------------------------------------------------------------------------
def _gate_ref(act, y, gate):
    if gate is None or act not in ("relu", "leaky_relu"):
        return ACTIVATIONS[act](y)
    one = torch.ones((), dtype=torch.float64)
    return y * torch.where(torch.as_tensor(gate), ACTIVATIONS[act](one), -ACTIVATIONS[act](-one))


@pytest.mark.parametrize("rate", [0.1, 0.5])
@pytest.mark.parametrize("R,D", [(13, 64), (256, 512), (100, 192)])
@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("act", ACTS)
def test_ln_act_dropout_fwd_bwd(act, ln, R, D, rate):
    """Dropout -> [LayerNorm] -> act on the policy's call shape (group_stride 0), then the backward on the forward's own out, xhat,
    rstd and (without LayerNorm) the dropped-out z written back in place; the masks come from serl_dropout_mask_fill."""
    from serl_b200 import _lib as L
    from serl_b200 import ops
    rng = np.random.default_rng(R + D + ACTS.index(act))
    z = (rng.standard_normal((R, D)) * 2 + 0.3).astype(np.float32)
    sc, bi = (1 + 0.2 * rng.standard_normal((1, D))).astype(np.float32), (0.1 * rng.standard_normal((1, D))).astype(np.float32)
    dt = rng.standard_normal((R, D)).astype(np.float32)
    key = cu(np.array([7, R * D], np.uint32).view(np.int32), torch.int32)
    mask = torch.empty(R, D, dtype=torch.uint8, device="cuda")
    ops.dropout_mask_fill(key.data_ptr(), 3, 1.0 - rate, mask, R * D)
    m = host(mask).astype(bool)
    assert 0 < m.mean() < 1
    zd, dtd = cu(z), cu(dt)
    scd, bid = cu(sc), cu(bi)
    out, xhat, rstd, dz, dy = _tail(R * D), _tail(R * D), _tail(R), _tail(R * D), _tail(R * D)
    a = getattr(L, "ACT_" + act.upper())
    inv_keep = 1.0 / (1.0 - rate)
    ops.ln_act_dropout_fwd(zd.data_ptr(), D, scd.data_ptr() if ln else None, bid.data_ptr() if ln else None, R, 0, mask, inv_keep,
                           out.data_ptr(), D, xhat.data_ptr(), rstd.data_ptr(), R, D, a, ln, LN_EPS)
    ops.ln_act_dropout_bwd(dtd.data_ptr(), D, out.data_ptr(), D, zd.data_ptr(), D, xhat.data_ptr(), rstd.data_ptr(),
                           scd.data_ptr() if ln else None, bid.data_ptr() if ln else None, R, 0, mask, inv_keep, dz.data_ptr(), dy.data_ptr(),
                           R, D, a, ln)
    for t, n in ((out, R * D), (xhat, R * D), (rstd, R), (dz, R * D), (dy, R * D)):
        np.testing.assert_array_equal(host(t)[n:], SENTINEL)
    zt = f64(z).requires_grad_(True)
    zm = torch.where(torch.as_tensor(m), zt * inv_keep, torch.zeros_like(zt))
    if ln:
        np.testing.assert_array_equal(host(zd), z)                                   # z itself is left alone
        y = layer_norm(zm, f64(sc), f64(bi))
    else:
        # the dropped-out z written back in place: z * fp32(1 / keep), one fp32 rounding, bit for bit
        np.testing.assert_array_equal(host(zd), np.where(m, z * np.float32(inv_keep), np.float32(0)))
        y = zm
    y.retain_grad()
    got_out = host(out)[:R * D].reshape(R, D)
    gate = (got_out > 0) if act == "relu" else (got_out >= 0)
    h = _gate_ref(act, y, gate)
    h.backward(f64(dt))
    assert rel_err(got_out, h.detach().numpy()) < TOL
    got_dz = host(dz)[:R * D].reshape(R, D)
    assert (got_dz[~m] == 0).all()
    if ln:
        assert rel_err(host(xhat)[:R * D].reshape(R, D), layer_norm(zm.detach(), 1.0, 0.0).numpy()) < TOL
        assert rel_err(host(dy)[:R * D].reshape(R, D), y.grad.numpy()) < LN_BWD_TOL
        assert rel_err(got_dz, zt.grad.numpy()) < LN_BWD_TOL
    else:
        assert rel_err(got_dz, zt.grad.numpy()) < TOL
