"""CPU: the references tests/test_vice_ops_gpu.py holds the VICE kernels to.  The permutation keys chosen for their ties really
tie in the first sort round at N = 2048, and vice_oracle.permutation keeps tied rows in index order (the stable rank sort of
vice_draws_kernel); the float64 LayerNorm + activation function, its forward-mode tangent and the reverse-mode gradients taken
through that tangent agree with central finite differences, at both activations and with dropout masks."""
import numpy as np
import pytest
import torch

import vice_oracle as V
from oracle import jax_prng as P

TIE_KEYS = ((0, 17220), (0, 19942), (0, 27595))


def _rank_sort(x, bits):
    """One round as vice_draws_kernel computes it: row i goes to rank #{bits < b_i} + #{j < i: bits_j == b_i}."""
    b = bits.astype(np.int64)
    n = b.size
    less = (b[None, :] < b[:, None]).sum(1)
    tie_before = ((b[None, :] == b[:, None]) & (np.arange(n)[None, :] < np.arange(n)[:, None])).sum(1)
    out = np.empty_like(x)
    out[less + tie_before] = x
    return out


@pytest.mark.parametrize("key", TIE_KEYS)
def test_tie_keys_tie_in_round_one_and_sort_stably(key):
    from serl_b200.agents.continuous.vice import permutation_rounds
    N = 2048
    k = np.array(key, np.uint32)
    assert permutation_rounds(N) == 2
    k2, sub = P.split(k)
    bits = P.random_bits(sub, (N,))
    vals, counts = np.unique(bits, return_counts=True)
    tied = vals[counts > 1]
    assert tied.size >= 1
    x1 = _rank_sort(np.arange(N), bits)
    for v in tied:                                          # tied rows keep their index order after round 1
        rows = np.flatnonzero(bits == v)
        pos = [int(np.flatnonzero(x1 == r)[0]) for r in rows]
        assert pos == sorted(pos) and np.all(np.diff(pos) == 1)
    x2 = _rank_sort(x1, P.random_bits(P.split(k2)[1], (N,)))
    assert np.array_equal(V.permutation(k, N), x2)
    # the reverse tie-break gives another permutation: only a key with a tie tells the two apart
    x1r = x1.copy()
    for v in tied:
        idx = [int(np.flatnonzero(x1 == r)[0]) for r in np.flatnonzero(bits == v)]
        x1r[idx] = x1[idx][::-1]
    assert not np.array_equal(_rank_sort(x1r, P.random_bits(P.split(k2)[1], (N,))), x2)


def test_rank_sort_restates_permutation():
    from serl_b200.agents.continuous.vice import permutation_rounds
    for n in (2, 16, 1624, 1626):
        k = P.split(np.array([3, n], np.uint32))[0]
        x, key = np.arange(n), k
        for _ in range(permutation_rounds(n)):
            key, sub = P.split(key)
            x = _rank_sort(x, P.random_bits(sub, (n,)))
        assert np.array_equal(V.permutation(k, n), x), n


def _fd(f, x, v, h=1e-5):
    return (f(x + h * v) - f(x - h * v)) / (2 * h)


@pytest.mark.parametrize("act", ["tanh", "leaky_relu"])
@pytest.mark.parametrize("masked", [False, True])
def test_ln_act_tangent_and_gradients_match_finite_differences(act, masked):
    rng = np.random.default_rng(7)
    R, D = 3, 256
    t = lambda *s, s0=1.0: torch.as_tensor(s0 * rng.standard_normal(s), dtype=torch.float64)
    z, zdot, pb = t(R, D, s0=1.5) + 0.2, t(R, D), t(D, s0=0.1)
    scale, bias = 1 + t(R, D, s0=0.3), t(R, D, s0=0.2)                   # one parameter row per input row
    mask = rng.random((R, D)) < 0.9 if masked else None
    ybar, ydotbar = t(R, D), t(R, D)
    y, ydot = V.ln_act_jvp(z, zdot, scale, bias, act, mask, pb)
    f = lambda zz: V.ln_act(zz, scale, bias, act, mask, pb)
    assert torch.allclose(y, f(z), rtol=0, atol=1e-14)
    fd = _fd(f, z, zdot)
    assert float((ydot - fd).abs().max()) <= 1e-7 * float(fd.abs().max())

    leaves = [x.clone().requires_grad_(True) for x in (z, zdot, scale, bias)]

    def objective(zz, zd, sc, bi):
        yy, yd = V.ln_act_jvp(zz, zd, sc, bi, act, mask, pb)
        return (ybar * yy).sum() + (ydotbar * yd).sum()

    grads = torch.autograd.grad(objective(*leaves), leaves)
    base = [x.detach() for x in leaves]
    for i, g in enumerate(grads):
        for _ in range(2):
            v = t(*base[i].shape)
            with torch.no_grad():
                fd = _fd(lambda xi: objective(*[xi if j == i else base[j] for j in range(4)]), base[i], v)
            got = float((g * v).sum())
            assert abs(got - float(fd)) <= 1e-6 * max(1.0, abs(float(fd))), (i, got, float(fd))
    if masked:                                              # dropped units get no gradient in the primal or the tangent
        assert float(grads[0][torch.as_tensor(~mask)].abs().max()) == 0.0
        assert float(grads[1][torch.as_tensor(~mask)].abs().max()) == 0.0


def test_leaky_relu_slope_at_zero_is_one():
    u = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    (g,) = torch.autograd.grad(V.act("leaky_relu", u).sum(), [u])
    assert torch.equal(g, torch.ones(3, dtype=torch.float64))
