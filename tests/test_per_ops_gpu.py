"""GPU: serl_critic_loss_weighted (prioritized replay's importance-weighted critic loss) against float64, and bit for bit against
serl_critic_loss when every weight is 1."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _case(E, B, seed, n_sub=0):
    rng = np.random.default_rng(seed)
    f = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32)).cuda()
    q, q_next, rewards = f(E, B), f(E, B), f(B)
    masks = torch.from_numpy((rng.random(B) < 0.9).astype(np.float32)).cuda()
    sub = torch.from_numpy(rng.choice(E, max(n_sub, 1), replace=False).astype(np.int32)).cuda()
    w = torch.from_numpy((rng.random(B) * 0.9 + 0.1).astype(np.float32)).cuda()
    return q, q_next, sub, rewards, masks, w


def _run(q, q_next, sub, n_sub, rewards, masks, E, B, weights=None, grad_scale=0.5):
    from serl_b200 import ops
    out = dict(target_q=torch.empty(B, device="cuda"), dq=torch.empty(E, B, device="cuda"), info=torch.zeros(4, device="cuda"),
               delta=torch.full((B,), float("nan"), device="cuda"))
    lagrange = torch.zeros(1, device="cuda")
    ops.critic_loss(q, q_next, sub, n_sub, rewards, masks, q, lagrange.data_ptr(), False, 0.99, grad_scale, out["target_q"],
                    out["dq"], out["info"].data_ptr(), E, B, weights=weights, delta=out["delta"] if weights is not None else None)
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("B", [1, 2, 255, 1024, 4096])
@pytest.mark.parametrize("E,n_sub", [(2, 0), (10, 2)])
def test_weighted_critic_loss_float64(E, n_sub, B):
    from oracle import per as P
    q, q_next, sub, rewards, masks, w = _case(E, B, seed=B + E, n_sub=n_sub)
    got = _run(q, q_next, sub, n_sub, rewards, masks, E, B, weights=w)
    qn = q_next.double().cpu().numpy()[sub.cpu().numpy()[:n_sub]] if n_sub else q_next.double().cpu().numpy()
    y = rewards.double().cpu().numpy() + 0.99 * masks.double().cpu().numpy() * qn.min(axis=0)
    loss, dq, delta = P.critic_loss(q.cpu().numpy(), y, w.cpu().numpy())
    np.testing.assert_allclose(got["target_q"], y, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got["info"][0], 0.5 * loss, rtol=1e-5)
    np.testing.assert_allclose(got["dq"], 0.5 * dq, rtol=1e-5, atol=1e-6 * np.abs(dq).max())
    np.testing.assert_allclose(got["delta"], delta, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("B", [1, 256, 4096])
def test_unit_weights_are_bitwise_the_unweighted_kernel(B):
    E = 2
    q, q_next, sub, rewards, masks, _ = _case(E, B, seed=7 * B)
    ones = torch.ones(B, device="cuda")
    a = _run(q, q_next, sub, 0, rewards, masks, E, B, weights=ones)
    b = _run(q, q_next, sub, 0, rewards, masks, E, B)
    for k in ("target_q", "dq", "info"):
        np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=k)
