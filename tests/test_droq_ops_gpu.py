"""GPU: the kernels a dropout-MLP agent adds, bit-exact or against float64.  The (B, H_i) keep masks of serl_dropout_mask_fill
against the oracle's bernoulli(fold_in(key, ncams + i), 1 - rate); serl_mlp_dropout_keys against the oracle's key chain; and the
masked LayerNorm / activation layers over an ensemble's E*B rows with the mask row period B (every member reads the same mask)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,H,fold,rate", [(1, 64, 0, 0.01), (8, 256, 2, 0.1), (257, 512, 3, 0.5), (1024, 256, 1, 0.9)])
def test_mask_fill_is_the_oracle_bernoulli(B, H, fold, rate):
    from droq_oracle import mlp_masks
    from oracle import jax_prng as P
    from serl_b200 import ops
    from serl_b200.params import MlpArch
    key = P.prng_key(1000 + B)
    k = torch.from_numpy(key.view(np.int32)).cuda()
    m = torch.full((B, H), 7, dtype=torch.uint8, device="cuda")
    ops.dropout_mask_fill(k.data_ptr(), fold, 1.0 - rate, m, B * H)
    ref = mlp_masks(key, fold, B, MlpArch((H,), "tanh", True, rate))[0]
    np.testing.assert_array_equal(m.cpu().numpy().astype(bool), ref)


@pytest.mark.parametrize("do_aug", [0, 1])
def test_mlp_dropout_keys_kernel(do_aug):
    from droq_oracle import update_keys
    from oracle import jax_prng as P
    from serl_b200 import _lib as L
    from serl_b200 import ops
    rng = P.prng_key(77)
    dev_rng = torch.from_numpy(rng.view(np.int32)).cuda().view(torch.uint32)
    keys = torch.zeros(2 * L.NUM_KEYS_MLP, dtype=torch.uint32, device="cuda")
    ops.rng_schedule(dev_rng, keys, do_aug, 1, mlp_dropout=True)
    got = keys.cpu().view(torch.int32).numpy().view(np.uint32)
    r = P.split(rng, 3)[0] if do_aug else rng
    calls = update_keys(r, ("critic", "actor", "temperature"), True)
    np.testing.assert_array_equal(got[2 * L.KEY_MLP_CRITIC_TARGET:][:2], calls[1][1])
    np.testing.assert_array_equal(got[2 * L.KEY_MLP_CRITIC_SUBSAMPLED:][:2], calls[2][1])
    np.testing.assert_array_equal(got[2 * L.KEY_MLP_ACTOR_CRITIC:][:2], calls[4][1])
    np.testing.assert_array_equal(got[2 * L.KEY_CRITIC_NEXT:][:2], calls[0][1])
    np.testing.assert_array_equal(got[2 * L.KEY_ACTOR_DROPOUT:][:2], calls[3][1])
    np.testing.assert_array_equal(got[2 * L.KEY_TEMP_NEXT:][:2], calls[5][1])


def _ref_layer(z, mask, rate, act, ln, scale, bias):
    from arch_oracle import ACTIVATIONS
    from oracle import drq as O
    x = torch.where(mask, z / (1.0 - rate), torch.zeros_like(z))
    if ln:
        x = O.layer_norm(x, scale, bias)
    return ACTIVATIONS[act](x)


@pytest.mark.parametrize("act,ln", [("tanh", True), ("relu", False), ("swish", True), ("gelu", False)])
@pytest.mark.parametrize("E,B,D", [(2, 1, 64), (10, 33, 256), (3, 256, 512)])
def test_ensemble_layer_with_shared_mask_matches_float64(act, ln, E, B, D):
    """Forward and backward over E*B member-major rows with one (B, D) mask (mask_rows = B), per-member LayerNorm parameters."""
    from serl_b200 import ops
    from serl_b200.engine import ACT_IDS
    g = torch.Generator(device="cuda").manual_seed(E * 1000 + B)
    rate, R = 0.2, E * B
    z = torch.randn(R, D, device="cuda", generator=g)
    dt = torch.randn(R, D, device="cuda", generator=g)
    scale = 1 + 0.3 * torch.randn(E, D, device="cuda", generator=g)
    bias = 0.3 * torch.randn(E, D, device="cuda", generator=g)
    mask = (torch.rand(B, D, device="cuda", generator=g) > rate).to(torch.uint8)
    out, xhat, rstd = torch.full_like(z, float("nan")), torch.full_like(z, float("nan")), torch.full((R,), float("nan"), device="cuda")
    zz = z.clone()
    sc, bi = (scale.data_ptr(), bias.data_ptr()) if ln else (None, None)
    ops.ln_act_dropout_fwd(zz.data_ptr(), D, sc, bi, B, D, mask, 1.0 / (1.0 - rate), out.data_ptr(), D, xhat.data_ptr() if ln else None,
                           rstd.data_ptr() if ln else None, R, D, ACT_IDS[act], ln, mask_rows=B)
    dz, dy = torch.full_like(z, float("nan")), torch.full_like(z, float("nan"))
    ops.ln_act_dropout_bwd(dt.data_ptr(), D, out.data_ptr(), D, zz.data_ptr(), D, xhat.data_ptr() if ln else None,
                           rstd.data_ptr() if ln else None, sc, bi, B, D, mask, 1.0 / (1.0 - rate), dz.data_ptr(),
                           dy.data_ptr() if ln else None, R, D, ACT_IDS[act], ln, mask_rows=B)
    torch.cuda.synchronize()
    z64 = z.double().cpu().view(E, B, D).requires_grad_(True)
    m = mask.bool().cpu()[None].expand(E, B, D)
    ref = _ref_layer(z64, m, rate, act, ln, scale.double().cpu()[:, None], bias.double().cpu()[:, None])
    (ref * dt.double().cpu().view(E, B, D)).sum().backward()
    np.testing.assert_allclose(out.cpu().numpy(), ref.detach().reshape(R, D).numpy(), rtol=1e-5, atol=5e-5)
    gref = z64.grad.reshape(R, D).numpy()
    tol = (5e-3 if act == "relu" else 2e-4) * np.abs(gref).max()
    assert np.abs(dz.cpu().numpy() - gref).max() <= tol
    # every member's dropped units carry no gradient
    assert (dz.view(E, B, D)[:, ~mask.bool()] == 0).all()
