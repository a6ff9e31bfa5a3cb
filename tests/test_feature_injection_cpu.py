"""CPU: `helpers.injected_features`, which feeds the float64 oracle a set of precomputed trunk features (on the GPU tests: the
engine's own).  Injecting the oracle's own float64 trunk output for the same crops must change nothing, bit for bit, and a crop
the table does not hold must raise."""
import numpy as np
import pytest
import torch

from helpers import injected_features
from oracle import drq as O
from oracle import jax_prng as P
from serl_b200.params import ENC, init_trainable, init_trunk, trainable_spec


def _setup(B=2, S=7, A=4, E=4, seed=0):
    rng = np.random.default_rng(seed)
    cams = ("front",)
    params = {k: torch.as_tensor(v) for k, v in init_trainable(rng, trainable_spec(cams, S, A, E, pixel=True), 1.0).items()}
    for k in params:                                        # biases / LayerNorm offsets off their init: every gradient path live
        params[k] = params[k] + 0.05 * torch.as_tensor(rng.standard_normal(params[k].shape).astype(np.float32))
    for k, v in init_trunk(rng).items():
        params[f"{ENC}/encoder_front/pretrained_encoder/{k}"] = torch.as_tensor(v)
    cfg = O.OracleConfig(cams=cams, ensemble=E, subsample=2)
    batch = dict(observations={"front": rng.integers(0, 256, (B, 1, 128, 128, 3), dtype=np.uint8),
                               "state": rng.standard_normal((B, 1, S)).astype(np.float32)},
                 next_observations={"front": rng.integers(0, 256, (B, 1, 128, 128, 3), dtype=np.uint8),
                                    "state": rng.standard_normal((B, 1, S)).astype(np.float32)},
                 actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.random(B).astype(np.float32),
                 masks=np.array([1.0, 0.0], np.float32)[:B])
    return params, cfg, batch


def _crops_and_feats(params, aug):
    """The engine's layout: obs crops in rows [0, B), next-obs crops in [B, 2B), and their float64 trunk features (one trunk
    call per half, as the oracle makes them)."""
    halves = [aug[k]["front"][:, 0] for k in ("observations", "next_observations")]
    feats = [O.trunk_forward(params, "front", torch.as_tensor(h), torch.float64) for h in halves]
    return {"front": np.concatenate(halves)}, {"front": torch.cat(feats)}


def test_injected_oracle_features_change_nothing():
    params, cfg, batch = _setup()
    plain = O.update_critics(O.OracleState.create(params, P.prng_key(3), torch.float64), cfg, batch)
    pix, feats = _crops_and_feats(params, plain["_aug"])
    with injected_features(pix, feats):
        inj = O.update_critics(O.OracleState.create(params, P.prng_key(3), torch.float64), cfg, batch)
    assert O._features.__module__ == "oracle.drq"                                      # restored on exit
    assert inj["critic"]["critic_loss"] == plain["critic"]["critic_loss"]
    assert torch.equal(inj["critic"]["_q"], plain["critic"]["_q"])
    assert torch.equal(inj["critic"]["_target_q"], plain["critic"]["_target_q"])
    g0, g1 = plain["_grads"]["critic"], inj["_grads"]["critic"]
    assert set(g0) == set(g1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    assert float(g0[f"{ENC}/encoder_front/SpatialLearnedEmbeddings_0/kernel"].abs().max()) > 0


def test_a_crop_with_one_changed_byte_raises():
    params, cfg, batch = _setup()
    plain = O.update_critics(O.OracleState.create(params, P.prng_key(3), torch.float64), cfg, batch)
    pix, feats = _crops_and_feats(params, plain["_aug"])
    pix["front"] = pix["front"].copy()
    pix["front"][1, 64, 64, 2] ^= 1                         # obs frame 1 no longer matches the oracle's crop
    with injected_features(pix, feats):
        with pytest.raises(AssertionError, match="front: 1 of 2 oracle frames match no engine crop"):
            O.update_critics(O.OracleState.create(params, P.prng_key(3), torch.float64), cfg, batch)
    assert O._features.__module__ == "oracle.drq"
