"""GPU: whole DroQ / REDQ-with-dropout steps (the critic and policy MLPs' dropout_rate) at the batch sizes where the fused heads'
masked kernels change regime, against the float64 oracle of tests/droq_oracle.py fed the engine's own trunk features.

Built like tests/test_drq_batches_gpu.py (RLPD halves from two synthetic rings, or one ring; helpers.injected_features takes the
trunk's rounding out of the comparison) and held to its bars: fused heads Q 1e-4, fp32 build Q 1e-5, every gradient leaf 2e-4 of
its max, info scalars |got - ref| / (|ref| + 0.1) at the Q bar.  Each case runs update_critics twice, update once and
update_high_utd once, and checks every MLP keep mask the device drew bit-exact against the oracle's: the online and target
critics', the policy's on s', the actor step's policy and critic (KEY_MLP_ACTOR_CRITIC) masks and the temperature pass's policy
masks.

What each case reaches:
  DroQ (E = 2, no subsampling)  B = 1: one-row M tile; 129 = 65 + 64: a 1-row second M tile; 257 = 129 + 128: a third;
                                1024 = 512 + 512 with utd_ratio 8: critic minibatches of 128, then the actor and temperature
                                passes over 1024 rows (eight M tiles of masked epilogues)
  REDQ + dropout (E = 10, 2)    rates 0.5 (critic) / 0.1 (policy) at the benchmark batch 256 = 128 + 128 and at 129: the online
                                critic's masks (key c2) differ from the target's (c1), and inv_keep = 2 shows in rstd and dz
  fp32 build                    B = 1 and 1025 = 513 + 512 at rate 0.5: the per-op ln_act_dropout_rows chain
Measured errors per case: DESIGN.md §5."""
import os
from unittest import mock

import numpy as np
import pytest
import torch

from helpers import injected_features, oracle_cfg_from_agent, oracle_state_from_agent
from test_drq_batches_gpu import INFO
from test_heads_grads_b256_gpu import FP32, FUSED, _agent, _bar, _critic_errs, _draw, _engine_rows, _high_utd_errs, _run

pytestmark = pytest.mark.gpu
TXS = ("critic", "actor", "temperature")
NET = {"hidden_dims": [256, 256], "activations": "tanh", "use_layer_norm": True}

#        precision, (ensemble, subsample), (critic rate, policy rate), (online rows, demo rows | None), utd_ratio, bars
CASES = {
    "droq-b1": ("fp16", (2, None), (0.01, 0.01), (1, None), 1, FUSED),
    "droq-b129": ("fp16", (2, None), (0.01, 0.01), (65, 64), 1, FUSED),
    "droq-b257": ("fp16", (2, None), (0.01, 0.01), (129, 128), 1, FUSED),
    "droq-b1024-utd8": ("fp16", (2, None), (0.01, 0.01), (512, 512), 8, FUSED),
    "redq-drop-b256": ("fp16", (10, 2), (0.5, 0.1), (128, 128), 1, FUSED),
    "redq-drop-b129": ("fp16", (10, 2), (0.5, 0.1), (65, 64), 1, FUSED),
    "droq-bf16-b129": ("bf16", (2, None), (0.01, 0.01), (65, 64), 1, FUSED),
    "fp32-b1": ("fp32", (2, None), (0.5, 0.5), (1, None), 1, FP32),
    "fp32-b1025": ("fp32", (2, None), (0.5, 0.5), (513, 512), 1, FP32),
}


def _create(cams, precision, ensemble, subsample, rc, rp):
    from serl_b200.agents.continuous.drq import DrQAgent

    def create(tr):
        return DrQAgent.create_drq(
            42, tr["observations"], tr["actions"], encoder_type="resnet-pretrained", use_proprio=True, image_keys=cams,
            policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5},
            temperature_init=1e-2, discount=0.96, backup_entropy=False, critic_ensemble_size=ensemble, critic_subsample_size=subsample,
            precision=precision, critic_network_kwargs=dict(NET, dropout_rate=rc), policy_network_kwargs=dict(NET, dropout_rate=rp))
    return create


HEAD_B, HEAD_W = "modules_critic/Dense_0/bias", "modules_critic/Dense_0/kernel"


def _value_head_bias(errs, agent, ograds):
    """The value head's bias gradient is sum_r dQ_r, which the critic loss drives toward zero: on some batches it is a small
    remainder of much larger terms, and its error over its own size measures that cancellation.  It is held against the
    value-head kernel gradient instead, sum_r dQ_r h_r with |h| < 1: the same dQ terms, summed without that cancellation."""
    st = agent._store
    got = float(st.view(st.grad, HEAD_B).cpu().numpy().astype(np.float64).ravel()[0])
    ref = float(ograds[HEAD_B].numpy().ravel()[0])
    scale = max(abs(ref), float(np.abs(ograds[HEAD_W].numpy()).max()))
    for k in list(errs):
        if k.endswith(f"grad {HEAD_B}"):
            errs[k] = abs(got - ref) / scale
    return errs


def _same(got, ref, what):
    assert got is not None and ref is not None and len(got) == len(ref), what
    for i, (g, r) in enumerate(zip(got, ref)):
        np.testing.assert_array_equal(g.cpu().numpy().astype(bool), np.asarray(r), err_msg=f"{what}: layer {i}")


def _policy_masks(eng):
    """(the actor pass's policy masks or None, the temperature pass's): the per-op chain runs both passes in eng.p_mask."""
    return (eng.p_mask, eng.fused.p_mask_t) if eng.fused is not None else (None, eng.p_mask)


def _check_actor_temp_masks(eng, calls, what):
    """calls: the oracle's [("policy", k_p), ("critic", k_c), ("policy", k)] of an actor + temperature update."""
    actor, temp = _policy_masks(eng)
    if actor is not None:
        _same(actor, calls[0][1], f"{what}: actor pass policy")
    _same(eng.c_mask, calls[1][1], f"{what}: actor pass critic (KEY_MLP_ACTOR_CRITIC)")
    _same(temp, calls[2][1], f"{what}: temperature pass policy")


@pytest.mark.parametrize("case", list(CASES))
def test_droq_steps_match_float64_across_batches(case):
    from droq_oracle import networks_of
    from oracle import drq as O
    precision, (E, sub), (rc, rp), halves, utd, bars = CASES[case]
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams, B = ("cam0", "cam1"), sum(h or 0 for h in halves)
    agent, its = _agent(cams, precision, halves, create=_create(cams, precision, E, sub, rc, rp))
    ocfg = oracle_cfg_from_agent(agent)
    worst, fails, modes = {}, [], []

    def bar(k):
        return bars["info"] if (k in INFO and "info" in bars) else _bar(bars, k)

    def record(what, errs):
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
        fails.extend(f"{what}: {k} {v:.2e} > {bar(k):.0e}" for k, v in errs.items() if not v <= bar(k))

    with networks_of(agent):
        for i in range(2):
            ostate = oracle_state_from_agent(agent)
            both, host = _draw(its)
            (agent, info), mode = _run(agent, lambda: agent.update_critics(both))
            modes.append(mode)
            eng = agent._engines[B]
            assert (eng.fused is not None) == (precision != "fp32"), case
            pix, feats = _engine_rows(eng, cams)
            with injected_features(pix, feats):
                oinfo = O.update_critics(ostate, ocfg, host)
            for cam in cams:                                           # crops bit-exact, in the engine's row order
                np.testing.assert_array_equal(pix[cam][:B], oinfo["_aug"]["observations"][cam][:, 0])
                np.testing.assert_array_equal(pix[cam][B:], oinfo["_aug"]["next_observations"][cam][:, 0])
            np.testing.assert_array_equal(agent.state.rng, ostate.rng)
            calls = oinfo["_mlp_masks"]                                # policy on s' (k_na), target critic (c1), online critic
            _same(eng.p_mask, calls[0][1], f"update_critics {i}: policy on s'")
            _same(eng.c_mask_tgt, calls[1][1], f"update_critics {i}: target critic")
            _same(eng.c_mask, calls[2][1], f"update_critics {i}: online critic")
            if sub is not None:                                        # c2 vs c1: the two problems of each critic launch differ
                assert not np.array_equal(np.asarray(calls[1][1][0]), np.asarray(calls[2][1][0]))
            record(f"update_critics {i} ({mode})", _value_head_bias(_critic_errs(agent, eng, info, oinfo), agent, oinfo["_grads"]["critic"]))

        ostate = oracle_state_from_agent(agent)
        both, host = _draw(its)
        rnd, new_rng = O.derive_update_randomness(ostate.rng, B, agent._cfg.action_dim, cams, True, ocfg.ensemble, ocfg.subsample or 0)
        (agent, info), mode = _run(agent, lambda: agent.update(both))
        modes.append(mode)
        eng = agent._engines[B]
        pix, feats = _engine_rows(eng, cams)
        with injected_features(pix, feats):
            oinfo = O.update(ostate, ocfg, host, rnd, frozenset(TXS), torch.float64, new_rng)
        np.testing.assert_array_equal(agent.state.rng, ostate.rng)
        calls = oinfo["_mlp_masks"]
        _same(eng.c_mask_tgt, calls[1][1], "update: target critic")
        _check_actor_temp_masks(eng, calls[3:], "update")
        errs = _high_utd_errs(agent, info, oinfo, oinfo)               # group 0: the same update's critic gradients
        errs["target_q"] = _critic_errs(agent, eng, info, oinfo)["target_q"]
        record(f"update ({mode})", _value_head_bias(errs, agent, oinfo["_grads"]["critic"]))

        ostate = oracle_state_from_agent(agent)
        both, host = _draw(its)
        (agent, info), mode = _run(agent, lambda: agent.update_high_utd(both, utd_ratio=utd))
        modes.append(mode)
        eng = agent._engines[B]
        pix, feats = _engine_rows(eng, cams)
        ucalls, update = [], O.update                                  # the oracle's critic steps inside update_high_utd, kept
        with mock.patch.object(O, "update", lambda *a, **k: ucalls.append(update(*a, **k)) or ucalls[-1]), injected_features(pix, feats):
            oinfo = O.update_high_utd(ostate, ocfg, host, utd)
    assert len(ucalls) == utd + 1
    np.testing.assert_array_equal(agent.state.rng, ostate.rng)
    _check_actor_temp_masks(eng, ucalls[utd]["_mlp_masks"], "update_high_utd")
    last = ucalls[utd - 1]["_mlp_masks"]                               # the last critic minibatch's engine keeps its critic masks
    mb = agent._engine(B // utd)
    _same(mb.c_mask_tgt, last[1][1], "update_high_utd: last minibatch target critic")
    if utd > 1:
        _same(mb.c_mask, last[2][1], "update_high_utd: last minibatch online critic")
    errs = _value_head_bias(_high_utd_errs(agent, info, oinfo, ucalls[utd - 1]), agent, ucalls[utd - 1]["_grads"]["critic"])
    # the actor loss here reads the critic after its Adam step, whose entries with fp32-noise gradients may move by up to ~2 lr
    # either way: a ~1e-6 absolute shift of Q (test_droq_gpu.py's allowance, atol 1e-5)
    errs["actor_loss"] = abs(float(info["actor"]["actor_loss"]) - oinfo["actor"]["actor_loss"]) / (abs(oinfo["actor"]["actor_loss"]) + 1.0)
    record(f"update_high_utd ({mode})", errs)
    agent.check_status()

    print(f"[{case}] B = {B}, modes {modes}")
    for name, keys in {"Q / target Q": ("q", "target_q"), "critic info": ("critic_loss", "predicted_qs", "target_qs"),
                       "actor / temperature info": ("actor_loss", "temperature", "entropy", "temperature_loss")}.items():
        print(f"[{case}] {name}: " + ", ".join(f"{k} {worst[k]:.2e}" for k in keys if k in worst))
    leaves = {k: v for k, v in worst.items() if "grad " in k}
    k = max(leaves, key=leaves.get)
    print(f"[{case}] worst gradient leaf: {leaves[k]:.2e} ({k})")
    assert not fails, "\n".join(fails)
