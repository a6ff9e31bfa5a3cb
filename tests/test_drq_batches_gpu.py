"""GPU: whole DrQ / SAC gradient steps at the batch sizes where their kernels change regime, against the float64 oracle.

The pixel cases reuse tests/test_heads_grads_b256_gpu.py: RLPD halves from two synthetic rings (or one ring), the oracle fed the
engine's own trunk features, and that file's bars (fused heads Q 1e-4, per-op chain and fp32 build Q 1e-5, gradient leaves 2e-4
of their max, info scalars |got - ref| / (|ref| + 0.1)).  Each runs update_critics twice and update_high_utd once, and checks the
crops bit-exact and that a twin agent's eager run of the first step gives bitwise the same gradients and parameters.

What each batch reaches (two cameras unless noted):
  fused heads (16-bit build)  B = 1 (one ring): one-row M tile and k-block; 64 = 32 + 32: sle_bwd_multi's 16 chunks, two whole
                              k-blocks; 65 = 33 + 32: a 1-row k tail; 129 = 65 + 64: a 1-row second M tile, encoder k-split 11;
                              257 = 129 + 128: a third M tile, k-split 7; 1024 = 512 + 512 with utd_ratio 4: critic minibatches
                              of 256, the actor step over 1024 rows; one camera at 385 = 193 + 192: k-split 11 with four M tiles.
  per-op chain (3xTF32)       B = 127 / 129: the ensemble forward's last split / first unsplit batch, weight-gradient split-K
                              from 128; 1024: the actor step's GEMMs over 1024 rows.
  fp32 build (SGEMM)          B = 1, 129, 704 (the ensemble forward's last split batch) and 705 (its first unsplit one), 1025 =
                              513 + 512: the loss kernels' first batch above one row per thread.
  state SAC                   2048 rows with update_high_utd(utd_ratio=8) (the reference's state example: critic minibatches of
                              256, the actor / temperature step over 2048 rows) on the SGEMM and on the 3xTF32 GEMM, and 1025
                              with utd_ratio 1.
Measured errors per case: DESIGN.md §5."""
import os

import numpy as np
import pytest
import torch

from helpers import injected_features, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions
from test_agent_gpu import Q_TOL, _compare_state, _perturb
from test_heads_grads_b256_gpu import FP32, FUSED, _agent, _bar, _critic_errs, _draw, _engine_rows, _high_utd_errs, _run

pytestmark = pytest.mark.gpu
CHAIN = {"SERL_FUSED_HEADS": "0", "SERL_FUSED_ACTOR": "0"}
INFO = ("critic_loss", "predicted_qs", "target_qs", "actor_loss", "temperature", "entropy", "temperature_loss")
# The per-op chain's info scalars above 128 rows.  Measured on an H100 80GB HBM3 (700 W): target_qs 1.35e-5 at B = 129 and
# 2.0e-5 at B = 1024, actor_loss 1.9e-5 at B = 1024, while Q stays within 8.2e-6 and every gradient leaf within 2.2e-5.  At
# B = 127, where the 3xTF32 ensemble forward still splits K, target_qs is 2.7e-6; the fp32 build's SGEMM at the same batches
# gives 1e-7.  These scalars are batch means, so an error shared by the rows does not average out: the chain's 3xTF32 GEMMs
# (the fused heads' arithmetic, whose info bar is 1e-4, measured 1.2e-5 to 1.9e-5 here) put them at 1-2e-5.  Q and leaves keep
# the 1e-5 / 2e-4 bars; the info scalars get 5e-5, 2.5x over the worst measured.
CHAIN_WIDE = dict(FP32, info=5e-5)

#         precision, cameras, (online rows, demo rows | None), utd_ratio, environment, bars
CASES = {
    "fused-b1": ("fp16", 2, (1, None), 1, {}, FUSED),
    "fused-b64": ("fp16", 2, (32, 32), 1, {}, FUSED),
    "fused-b65": ("fp16", 2, (33, 32), 1, {}, FUSED),
    "fused-b129": ("fp16", 2, (65, 64), 1, {}, FUSED),
    "fused-b257": ("fp16", 2, (129, 128), 1, {}, FUSED),
    "fused-b1024-utd4": ("fp16", 2, (512, 512), 4, {}, FUSED),
    "fused-single-b385": ("fp16", 1, (193, 192), 1, {}, FUSED),
    "chain-b127": ("fp16", 2, (64, 63), 1, CHAIN, FP32),
    "chain-b129": ("fp16", 2, (65, 64), 1, CHAIN, CHAIN_WIDE),
    "chain-b1024": ("fp16", 2, (512, 512), 1, CHAIN, CHAIN_WIDE),
    "fp32-b1": ("fp32", 2, (1, None), 1, {}, FP32),
    "fp32-b129": ("fp32", 2, (65, 64), 1, {}, FP32),
    "fp32-b704": ("fp32", 2, (352, 352), 1, {}, FP32),
    "fp32-b705": ("fp32", 2, (353, 352), 1, {}, FP32),
    "fp32-b1025": ("fp32", 2, (513, 512), 1, {}, FP32),
}


def _twin(agent, cams, precision):
    """A second agent built like test_heads_grads_b256_gpu._agent's, holding the same parameters, CUDA graphs off."""
    from serl_b200.utils.launcher import make_drq_agent
    tr = random_transitions(np.random.default_rng(0), 1, cams)[0]
    twin = make_drq_agent(42, tr["observations"], tr["actions"], image_keys=cams, encoder_type="resnet-pretrained", precision=precision)
    twin.use_cuda_graphs = False
    twin._store.params.copy_(agent._store.params)
    twin._store.target.copy_(agent._store.target)
    twin._store.version += 1
    assert np.array_equal(twin.state.rng, agent.state.rng)
    return twin


def _assert_same_step(agent, twin, what):
    a, b = agent._store, twin._store
    for name in ("grad", "params", "target", "m", "v"):
        assert torch.equal(getattr(a, name), getattr(b, name)), f"{what}: two eager runs differ in {name}"


@pytest.mark.parametrize("case", list(CASES))
def test_drq_step_matches_float64_across_batches(case, monkeypatch):
    from oracle import drq as O
    precision, ncam, halves, utd, env, bars = CASES[case]
    for k, v in env.items():                                          # before the engine is built: it picks its head path then
        monkeypatch.setenv(k, v)
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams, B = ("cam0", "cam1")[:ncam], sum(h or 0 for h in halves)
    agent, its = _agent(cams, precision, halves)
    ocfg = oracle_cfg_from_agent(agent)
    worst, fails, modes = {}, [], []

    def bar(k):
        return bars["info"] if (k in INFO and "info" in bars) else _bar(bars, k)

    def record(what, errs):
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
        fails.extend(f"{what}: {k} {v:.2e} > {bar(k):.0e}" for k, v in errs.items() if not v <= bar(k))

    for i in range(2):
        ostate = oracle_state_from_agent(agent)
        both, host = _draw(its)
        twin = _twin(agent, cams, precision) if i == 0 else None
        (agent, info), mode = _run(agent, lambda: agent.update_critics(both))
        modes.append(mode)
        if twin is not None:
            twin.update_critics(both)
            _assert_same_step(agent, twin, f"{case} update_critics")
            del twin
            torch.cuda.empty_cache()
        eng = agent._engines[B]
        assert (eng.fused is not None) == (precision != "fp32" and not env), case
        pix, feats = _engine_rows(eng, cams)
        with injected_features(pix, feats):
            oinfo = O.update_critics(ostate, ocfg, host)
        for cam in cams:                                               # crops bit-exact, in the engine's row order
            np.testing.assert_array_equal(pix[cam][:B], oinfo["_aug"]["observations"][cam][:, 0])
            np.testing.assert_array_equal(pix[cam][B:], oinfo["_aug"]["next_observations"][cam][:, 0])
        np.testing.assert_array_equal(agent.state.rng, ostate.rng)
        record(f"update_critics {i} ({mode})", _critic_errs(agent, eng, info, oinfo))

    ostate = oracle_state_from_agent(agent)
    both, host = _draw(its)
    (agent, info), mode = _run(agent, lambda: agent.update_high_utd(both, utd_ratio=utd))
    modes.append(mode)
    pix, feats = _engine_rows(agent._engines[B], cams)
    calls, update = [], O.update                                       # the oracle's critic steps inside update_high_utd, kept
    monkeypatch.setattr(O, "update", lambda *a, **k: calls.append(update(*a, **k)) or calls[-1])
    with injected_features(pix, feats):
        oinfo = O.update_high_utd(ostate, ocfg, host, utd)
    monkeypatch.setattr(O, "update", update)
    assert len(calls) == utd + 1
    np.testing.assert_array_equal(agent.state.rng, ostate.rng)
    # group 0 still holds the gradient of the last critic minibatch
    record(f"update_high_utd ({mode})", _high_utd_errs(agent, info, oinfo, calls[utd - 1]))
    agent.check_status()

    print(f"[{case}] B = {B}, modes {modes}")
    for name, keys in {"Q / target Q": ("q", "target_q"), "critic info": ("critic_loss", "predicted_qs", "target_qs"),
                       "actor / temperature info": ("actor_loss", "temperature", "entropy", "temperature_loss")}.items():
        print(f"[{case}] {name}: " + ", ".join(f"{k} {worst[k]:.2e}" for k in keys if k in worst))
    leaves = {k: v for k, v in worst.items() if "grad " in k}
    k = max(leaves, key=leaves.get)
    print(f"[{case}] worst gradient leaf: {leaves[k]:.2e} ({k})")
    assert not fails, "\n".join(fails)


# ---- state SAC (no trunk): the two builds differ only in the GEMM carrier of the heads ----------------------------------------
@pytest.mark.parametrize("gemm,B,utd", [("f32", 2048, 8), ("tf32x3", 2048, 8), ("f32", 1025, 1)])
def test_state_sac_update_high_utd_across_batches(gemm, B, utd, monkeypatch):
    """As test_agent_gpu.test_state_sac_update_high_utd_matches_oracle, at the reference state example's 2048 rows and at 1025."""
    from oracle import drq as O
    from serl_b200.ops import Workspace
    from serl_b200.utils.launcher import make_sac_agent
    monkeypatch.setenv("SERL_HEADS_GEMM", gemm)
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    S, A = 10, 4
    rng = np.random.default_rng(B)
    obs0, act0 = rng.standard_normal(S).astype(np.float32), rng.uniform(-1, 1, A).astype(np.float32)
    agents = []
    for _ in range(2):                                                  # the second one: the same step again, for bitwise equality
        a = make_sac_agent(42, obs0, act0)
        a.use_cuda_graphs = False
        _perturb(a, seed=4)
        a._store.counts.fill_(700)                                      # inside the warm-up ramp so lr != 0
        agents.append(a)
    agent, twin = agents
    assert agent._engine(B).ws.gemm_fn == Workspace.GEMM_IMPLS[gemm]
    ostate, ocfg = oracle_state_from_agent(agent), oracle_cfg_from_agent(agent)
    ocfg.discount = 0.99
    batch = dict(observations=rng.standard_normal((B, S)).astype(np.float32), next_observations=rng.standard_normal((B, S)).astype(np.float32),
                 actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.random(B).astype(np.float32),
                 masks=(rng.random(B) > 0.1).astype(np.float32), dones=np.zeros(B, bool))
    agent, info = agent.update_high_utd(batch, utd_ratio=utd)
    twin.update_high_utd(batch, utd_ratio=utd)
    _assert_same_step(agent, twin, f"state sac {gemm} B={B}")
    ob = dict(batch, observations={"state": batch["observations"]}, next_observations={"state": batch["next_observations"]})
    oinfo = O.update_high_utd(ostate, ocfg, ob, utd, augment=False)
    errs = {"critic_loss": abs(float(info["critic"]["critic_loss"]) - oinfo["critic"]["critic_loss"]) / abs(oinfo["critic"]["critic_loss"]),
            "actor_loss": abs(float(info["actor"]["actor_loss"]) - oinfo["actor"]["actor_loss"]) / (abs(oinfo["actor"]["actor_loss"]) + 0.1),
            "temperature_loss": abs(float(info["temperature"]["temperature_loss"]) - oinfo["temperature"]["temperature_loss"])
            / (abs(oinfo["temperature"]["temperature_loss"]) + 0.1)}
    print(f"[state sac {gemm} B={B} utd={utd}] " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v <= Q_TOL for v in errs.values()), errs
    np.testing.assert_allclose(float(info["actor_lr"]), 3e-4 * (700 + utd) / 2000, rtol=1e-6)
    _compare_state(agent, ostate, oinfo, f"state sac {gemm} B={B}")
    assert agent.state.step == utd + 1
