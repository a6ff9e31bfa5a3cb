"""GPU: critic, actor and temperature gradients at the benchmark batch (256 rows, RLPD halves, two 128x128 cameras, graph replay)
against the float64 oracle fed the engine's OWN frozen-trunk features (helpers.injected_features).

With the trunk's rounding out of the comparison, what is measured is the heads, losses and reductions alone, so the 16-bit
build's heads are held to fp32-class bars: its fused heads and its per-op chain both run 3xTF32 GEMMs.  At B = 256 the
weight-gradient GEMMs run eight 32-wide k-blocks through the TMA stage ring, the forward and input-gradient GEMMs span two 128-row
M tiles, the encoder GEMM uses its B = 256 k-split and the small-gradient reductions run over 2560 rows: a fault in any of these
moves a gradient leaf long before it moves Q or the loss.  The injected features are checked too: a sample of rows of each
512-frame camera pass against the float64 trunk.

Errors: max|got - ref| / max|ref| per gradient leaf and for Q / target Q; info scalars |got - ref| / (|ref| + 0.1), i.e. the fp32
tests' rtol / atol = 1e-5 / 1e-6 rule at the 1e-5 bar.  Measured worst on an H100 80GB HBM3 (400 W power limit):
  fused (all four cases)  Q 6.0e-6, info 1.9e-5 (target_qs, entropy), gradient leaves 2.2e-5 (modules_actor/Dense_0/bias)
  per-op chain            Q 4.8e-6, info 8.4e-6 (target_qs), gradient leaves 8.4e-6
  fp32 build              Q 6.2e-7, info 1.1e-6, gradient leaves 6.2e-7
  trunk row sample        fp16 9.2e-4, fp32 1.9e-6
The negative control (two feature rows of camera 0 in the second M tile swapped) moves Q by 1.5e-1 and the encoder / critic
gradient leaves by up to 2.5e-2."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

from helpers import (fake_env, injected_features, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, rel_err,
                     to_numpy_tree)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP32 = {"q": 1e-5, "grad": 2e-4}                  # the fp32 build's bars (DESIGN.md §5): fp32 build and the per-op chain
FUSED = {"q": 1e-4, "grad": 2e-4}                 # fused heads (3xTF32 tgemm): 5x over the worst measured Q / info error
TRUNK_ROWS = [0, 1, 127, 128, 255, 256, 383, 511]  # first / last rows of each half of a 512-frame camera pass and between
TRUNK_TOL = {"fp16": 5e-3, "fp32": 2e-5}
PROPRIO = [f"modules_actor/encoder/{k}" for k in ("Dense_0/kernel", "Dense_0/bias", "LayerNorm_0/scale", "LayerNorm_0/bias")]

#        precision, cameras, rows per ring, update_critics calls, update_high_utd calls, pipelined, environment, bars
CASES = {
    "fused-dual": ("fp16", 2, 128, 3, 3, False, {}, FUSED),
    "fused-dual-pipelined": ("fp16", 2, 128, 6, 0, True, {}, FUSED),
    "fused-single": ("fp16", 1, 128, 3, 3, False, {}, FUSED),
    "fused-ragged": ("fp16", 2, 100, 2, 1, False, {}, FUSED),
    "chain-dual": ("fp16", 2, 128, 2, 1, False, {"SERL_FUSED_HEADS": "0", "SERL_FUSED_ACTOR": "0"}, FP32),
    "fp32-dual": ("fp32", 2, 128, 2, 1, False, {}, FP32),
}


def _agent(cams, precision, half, create=None):
    """half: the rows drawn from each ring, or (online rows, demo rows); demo rows None: one ring, no RLPD split.  create(sample
    transition) builds the agent (default: make_drq_agent's ResNet-10 DrQ agent at `precision`)."""
    halves = (half, half) if isinstance(half, int) else tuple(half)
    sys.path.insert(0, ROOT)
    from bench import fill_ring_synthetic
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    env = fake_env(cams)
    rb = make_replay_buffer(env, capacity=3000, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=11)
    demo = make_replay_buffer(env, capacity=20 * 101, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=12)
    fill_ring_synthetic(rb, seed=1)
    fill_ring_synthetic(demo, seed=2)
    tr = random_transitions(np.random.default_rng(0), 1, cams)[0]
    if create is None:
        agent = make_drq_agent(42, tr["observations"], tr["actions"], image_keys=cams, encoder_type="resnet-pretrained", precision=precision)
    else:
        agent = create(tr)
    g = torch.Generator(device="cuda").manual_seed(0)             # biases / LayerNorm offsets off their zero init: every gradient path live
    st = agent._store
    st.params.add_(torch.randn(st.n, device="cuda", generator=g) * 0.05)
    st.target.copy_(st.params + torch.randn(st.n, device="cuda", generator=g) * 0.005)
    st.version += 1
    lam = st.leaf["modules_temperature/lagrange"].offset
    st.params[lam] = -4.0
    st.target[lam] = -4.0
    its = [r.get_iterator(sample_args={"batch_size": h, "pack_obs_and_next_obs": True}) for r, h in zip((rb, demo), halves) if h]
    return agent, its


def _draw(its):
    """An RLPD batch (online rows first), or one ring's batch, as a lazy handle and as the oracle's unpacked host batch."""
    from oracle.replay import concat_batches as oconcat
    from oracle.replay import unpack
    from serl_b200.utils.train_utils import concat_batches
    bs = [next(it) for it in its]
    hs = [to_numpy_tree({k: v for k, v in b.to_dict().items() if k != "_indices"}) for b in bs]
    if len(bs) == 1:
        return bs[0], unpack(hs[0])
    return concat_batches(bs[0], bs[1], axis=0), unpack(oconcat(hs[0], hs[1], axis=0))


def _run(agent, call):
    """call() and how the step ran: "eager", "capture" (captured, then replayed) or "replay" (no library launch from the host)."""
    from serl_b200 import _lib as L
    graphs = lambda: sum(isinstance(v, tuple) for v in agent._graphs.values())
    g0, n0 = graphs(), L.launch_count()
    out = call()
    return out, ("capture" if graphs() > g0 else "replay" if L.launch_count() == n0 else "eager")


def _engine_rows(eng, cams):
    return {c: eng.pix[c].cpu().numpy() for c in cams}, {c: eng.feats[c].cpu() for c in cams}


def _scalar_err(got, ref):
    return abs(float(got) - float(ref)) / (abs(float(ref)) + 0.1)


def _leaf_err(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-12))


def _critic_errs(agent, eng, info, oinfo):
    st = agent._store
    grad = st.grad.cpu()
    e = {"q": rel_err(eng.q.cpu().numpy(), oinfo["critic"]["_q"].numpy()),
         "target_q": rel_err(eng.target_q.cpu().numpy(), oinfo["critic"]["_target_q"].numpy())}
    for k in ("critic_loss", "predicted_qs", "target_qs"):
        e[k] = _scalar_err(info["critic"][k], oinfo["critic"][k])
    for leaf in st.spec:
        if leaf.group == 0:
            e[f"grad {leaf.path}"] = _leaf_err(st.view(grad, leaf.path).numpy(), oinfo["_grads"]["critic"][leaf.path].numpy())
    return e


def _high_utd_errs(agent, info, oinfo, ocritic):
    """Info scalars, every group-1 / group-2 leaf, the actor-tx twin of the proprio encoder, and group 0: the actor step writes no
    parameter gradient there, so after the call it still holds the critic step's (image heads included) - against the oracle's."""
    st = agent._store
    grad = st.grad.cpu()
    e = {}
    for net, keys in (("critic", ("critic_loss", "predicted_qs", "target_qs")), ("actor", ("actor_loss", "temperature", "entropy")),
                      ("temperature", ("temperature_loss",))):
        for k in keys:
            e[k] = _scalar_err(info[net][k], oinfo[net][k])
    for leaf in st.spec:
        if leaf.group == 0:
            e[f"critic-step grad {leaf.path}"] = _leaf_err(st.view(grad, leaf.path).numpy(), ocritic["_grads"]["critic"][leaf.path].numpy())
        else:
            ref = oinfo["_grads"]["actor" if leaf.group == 1 else "temperature"][leaf.path].numpy()
            e[f"grad {leaf.path}"] = _leaf_err(st.view(grad, leaf.path).numpy(), ref)
    for path in PROPRIO:
        ref = oinfo["_grads"]["actor"][path].numpy()
        assert np.abs(ref).max() > 0, f"oracle: the actor loss must reach {path}"
        e[f"actor-tx grad {path}"] = _leaf_err(st.aux_view(grad, path).numpy(), ref)
    return e


def _bar(bars, name):
    return bars["grad"] if "grad " in name else bars["q"]


def _over(errs, bars):
    return {k: v for k, v in errs.items() if not v <= _bar(bars, k)}


@pytest.mark.parametrize("case", list(CASES))
def test_gradients_at_benchmark_batch_match_float64_on_engine_features(case, monkeypatch):
    from oracle import drq as O
    precision, ncam, half, n_crit, n_utd, pipelined, env, bars = CASES[case]
    for k, v in env.items():                                          # before the engine is built: it picks its head path then
        monkeypatch.setenv(k, v)
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams, B = ("cam0", "cam1")[:ncam], 2 * half
    agent, its = _agent(cams, precision, half)
    agent.pipeline_critic_steps = pipelined
    ocfg = oracle_cfg_from_agent(agent)
    worst, fails, modes = {}, [], {"update_critics": [], "update_high_utd": []}

    def record(what, errs):
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
        fails.extend(f"{what}: {k} {v:.2e} > {_bar(bars, k):.0e}" for k, v in _over(errs, bars).items())

    for i in range(n_crit):
        ostate = oracle_state_from_agent(agent)
        both, host = _draw(its)
        (agent, info), mode = _run(agent, lambda: agent.update_critics(both))
        modes["update_critics"].append(mode)
        eng = agent._last_engine if pipelined else agent._engines[B]
        assert (eng.fused is not None) == (precision != "fp32" and not env), case
        pix, feats = _engine_rows(eng, cams)
        if i == 0 and case in ("fused-dual", "fp32-dual"):
            for cam in cams:                                           # the features injected below are the trunk's, and sound
                f = feats[cam]
                assert f.shape[0] == 512 and bool(torch.isfinite(f).all()) and float(f.abs().max()) > 0, cam
                ref = O.trunk_forward(ostate.params, cam, torch.as_tensor(pix[cam][TRUNK_ROWS]), torch.float64).numpy()
                e = _leaf_err(f[TRUNK_ROWS].numpy(), ref)
                print(f"[{case}] trunk rows {TRUNK_ROWS} of {cam}: {e:.2e}")
                assert e < TRUNK_TOL[precision], (cam, e)
        neg_state = copy.deepcopy(ostate) if (i == 0 and case == "fused-dual") else None
        with injected_features(pix, feats):
            oinfo = O.update_critics(ostate, ocfg, host)
        for cam in cams:                                               # crops bit-exact, in the engine's row order
            np.testing.assert_array_equal(pix[cam][:B], oinfo["_aug"]["observations"][cam][:, 0])
            np.testing.assert_array_equal(pix[cam][B:], oinfo["_aug"]["next_observations"][cam][:, 0])
        np.testing.assert_array_equal(agent.state.rng, ostate.rng)
        errs = _critic_errs(agent, eng, info, oinfo)
        record(f"update_critics {i} ({mode})", errs)
        if neg_state is not None:
            # negative control: two obs rows of camera 0 in the second 128-row M tile trade features; the same bars must see it
            swapped = dict(feats)
            swapped[cams[0]] = feats[cams[0]].clone()
            swapped[cams[0]][[200, 201]] = feats[cams[0]][[201, 200]]
            with injected_features(pix, swapped):
                oneg = O.update_critics(neg_state, ocfg, host)
            flagged = _over(_critic_errs(agent, eng, info, oneg), bars)
            print(f"[{case}] negative control (rows 200 <-> 201 of {cams[0]}) flagged {len(flagged)} checks: "
                  + ", ".join(f"{k} {v:.1e}" for k, v in sorted(flagged.items(), key=lambda t: -t[1])))
            assert flagged, "swapping two feature rows in the second M tile went unnoticed"

    for i in range(n_utd):
        ostate = oracle_state_from_agent(agent)
        both, host = _draw(its)
        (agent, info), mode = _run(agent, lambda: agent.update_high_utd(both, utd_ratio=1))
        modes["update_high_utd"].append(mode)
        eng = agent._engines[B]
        pix, feats = _engine_rows(eng, cams)
        calls, update = [], O.update                                   # the oracle's critic step inside update_high_utd, kept
        monkeypatch.setattr(O, "update", lambda *a, **k: calls.append(update(*a, **k)) or calls[-1])
        with injected_features(pix, feats):
            oinfo = O.update_high_utd(ostate, ocfg, host, 1)
        monkeypatch.setattr(O, "update", update)
        assert len(calls) == 2
        np.testing.assert_array_equal(agent.state.rng, ostate.rng)
        for k, v in oinfo["_grads"]["actor"].items():                 # the image heads sit behind the policy's stop_gradient
            if "/encoder_" in k:
                assert float(v.abs().max()) == 0.0, k
        record(f"update_high_utd {i} ({mode})", _high_utd_errs(agent, info, oinfo, calls[0]))

    order = ["eager", "capture", "replay"]
    if pipelined:                                                      # W, then the two P variants: eager, capture, replay
        assert modes["update_critics"] == ["eager"] * 3 + ["capture"] * 2 + ["replay"], modes
    else:
        assert modes["update_critics"] == order[:n_crit] and modes["update_high_utd"] == order[:n_utd], modes
    agent.check_status()
    groups = {"Q / target Q": ("q", "target_q"), "critic info": ("critic_loss", "predicted_qs", "target_qs"),
              "actor / temperature info": ("actor_loss", "temperature", "entropy", "temperature_loss")}
    for name, keys in groups.items():
        if any(k in worst for k in keys):
            print(f"[{case}] {name}: " + ", ".join(f"{k} {worst[k]:.2e}" for k in keys if k in worst))
    for prefix in ("grad modules_actor/encoder", "grad modules_critic", "grad modules_actor/network", "grad modules_actor/Dense",
                   "grad modules_temperature", "actor-tx grad", "critic-step grad"):
        sel = {k: v for k, v in worst.items() if k.startswith(prefix)}
        if sel:
            k = max(sel, key=sel.get)
            print(f"[{case}] worst {prefix}*: {sel[k]:.2e} ({k})")
    assert not fails, "\n".join(fails)
