"""GPU: DrQ gradient steps with the trainable "resnet" and "small" encoders at the batch sizes where their kernels change
regime, on the 16-bit builds as on fp32, against the float64 oracle run end to end (tests/resnet_encoder_oracle.py,
tests/small_encoder_oracle.py: the oracle trains its own encoder on the crops).

Each case follows tests/test_drq_batches_gpu.py: RLPD halves from two synthetic rings (or one ring), update_critics twice and
update_high_utd once; the crops bit-exact; a twin agent's eager run of the first step bitwise equal in grad / params / target /
m / v; Q and target Q (max|got - ref| / max|ref|), the info scalars (|got - ref| / (|ref| + 0.1)), every gradient leaf and the
post-Adam parameters (test_resnet_encoder_gpu._compare_state).  The 16-bit builds run the encoder convs as 3xTF32 wgmma from
the fp32 masters and the heads as 3xTF32 GEMMs, fp32-class arithmetic, so they take fp32-class bars: Q / target Q / info 1e-4
(fp32 build 1e-5, its info scalars 2e-5: at one row each is one row's value), gradient leaves 2e-4 of their max, conv and
GroupNorm leaves the 5e-3 ReLU bar (a pre-activation that rounds to the other side of 0 flips a unit).  Scalars computed on
encoder weights an Adam step of the same call already moved (the actor / temperature step of update_high_utd, the critic
minibatches after the first) take test_resnet_encoder_gpu.POST_ADAM_TOL, 1e-4.  On the 16-bit builds below 64 rows per critic
minibatch (FEW_ROWS_16) a flipped unit weighs more: it moves a conv leaf's gradient by about 1/sqrt(K) of its max, K the layer's
pixels over the batch (16 for block 3 at B = 1), and Adam carries that into everything computed after the critic step's update;
DESIGN.md §3 has the mechanism and the measured errors.

What each case reaches (wgrad splits per conv: min(264 / tiles, K / 128), at least 1; M tiles of 128 rows):
  resnet-fp16-b1        every 4x4 / 8x8 conv in one partial M tile; wgrad splits 1 on blocks 2-3 and the block-3 projection,
                        32 on the stem, 8 on block 0; one grid pass of the max-pool backward
  resnet-fp16-b18-utd2  critic minibatches of 9: the 4x4 forwards and each parity class of block 3's stride-2 dgrads have
                        M = 144 (a 16-row second tile); block 2 Conv_0 / Conv_1 wgrad at 4 / 3 splits; the actor step over 18
  resnet-fp16-b256      the benchmark's shape: every wgrad at its cap (stem 132, block 0 52, block 1 26 / 14 / 132, block 2 7 /
                        3 / 66, block-3 projection 16; rounding k_split up to 32 runs the block-1 / block-2 projections in
                        128 / 64 of them); the max-pool backward strides its grid about 120 times
  resnet-bf16-b9        the other 16-bit build, one camera
  resnet-fp32-b1/-b256  the CUDA-core dgrad / wgrad and the conv_igemm_f32 forward at one row and at the benchmark batch
  small-fp16-b1/-b256   the "small" encoder's tensor-core convs at one row (wgrad splits 16 / 4 / 1 / 1 by layer,
                        ops.sconv_wgrad_splits) and at 256 (528 / 105 / 26 / 6)
Plus the fp16 resnet encoder at B = 16 on two cameras: CUDA-graph replay and the cross-step pipeline bitwise equal to serial
eager steps.  Measured errors and the oracle's wall time per case: DESIGN.md §3."""
import os
import sys
import time

import numpy as np
import pytest
import torch

from helpers import fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions
from resnet_encoder_oracle import resnet_encoder_oracle
from small_encoder_oracle import small_encoder_oracle
from test_agent_gpu import _perturb
from test_heads_grads_b256_gpu import ROOT, _critic_errs, _draw, _high_utd_errs, _run
from test_resnet_encoder_gpu import POST_ADAM_TOL, RELU_G_TOL, _compare_state, _relu_leaf
from test_resnet_encoder_gpu import _setup as _resnet_setup

pytestmark = pytest.mark.gpu
BARS = {"fp16": {"q": 1e-4, "grad": 2e-4, "relu": RELU_G_TOL}, "bf16": {"q": 1e-4, "grad": 2e-4, "relu": RELU_G_TOL},
        "fp32": {"q": 1e-5, "info": 2e-5, "grad": 2e-4, "relu": RELU_G_TOL}}
# 16-bit builds at critic minibatches below 64 rows: conv / GroupNorm leaves and their Adam steps (_compare_state), the
# info scalars, and what update_high_utd computes on encoder weights its critic step's Adam update already moved ("post")
FEW_ROWS_16 = {"relu": 0.15, "relu_frac": 5e-3, "relu_steps": 3.0, "info": 2e-4, "post_info": 3e-3, "post_grad": 5e-3}
INFO = ("critic_loss", "predicted_qs", "target_qs", "actor_loss", "temperature", "entropy", "temperature_loss")

#         encoder, precision, cameras, (online rows, demo rows | None), utd_ratio
CASES = {
    "resnet-fp16-b1": ("resnet", "fp16", 2, (1, None), 1),
    "resnet-fp16-b18-utd2": ("resnet", "fp16", 2, (9, 9), 2),
    "resnet-fp16-b256": ("resnet", "fp16", 2, (128, 128), 1),
    "resnet-bf16-b9": ("resnet", "bf16", 1, (9, None), 1),
    "resnet-fp32-b1": ("resnet", "fp32", 2, (1, None), 1),
    "resnet-fp32-b256": ("resnet", "fp32", 1, (128, 128), 1),
    "small-fp16-b1": ("small", "fp16", 2, (1, None), 1),
    "small-fp16-b256": ("small", "fp16", 2, (128, 128), 1),
}


def _make(encoder, cams, precision, seed=42):
    from serl_b200.utils.launcher import make_drq_agent
    tr = random_transitions(np.random.default_rng(0), 1, cams)[0]
    return make_drq_agent(seed, tr["observations"], tr["actions"], image_keys=cams, encoder_type=encoder, precision=precision)


def _agent(encoder, cams, precision, halves):
    """test_heads_grads_b256_gpu._agent's rings and draws with a trainable encoder; parameters off their init (_perturb)."""
    sys.path.insert(0, ROOT)
    from bench import fill_ring_synthetic
    from serl_b200.utils.launcher import make_replay_buffer
    env = fake_env(cams)
    rb = make_replay_buffer(env, capacity=3000, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=11)
    demo = make_replay_buffer(env, capacity=20 * 101, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=12)
    fill_ring_synthetic(rb, seed=1)
    fill_ring_synthetic(demo, seed=2)
    agent = _make(encoder, cams, precision)
    _perturb(agent, seed=7)
    its = [r.get_iterator(sample_args={"batch_size": h, "pack_obs_and_next_obs": True}) for r, h in zip((rb, demo), halves) if h]
    return agent, its


def _twin(agent, encoder, cams, precision):
    """A second agent built like _agent's, holding the same parameters, CUDA graphs off."""
    twin = _make(encoder, cams, precision)
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


def _is_relu(name):
    path = name.split("grad ", 1)[-1]
    return "grad " in name and "/encoder_" in path and _relu_leaf(path)


@pytest.mark.parametrize("case", list(CASES))
def test_trainable_encoder_step_matches_float64_across_batches(case, monkeypatch):
    from oracle import drq as O
    encoder, precision, ncam, halves, utd = CASES[case]
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams, B = ("cam0", "cam1")[:ncam], sum(h or 0 for h in halves)
    agent, its = _agent(encoder, cams, precision, halves)
    bars = dict(BARS[precision], **(FEW_ROWS_16 if precision != "fp32" and B // utd < 64 else {}))

    def compare_state(what):
        try:
            _compare_state(agent, ostate, oinfo, f"{case} {what}", relu_frac=bars.get("relu_frac", 1e-3),
                           relu_steps=bars.get("relu_steps", 2.5))
        except AssertionError as e:
            fails.append(str(e).splitlines()[0])
    ocfg = oracle_cfg_from_agent(agent)
    worst, fails, modes, oracle_s = {}, [], [], [0.0]

    def bar(k, post=False):
        if _is_relu(k):
            return bars["relu"]
        if "grad " in k:
            return bars["post_grad"] if post and "post_grad" in bars else bars["grad"]
        q = bars.get("info", bars["q"]) if k in INFO else bars["q"]
        return max(q, bars.get("post_info", POST_ADAM_TOL)) if post else q

    def record(what, errs, post=lambda k: False):
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
        fails.extend(f"{what}: {k} {v:.2e} > {bar(k, post(k)):.0e}" for k, v in errs.items() if not v <= bar(k, post(k)))

    def oracle(fn, *a):
        t0 = time.perf_counter()
        out = fn(*a)
        oracle_s[0] += time.perf_counter() - t0
        return out

    with (resnet_encoder_oracle() if encoder == "resnet" else small_encoder_oracle()):
        for i in range(2):
            ostate = oracle_state_from_agent(agent)
            both, host = _draw(its)
            twin = _twin(agent, encoder, cams, precision) if i == 0 else None
            (agent, info), mode = _run(agent, lambda: agent.update_critics(both))
            modes.append(mode)
            if twin is not None:
                twin.update_critics(both)
                _assert_same_step(agent, twin, f"{case} update_critics")
                del twin
                torch.cuda.empty_cache()
            eng = agent._engines[B]
            assert eng.fused is None
            pix = {c: eng.pix[c].cpu().numpy() for c in cams}
            oinfo = oracle(O.update_critics, ostate, ocfg, host)
            for cam in cams:                                           # crops bit-exact, in the engine's row order
                np.testing.assert_array_equal(pix[cam][:B], oinfo["_aug"]["observations"][cam][:, 0])
                np.testing.assert_array_equal(pix[cam][B:], oinfo["_aug"]["next_observations"][cam][:, 0])
            np.testing.assert_array_equal(agent.state.rng, ostate.rng)
            record(f"update_critics {i} ({mode})", _critic_errs(agent, eng, info, oinfo))
            compare_state(f"update_critics {i}")

        ostate = oracle_state_from_agent(agent)
        both, host = _draw(its)
        (agent, info), mode = _run(agent, lambda: agent.update_high_utd(both, utd_ratio=utd))
        modes.append(mode)
        calls, update = [], O.update                                   # the oracle's critic steps inside update_high_utd, kept
        monkeypatch.setattr(O, "update", lambda *a, **k: calls.append(update(*a, **k)) or calls[-1])
        oinfo = oracle(O.update_high_utd, ostate, ocfg, host, utd)
        monkeypatch.setattr(O, "update", update)
        assert len(calls) == utd + 1
        np.testing.assert_array_equal(agent.state.rng, ostate.rng)
        # group 0 still holds the gradient of the last critic minibatch; every critic minibatch after the first, and the actor /
        # temperature step, run on encoder weights the critic step's Adam update already moved
        pre = () if utd > 1 else ("critic_loss", "predicted_qs", "target_qs", "critic-step grad ")
        record(f"update_high_utd ({mode})", _high_utd_errs(agent, info, oinfo, calls[utd - 1]), post=lambda k: not k.startswith(pre))
        if not (utd > 1 and "post_grad" in bars):      # a post-Adam minibatch's leaves, held to post_grad, can take Adam's opposite step
            compare_state("update_high_utd")
    agent.check_status()

    print(f"[{case}] B = {B}, modes {modes}, oracle {oracle_s[0]:.1f} s")
    for name, keys in {"Q / target Q": ("q", "target_q"), "critic info": ("critic_loss", "predicted_qs", "target_qs"),
                       "actor / temperature info": ("actor_loss", "temperature", "entropy", "temperature_loss")}.items():
        print(f"[{case}] {name}: " + ", ".join(f"{k} {worst[k]:.2e}" for k in keys if k in worst))
    for what, sel in (("conv / GroupNorm", _is_relu), ("other", lambda k: "grad " in k and not _is_relu(k))):
        leaves = {k: v for k, v in worst.items() if sel(k)}
        k = max(leaves, key=leaves.get)
        print(f"[{case}] worst {what} gradient leaf: {leaves[k]:.2e} ({k})")
    assert not fails, "\n".join(fails)


def test_resnet_fp16_pipeline_and_graphs_equal_serial_eager():
    """As test_resnet_encoder_gpu.test_pipeline_and_graphs_equal_serial_eager on the fp16 build: the tensor-core convs, the
    GroupNorm / max-pool backward and every reduction run in a fixed order, so graph replay and the pipeline are bitwise equal."""
    cams, B = ("front", "wrist"), 16
    runs = {}
    for name, graphs, pipe in (("eager", False, False), ("graph", True, False), ("pipe", True, True)):
        agent, rb = _resnet_setup(cams, precision="fp16")
        agent.use_cuda_graphs = graphs
        agent.pipeline_critic_steps = pipe
        it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
        losses = []
        for _ in range(4):
            agent, i = agent.update_critics(next(it))
            losses.append(float(i["critic"]["critic_loss"]))
        agent, i = agent.update_high_utd(next(it), utd_ratio=2)
        losses.append(float(i["actor"]["actor_loss"]))
        agent.check_status()
        st = agent._store
        runs[name] = (losses, st.params.clone(), st.target.clone(), st.m.clone(), st.v.clone(), agent.state.rng)
    ref = runs["eager"]
    for name in ("graph", "pipe"):
        losses, params, target, m, v, rng = runs[name]
        np.testing.assert_array_equal(rng, ref[5])
        assert losses == ref[0], (name, losses, ref[0])
        assert torch.equal(params, ref[1]) and torch.equal(target, ref[2]) and torch.equal(m, ref[3]) and torch.equal(v, ref[4]), name
