"""GPU: VICEAgent at the batch sizes where its kernels change regime, against tests/vice_oracle.py fed the agent's own trunk
features.  update_vice at B = 2 (6 LayerNorm rows: one partial 8-row block), 256, 814 (N = 1628: the smallest batch whose
permutation takes two sort rounds) and 1024 (the largest), with one camera and on the fp16 build; besides the draws, infos and
gradients of tests/test_vice_gpu.py, its dropout masks and mixup logits are compared too.  vice_reward against the oracle's
sigmoid at one observation and at 13 and 257 rows.  The reward relabelling on scripts/bench_vice.py's configuration (fp16, two
128x128 cameras, batch 256 as RLPD halves of two rings, cross-step pipeline and CUDA graphs) step by step, a twin agent with the
pipeline off, and update_high_utd(utd_ratio=4).  Measured errors: DESIGN.md §5."""
import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions
from test_vice_gpu import BARS, _adam_bar_ok

pytestmark = pytest.mark.gpu

CAMS = ("wrist", "side")
KEEP = 0.9


def _agent(precision, cams=CAMS, seed=0):
    from serl_b200.agents.continuous.vice import VICEAgent
    obs = {c: np.zeros((1, 128, 128, 3), np.uint8) for c in cams}
    obs["state"] = np.zeros((1, 7), np.float32)
    agent = VICEAgent.create_vice(seed, obs, np.zeros(4, np.float32), encoder_type="resnet-pretrained", image_keys=cams,
                                  precision=precision)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)           # biases / scales off their init so every path is exercised
    agent._vice.params.add_(torch.randn(agent._vice.n, device="cuda", generator=g) * 0.05)
    agent._vice.target.copy_(agent._vice.params)
    return agent


def _batch(rng, B, cams=CAMS):
    trs = random_transitions(rng, B, cams)
    st = lambda k: {**{c: np.stack([t[k][c] for t in trs]) for c in cams}, "state": np.stack([t[k]["state"] for t in trs])}
    return {"observations": st("observations"), "next_observations": st("next_observations"),
            "actions": np.stack([t["actions"] for t in trs]), "rewards": np.array([t["rewards"] for t in trs], np.float32),
            "masks": np.array([t["masks"] for t in trs], np.float32), "dones": np.array([t["dones"] for t in trs])}


def _logits(vice_params, cams, feats):
    import vice_oracle as V
    return V.forward({k: torch.as_tensor(v).double() for k, v in vice_params.items()}, cams,
                     {c: torch.as_tensor(np.asarray(f, np.float32)).double() for c, f in feats.items()}).numpy()


@pytest.mark.parametrize("precision,cams,B", [("fp32", CAMS, 2), ("fp32", CAMS, 256), ("fp32", CAMS, 814), ("fp32", CAMS, 1024),
                                              ("fp32", ("image",), 256), ("fp16", CAMS, 256)])
def test_update_vice_matches_oracle_across_batches(precision, cams, B):
    import vice_oracle as V
    from oracle import drq as O
    from oracle import jax_prng as P
    from serl_b200.agents.continuous.vice import permutation_rounds
    tol, gtol = BARS[precision]
    nc, N = len(cams), 2 * B
    agent = _agent(precision, cams, seed=B)
    batch = _batch(np.random.default_rng(B + 1), B, cams)
    vp = agent._vice
    params = vp.dump(vp.params)
    k = V.keys(agent.state.rng, nc)
    agent, info = agent.update_vice(batch)
    assert np.array_equal(agent.state.rng, k["final"])
    b = agent._vice_scratch(B)
    raw = {cam: b["raw"][j].view(N, 4, 4, 512).cpu().numpy().astype(np.float64) for j, cam in enumerate(cams)}
    grads, oinfo = V.update_vice_grads(params, cams, raw, k)
    assert permutation_rounds(N) == (2 if N >= 1626 else 1)
    for j, (lam, perm, eps) in enumerate(oinfo["draws"]):
        assert np.float32(lam) == b["lam"][j].item()
        assert np.array_equal(b["perm"][j].cpu().numpy(), perm), j
        assert np.array_equal(b["eps"][j].cpu().numpy(), eps), j
    # dropout masks: keyed (N, n) masks of the mixup rows, one broadcast row for the penalty rows and their tangents
    smask, hmask = b["smask"].cpu().numpy().astype(bool), b["hmask"].cpu().numpy().astype(bool)
    for j, cam in enumerate(cams):
        assert np.array_equal(smask[j, :N], oinfo["sle_masks"][cam]), cam
        assert (smask[j, N:] == P.bernoulli(P.fold_in(k["vice"], j), KEEP, (4096,))[None]).all(), cam
    assert np.array_equal(hmask[:N], oinfo["hidden_mask"])
    assert (hmask[N:] == P.bernoulli(P.fold_in(k["vice"], nc), KEEP, (256,))[None]).all()
    ref_logit = oinfo["logits"].detach().numpy()
    lerr = float(np.abs(b["logit"][:N].cpu().numpy() - ref_logit).max()) / max(np.abs(ref_logit).max(), 1.0)
    print(f"VICE_BATCH_ERR {precision} cams={nc} B={B} logits {lerr:.3e}")
    assert lerr <= tol, lerr
    for key, got in (("bce", info["vice"]["bce_loss"]), ("grad_norm", info["vice"]["grad_norm"]), ("total", vp.info[3])):
        ref = float(oinfo[key])
        err = abs(float(got) - ref) / max(abs(ref), 1.0)
        print(f"VICE_BATCH_ERR {precision} cams={nc} B={B} {key} {err:.3e}")
        assert err <= tol, (key, float(got), ref)
    g = vp.dump(vp.grad)
    worst = 0.0
    for path, ref in grads.items():
        ref = ref.numpy()
        scale = np.abs(ref).max()
        assert scale > 0, path
        err = np.abs(g[path] - ref).max() / scale
        worst = max(worst, err)
        assert err <= gtol, (path, err)
    print(f"VICE_BATCH_ERR {precision} cams={nc} B={B} grad_leaves {worst:.3e}")
    opt = {"count": 0, "mu": {k_: torch.zeros_like(v) for k_, v in grads.items()}, "nu": {k_: torch.zeros_like(v) for k_, v in grads.items()}}
    upd = O.adam_tx_update(grads, opt, 3e-4)
    new = vp.dump(vp.params)
    for path in grads:
        assert _adam_bar_ok(new[path], params[path] + upd[path].numpy(), grads[path].numpy(), 3e-4), path


@pytest.mark.parametrize("B", [None, 13, 257])
def test_vice_reward_values(B):
    import vice_oracle as V
    agent = _agent("fp32", seed=61)
    rng = np.random.default_rng(62)
    n = 1 if B is None else B
    obs = {c: rng.integers(0, 256, (n, 1, 128, 128, 3), dtype=np.uint8) for c in CAMS}
    obs["state"] = rng.standard_normal((n, 1, 7)).astype(np.float32)
    if B is None:
        obs = {k: v[0] for k, v in obs.items()}
    got = agent.vice_reward(obs)
    assert got.shape == (() if B is None else (B,))
    eng = agent._infer_engine(n)
    feats = {c: eng.feats[c].view(n, 4, 4, 512).cpu().numpy() for c in CAMS}
    want = V.vice_reward(agent._vice.dump(agent._vice.params), CAMS, feats).numpy()
    err = float(np.abs(got.cpu().numpy().reshape(-1) - want).max())
    print(f"VICE_BATCH_ERR vice_reward B={B} {err:.3e}")
    assert err <= 1e-6


# ---- relabelling on scripts/bench_vice.py's configuration ---------------------------------------------------------------
def _rings(cams):
    from serl_b200.utils.launcher import make_replay_buffer
    env = fake_env(cams)
    rb = make_replay_buffer(env, capacity=300, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=3)
    demo = make_replay_buffer(env, capacity=120, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=4)
    trs = random_transitions(np.random.default_rng(1), 420, cams)
    for tr in trs[:300]:
        rb.insert(tr)
    for tr in trs[300:]:
        demo.insert(tr)
    return rb, demo, trs


def _relabel_check(agent, eng, vice_params, B):
    """eng.rewards against the float64 threshold of eng's own next-observation features (rows [B, 2B)); returns (rewards, logits)"""
    logits = _logits(vice_params, CAMS, {c: eng.feats[c].view(2 * B, 4, 4, 512)[B:].cpu().numpy() for c in CAMS})
    got = eng.rewards.cpu().numpy()
    far = np.abs(logits) > 1e-5
    assert np.array_equal(got[far], (logits[far] >= 0).astype(np.float32))
    return got, logits


def test_relabel_on_the_bench_vice_configuration():
    from serl_b200.utils.launcher import make_vice_agent
    from serl_b200.utils.train_utils import concat_batches
    B = 256
    agents, its = [], []
    for pipelined in (True, False):
        rb, demo, trs = _rings(CAMS)
        a = make_vice_agent(42, trs[0]["observations"], trs[0]["actions"], image_keys=CAMS, vice_image_keys=CAMS,
                            encoder_type="resnet-pretrained", precision="fp16")
        a.pipeline_critic_steps = pipelined
        agents.append(a)
        its.append([r.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True}) for r in (rb, demo)])
    # spread the logits and centre them on the next observations, so that both reward classes occur
    probe = agents[0].vice_reward({**{c: np.stack([t["next_observations"][c] for t in trs[::3]]) for c in CAMS},
                                   "state": np.stack([t["next_observations"]["state"] for t in trs[::3]])})
    p = probe.double().clamp(1e-12, 1 - 1e-12).cpu().numpy()
    med = np.median(np.log(p / (1 - p)))
    vp0 = agents[0]._vice.dump(agents[0]._vice.params)
    w, b0 = vp0["modules_vice/Dense_0/kernel"], vp0["modules_vice/Dense_0/bias"]
    head = {"modules_vice/Dense_0/kernel": 4 * w, "modules_vice/Dense_0/bias": (4 * (b0 - med)).astype(np.float32)}   # 4 (logit - median)
    for a in agents:
        a._vice.load(a._vice.params, head)
    ones, total = 0.0, 0
    for step in range(8):                                          # W eager, P eager, P capture, P replay ...
        got = []
        for a, (it, dit) in zip(agents, its):
            vice0 = a._vice.dump(a._vice.params)
            a, _ = a.update_critics(concat_batches(next(it), next(dit), axis=0))
            eng = a._last_engine if a.pipeline_critic_steps else a._engines[B]
            got.append(_relabel_check(a, eng, vice0, B))
        (r_pipe, l_pipe), (r_ser, l_ser) = got
        # the twins' features differ by the order of the fp16 trunk's GroupNorm sums: compare away from 0 by that margin
        far = (np.abs(l_pipe) > 1e-3 * np.abs(l_pipe).max()) & (np.abs(l_ser) > 1e-3 * np.abs(l_ser).max())
        assert np.array_equal(r_pipe[far], r_ser[far]), step
        assert 0 < r_pipe.mean() < 1, (step, r_pipe.mean())
        ones, total = ones + r_pipe.sum(), total + B
    print(f"VICE_BATCH_ERR relabel share of ones {ones / total:.3f}")
    assert 0.2 <= ones / total <= 0.8, ones / total
    # update_high_utd(utd_ratio=4) on the pipelined agent's rings: relabelled once, before the minibatches
    a, (it, dit) = agents[0], its[0]
    vice0 = a._vice.dump(a._vice.params)
    a, info = a.update_high_utd(concat_batches(next(it), next(dit), axis=0), utd_ratio=4)
    got, _ = _relabel_check(a, a._engine(B), vice0, B)
    assert 0 < got.mean() < 1
    assert np.array_equal(a._engine(B // 4).rewards.cpu().numpy(), got[3 * B // 4:])
    assert abs(float(info["vice_rewards"]) - float(got.mean())) <= 1e-7
    for a in agents:
        a.check_status()
