"""GPU: agents on stacks of T frames (ChunkingWrapper(obs_horizon=T)), the encoder input "B T H W C -> B H W (T C)".

- The sampler's channel-stacked output (serl_batch_out.stacked) holds, bit for bit, the reference-layout (B, T, H, W, C) output of
  the same draw and crops rearranged; the reference layout is pinned to the oracle's gather + per-frame crop by
  test_replay_sampler_paths_gpu.py and the golden rings.  Covered: T in {2, 3, 4, 8}, one and two cameras, 16-byte rows (the
  one-CTA-per-row kernel) and 36x36 frames (108-byte rows: the bytewise kernel), an RLPD two-part batch, n_step = 3, a prioritized
  ring, episode-start filler slots and windows that wrap around the ring's end.
- DrQ "small" and "resnet" at T = 3: update_critics twice and update_high_utd against the float64 oracle with the bars of
  test_trainable_encoder_batches_gpu.py, on the fp32, fp16 and bf16 builds, at a few rows and at 256.  The encoder maps the critic
  step saves are compared with the oracle's sign by sign: a ReLU flip is accepted only at fp32 rounding level of 0, and a step with
  one holds its conv / GroupNorm gradient leaves to the few-rows ReLU bar (_relu_flips).
- The pipelined CUDA-graph update_critics sequence equals the eager serial one bitwise; sample_actions / forward_* on one and on a
  batch of stacked observations match the oracle; a checkpoint round trip restores the parameters and the next step.
- BC update at T = 3 on both encoders against the BC oracle.
"""
import os
import sys

import numpy as np
import pytest
import torch

import test_bc_encoders_gpu as tbc
import test_trainable_encoder_batches_gpu as tte
from frame_stack_oracle import resnet_stack_oracle, stack
from helpers import fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, rel_err
from small_encoder_oracle import small_encoder_oracle
from test_agent_gpu import _perturb
from test_heads_grads_b256_gpu import ROOT, _critic_errs, _draw, _high_utd_errs
from test_resnet_encoder_gpu import POST_ADAM_TOL, _compare_state

pytestmark = pytest.mark.gpu
T3 = 3


def _ring(cams, hw, T, cap, seed, **kw):
    sys.path.insert(0, ROOT)
    from bench import fill_ring_synthetic
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(cams, hw, T=T), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams),
                            seed=seed, **kw)
    fill_ring_synthetic(rb, seed=seed)
    if rb.prioritized:                                     # random priorities on the valid slots
        from serl_b200 import ops
        g = torch.Generator(device="cuda").manual_seed(seed)
        rb.tree[:cap] = torch.rand(cap, device="cuda", generator=g) * rb.valid.float() + 0.0
        ops.priority_rebuild(rb.priority_tree())
    return rb


def _launch(parts, cams, hw, T, stacked, keys, nstep_bufs=None):
    from serl_b200 import _lib as L
    B = sum(p["batch"] for p in parts)
    dev = "cuda"
    shape = (B, hw, hw, 3 * T) if stacked else (B, T, hw, hw, 3)
    pix = {c: torch.full(shape, 7, dtype=torch.uint8, device=dev) for c in cams}
    npix = {c: torch.full(shape, 7, dtype=torch.uint8, device=dev) for c in cams}
    S = parts[0]["ring"].S * T
    st, nst = torch.zeros(B, S, device=dev), torch.zeros(B, S, device=dev)
    ac, rw, mk = torch.zeros(B, 4, device=dev), torch.zeros(B, device=dev), torch.zeros(B, device=dev)
    dn, idx = torch.zeros(B, dtype=torch.uint8, device=dev), torch.zeros(B, dtype=torch.int32, device=dev)
    off = torch.zeros(2, B * T, 2, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    prio = torch.zeros(B, device=dev)
    out = L.BatchOut()
    for j, c in enumerate(cams):
        out.obs_pix[j], out.next_pix[j] = pix[c].data_ptr(), npix[c].data_ptr()
    out.obs_state, out.next_state, out.actions = st.data_ptr(), nst.data_ptr(), ac.data_ptr()
    out.rewards, out.masks, out.dones, out.idx, out.status = rw.data_ptr(), mk.data_ptr(), dn.data_ptr(), idx.data_ptr(), status.data_ptr()
    out.off_obs, out.off_next, out.stacked = off[0].data_ptr(), off[1].data_ptr(), int(stacked)
    row = 0
    for p in parts:
        p["ring"].launch_sample(p, out, crop_total=B * T, out_row_offset=row, key_obs=keys[0].data_ptr(), key_next=keys[1].data_ptr(),
                                prio_out=prio if p["ring"].prioritized else None)
        row += p["batch"]
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    return pix, npix, (st, nst, ac, rw, mk, dn, idx, off)


SAMPLER_CASES = {                     # T, cameras, frame size, RLPD, n_step, prioritized, explicit wrap-around slots
    "t2-cam2-rlpd": (2, 2, 128, True, 1, False, False),
    "t3-cam1-nstep3": (3, 1, 128, False, 3, False, False),
    "t3-cam2-prio": (3, 2, 128, False, 1, True, False),
    "t4-cam1-wrap": (4, 1, 128, False, 1, False, True),
    "t8-cam2-rlpd-nstep3": (8, 2, 128, True, 3, False, False),
    "t3-cam2-36x36-bytewise": (3, 2, 36, True, 1, False, False),
    "t8-cam1-36x36-wrap": (8, 1, 36, False, 1, False, True),
}


@pytest.mark.parametrize("case", list(SAMPLER_CASES))
def test_sampler_stacked_layout_is_the_reference_layout_rearranged(case):
    T, ncam, hw, rlpd, n_step, prio, wrap = SAMPLER_CASES[case]
    cams = ("cam0", "cam1")[:ncam]
    rings = [_ring(cams, hw, T, 707, 3, **({"priority_alpha": 0.6} if prio else {}))]
    if rlpd:
        rings.append(_ring(cams, hw, T, 303, 4))
    args = {"batch_size": 37}
    if n_step > 1:
        args.update(n_step=n_step, discount=0.9)
    parts = []
    for r in rings:
        h = next(r.get_iterator(sample_args=args))
        parts += [dict(p) for p in h.parts]
    if wrap:                           # slots < T: windows that wrap to the ring's end; slots after a filler: episode starts
        slots = np.array([1, 2, T - 1, 102, 103, 203, 5, 300, 0 if T > 1 else 1] * 5, dtype=np.int32)[:parts[0]["batch"]]
        slots = np.where(rings[0]._valid_host[slots], slots, slots + 1).astype(np.int32)
        parts[0]["indx"] = torch.as_tensor(slots, device="cuda")
    kr = np.random.default_rng(T)
    keys = [torch.from_numpy(kr.integers(0, 2 ** 32, 2, dtype=np.uint32)).cuda() for _ in range(2)]
    ref_o, ref_n, ref_rest = _launch(parts, cams, hw, T, False, keys)
    got_o, got_n, got_rest = _launch(parts, cams, hw, T, True, keys)
    for c in cams:
        np.testing.assert_array_equal(got_o[c].cpu().numpy(), stack(ref_o[c].cpu().numpy()), err_msg=f"{case} obs {c}")
        np.testing.assert_array_equal(got_n[c].cpu().numpy(), stack(ref_n[c].cpu().numpy()), err_msg=f"{case} next_obs {c}")
    for a, b in zip(ref_rest, got_rest):
        assert torch.equal(a, b), case
    o = ref_rest[-1][0].cpu().numpy().reshape(-1, T, 2)
    assert (o != o[:, :1]).any()                             # the frames of a stack take their own shifts


# ---- DrQ at T = 3 against the float64 oracle ------------------------------------------------------------------------------------
#         encoder, precision, cameras, (online rows, demo rows | None), utd_ratio
DRQ_CASES = {
    "small-fp32-b5": ("small", "fp32", 2, (5, None), 1),
    "small-fp16-b256": ("small", "fp16", 2, (128, 128), 1),
    "small-bf16-b8-utd2": ("small", "bf16", 1, (4, 4), 2),
    "resnet-fp32-b2": ("resnet", "fp32", 1, (2, None), 1),
    "resnet-fp16-b256": ("resnet", "fp16", 2, (128, 128), 1),
    "resnet-bf16-b9": ("resnet", "bf16", 1, (9, None), 1),
}


def _make(encoder, cams, precision, T=T3, seed=42):
    from serl_b200.utils.launcher import make_drq_agent
    tr = random_transitions(np.random.default_rng(0), 1, cams, T=T)[0]
    return make_drq_agent(seed, tr["observations"], tr["actions"], image_keys=cams, encoder_type=encoder, precision=precision)


def _oracle_ctx(encoder, T=T3):
    return resnet_stack_oracle(T) if encoder == "resnet" else small_encoder_oracle()


# A unit whose float64 pre-activation lies within rounding of 0 can land on the other side of its ReLU.  At a few rows that one
# unit moves a conv leaf's gradient by up to about 1/sqrt(K) of its max (K: the layer's positions over the batch), so a step whose
# saved maps show such flips, each no larger than the map's own disagreement with the oracle on its agreeing units (and at least
# ROUNDING_FLIP of its max), holds its conv / GroupNorm gradient leaves to FEW_ROWS_16's ReLU bar.  A larger flip fails the test.
ROUNDING_FLIP = 1e-6


def _relu_flips(eng, encoder, cams, B, params):
    """(count, largest ratio of a flipped unit's |value| to its map's rounding bound) of the ReLU sign disagreements between the
    post-ReLU maps the critic step saved for its obs rows and the oracle's on the same crops (eng.pix) and the step's starting
    parameters; the bound is max(ROUNDING_FLIP, the largest |difference| on the units that agree) times the map's max."""
    import resnet_encoder_oracle as R
    from small_encoder_oracle import conv_stack
    n, worst = 0, 0.0
    for cam in cams:
        x = eng.pix[cam][:B].cpu().numpy()
        if encoder == "resnet":
            _, acts = R.trunk(params, cam, x, keep=True)
            ra = eng.res_saved[cam]
            pairs = [(ra.a_stem, acts["stem"])] + [(ra.blocks[b]["out"], acts[f"ResNetBlock_{b}"]) for b in range(len(ra.blocks))]
        else:
            _, maps = conv_stack(params, cam, x, keep=True)
            pairs = list(zip(eng.small_saved[cam].y, maps))
        for got, ref in pairs:
            g, r = got[:B].double().cpu(), ref.detach()
            flip = (g > 0) != (r > 0)
            if flip.any():
                n += int(flip.sum())
                rmax = r.abs().max()
                bound = max(ROUNDING_FLIP, ((g - r).abs()[~flip].max() / rmax).item()) * rmax
                worst = max(worst, (torch.maximum(g.abs(), r.abs())[flip].max() / bound).item())
    return n, worst


@pytest.mark.parametrize("case", list(DRQ_CASES))
def test_drq_stacked_steps_match_float64(case, monkeypatch):
    from oracle import drq as O
    encoder, precision, ncam, halves, utd = DRQ_CASES[case]
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams, B = ("cam0", "cam1")[:ncam], sum(h or 0 for h in halves)
    rings = [_ring(cams, 128, T3, 3000, 11), _ring(cams, 128, T3, 20 * 101, 12)]
    its = [r.get_iterator(sample_args={"batch_size": h, "pack_obs_and_next_obs": True}) for r, h in zip(rings, halves) if h]
    agent = _make(encoder, cams, precision)
    _perturb(agent, seed=7)
    bars = dict(tte.BARS[precision], **(tte.FEW_ROWS_16 if precision != "fp32" and B // utd < 64 else {}))
    ocfg = oracle_cfg_from_agent(agent)
    fails = []

    def bar(k, post=False):
        if tte._is_relu(k):
            return bars["rounding_flip_relu"] if "rounding_flip_relu" in bars else bars["relu"]
        if "grad " in k:
            return bars["post_grad"] if post and "post_grad" in bars else bars["grad"]
        q = bars.get("info", bars["q"]) if k in tte.INFO else bars["q"]
        return max(q, bars.get("post_info", POST_ADAM_TOL)) if post else q

    def record(what, errs, post=lambda k: False):
        fails.extend(f"{what}: {k} {v:.2e} > {bar(k, post(k)):.0e}" for k, v in errs.items() if not v <= bar(k, post(k)))

    def compare_state(what, ostate, oinfo):
        try:
            _compare_state(agent, ostate, oinfo, f"{case} {what}", relu_frac=bars.get("relu_frac", 1e-3), relu_steps=bars.get("relu_steps", 2.5))
        except AssertionError as e:
            fails.append(str(e).splitlines()[0])

    with _oracle_ctx(encoder):
        for i in range(2):
            ostate = oracle_state_from_agent(agent)
            params0 = {k: v.clone() for k, v in ostate.params.items()}
            both, host = _draw(its)
            agent, info = agent.update_critics(both)
            eng = agent._engines[B]
            oinfo = O.update_critics(ostate, ocfg, host)
            for cam in cams:                                           # crops bit-exact, stacked on the channel axis
                pix = eng.pix[cam].cpu().numpy()
                np.testing.assert_array_equal(pix[:B], stack(oinfo["_aug"]["observations"][cam]))
                np.testing.assert_array_equal(pix[B:], stack(oinfo["_aug"]["next_observations"][cam]))
            np.testing.assert_array_equal(agent.state.rng, ostate.rng)
            flips, worst = _relu_flips(eng, encoder, cams, B, params0)
            assert worst <= 1.0, f"update_critics {i}: a ReLU flip at {worst:.2e} times its map's rounding bound"
            if flips:
                print(f"[{case}] update_critics {i}: {flips} ReLU flip(s) at rounding level ({worst:.1e} of the bound)")
                bars["rounding_flip_relu"] = max(bars["relu"], tte.FEW_ROWS_16["relu"])
            record(f"update_critics {i}", _critic_errs(agent, eng, info, oinfo))
            bars.pop("rounding_flip_relu", None)
            compare_state(f"update_critics {i}", ostate, oinfo)
        ostate = oracle_state_from_agent(agent)
        both, host = _draw(its)
        agent, info = agent.update_high_utd(both, utd_ratio=utd)
        calls, update = [], O.update
        monkeypatch.setattr(O, "update", lambda *a, **k: calls.append(update(*a, **k)) or calls[-1])
        oinfo = O.update_high_utd(ostate, ocfg, host, utd)
        monkeypatch.setattr(O, "update", update)
        np.testing.assert_array_equal(agent.state.rng, ostate.rng)
        pre = () if utd > 1 else ("critic_loss", "predicted_qs", "target_qs", "critic-step grad ")
        record("update_high_utd", _high_utd_errs(agent, info, oinfo, calls[utd - 1]), post=lambda k: not k.startswith(pre))
        if not (utd > 1 and "post_grad" in bars):
            compare_state("update_high_utd", ostate, oinfo)
    agent.check_status()
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("encoder", ["small", "resnet"])
def test_stacked_pipeline_and_graphs_equal_serial_eager(encoder):
    """update_critics x4 (pipelined, CUDA graphs), update_high_utd and update at T = 3: bitwise the eager serial run."""
    cams, B = ("front", "wrist"), 16
    runs = {}
    for name, graphs, pipe in (("eager", False, False), ("graph", True, False), ("pipe", True, True)):
        rb = _ring(cams, 128, T3, 500, 5)
        agent = _make(encoder, cams, "fp16")
        _perturb(agent, seed=7)
        agent.use_cuda_graphs, agent.pipeline_critic_steps = graphs, pipe
        it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
        losses = []
        for _ in range(4):
            agent, i = agent.update_critics(next(it))
            losses.append(float(i["critic"]["critic_loss"]))
        agent, i = agent.update_high_utd(next(it), utd_ratio=2)
        losses.append(float(i["actor"]["actor_loss"]))
        for _ in range(2):
            agent, i = agent.update(next(it))
            losses.append(float(i["critic"]["critic_loss"]))
        agent.check_status()
        st = agent._store
        runs[name] = (losses, st.params.clone(), st.target.clone(), st.m.clone(), st.v.clone(), agent.state.rng)
    ref = runs["eager"]
    for name in ("graph", "pipe"):
        losses, params, target, m, v, rng = runs[name]
        np.testing.assert_array_equal(rng, ref[5])
        assert losses == ref[0], (name, losses, ref[0])
        assert torch.equal(params, ref[1]) and torch.equal(target, ref[2]) and torch.equal(m, ref[3]) and torch.equal(v, ref[4]), name


@pytest.mark.parametrize("encoder", ["small", "resnet"])
def test_stacked_inference_and_checkpoint(encoder, tmp_path):
    from oracle import drq as O
    from serl_b200.params import flatten
    from serl_b200.utils import checkpoints
    cams = ("front", "wrist")
    agent = _make(encoder, cams, "fp32")
    _perturb(agent, seed=3)
    trs = random_transitions(np.random.default_rng(9), 6, cams, T=T3)
    obs = {k: np.stack([t["observations"][k] for t in trs]) for k in (*cams, "state")}
    acts = np.stack([t["actions"] for t in trs])
    shapes = {k: v.shape for k, v in flatten(agent.state.params).items()}
    for cam in cams:
        p = f"modules_actor/encoder/encoder_{cam}"
        assert shapes[f"{p}/Conv_0/kernel" if encoder == "small" else f"{p}/conv_init/kernel"] == \
            ((3, 3, 3 * T3, 32) if encoder == "small" else (7, 7, 3 * T3, 64))
    batched = agent.sample_actions(obs, argmax=True)
    one = agent.sample_actions({k: v[2] for k, v in obs.items()}, argmax=True)
    assert rel_err(one, batched[2]) <= 1e-5
    ostate, ocfg = oracle_state_from_agent(agent), oracle_cfg_from_agent(agent)
    with _oracle_ctx(encoder):
        ref = O.sample_actions(ostate, ocfg, obs, argmax=True).numpy()
        assert rel_err(batched, ref) <= 1e-5, rel_err(batched, ref)
        import forward_oracle as FO
        q = agent.forward_critic(obs, acts, None, train=False).cpu().numpy()
        qref = FO.critic(agent, ostate.params, obs, acts).detach().numpy()
        assert rel_err(q, qref) <= 1e-5, rel_err(q, qref)
    q1 = agent.forward_target_critic({k: v[1] for k, v in obs.items()}, acts[1], np.array([0, 1], np.uint32)).cpu().numpy()
    qt = agent.forward_target_critic(obs, acts, np.array([0, 1], np.uint32)).cpu().numpy()
    assert rel_err(q1, qt[:, 1]) <= 1e-5
    dist = agent.forward_policy(obs, train=False)
    np.testing.assert_array_equal(dist.mode().cpu().numpy(), batched)
    # checkpoint round trip: the restored agent holds the same parameters and takes the same next step
    rb = _ring(cams, 128, T3, 400, 8)
    it = rb.get_iterator(sample_args={"batch_size": 8, "pack_obs_and_next_obs": True})
    agent, _ = agent.update_critics(next(it))
    checkpoints.save_checkpoint(str(tmp_path), agent.state, step=1)
    restored = _make(encoder, cams, "fp32", seed=5)
    restored.replace(state=checkpoints.restore_checkpoint(str(tmp_path), restored.state))
    st, sr = agent._store, restored._store
    own = torch.zeros(st.n, dtype=torch.bool, device=st.params.device)      # the leaves (not the alignment padding or info gap)
    for leaf in st.spec:
        own[leaf.offset:leaf.offset + leaf.size] = True
    for name in ("params", "target", "m", "v"):
        assert torch.equal(getattr(st, name)[own], getattr(sr, name)[own]), name
    batch = next(it)
    agent, ia = agent.update_critics(batch)
    restored, ib = restored.update_critics(batch)
    assert float(ia["critic"]["critic_loss"]) == float(ib["critic"]["critic_loss"])
    assert torch.equal(st.params[own], sr.params[own])


# ---- BC at T = 3 against the BC oracle ------------------------------------------------------------------------------------------
BC_CASES = {
    "small-fp32-b3": ("small", "fp32", 2, 3, True, tbc.LAUNCHER),
    "small-fp16-b64": ("small", "fp16", 1, 64, False, tbc.DROPOUT),
    "resnet-fp32-b2": ("resnet", "fp32", 1, 2, True, tbc.DROPOUT),
    "resnet-bf16-b64": ("resnet", "bf16", 1, 64, False, tbc.LAUNCHER),
}


@pytest.mark.parametrize("case", list(BC_CASES))
def test_bc_stacked_update_and_sample_actions_match_float64(case, monkeypatch):
    from serl_b200.agents.continuous.bc import BCAgent
    encoder, precision, ncam, B, proprio, mlp = BC_CASES[case]
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams = ("front", "wrist")[:ncam]
    tr = random_transitions(np.random.default_rng(0), 1, cams, T=T3)[0]
    agent = BCAgent.create(3, tr["observations"], tr["actions"], encoder_type=encoder, image_keys=cams, use_proprio=proprio,
                           network_kwargs=mlp, policy_kwargs={"std_parameterization": "exp", "std_min": 1e-5, "std_max": 5},
                           precision=precision)
    g = torch.Generator(device="cuda").manual_seed(3)
    agent._params.add_(torch.randn(agent._n, device="cuda", generator=g) * 0.05)
    trs = random_transitions(np.random.default_rng(10), B, cams, T=T3)
    obs = {**{c: np.stack([t["observations"][c] for t in trs]) for c in cams}, "state": np.stack([t["observations"]["state"] for t in trs])}
    batch = {"observations": obs, "actions": np.stack([t["actions"] for t in trs]).astype(np.float32)}
    monkeypatch.setattr(tbc, "_images", lambda b, cams: {c: stack(b["observations"][c]) for c in cams})
    bars = {"loss": tbc.FEW_ROWS_16_LOSS_TOL if precision != "fp32" and B < 64 else tbc.LOSS_TOL[precision]}
    with (resnet_stack_oracle(T3) if encoder == "resnet" else small_encoder_oracle()):
        tbc._step_against_oracle(agent, batch, None, bars, explicit_rng=np.random.default_rng(B))
        agent.explicit_dropout = None
        o = tbc._opts(agent)
        params = {k: torch.as_tensor(np.asarray(v)).double() for k, v in tbc._flat(agent.state.params).items()}
        enc = tbc.encode(params, encoder, cams, {c: stack(obs[c]) for c in cams},
                         torch.as_tensor(obs["state"]) if proprio else None, None)
        mu, _ = tbc.policy(params, enc, o)
    got = agent.sample_actions(obs, argmax=True)
    tol = tbc.LOSS_TOL[precision] * 10
    assert rel_err(got, tbc.mode(mu, o["squash"]).numpy()) <= tol
    assert rel_err(agent.sample_actions({k: v[0] for k, v in obs.items()}, argmax=True), got[0]) <= tol
