"""CPU: the per-network optimizer options (make_optimizer's learning_rate, warmup_steps, cosine_decay_steps, clip_grad_norm;
common/optimizers.py:6-56).  The oracle's restated schedule and clip at closed-form points and against a literal float64
restatement; how the agents resolve the kwargs against their own arguments; and, on the dry device, which launches a step
makes (the norm pass only when a live tx clips) and that data parallelism keeps ONE collective per step."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR = 3e-4


# ---- oracle: schedule ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,D", [(10, 50), (4, 11), (0, 20)])
def test_cosine_schedule_closed_form_points(w, D):
    from oracle.optim import lr_schedule
    if w:
        assert lr_schedule(w // 2, LR, w, D) == pytest.approx(LR * (w // 2) / w, rel=1e-12)
        assert lr_schedule(0, LR, w, D) == 0.0
    assert lr_schedule(w, LR, w, D) == pytest.approx(LR, rel=1e-12)
    if (w + D) % 2 == 0:
        assert lr_schedule((w + D) // 2, LR, w, D) == pytest.approx(LR / 2, rel=1e-12)
    for c in (D, D + 1, D + 5, 10 * D):
        assert lr_schedule(c, LR, w, D) == pytest.approx(0.0, abs=1e-20)
    for c in range(w, D):                                      # optax warmup_cosine_decay_schedule, written out
        ref = LR * 0.5 * (1 + math.cos(math.pi * (c - w) / (D - w)))
        assert lr_schedule(c, LR, w, D) == pytest.approx(ref, rel=1e-12)


def test_schedule_without_decay_is_unchanged():
    from oracle.optim import lr_schedule
    assert [lr_schedule(c, LR, 4) for c in range(6)] == [LR * c / 4 for c in range(4)] + [LR, LR]
    assert lr_schedule(0, LR, 0) == LR and lr_schedule(7, LR, 0, None) == LR


# ---- oracle: clip_by_global_norm -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_norm", [1e-3, 0.5, 1e3])
def test_clip_by_global_norm_matches_float64_restatement(max_norm):
    from oracle.optim import clip_by_global_norm
    rng = np.random.default_rng(1)
    grads = {"a": rng.standard_normal((3, 4)) * 0.1, "b": rng.standard_normal(5) * 0.1, "c": np.array(0.02)}
    norm = math.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in grads.values()))
    out, got_norm = clip_by_global_norm({k: torch.as_tensor(v) for k, v in grads.items()}, max_norm)
    assert float(got_norm) == pytest.approx(norm, rel=1e-14)
    for k, g in grads.items():
        ref = g if norm < max_norm else (g / norm) * max_norm
        np.testing.assert_allclose(out[k].numpy(), ref, rtol=1e-14, atol=0)
    if norm >= max_norm:
        assert math.sqrt(sum(float((v.numpy() ** 2).sum()) for v in out.values())) == pytest.approx(max_norm, rel=1e-12)


def test_oracle_update_clips_each_tx_on_its_own_gradient_tree():
    """A state-SAC oracle step: the critic tx clips on the critic-loss gradient only, the actor tx on the actor-loss one; the
    tx that is not clipped takes the same Adam step as without the option."""
    from oracle import drq as O
    from oracle import jax_prng as P
    from oracle import optim
    from serl_b200.params import init_trainable, trainable_spec
    rng = np.random.default_rng(0)
    S, A, E, B = 5, 3, 4, 16
    params = {k: torch.as_tensor(v) for k, v in init_trainable(rng, trainable_spec((), S, A, E, pixel=False), 1e-2).items()}
    batch = dict(observations={"state": rng.standard_normal((B, S)).astype(np.float32)},
                 next_observations={"state": rng.standard_normal((B, S)).astype(np.float32)},
                 actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rng.random(B).astype(np.float32),
                 masks=np.ones(B, np.float32))
    nets = frozenset({"actor", "critic", "temperature"})

    def step(**opts):
        st = O.OracleState.create(params, P.prng_key(3), torch.float64)
        cfg = O.OracleConfig(cams=(), discount=0.99, target_entropy=-A / 2, ensemble=E, subsample=2, pixel=False)
        rnd, new_rng = O.derive_update_randomness(st.rng, B, A, (), False, E, 2, nets=tuple(nets))
        return st, optim.update(st, cfg, batch, rnd, nets, torch.float64, new_rng, opts=optim.OptimizerOptions(**opts))

    s0, i0 = step()
    # without options the restated optimizer tail is drq.update's own, bit for bit
    sd = O.OracleState.create(params, P.prng_key(3), torch.float64)
    rnd, new_rng = O.derive_update_randomness(sd.rng, B, A, (), False, E, 2, nets=tuple(nets))
    idr = O.update(sd, O.OracleConfig(cams=(), discount=0.99, target_entropy=-A / 2, ensemble=E, subsample=2, pixel=False),
                   batch, rnd, nets, torch.float64, new_rng)
    for k in sd.params:
        assert torch.equal(s0.params[k], sd.params[k]) and torch.equal(s0.target_params[k], sd.target_params[k])
        for n in sd.opt:
            assert torch.equal(s0.opt[n]["mu"][k], sd.opt[n]["mu"][k]) and torch.equal(s0.opt[n]["nu"][k], sd.opt[n]["nu"][k])
    assert [s0.opt[n]["count"] for n in sd.opt] == [sd.opt[n]["count"] for n in sd.opt] and s0.step == sd.step
    assert all(i0[f"{n}_lr"] == idr[f"{n}_lr"] for n in sd.opt)
    s1, i1 = step(clip_grad_norm={"critic": 1e-6})
    critic_norm = float(optim.global_norm(i0["_grads"]["critic"]))
    assert float(i1["_grad_norm"]["critic"]) == pytest.approx(critic_norm, rel=1e-14) and "actor" not in i1["_grad_norm"]
    # first Adam step: update = -lr * g / (|g| + eps') elementwise, so clipping by a scalar barely moves it - the moments show it
    mu0, mu1 = s0.opt["critic"]["mu"], s1.opt["critic"]["mu"]
    for k in mu0:
        torch.testing.assert_close(mu1[k], mu0[k] * (1e-6 / critic_norm), rtol=1e-12, atol=0)
        torch.testing.assert_close(s1.opt["actor"]["mu"][k], s0.opt["actor"]["mu"][k], rtol=0, atol=0)


# ---- agent construction ---------------------------------------------------------------------------------------------------
def _sac_cfg(**kw):
    """AgentConfig of a state SAC agent, without building device state."""
    from serl_b200.agents.continuous.sac import optimizer_settings
    txk = {tx: kw.pop(f"{tx}_optimizer_kwargs", None) for tx in ("critic", "actor", "temperature")}
    return optimizer_settings(txk, kw.pop("learning_rate", None), {"critic": kw.pop("critic_warmup", None), "actor": kw.pop("actor_warmup", None)},
                              {"critic": 2000, "actor": 2000, "temperature": 0})


def test_optimizer_kwargs_resolution():
    default = _sac_cfg()
    assert default == dict(lr=(LR,) * 3, warmup=(2000, 2000, 0), decay=(None,) * 3, clip=(None,) * 3)
    assert _sac_cfg(critic_optimizer_kwargs={"learning_rate": 3e-4, "clip_grad_norm": None}) == default
    got = _sac_cfg(critic_optimizer_kwargs={"learning_rate": 1e-3, "clip_grad_norm": 10.0},
                   actor_optimizer_kwargs={"warmup_steps": 5, "cosine_decay_steps": 100},
                   temperature_optimizer_kwargs={"clip_grad_norm": 0.5})
    assert got == dict(lr=(1e-3, LR, LR), warmup=(2000, 5, 0), decay=(None, 100, None), clip=(10.0, None, 0.5))
    # an explicit argument fills what the dict leaves out, and must agree with what it states
    assert _sac_cfg(learning_rate=1e-3, critic_optimizer_kwargs={"clip_grad_norm": 1.0})["lr"] == (1e-3,) * 3
    assert _sac_cfg(learning_rate=1e-3, actor_optimizer_kwargs={"learning_rate": 1e-3})["lr"] == (1e-3,) * 3
    with pytest.raises(ValueError, match="disagrees"):
        _sac_cfg(learning_rate=1e-3, actor_optimizer_kwargs={"learning_rate": 3e-4})
    with pytest.raises(ValueError, match="disagrees"):
        _sac_cfg(critic_warmup=100, critic_optimizer_kwargs={"warmup_steps": 0})
    with pytest.raises(ValueError, match="cosine_decay_steps"):
        _sac_cfg(actor_optimizer_kwargs={"cosine_decay_steps": 2000})              # decay must exceed the 2000-step warm-up
    with pytest.raises(ValueError, match="clip_grad_norm"):
        _sac_cfg(critic_optimizer_kwargs={"clip_grad_norm": 0.0})
    with pytest.raises(NotImplementedError, match="weight_decay"):
        _sac_cfg(critic_optimizer_kwargs={"weight_decay": 1e-4})
    with pytest.raises(NotImplementedError, match="return_lr_schedule"):
        _sac_cfg(actor_optimizer_kwargs={"return_lr_schedule": True})
    with pytest.raises(TypeError, match="unexpected keys"):
        _sac_cfg(actor_optimizer_kwargs={"momentum": 0.9})
    assert _sac_cfg(critic_optimizer_kwargs={"weight_decay": None})["lr"] == (LR,) * 3


# ---- dry device: launches -------------------------------------------------------------------------------------------------
@pytest.fixture()
def dry(monkeypatch):
    from serl_b200 import _lib as L
    calls = []
    real_call = L.call

    def fake_call(name, *args):
        if name.startswith("serl_host_"):
            return real_call(name, *args)
        calls.append((name, args))
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    monkeypatch.setattr(L, "call", fake_call)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(L, "new_event", lambda: Ev())
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: len(calls))
    return calls


def _drq(**opt):
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    cams = ("front",)
    rb = make_replay_buffer(fake_env(cams, 128), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams), device="cpu", seed=5)
    trs = random_transitions(np.random.default_rng(0), 30, cams, 128)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu", **opt)
    return agent, rb


def _names(calls):
    return [n for n, _ in calls]


def _opt_calls(calls):
    return [n for n in _names(calls) if n in ("serl_adam_polyak", "serl_adam_polyak_opts", "serl_grad_global_norms")]


def test_norm_pass_only_when_a_live_tx_clips(dry):
    agent, rb = _drq()
    del dry[:]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    assert _opt_calls(dry) == ["serl_adam_polyak"]                      # no option: the parent's launch sequence
    agent, rb = _drq(critic_optimizer_kwargs={"learning_rate": 3e-4, "clip_grad_norm": None})
    del dry[:]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    assert _opt_calls(dry) == ["serl_adam_polyak"]

    agent, rb = _drq(critic_optimizer_kwargs={"clip_grad_norm": 1.0})
    del dry[:]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    assert _opt_calls(dry) == ["serl_grad_global_norms", "serl_adam_polyak_opts"]
    assert _names(dry)[-2:] == ["serl_grad_global_norms", "serl_adam_polyak_opts"]     # after every gradient kernel
    d, want = dry[-2][1][0]._obj, list(dry[-2][1][1])
    assert want == [1, 0, 0]
    st = agent._store
    from serl_b200.params import INFO_GAP, PROPRIO_LEAVES
    # the flat layout the norm pass reads: tx 0 = [0, seg_end[0]); the info gap after it is in no norm; tx 1 = group 1 plus
    # the actor-tx twin of the proprio encoder leaves at [aux_lo, aux_hi) + aux_off; tx 2 = group 2
    assert list(d.seg_end) == list(st.seg_end) and d.gap == INFO_GAP == st.seg_end[0] + INFO_GAP - st.info_off
    assert (d.aux_lo, d.aux_hi, d.aux_off) == (st.aux_lo, st.aux_hi, st.aux_off)
    assert d.aux_lo == st.leaf[PROPRIO_LEAVES[0]].offset and d.aux_hi + d.aux_off == st.n and d.n == st.n_main
    o = dry[-1][1][1]._obj
    assert list(o.clip) == [1.0, 0.0, 0.0] and list(o.decay_steps) == [0, 0, 0]
    assert o.norms == agent._engine(4).grad_norms.data_ptr()

    # actor clipping: a critic step leaves the actor tx's gradient zero, so there is nothing to clip
    agent, rb = _drq(actor_optimizer_kwargs={"clip_grad_norm": 1.0})
    del dry[:]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    assert _opt_calls(dry) == ["serl_adam_polyak_opts"]
    del dry[:]
    agent.update_high_utd(rb.sample(4, pack_obs_and_next_obs=True), utd_ratio=1)
    assert _opt_calls(dry) == ["serl_adam_polyak_opts", "serl_grad_global_norms", "serl_adam_polyak_opts"]
    assert list(dry[[n for n, _ in dry].index("serl_grad_global_norms")][1][1]) == [0, 1, 0]

    # a cosine schedule alone needs no norm pass
    agent, rb = _drq(temperature_optimizer_kwargs={"cosine_decay_steps": 10})
    del dry[:]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    assert _opt_calls(dry) == ["serl_adam_polyak_opts"] and list(dry[-1][1][1]._obj.decay_steps) == [0, 0, 10]


def test_state_sac_high_utd_launches_with_clipping(dry):
    from serl_b200.utils.launcher import make_sac_agent
    rng = np.random.default_rng(0)
    agent = make_sac_agent(0, rng.standard_normal(10).astype(np.float32), np.zeros(4, np.float32), device="cpu",
                           critic_optimizer_kwargs={"clip_grad_norm": 1.0, "warmup_steps": 2000})
    B = 32
    batch = dict(observations=rng.standard_normal((B, 10)).astype(np.float32), next_observations=rng.standard_normal((B, 10)).astype(np.float32),
                 actions=np.zeros((B, 4), np.float32), rewards=np.zeros(B, np.float32), masks=np.ones(B, np.float32), dones=np.zeros(B, bool))
    del dry[:]
    agent.update_high_utd(batch, utd_ratio=4)
    assert _opt_calls(dry) == ["serl_grad_global_norms", "serl_adam_polyak_opts"] * 4 + ["serl_adam_polyak_opts"]
    assert agent.state.step == 5


# ---- data parallel (gloo, world 2): still ONE collective per step, and the norm reads the all-reduced buffer ---------------
def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from serl_b200 import _lib as L
    real = L.call
    events = []

    def fake(name, *a):
        if name.startswith("serl_host_"):
            return real(name, *a)
        events.append(name)
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    L.call, L.require_cuda, L.stream_ptr, L.new_event, L.pin = fake, (lambda d: None), (lambda: 0), (lambda: Ev()), (lambda t: t)
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    cams = ("front",)
    rb = make_replay_buffer(fake_env(cams, 128), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams), device="cpu",
                            seed=100 + rank)
    trs = random_transitions(np.random.default_rng(rank), 30, cams, 128)
    for tr in trs:
        rb.insert(tr)
    clip = {"clip_grad_norm": 1.0}
    agent = make_drq_agent(7, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu",
                           critic_optimizer_kwargs=clip, actor_optimizer_kwargs=clip, temperature_optimizer_kwargs=clip)
    agent.data_parallel = True
    agent.use_cuda_graphs = False
    real_ar = dist.all_reduce
    dist.all_reduce = lambda t, *a, **k: (events.append(("all_reduce", t.numel())), real_ar(t, *a, **k))[1]
    seqs = []
    for call in (lambda b: agent.update_critics(b), lambda b: agent.update(b, pmap_axis="devices"),
                 lambda b: agent.update_high_utd(b, utd_ratio=1)):
        del events[:]
        call(rb.sample(4, pack_obs_and_next_obs=True))
        seqs.append([e for e in events if isinstance(e, tuple) or e in ("serl_grad_global_norms", "serl_adam_polyak_opts", "serl_adam_polyak")])
    st = agent._store
    torch.save(dict(seqs=seqs, n=st.n, cut=st.info_off + 4), out.format(rank))
    dist.destroy_process_group()


def test_data_parallel_keeps_one_collective_and_norms_after_it(tmp_path):
    import torch.multiprocessing as mp
    world, port = 2, 33000 + os.getpid() % 2000
    out = str(tmp_path / "rank{}.pt")
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    r0 = torch.load(out.format(0))
    n, cut = r0["n"], r0["cut"]
    step = ["serl_grad_global_norms", "serl_adam_polyak_opts"]
    assert r0["seqs"][0] == [("all_reduce", cut)] + step                               # critic step
    assert r0["seqs"][1] == [("all_reduce", n)] + step                                 # all three networks
    assert r0["seqs"][2] == [("all_reduce", cut)] + step + [("all_reduce", n - cut)] + step
    assert torch.load(out.format(1))["seqs"] == r0["seqs"]
