"""CPU (dry device): one FrozenTrunk per agent.  Its 16-bit packing is made once per camera and read by every runner it hands
out, a fault flag raised by any runner's kernels reaches the agent's check_status, and a 16-bit runner holds no fp32 scratch."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

CAMS = ("front", "wrist")


@pytest.fixture()
def dry(monkeypatch):
    """Kernel launches replaced by a recorder of (entry point, weight addresses its descriptor names)."""
    from serl_b200 import _lib as L
    calls = []
    real_call = L.call

    def fake_call(name, *args):
        if name.startswith("serl_host_"):
            return real_call(name, *args)
        d = args[0]._obj if args and isinstance(args[0], type(C.byref(C.c_int()))) else None
        calls.append((name, tuple(getattr(d, f) for f in ("w", "w_proj") if getattr(d, f, None))))
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


def _agent_and_ring(precision="fp16"):
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    rb = make_replay_buffer(fake_env(CAMS, 128), capacity=64, type="memory_efficient_replay_buffer", image_keys=list(CAMS), device="cpu", seed=5)
    trs = random_transitions(np.random.default_rng(0), 40, CAMS, 128)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=CAMS, encoder_type="resnet-pretrained", device="cpu",
                           precision=precision)
    return agent, rb, trs


def _exercise_every_engine(agent, rb, trs):
    """A training engine (batch 8), the step pipeline's ping-pong pair (batch 4) and an inference engine (one observation)."""
    agent.update_high_utd(rb.sample(8, pack_obs_and_next_obs=True), utd_ratio=1)
    agent.pipeline_critic_steps = True
    agent._graph_key = lambda tag, batch: ("dry",)                  # the dry device cannot capture graphs: pipelined path, eager bodies
    agent.use_cuda_graphs = False
    it = rb.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    for _ in range(2):
        agent.update_critics(next(it))
    agent.sample_actions(trs[0]["observations"], argmax=True)


def test_16bit_weights_are_packed_once_per_camera_and_shared_by_every_runner(dry, monkeypatch):
    from serl_b200 import trunk_bf16
    packs = []
    real_pack = trunk_bf16.pack_trunk
    monkeypatch.setattr(trunk_bf16, "pack_trunk", lambda w, dt: packs.append(dt) or real_pack(w, dt))
    agent, rb, trs = _agent_and_ring()
    del dry[:]
    _exercise_every_engine(agent, rb, trs)
    assert len(packs) == len(CAMS)
    trunk = agent._frozen_trunk
    runners = trunk._runners
    assert len(runners) == 4 and all(set(r.plans) == set(CAMS) for r in runners)
    stems = [w for name, w in dry if name == "serl_stem_conv_pool_tc_h16"]
    assert len(stems) == 5 * len(CAMS)                              # batch 8 once, the pair three times (cold start + 2 steps), inference once
    packed = {t.data_ptr() for cam in CAMS for k, t in trunk.packed(cam).items() if k.endswith("kernel")}
    read = {p for name, ws in dry if name.startswith(("serl_stem_", "serl_conv")) for p in ws}
    assert read == packed and len(packs) == len(CAMS)


@pytest.mark.parametrize("kind", ["drq", "vice"])
def test_a_trunk_fault_flag_raises_in_check_status(dry, kind):
    from serl_b200 import _lib as L
    if kind == "drq":
        agent, rb, _ = _agent_and_ring()
        agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
        runner = agent._engines[4].trunk
    else:
        from serl_b200.utils.launcher import make_vice_agent
        trs = random_transitions(np.random.default_rng(0), 4, CAMS, 128)
        agent = make_vice_agent(7, trs[0]["observations"], trs[0]["actions"], image_keys=CAMS, vice_image_keys=CAMS,
                                encoder_type="resnet-pretrained", device="cpu", precision="fp16")
        runner = agent._vice_scratch(4)["trunk"]                     # update_vice's own trunk pass over 2B images
    agent.check_status()
    runner.error.fill_(1)
    with pytest.raises(L.SerlError, match="frozen trunk"):
        agent.check_status()


def test_16bit_runner_holds_no_fp32_trunk_scratch(dry):
    agent, rb, trs = _agent_and_ring()
    _exercise_every_engine(agent, rb, trs)
    runners = agent._frozen_trunk._runners
    assert len(runners) == 4
    for r in runners:
        assert r._f32 is None
        held = [(k, t) for k, t in vars(r).items()] + [(k, t) for p in r.plans.values() for k, t in vars(p).items()]
        fp32 = {k for k, t in held if isinstance(t, torch.Tensor) and t.dtype == torch.float32}
        assert fp32 <= {"stats", "aff"}, fp32                       # only the GroupNorm sums and affines of the 16-bit convs
