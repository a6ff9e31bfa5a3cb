"""CPU, world_size 2, gloo: the data-parallel host logic of `SACAgent._update_on_engine` - ONE all-reduce per `update`,
which contiguous range of the flat gradient buffer it covers for a critic vs an actor/temperature step (gradient
segment + the info scalars that sit next to it, + the actor-tx twin of the proprio encoder), mean semantics (kernels
pre-scale gradients and infos by 1/world, the collective sums), and that both ranks end with identical buffers.
Kernels are replaced by a recorder (dry run)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out, fused=False):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    if fused:                                                # read when the engine is built
        os.environ.update(SERL_FUSED_HEADS="force")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from serl_b200 import _lib as L
    real = L.call
    scales = []

    def fake(name, *a):
        if name.startswith("serl_host_"):
            return real(name, *a)
        if name == "serl_critic_loss":
            scales.append(("critic", float(a[10])))          # grad_scale argument
        if name == "serl_actor_loss":
            scales.append(("actor", float(a[12])))
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    L.call, L.require_cuda, L.stream_ptr, L.new_event, L.pin = fake, (lambda d: None), (lambda: 0), (lambda: Ev()), (lambda t: t)
    from helpers import fake_env, random_transitions
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    cams = ("front",)
    rb = make_replay_buffer(fake_env(cams, 128), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams), device="cpu",
                            seed=100 + rank)
    trs = random_transitions(np.random.default_rng(rank), 30, cams, 128)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(7, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu",
                           precision="fp16" if fused else "fp32")
    agent.data_parallel = True
    agent.use_cuda_graphs = False
    st = agent._store
    eng = agent._engine(4)
    # rank-specific gradients / infos stand in for what the (no-op) kernels would have written
    st.grad.copy_(torch.arange(st.n, dtype=torch.float32) * (rank + 1))
    n_coll = []
    real_ar = dist.all_reduce
    dist.all_reduce = lambda t, *a, **k: (n_coll.append(t.numel()), real_ar(t, *a, **k))[1]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    g_after_critic = st.grad.clone()
    n_critic = list(n_coll)
    st.grad.copy_(torch.arange(st.n, dtype=torch.float32) * (rank + 1))
    agent.update_high_utd(rb.sample(4, pack_obs_and_next_obs=True), utd_ratio=1)
    g_utd = st.grad.clone()
    del n_coll[:]
    st.grad.copy_(torch.arange(st.n, dtype=torch.float32) * (rank + 1))
    agent.update(rb.sample(4, pack_obs_and_next_obs=True), pmap_axis="devices")       # all three networks: still ONE collective
    torch.save(dict(seg=st.seg_end, n=st.n, info_off=st.info_off, fused=eng.fused is not None, g_critic=g_after_critic, g_utd=g_utd,
                    g_all=st.grad.clone(), n_critic=n_critic, n_all=list(n_coll), scales=scales), out.format(rank))
    dist.destroy_process_group()


def test_allreduce_segments_and_mean(tmp_path):
    world, port = 2, 29000 + os.getpid() % 2000
    out = str(tmp_path / "rank{}.pt")
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    r0, r1 = torch.load(out.format(0)), torch.load(out.format(1))
    n, io = r0["n"], r0["info_off"]
    cut = io + 4                                      # [0, cut): critic-tx segment + critic infos; [cut, n): everything the actor/temperature step owns
    base = torch.arange(n, dtype=torch.float32)
    # critic step: ONE collective over [0, cut): sum over ranks of base*(rank+1) = 3*base; the rest is untouched
    assert r0["n_critic"] == [cut]
    for r, k in ((r0, 1.0), (r1, 2.0)):
        torch.testing.assert_close(r["g_critic"][:cut], 3.0 * base[:cut])
        torch.testing.assert_close(r["g_critic"][cut:], k * base[cut:])
    torch.testing.assert_close(r0["g_critic"][:cut], r1["g_critic"][:cut], rtol=0, atol=0)          # replicas identical
    # update_high_utd: the critic range, then [cut, n) = actor/temperature infos + groups 1, 2 + the actor-tx twin (aux tail)
    torch.testing.assert_close(r0["g_utd"], 3.0 * base)
    torch.testing.assert_close(r0["g_utd"], r1["g_utd"], rtol=0, atol=0)
    # update(all three networks): one collective over the whole buffer
    assert r0["n_all"] == [n]
    torch.testing.assert_close(r0["g_all"], 3.0 * base)
    # kernels were asked to pre-scale gradients (and infos) by 1/world
    assert r0["scales"] and all(abs(v - 0.5) < 1e-12 for _, v in r0["scales"])
    assert {k for k, _ in r0["scales"]} == {"critic", "actor"}


def test_fused_critic_step_reduces_the_same_range_in_one_collective(tmp_path):
    """The fused heads (forced onto the dry device) exchange what the per-op chain does: a critic step sums [critic-tx segment |
    critic infos] in ONE collective and leaves the rest alone, replicas identical; update_high_utd and update keep the ranges
    of test_allreduce_segments_and_mean."""
    world, port = 2, 31000 + os.getpid() % 2000
    out = str(tmp_path / "rank{}.pt")
    mp.spawn(_worker, args=(world, port, out, True), nprocs=world, join=True)
    r0, r1 = torch.load(out.format(0)), torch.load(out.format(1))
    n, io = r0["n"], r0["info_off"]
    cut = io + 4
    assert r0["fused"]
    assert r0["n_critic"] == [cut]
    base = torch.arange(n, dtype=torch.float32)
    for r, k in ((r0, 1.0), (r1, 2.0)):
        torch.testing.assert_close(r["g_critic"][:cut], 3.0 * base[:cut])
        torch.testing.assert_close(r["g_critic"][cut:], k * base[cut:])
    torch.testing.assert_close(r0["g_critic"][:cut], r1["g_critic"][:cut], rtol=0, atol=0)          # replicas identical
    torch.testing.assert_close(r0["g_utd"], 3.0 * base)
    torch.testing.assert_close(r0["g_utd"], r1["g_utd"], rtol=0, atol=0)
    assert r0["n_all"] == [n]
