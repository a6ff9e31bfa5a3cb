"""Prioritized replay: critic-step throughput and kernel times on bench.py's flagship workload.

    python scripts/bench_per.py [--steps 200] [--windows 3] [--out DIR]

The workload is bench.py's (`Workload`): DrQ update_critics, fp16, two 128x128x3 cameras, batch 256 RLPD (128 rows from a
200k-slot online ring, 128 from a uniform demo ring), pretrained ResNet-10 and CUDA graphs.  Three arms share the agent
type and the demo ring's content:
  uniform+pipeline   the uniform online ring, pipeline_critic_steps=True (bench.py's setting);
  uniform serial     the same ring, pipeline off;
  prioritized        an online ring with the same content built with priority_alpha=0.6 (a prioritized batch always runs the
                     serial step: its draw reads the priorities the previous step wrote).
Timed windows of `--steps` steps alternate between the arms, CUDA events around each window.  A separate torch.profiler run
(CUDA activity) of 20 steps per arm sums the device time of the sampler kernels and of the priority writes per step.  A third
part times one launch each of the uniform and the prioritized draw on state-only rings of 200k and 1M slots (the same kernel,
so the difference is the tree descent) and of priority_set_kernel writing 128 slots, with CUDA events over 200 launches.
Prints one JSON line; with --out, also writes it and the profiler tables there.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

KERNELS = {"sampler": re.compile(r"sample_(frames|gather_crop)\w*kernel"), "priority_set": re.compile(r"priority_set_kernel"),
           "priority_weights": re.compile(r"priority_weights_kernel")}


def _prioritize(rb):
    """Leaves of a ring whose slots were written directly (bench.fill_ring_synthetic): m = 1 on every valid slot."""
    from serl_b200 import ops
    cap = rb._capacity
    rb.tree[:cap] = rb.valid.float()
    ops.priority_rebuild(rb.priority_tree())


def _draw_launch_us(cap, alpha, batch=128, reps=200):
    """Mean device time of one state-only draw + gather launch of `batch` rows from a full ring of `cap` slots."""
    import torch
    from helpers import Box
    from serl_b200 import _lib as L
    from serl_b200 import ops
    from serl_b200.data.replay_buffer import ReplayBuffer
    rb = ReplayBuffer(Box((7,)), Box((4,)), cap, seed=1, priority_alpha=alpha)
    rb.valid.fill_(1)
    rb._valid_host[:] = True
    rb._size = cap
    rb.size_dev.fill_(cap)
    if alpha is not None:
        g = torch.Generator(device="cuda").manual_seed(0)
        rb.tree[:cap] = torch.rand(cap, device="cuda", generator=g) + 0.01
        ops.priority_rebuild(rb.priority_tree())
    e = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device="cuda")
    st, nst, ac, rw, mk, dn, idx = e(batch, 7), e(batch, 7), e(batch, 4), e(batch), e(batch), e(batch, dt=torch.uint8), e(batch, dt=torch.int32)
    prio, status = e(batch), torch.zeros(1, dtype=torch.int32, device="cuda")
    out = L.BatchOut()
    out.obs_state, out.next_state, out.actions, out.rewards, out.masks = st.data_ptr(), nst.data_ptr(), ac.data_ptr(), rw.data_ptr(), mk.data_ptr()
    out.dones, out.idx, out.status = dn.data_ptr(), idx.data_ptr(), status.data_ptr()

    def launch(step):
        part = dict(ring=rb, seed=rb._seed, step=step, batch=batch, indx=None)
        rb.launch_sample(part, out, crop_total=batch, out_row_offset=0, record_event=False, prio_out=prio if alpha is not None else None)

    for s in range(10):
        launch(s)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for s in range(reps):
        launch(s)
    b.record()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    return 1e3 * a.elapsed_time(b) / reps


def _priority_set_us(cap, n=128, reps=200):
    import torch
    from serl_b200 import ops
    from serl_b200.data.replay_buffer import _tree_nodes
    tree = torch.zeros(_tree_nodes(cap), device="cuda")
    mx = torch.ones(1, device="cuda")
    t = ops.priority_tree(tree, mx, cap)
    g = torch.Generator(device="cuda").manual_seed(0)
    slots = torch.randint(0, cap, (reps + 10, n), device="cuda", generator=g, dtype=torch.int32)
    td = torch.randn(reps + 10, n, device="cuda", generator=g)
    for r in range(10):
        ops.priority_set(t, slots[r], n, td=td[r], alpha=0.6, eps=1e-6)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for r in range(10, reps + 10):
        ops.priority_set(t, slots[r], n, td=td[r], alpha=0.6, eps=1e-6)
    b.record()
    torch.cuda.synchronize()
    return 1e3 * a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="critic steps per timed window")
    ap.add_argument("--windows", type=int, default=3, help="timed windows per arm, alternating")
    ap.add_argument("--precision", default="fp16", choices=["fp32", "bf16", "fp16"])
    ap.add_argument("--out", default=None, help="directory for the JSON line and the profiler tables")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_per.py measures on a CUDA device; none is available")
    import bench
    from bench_nstep import gpu_conditions
    from helpers import fake_env
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    from serl_b200.utils.train_utils import concat_batches

    torch.cuda.set_device(0)
    w = bench.Workload(argparse.Namespace(precision=args.precision), 2, True, 200_000, 256)
    half = w.B // 2
    prb = make_replay_buffer(fake_env(w.cams), capacity=w.rb._capacity, type="memory_efficient_replay_buffer", image_keys=list(w.cams),
                             seed=1000, priority_alpha=0.6)
    bench.fill_ring_synthetic(prb, seed=0)
    _prioritize(prb)
    tr = w.transitions[0]
    agents = {k: make_drq_agent(42, tr["observations"], tr["actions"], image_keys=w.cams, encoder_type="resnet-pretrained",
                                precision=args.precision) for k in ("uniform+pipeline", "uniform serial", "prioritized")}
    agents["uniform+pipeline"].pipeline_critic_steps = True
    sa = {"batch_size": half, "pack_obs_and_next_obs": True}
    src = {k: (w.rb if k != "prioritized" else prb).get_iterator(sample_args=sa) for k in agents}
    dsrc = {k: w.demo.get_iterator(sample_args={**sa, "batch_size": w.B - half}) for k in agents}

    def run(k, steps):
        agent = agents[k]
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            agents[k], _ = agent.update_critics(concat_batches(next(src[k]), next(dsrc[k]), axis=0))
            agent = agents[k]
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b)

    for k in agents:
        run(k, 12)
    rates = {k: [] for k in agents}
    t0 = time.time()
    for _ in range(args.windows):
        for k in agents:
            rates[k].append(1e3 * args.steps / run(k, args.steps))
    wall = time.time() - t0
    for a in agents.values():
        a.check_status()

    kern, tables, prof_steps = {}, {}, 20
    for k in agents:
        run(k, 4)
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            run(k, prof_steps)
        per = {}
        for name, pat in KERNELS.items():
            us, names = 0.0, set()
            for e in prof.key_averages():
                if pat.search(e.key):
                    us += e.device_time_total
                    names.add(e.key)
            per[name] = {"us_per_step": us / prof_steps, "kernels": sorted(names)}
        kern[k] = per
        tables[k] = prof.key_averages().table(sort_by="device_time_total", row_limit=25)

    launches = {}
    for cap in (200_000, 1_000_000):
        launches[str(cap)] = {"uniform_draw_us": _draw_launch_us(cap, None), "prioritized_draw_us": _draw_launch_us(cap, 0.6),
                              "priority_set_128_us": _priority_set_us(cap)}

    med = lambda v: sorted(v)[len(v) // 2]
    line = {"metric": "critic steps/s: uniform+pipeline, uniform serial, prioritized (alternating windows)", "gpu": gpu_conditions(),
            "precision": args.precision,
            "workload": "bench.py: DrQ update_critics, 2x 128x128x3 cameras, batch 256 RLPD (200k online ring, uniform demo ring), CUDA graphs",
            "steps_per_window": args.steps, "windows": args.windows, "wall_s": wall,
            "steps_per_s": {k: {"median": med(v), "all": v} for k, v in rates.items()},
            "kernel_us_per_step": kern,
            "single_launch_us (state-only rings, batch 128; priority_set: 128 slots)": launches}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_per.json"), "w") as f:
            f.write(json.dumps(line) + "\n")
        for k, t in tables.items():
            with open(os.path.join(args.out, f"bench_per_profile_{k.replace(' ', '_').replace('+', '_')}.txt"), "w") as f:
                f.write(t)
    w.close()


if __name__ == "__main__":
    main()
