"""Cost of feeding a data-parallel learner from one actor: critic-step throughput of bench.py's workload (fp16, two 128x128
cameras, global batch 256 drawn 50/50 from a 200k online ring and a demo ring, cross-step pipeline and CUDA graphs) while an
actor thread on rank 0 inserts synthetic transitions into a `DataParallelDataStore` at a fixed rate.

Both rings are wrapped (the learner loop of INTEGRATION.md), so every draw syncs: rank 0's pending transitions are pickled and
broadcast over the store's gloo group and inserted into every replica.  Each rank holds a full 200k replica, filled with the
same synthetic frames as bench.py's ring.  The rates run in alternating timed windows (default three windows of 200 steps per
rate); the script prints one JSON line with, per rate: steps/s (median over windows, each window timed with CUDA events and
taken on the slowest rank), the median time per step spent inside sync() (both rings, slowest rank) and the payload bytes per
sync of the online ring.  With one process the store is a pass-through: the actor inserts straight into the ring.

    torchrun --nproc-per-node N scripts/bench_dp_ingest.py [--rates 0,10,100] [--windows 3] [--steps 200] [--warmup 10]
    python scripts/bench_dp_ingest.py ...                                  (one GPU)
"""
from __future__ import annotations

import argparse
import json
import os
import pickle
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _gpu():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:                                   # noqa: BLE001
        return "unknown"


class Actor(threading.Thread):
    """Inserts transitions into the store at `rate` Hz (0: idle) until stopped."""

    def __init__(self, store, transitions):
        super().__init__(daemon=True)
        self.store, self.transitions, self.rate, self.sent = store, transitions, 0.0, 0
        self.stop = threading.Event()

    def run(self):
        nxt = time.perf_counter()
        while not self.stop.is_set():
            if self.rate <= 0:
                time.sleep(0.001)
                nxt = time.perf_counter()
                continue
            self.store.insert(self.transitions[self.sent % len(self.transitions)])
            self.sent += 1
            nxt += 1.0 / self.rate
            time.sleep(max(0.0, nxt - time.perf_counter()))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rates", default="0,10,100", help="actor insert rates in Hz, comma-separated")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    rates = [float(r) for r in a.rates.split(",")]
    import torch
    import torch.distributed as dist
    from bench import fill_ring_synthetic
    from helpers import fake_env, random_transitions
    from serl_b200.utils.launcher import init_data_parallel, make_drq_agent, make_replay_buffer
    from serl_b200.utils.train_utils import concat_batches
    rank, world = init_data_parallel()
    batch, cams = 256, ("cam0", "cam1")
    env = fake_env(cams)
    kw = dict(type="memory_efficient_replay_buffer", image_keys=list(cams), data_parallel=True)
    rb = make_replay_buffer(env, capacity=200_000, seed=1000, **kw)
    demo = make_replay_buffer(env, capacity=20 * 101, seed=1500, **kw)
    fill_ring_synthetic(rb.store, seed=0)                     # the same contents on every rank: replicas
    fill_ring_synthetic(demo.store, seed=100)
    transitions = random_transitions(np.random.default_rng(0), 16, cams, mean_ep=1000)
    agent = make_drq_agent(42, transitions[0]["observations"], transitions[0]["actions"], image_keys=cams,
                           encoder_type="resnet-pretrained", precision="fp16")
    agent.data_parallel = world > 1
    agent.pipeline_critic_steps = True
    sync_s = []                                               # host seconds inside sync(), both rings, of the current step

    def timed(sync):
        def run():
            t = time.perf_counter()
            try:
                return sync()
            finally:
                sync_s.append(time.perf_counter() - t)
        return run

    rb.sync, demo.sync = timed(rb.sync), timed(demo.sync)
    half = {"batch_size": batch // 2, "pack_obs_and_next_obs": True}
    it, dit = rb.get_iterator(sample_args=half), demo.get_iterator(sample_args=half)
    next_batch = lambda: concat_batches(next(it), next(dit), axis=0)
    actor = Actor(rb, transitions) if rank == 0 else None
    if actor is not None:
        actor.start()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def window(rate, steps):
        if actor is not None:
            actor.rate = rate
        barrier()
        b0 = rb.sync_bytes
        del sync_s[:]
        per_step = []
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(steps):
            k = len(sync_s)
            agent.update_critics(next_batch())
            per_step.append(sum(sync_s[k:]))
        t1.record()
        barrier()
        n_sync = len(sync_s) // 2                             # one sync per ring per step
        stats = torch.tensor([t0.elapsed_time(t1), 1e3 * statistics.median(per_step)], dtype=torch.float64, device="cuda")
        if world > 1:
            dist.all_reduce(stats, op=dist.ReduceOp.MAX)
        ms, sync_ms = stats.tolist()
        return 1e3 * steps / ms, sync_ms, (rb.sync_bytes - b0) / max(n_sync, 1)

    for _ in range(a.warmup + 6):                             # pipeline graph variants: eager once, captured on second use
        agent.update_critics(next_batch())
    for r in rates:                                           # untimed: each rate once, so the first timed window is not special
        window(r, 20)
    res = {r: {"steps_per_s": [], "sync_ms_per_step": [], "payload_bytes_per_sync": []} for r in rates}
    for _ in range(a.windows):
        for r in rates:
            sps, sms, pb = window(r, a.steps)
            res[r]["steps_per_s"].append(sps)
            res[r]["sync_ms_per_step"].append(sms)
            res[r]["payload_bytes_per_sync"].append(pb)
    if actor is not None:
        actor.stop.set()
        actor.join(timeout=10)
    agent.check_status()
    agent._graphs.clear()                                     # captured NCCL kernels must not outlive the process group
    torch.cuda.synchronize()
    if rank == 0:
        tr_bytes = len(pickle.dumps(transitions[0], protocol=pickle.HIGHEST_PROTOCOL))
        out = {"workload": "bench.py critic step, fp16, 2x 128x128 cameras, global batch 256 RLPD, 200k replica per rank, "
                           "pipeline + CUDA graphs, both rings DataParallelDataStore", "gpu": _gpu(), "world": world,
               "windows": a.windows, "steps_per_window": a.steps, "pickled_transition_bytes": tr_bytes,
               "rates": {f"{r:g}Hz": {**v, "steps_per_s_median": statistics.median(v["steps_per_s"]),
                                      "sync_ms_per_step_median": statistics.median(v["sync_ms_per_step"]),
                                      "payload_bytes_per_sync_median": statistics.median(v["payload_bytes_per_sync"])}
                         for r, v in res.items()}}
        print(json.dumps(out), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
