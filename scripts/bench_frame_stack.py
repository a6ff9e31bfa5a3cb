"""What stacking frames costs: DrQ "small" update_critics at obs_horizon T = 1 and T = 3 on bench.py's workload (fp16, two 128x128
cameras, batch 256 RLPD from a 200k-slot online ring and a demo ring, cross-step pipeline + CUDA graphs).

    python scripts/bench_frame_stack.py [--steps 200] [--windows 5] [--capacity 200000] [--out DIR]

Prints one JSON line: the card and its power limit (read in the same run), steps/s of each setting over alternating timed windows
(median and spread), and each setting's per-step sampler kernel time from a separate torch.profiler run.  Needs a GPU; writes
only under --out (default: a temporary directory).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


class Setup:
    def __init__(self, T, capacity, B=256, cams=("front", "wrist")):
        from bench import fill_ring_synthetic
        from helpers import fake_env, random_transitions
        from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
        from serl_b200.utils.train_utils import concat_batches
        env = fake_env(cams, T=T)
        self.rb = make_replay_buffer(env, capacity=capacity, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=11)
        self.demo = make_replay_buffer(env, capacity=20 * 101, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=12)
        fill_ring_synthetic(self.rb, seed=1)
        fill_ring_synthetic(self.demo, seed=2)
        tr = random_transitions(np.random.default_rng(0), 1, cams, T=T)[0]
        self.agent = make_drq_agent(42, tr["observations"], tr["actions"], image_keys=list(cams), encoder_type="small", precision="fp16")
        self.agent.pipeline_critic_steps = True
        it = self.rb.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True})
        dit = self.demo.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True})
        self.next_batch = lambda: concat_batches(next(it), next(dit), axis=0)

    def steps(self, n):
        for _ in range(n):
            self.agent, _ = self.agent.update_critics(self.next_batch())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--capacity", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_frame_stack.py measures on the GPU"
    out = a.out or tempfile.mkdtemp(prefix="bench_frame_stack_")
    os.makedirs(out, exist_ok=True)
    setups = {T: Setup(T, a.capacity) for T in (1, 3)}
    for s in setups.values():
        s.steps(a.warmup)
    torch.cuda.synchronize()
    rates = {T: [] for T in setups}
    for _ in range(a.windows):                                 # alternating windows: both settings see the same host noise
        for T, s in setups.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s.steps(a.steps)
            torch.cuda.synchronize()
            rates[T].append(a.steps / (time.perf_counter() - t0))
    for s in setups.values():
        s.agent.check_status()
    sampler_us = {}
    from torch.profiler import ProfilerActivity, profile
    for T, s in setups.items():                                # separate profiled run per setting
        n = 20
        s.agent.use_cuda_graphs = False                        # eager launches: every sampler kernel is its own trace event
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s.steps(n)
            torch.cuda.synchronize()
        tot = sum(e.device_time_total for e in prof.key_averages() if "sample_frames" in e.key or "sample_gather_crop" in e.key)
        sampler_us[T] = tot / n
        prof.export_chrome_trace(os.path.join(out, f"trace_T{T}.json"))
    res = {"card": card(), "workload": "DrQ small update_critics, fp16, 2x 128x128 cameras, batch 256 RLPD, pipeline + CUDA graphs",
           "steps_per_window": a.steps, "windows": a.windows}
    for T in setups:
        r = np.array(rates[T])
        res[f"T{T}_steps_per_s_median"] = round(float(np.median(r)), 2)
        res[f"T{T}_steps_per_s_min_max"] = [round(float(r.min()), 2), round(float(r.max()), 2)]
        res[f"T{T}_sampler_us_per_step"] = round(sampler_us[T], 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
