"""Critic-step throughput of the pixel-only DrQ agent (use_proprio=False) next to the proprio agent on bench.py's workload: fp16,
two 128x128 cameras, batch 256 (RLPD halves from a 200k online ring and a demo ring), cross-step pipeline and CUDA graphs on.

One pair of rings, built and filled as bench.py builds them (they store a state vector), serves both agents, each through its own
iterators.  The pixel-only agent's sampler writes the state rows to scratch, so the sampler does the same work in both arms and
the difference is the heads (no proprio finish problems, first-layer K smaller by 64).  The two agents run in alternating timed
windows (default three of 100 steps each; a window's first step restarts the pipeline, in both arms alike); the script prints one
JSON line with the per-arm medians of steps/s and the library kernel launches per step.

    python scripts/bench_pixel_only.py [--windows 3] [--steps 100] [--warmup 10]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import types

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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    import torch
    from bench import Workload
    from pixel_only import make_agent
    from serl_b200.utils.train_utils import concat_batches
    torch.cuda.set_device(0)
    w = Workload(types.SimpleNamespace(precision="fp16"), 2, True, 200_000, 256)     # rings + the proprio agent of bench.py
    tr = w.transitions[0]
    agents = {"proprio": w.agent,
              "pixel_only": make_agent(42, tr["observations"], tr["actions"], w.cams, use_proprio=False, precision="fp16")}
    half = w.B // 2
    arms = {}
    for name, agent in agents.items():
        it = w.rb.get_iterator(sample_args={"batch_size": half, "pack_obs_and_next_obs": True})
        dit = w.demo.get_iterator(sample_args={"batch_size": w.B - half, "pack_obs_and_next_obs": True})
        agent.pipeline_critic_steps = True
        assert agent._engine(w.B).fused is not None, name
        arms[name] = (agent, lambda it=it, dit=dit: concat_batches(next(it), next(dit), axis=0), [], [], {})
        for _ in range(a.warmup + 6):                   # graph variants of the pipeline: eager once, captured on second use
            agent.update_critics(arms[name][1]())
    for _ in range(2):                                  # untimed alternations: the restart variant is captured before timing
        for agent, next_batch, *_ in arms.values():
            for _ in range(3):
                agent.update_critics(next_batch())
    torch.cuda.synchronize()
    for _ in range(a.windows):
        for name, (agent, next_batch, rates, launches, last) in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0 = agent.kernel_launches
            torch.cuda.synchronize()
            t0.record()
            for _ in range(a.steps):
                _, last["info"] = agent.update_critics(next_batch())
            t1.record()
            torch.cuda.synchronize()
            rates.append(1e3 * a.steps / t0.elapsed_time(t1))
            launches.append((agent.kernel_launches - l0) / a.steps)
    out = {"workload": "bench.py critic step, fp16, 2x 128x128 cameras, batch 256 RLPD, 200k ring, pipeline + CUDA graphs",
           "gpu": _gpu(), "windows": a.windows, "steps_per_window": a.steps}
    for name, (agent, _, rates, launches, last) in arms.items():
        agent.check_status()
        out[name] = {"steps_per_s_median": statistics.median(rates), "steps_per_s": rates,
                     "gpu_launches_per_step": statistics.median(launches), "critic_loss": float(last["info"]["critic"]["critic_loss"])}
    out["pixel_only_over_proprio"] = out["pixel_only"]["steps_per_s_median"] / out["proprio"]["steps_per_s_median"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
