"""VICE on bench.py's workload: fp16, two 128x128 cameras, batch 256 (RLPD halves from a 200k online ring and a demo ring).

* `update_critics` of the VICE agent (reward relabelling from the step's own trunk features) next to bench.py's DrQ agent, on one
  pair of rings, each agent through its own iterators, cross-step pipeline and CUDA graphs on, in alternating timed windows
  (default three of 100 steps each);
* `update_vice` steps/s at batch 256: 128 next observations from the online ring, 128 goals from the demo ring.

Prints one JSON line with the GPU's name and power limit (read in the same run), per-arm medians of steps/s and kernel launches
per step.

    python scripts/bench_vice.py [--windows 3] [--steps 100] [--warmup 10] [--vice-steps 20]
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
    ap.add_argument("--vice-steps", type=int, default=20)
    a = ap.parse_args()
    import torch
    from bench import Workload
    from serl_b200.utils.launcher import make_vice_agent
    from serl_b200.utils.train_utils import concat_batches
    torch.cuda.set_device(0)
    w = Workload(types.SimpleNamespace(precision="fp16"), 2, True, 200_000, 256)     # rings + the DrQ agent of bench.py
    tr = w.transitions[0]
    vice = make_vice_agent(42, tr["observations"], tr["actions"], image_keys=w.cams, vice_image_keys=w.cams,
                           encoder_type="resnet-pretrained", precision="fp16")
    agents = {"drq": w.agent, "vice": vice}
    half = w.B // 2
    arms = {}
    for name, agent in agents.items():
        it = w.rb.get_iterator(sample_args={"batch_size": half, "pack_obs_and_next_obs": True})
        dit = w.demo.get_iterator(sample_args={"batch_size": w.B - half, "pack_obs_and_next_obs": True})
        agent.pipeline_critic_steps = True
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
        out[f"update_critics_{name}"] = {"steps_per_s_median": statistics.median(rates), "steps_per_s": rates,
                                         "gpu_launches_per_step": statistics.median(launches),
                                         "critic_loss": float(last["info"]["critic"]["critic_loss"])}
    out["vice_over_drq"] = out["update_critics_vice"]["steps_per_s_median"] / out["update_critics_drq"]["steps_per_s_median"]
    it = w.rb.get_iterator(sample_args={"batch_size": half, "pack_obs_and_next_obs": True})
    git = w.demo.get_iterator(sample_args={"batch_size": w.B - half, "pack_obs_and_next_obs": True})
    for _ in range(3):
        vice.update_vice(concat_batches(next(it), next(git), axis=0))
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = vice.kernel_launches
    t0.record()
    for _ in range(a.vice_steps):
        _, info = vice.update_vice(concat_batches(next(it), next(git), axis=0))
    t1.record()
    torch.cuda.synchronize()
    out["update_vice"] = {"steps_per_s": 1e3 * a.vice_steps / t0.elapsed_time(t1), "steps": a.vice_steps,
                          "gpu_launches_per_step": (vice.kernel_launches - l0) / a.vice_steps,
                          "bce_loss": float(info["vice"]["bce_loss"]), "grad_norm": float(info["vice"]["grad_norm"])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
