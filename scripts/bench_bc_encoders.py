"""BCAgent.update steps/s for each encoder type ("resnet-pretrained", "small", "resnet") on one GPU, eager and replayed as CUDA
graphs: the launcher's network (make_bc_agent: tanh [256, 256], proprio, "exp" std), two 128x128 cameras, batch 256, batches
drawn from a memory_efficient_replay_buffer iterator (bc_policy.py's loop; a ring batch is what the step captures).  The six
configurations are timed in alternating windows, so that drift of a shared GPU falls on all of them.  Prints a markdown table and
one JSON line, both with the card name and power limit.

    python scripts/bench_bc_encoders.py [--steps 30] [--windows 3] [--precision fp16]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ENCODERS = ("resnet-pretrained", "small", "resnet")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def _env(cams, hw, S, A):
    box = lambda shape, dtype=np.float32: types.SimpleNamespace(shape=tuple(shape), dtype=np.dtype(dtype))
    obs = types.SimpleNamespace(spaces={**{c: box((1, hw, hw, 3), np.uint8) for c in cams}, "state": box((1, S))})
    return types.SimpleNamespace(observation_space=obs, action_space=box((A,)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--precision", default="fp16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bc_encoders: needs a CUDA device")
    from bench import fill_ring_synthetic
    from serl_b200.utils.launcher import make_bc_agent, make_replay_buffer
    cams, B, A, S, hw = ("front", "wrist"), args.batch, 7, 19, 128
    sample = {**{c: np.zeros((1, hw, hw, 3), np.uint8) for c in cams}, "state": np.zeros((1, S), np.float32)}
    runs = {}
    for i, enc in enumerate(ENCODERS):
        for graphs in (False, True):
            rb = make_replay_buffer(_env(cams, hw, S, A), capacity=20 * 101, type="memory_efficient_replay_buffer", image_keys=list(cams),
                                    seed=11 + i)
            fill_ring_synthetic(rb, seed=i)
            agent = make_bc_agent(0, sample, np.zeros(A, np.float32), image_keys=cams, encoder_type=enc, precision=args.precision)
            agent.use_cuda_graphs = graphs
            runs[(enc, graphs)] = (agent, rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True}))
    for agent, it in runs.values():
        for _ in range(args.warmup):
            agent.update(next(it))
    torch.cuda.synchronize()
    rates = {k: [] for k in runs}
    for _ in range(args.windows):
        for k, (agent, it) in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                agent.update(next(it))
            torch.cuda.synchronize()
            rates[k].append(args.steps / (time.perf_counter() - t0))
    for agent, _ in runs.values():
        agent.check_status()
        assert agent.use_cuda_graphs == bool(agent._graphs)
    name, power = _card()
    med = {k: statistics.median(v) for k, v in rates.items()}
    print(f"BCAgent.update, {args.precision} build, {len(cams)} x {hw}x{hw} cameras, batch {B}, launcher network, {name} at {power}")
    print("| encoder_type | eager steps/s | CUDA graphs steps/s |")
    print("|---|---|---|")
    for enc in ENCODERS:
        print(f"| {enc} | {med[(enc, False)]:.1f} | {med[(enc, True)]:.1f} |")
    print(json.dumps({"metric": "bc_update_steps_per_s", "precision": args.precision, "batch": B, "cameras": len(cams), "steps": args.steps,
                      "windows": {f"{e}/{'graphs' if g else 'eager'}": v for (e, g), v in rates.items()},
                      "median": {f"{e}/{'graphs' if g else 'eager'}": v for (e, g), v in med.items()}, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
