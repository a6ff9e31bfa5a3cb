"""BCAgent.update steps/s in bc_policy.py's training loop (batches drawn from a memory_efficient_replay_buffer iterator with
pack_obs_and_next_obs=True), batch 256, for the fp32 and fp16 builds with one and two 128x128 cameras, and three ways to run
the step:
  - "dict":     the handle materialised with to_dict() and copied into the step's buffers (how every handle ran before the step
                loaded its batch on the device);
  - "eager":    the sampler writes the batch into the step's buffers, kernels launched one by one (use_cuda_graphs=False);
  - "captured": the same step replayed as one CUDA graph.
The variants of one configuration are timed in alternating windows on the same card, so that drift of a shared GPU falls on all
of them.  Prints one JSON line with the card name and power limit.

    python scripts/bench_bc_loop.py [--steps 30] [--windows 3] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from bench_bc_options import _card  # noqa: E402

VARIANTS = ("dict", "eager", "captured")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bc_loop: needs a CUDA device")
    from helpers import fake_env, random_transitions
    from serl_b200.utils.launcher import make_bc_agent, make_replay_buffer
    B = args.batch
    results = {}
    for precision in ("fp32", "fp16"):
        for cams in (("front",), ("front", "wrist")):
            trs = random_transitions(np.random.default_rng(0), 200, cams)
            runs = {}
            for v in VARIANTS:
                agent = make_bc_agent(0, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained",
                                      precision=precision)
                agent.use_cuda_graphs = v == "captured"
                rb = make_replay_buffer(fake_env(cams), capacity=256, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=0)
                for tr in trs:
                    rb.insert(tr)
                it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
                step = (lambda a, i: a.update(next(i).to_dict())) if v == "dict" else (lambda a, i: a.update(next(i)))
                runs[v] = (agent, it, step)
                for _ in range(args.warmup):
                    step(agent, it)
            torch.cuda.synchronize()
            rates = {v: [] for v in VARIANTS}
            for _ in range(args.windows):
                for v, (agent, it, step) in runs.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(args.steps):
                        step(agent, it)
                    torch.cuda.synchronize()
                    rates[v].append(args.steps / (time.perf_counter() - t0))
            for agent, _, _ in runs.values():
                agent.check_status()
            results[f"{precision}/{len(cams)}cam"] = {"windows": rates, "median": {v: statistics.median(r) for v, r in rates.items()}}
            del runs
    name, power = _card()
    print(json.dumps({"metric": "bc_update_steps_per_s", "batch": B, "steps": args.steps, "results": results, "gpu": name,
                      "power_limit": power}))


if __name__ == "__main__":
    main()
