"""What gradient clipping costs in the DrQ critic step, on one GPU.

    python scripts/bench_optimizer_options.py [--clip-grad-norm 1.0] [--steps 100] [--rounds 3] [--precision fp16] [--out result.json]

bench.py's workload (BASELINE configs[2]: two 128x128x3 cameras, batch 256 drawn 50/50 from the online and demo rings,
cross-step pipeline on, whole step replayed as a CUDA graph) with two agents of the same seed on the same rings: one with
the default optimizers and one with `clip_grad_norm` on every tx, which adds the global-norm pass over the flat gradient
buffer and the options variant of the fused Adam.  The two are timed in alternating windows of `--steps` steps (CUDA events,
closed by a device synchronise) after a warm-up that captures every graph variant.  The output is one JSON line with
steps/s per window and arm, the medians, the overhead, and the card's name, power limit and max SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clip-grad-norm", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="fp16", choices=["fp32", "bf16", "fp16"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import bench
    from serl_b200.utils.launcher import make_drq_agent
    w = bench.Workload(args, 2, True, 200_000, 256)
    clip = {"clip_grad_norm": args.clip_grad_norm}
    agents = {"default": w.agent,
              "clip": make_drq_agent(42, w.transitions[0]["observations"], w.transitions[0]["actions"], image_keys=w.cams,
                                     encoder_type="resnet-pretrained", precision=args.precision,
                                     **{f"{tx}_optimizer_kwargs": clip for tx in ("actor", "critic", "temperature")})}
    for name, agent in agents.items():
        agent.pipeline_critic_steps = True
        w.agent = agent
        for _ in range(12):                      # serial, pipeline start and both steady-state variants: eager once, then captured
            agent.update_critics(w.next_batch())
    rates = {name: [] for name in agents}
    for r in range(args.rounds):
        for name in (("default", "clip") if r % 2 == 0 else ("clip", "default")):
            w.agent = agents[name]
            w.agent.update_critics(w.next_batch())           # each window starts the agent's pipeline afresh, untimed
            rates[name].append(1e3 * args.steps / w.timed_steps(args.steps))
    med = {name: statistics.median(v) for name, v in rates.items()}
    out = {"workload": "bench.py configs[2] critic step (2 cameras, batch 256, RLPD 50/50, pipeline, CUDA graph)",
           "precision": args.precision, "clip_grad_norm": args.clip_grad_norm, "card": card(), "steps_per_window": args.steps,
           "steps_per_s": rates, "median_steps_per_s": med, "overhead_pct": 100.0 * (med["default"] / med["clip"] - 1.0)}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    w.close()


if __name__ == "__main__":
    main()
