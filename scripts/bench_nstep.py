"""n-step replay targets: critic-step throughput and sampler kernel time, n_step = 1 vs 3, on bench.py's flagship workload.

    python scripts/bench_nstep.py [--steps 200] [--windows 4] [--out DIR]

The workload is bench.py's (`Workload`): DrQ update_critics, fp16, two 128x128x3 cameras, batch 256 RLPD (128 rows from a
200k-slot online ring, 128 from a demo ring), pretrained ResNet-10, the cross-step pipeline and CUDA graphs.  The same agent
draws from two pairs of iterators over the same rings, one with sample_args n_step = 1 and one with n_step = 3 (the agent's
discount); timed windows of `--steps` steps alternate between them, CUDA events around each window.  A separate profiled run
(torch.profiler, CUDA activity) of 20 steps per setting sums the device time of the sampler kernels per step.  Prints one JSON
line; with --out, also writes it and the profiler tables there.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SAMPLER = re.compile(r"sample_(frames|gather_crop)\w*kernel")


def gpu_conditions():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:                      # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")])) if "," in out else {"nvidia-smi": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="critic steps per timed window")
    ap.add_argument("--windows", type=int, default=4, help="timed windows per setting, alternating n_step = 1 and 3")
    ap.add_argument("--n-step", type=int, default=3)
    ap.add_argument("--precision", default="fp16", choices=["fp32", "bf16", "fp16"])
    ap.add_argument("--out", default=None, help="directory for the JSON line and the profiler tables")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_nstep.py measures on a CUDA device; none is available")
    import bench
    from serl_b200.utils.train_utils import concat_batches

    torch.cuda.set_device(0)
    w = bench.Workload(argparse.Namespace(precision=args.precision), 2, True, 200_000, 256)
    agent, half = w.agent, w.B // 2
    disc = agent.config["discount"]
    sources = {}
    for n in (1, args.n_step):
        sa = {"batch_size": half, "pack_obs_and_next_obs": True}
        if n > 1:
            sa.update(n_step=n, discount=disc)
        it, dit = w.rb.get_iterator(sample_args=sa), w.demo.get_iterator(sample_args={**sa, "batch_size": w.B - half})
        sources[n] = (lambda it=it, dit=dit: concat_batches(next(it), next(dit), axis=0))

    def run(n, steps):
        nb = sources[n]
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            _, info = agent.update_critics(nb())
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b)

    for n in sources:                                        # every graph variant of both settings captured before timing
        run(n, 12)
    rates = {n: [] for n in sources}
    t0 = time.time()
    for _ in range(args.windows):
        for n in sources:
            rates[n].append(1e3 * args.steps / run(n, args.steps))
    wall = time.time() - t0
    agent.check_status()

    kern = {}
    tables = {}
    prof_steps = 20
    for n in sources:
        run(n, 4)
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            run(n, prof_steps)
        us, names = 0.0, set()
        for e in prof.key_averages():
            if SAMPLER.search(e.key):
                us += e.device_time_total
                names.add(e.key)
        kern[n] = {"us_per_step": us / prof_steps, "kernels": sorted(names)}
        tables[n] = prof.key_averages().table(sort_by="device_time_total", row_limit=25)

    med = lambda v: sorted(v)[len(v) // 2]
    line = {"metric": "critic steps/s, n_step 1 vs 3 (alternating windows)", "gpu": gpu_conditions(), "precision": args.precision,
            "workload": "bench.py: DrQ update_critics, 2x 128x128x3 cameras, batch 256 RLPD, pipeline + CUDA graphs",
            "steps_per_window": args.steps, "windows": args.windows, "wall_s": wall,
            "steps_per_s": {str(n): {"median": med(v), "all": v} for n, v in rates.items()},
            "sampler_kernel_us_per_step": {str(n): v for n, v in kern.items()}}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_nstep.json"), "w") as f:
            f.write(json.dumps(line) + "\n")
        for n, t in tables.items():
            with open(os.path.join(args.out, f"bench_nstep_profile_n{n}.txt"), "w") as f:
                f.write(t)
    w.close()


if __name__ == "__main__":
    main()
