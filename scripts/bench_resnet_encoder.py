"""Critic-step throughput of the DrQ agent with the trainable "resnet" encoder (a ResNet-10 trained end to end) next to the
"resnet-pretrained" agent (frozen trunk) on bench.py's workload: fp16, two 128x128 cameras, batch 256 (RLPD halves from a 200k
online ring and a demo ring), cross-step pipeline and CUDA graphs on (for the trainable encoder the pipeline prefetches the
sampler only: its convs depend on the parameters each step writes).

The two agents share bench.py's rings, each through its own iterators, and run in alternating timed windows (default three of
100 steps each).  The script prints one JSON line: the per-arm medians of steps/s, the library kernel launches per step, and the
GPU's name and power limit read in the same run.  The numbers in README.md were taken with `--windows 3 --steps 30` (and
`--profile --steps 5 --warmup 2`).

    python scripts/bench_resnet_encoder.py [--windows 3] [--steps 100] [--warmup 10]
    python scripts/bench_resnet_encoder.py --profile [--steps 20]

--profile runs only the trainable arm, eagerly, under torch.profiler, and prints the per-launch times of the encoder's conv,
GroupNorm and max-pool kernels and the achieved TFLOP/s of the conv work a step needs (computed from the layer shapes below).

Useful work per critic step, from the shapes (not measured): forward 290.2 M MAC per 128x128 image, run on 3 B images per
camera (online obs, online next obs, target next obs); wgrad 290.2 M MAC and dgrad 251.7 M MAC (no stem dgrad) on the B obs
images: 2.83 GFLOP per row per camera, 1.45 TFLOP per step at batch 256 with two cameras.  At the data sheet's 495 TFLOP/s
dense TF32 and three MMAs per 3xTF32 product that is >= 8.8 ms of tensor-core time per step: a bound, not a measurement.
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

def conv_macs(hw: int = 128):
    """(leaf, multiply-adds per image) of each conv of the trainable ResNet-10, in forward order."""
    from serl_b200.engine import resnet_convs
    out = []
    for leaf, k, st, lo, hi, H, ci, co in resnet_convs(hw):
        o = (H + lo + hi - k) // st + 1
        out.append((leaf, o * o * co * k * k * ci))
    return out


def conv_flops_per_step(B: int, cams: int) -> float:
    """Useful FLOPs (2 per multiply-add) of the encoder convs in one critic step: forward on 3B images per camera, wgrad of every
    conv and dgrad of every conv but the stem on the B obs images."""
    mac = [m for _, m in conv_macs()]
    return 2.0 * cams * B * (3 * sum(mac) + sum(mac) + sum(mac[1:]))


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
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    from bench import Workload
    from serl_b200.utils.launcher import make_drq_agent
    from serl_b200.utils.train_utils import concat_batches
    torch.cuda.set_device(0)
    w = Workload(types.SimpleNamespace(precision="fp16"), 2, True, 200_000, 256)     # rings + the resnet-pretrained agent of bench.py
    tr = w.transitions[0]
    res = make_drq_agent(42, tr["observations"], tr["actions"], image_keys=w.cams, encoder_type="resnet", precision="fp16")
    agents = {"resnet": res} if a.profile else {"resnet_pretrained": w.agent, "resnet": res}
    half = w.B // 2
    arms = {}
    for name, agent in agents.items():
        it = w.rb.get_iterator(sample_args={"batch_size": half, "pack_obs_and_next_obs": True})
        dit = w.demo.get_iterator(sample_args={"batch_size": w.B - half, "pack_obs_and_next_obs": True})
        agent.pipeline_critic_steps = not a.profile
        agent.use_cuda_graphs = not a.profile
        arms[name] = (agent, lambda it=it, dit=dit: concat_batches(next(it), next(dit), axis=0), [], [], {})
        for _ in range(a.warmup + 6):                   # graph variants of the pipeline: eager once, captured on second use
            agent.update_critics(arms[name][1]())
    torch.cuda.synchronize()
    out = {"workload": "bench.py critic step, fp16, 2x 128x128 cameras, batch 256 RLPD, 200k ring"
                       + (", eager steps under torch.profiler" if a.profile else ", pipeline + CUDA graphs"),
           "gpu": _gpu()}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        next_batch = arms["resnet"][1]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                res.update_critics(next_batch())
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if any(n in ev.key for n in ("rconv", "rn_", "conv_igemm", "groupnorm", "maxpool")):
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                kern[ev.key] = {"launches_per_step": ev.count / a.steps, "us_per_launch": t / max(ev.count, 1),
                                "us_per_step": t / a.steps}
        conv_us = sum(k["us_per_step"] for n, k in kern.items() if "rconv_kernel" in n)
        flops = conv_flops_per_step(w.B, len(w.cams))
        out.update(kernels=kern, conv_us_per_step=conv_us, conv_gflop_per_step=flops / 1e9,
                   conv_tflops_achieved=flops / (conv_us * 1e-6) / 1e12,
                   encoder_us_per_step=sum(k["us_per_step"] for k in kern.values()))
        print(json.dumps(out))
        return
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
    out.update(windows=a.windows, steps_per_window=a.steps)
    for name, (agent, _, rates, launches, last) in arms.items():
        agent.check_status()
        out[name] = {"steps_per_s_median": statistics.median(rates), "steps_per_s": rates,
                     "gpu_launches_per_step": statistics.median(launches), "critic_loss": float(last["info"]["critic"]["critic_loss"])}
    out["resnet_over_resnet_pretrained"] = out["resnet"]["steps_per_s_median"] / out["resnet_pretrained"]["steps_per_s_median"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
