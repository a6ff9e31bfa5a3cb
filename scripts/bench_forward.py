"""Latency of the agents' public forward passes on one GPU.

    python scripts/bench_forward.py [--precision fp16] [--reps 50] [--out result.json]

Dual-camera DrQ agent (128x128 images, the launcher networks, ensemble 10), random observations:

* `forward_critic` latency at batch 1 and 256 (one (B, A) action per state);
* multi-action Q: `forward_critic` with (B, N, A) candidate actions at N = 16 and 64 (B = 32 and 256) against N single-action
  calls on the same states - Q-values per second for both and the speed-up, with the largest relative difference between them;
* unbatched `sample_actions` latency (one observation from the host, actions back on the host, as an actor loop calls it).

Each figure is the median of `--reps` calls, each timed by a host clock around the call and a device synchronise, after warm-up
calls of every shape.  The card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="fp16")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_forward.py measures on a GPU"
    from helpers import random_transitions
    from serl_b200.utils.launcher import make_drq_agent
    cams, A = ("front", "wrist"), 4
    trs = random_transitions(np.random.default_rng(0), 2, cams)
    agent = make_drq_agent(0, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained",
                           precision=args.precision)
    rng = np.random.default_rng(1)
    key = np.array([0, 1], np.uint32)

    def obs(B):
        o = {c: torch.as_tensor(rng.integers(0, 256, (B, 1, 128, 128, 3), dtype=np.uint8), device="cuda") for c in cams}
        o["state"] = torch.as_tensor(rng.standard_normal((B, 1, 7)).astype(np.float32), device="cuda")
        return o

    res = {"card": card(), "precision": args.precision, "cameras": len(cams), "ensemble": agent._cfg.ensemble, "reps": args.reps}
    for B in (1, 256):
        o, a = obs(B), torch.as_tensor(rng.uniform(-1, 1, (B, A)).astype(np.float32), device="cuda")
        res[f"forward_critic_ms_B{B}"] = 1e3 * timed(lambda: agent.forward_critic(o, a, key), args.reps)
    for B in (32, 256):
        o = obs(B)
        for N in (16, 64):
            a = torch.as_tensor(rng.uniform(-1, 1, (B, N, A)).astype(np.float32), device="cuda")
            singles = [a[:, n].contiguous() for n in range(N)]
            reps = max(3, args.reps // (4 if N == 64 else 2))
            t_multi = timed(lambda: agent.forward_critic(o, a, key), reps)
            t_single = timed(lambda: [agent.forward_critic(o, s, key) for s in singles], reps)
            q_multi = agent.forward_critic(o, a, key)
            q_single = torch.stack([agent.forward_critic(o, s, key) for s in singles], -1)
            diff = float((q_multi - q_single).abs().max() / q_single.abs().max())
            res[f"multi_action_B{B}_N{N}"] = {"multi_ms": 1e3 * t_multi, "n_single_calls_ms": 1e3 * t_single,
                                              "multi_q_per_s": B * N / t_multi, "single_q_per_s": B * N / t_single,
                                              "speedup": t_single / t_multi, "max_rel_diff": diff}
    one = {k: v[0].cpu().numpy() for k, v in obs(1).items()}
    res["sample_actions_unbatched_ms"] = 1e3 * timed(lambda: agent.sample_actions(one, seed=key), args.reps)
    res["sample_actions_unbatched_argmax_ms"] = 1e3 * timed(lambda: agent.sample_actions(one, argmax=True), args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
