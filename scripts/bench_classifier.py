"""Reward-classifier throughput and actor-side latency on one GPU.

    python scripts/bench_classifier.py [--batch 256] [--out result.json]

* train steps/s at batch B for 1 and 2 cameras, fp16 and fp32 builds: each step is sample_classifier_batch (two sampler
  launches from a positive and a negative HBM replay ring) + train_step; windows of >= 1 s of steps closed by a device
  synchronise after a warm-up, median of 3 windows;
* the per-env-step cost on the actor: one unbatched (1, 128, 128, 3) host observation through load_classifier_func's callable,
  H2D copy and `.item()` included (median of 200 calls);
* the card's name, power limit and max SM clock, read in the same run.
"""
import argparse
import json
import os
import statistics
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def make_buffers(cams, n, seed):
    from helpers import fake_env, random_transitions
    from serl_b200.utils.launcher import make_replay_buffer
    rng = np.random.default_rng(seed)
    out = []
    for s in (seed, seed + 1):
        rb = make_replay_buffer(fake_env(cams), capacity=n + 64, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=s)
        for tr in random_transitions(rng, n, cams, mean_ep=50):
            rb.insert(tr)
        out.append(rb)
    return out


def train_rate(cams, precision, B, pos, neg):
    from serl_b200.networks.reward_classifier import create_classifier, sample_classifier_batch, train_step
    sample = {c: np.zeros((1, 128, 128, 3), np.uint8) for c in cams}
    clf = create_classifier(np.array([0, 1], np.uint32), sample, cams, precision=precision)
    key = np.array([0, 0], np.uint32)

    def step(i):
        key[1] = i
        batch = sample_classifier_batch(pos, neg, B, key)
        return train_step(clf, batch, key)

    for i in range(5):
        step(i)
    torch.cuda.synchronize()
    rates, i, loss = [], 5, None
    for _ in range(3):
        n, t0 = 0, time.perf_counter()
        while True:
            _, loss, acc = step(i)
            i += 1
            n += 1
            if n % 8 == 0:
                torch.cuda.synchronize()
                if time.perf_counter() - t0 >= 1.0:
                    break
        rates.append(n / (time.perf_counter() - t0))
    clf.check_status()
    return statistics.median(rates), rates, float(loss)


def actor_latency(cams, precision, calls=200):
    from serl_b200.networks.reward_classifier import create_classifier, load_classifier_func
    from serl_b200.utils.checkpoints import save_checkpoint
    sample = {c: np.zeros((1, 128, 128, 3), np.uint8) for c in cams}
    clf = create_classifier(np.array([0, 2], np.uint32), sample, cams, precision=precision)
    with tempfile.TemporaryDirectory() as d:
        save_checkpoint(d, clf, step=0)
        f = load_classifier_func(np.array([0, 2], np.uint32), sample, cams, d, precision=precision)
    rng = np.random.default_rng(0)
    obs = [{c: rng.integers(0, 256, (1, 128, 128, 3), dtype=np.uint8) for c in cams} for _ in range(8)]
    for k in range(10):
        f(obs[k % 8]).item()
    ts = []
    for k in range(calls):
        t0 = time.perf_counter()
        f(obs[k % 8]).item()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--buffer", type=int, default=512, help="transitions per replay ring")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_classifier.py needs a CUDA device"
    import __graft_entry__ as G
    G.build()
    res = {"card": card(), "batch": a.batch, "train_steps_per_s": {}, "actor_latency_ms": {}}
    for cams in (("front",), ("front", "wrist")):
        pos, neg = make_buffers(cams, a.buffer, 11)
        for precision in ("fp16", "fp32"):
            name = f"{len(cams)}cam_{precision}"
            med, rates, loss = train_rate(cams, precision, a.batch, pos, neg)
            res["train_steps_per_s"][name] = {"median": round(med, 2), "windows": [round(r, 2) for r in rates], "last_loss": loss}
            res["actor_latency_ms"][name] = round(actor_latency(cams, precision), 3)
            print(name, res["train_steps_per_s"][name], f"actor {res['actor_latency_ms'][name]} ms", flush=True)
        del pos, neg
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
