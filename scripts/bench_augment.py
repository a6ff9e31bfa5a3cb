"""Image augmentations (serl_b200.vision.data_augmentations): device time and effective bandwidth per call.

    python scripts/bench_augment.py [--batch 256] [--calls 200] [--windows 5] [--out DIR]

Each function runs on a (batch, 128, 128, 3) batch with one key per image (batched_random_crop: one key split n ways): uint8 for
the crops, float32 for the rest.  The colour jitter runs with every op enabled and apply / jitter probability 1 (its heaviest
path: contrast's mean over each image, then the four ops); the blur with the defaults (blur_divider 10: radius 6, 13 taps) and
apply_prob 1; solarize with apply_prob 1.  Per function: a warm-up, then `--calls` back-to-back calls captured in one CUDA graph
(so the host's per-call Python does not pace the device) and replayed `--windows` times with CUDA events around each replay; the
median window over `--calls` gives the device time per call.  Effective GB/s counts the input read once and the
output written once (the colour kernel's second read of an image is not counted).  Prints a table and one JSON line; with
--out, also writes the JSON there.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--calls", type=int, default=200, help="calls per timed window")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment.py measures on a CUDA device; none is available")
    from serl_b200.vision import data_augmentations as DA

    torch.cuda.set_device(0)
    n, shape = args.batch, (args.batch, 128, 128, 3)
    g = torch.Generator(device="cuda").manual_seed(0)
    u8 = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=g)
    f32 = torch.rand(shape, dtype=torch.float32, device="cuda", generator=g)
    keys = torch.randint(-2**31, 2**31 - 1, (n, 2), dtype=torch.int32, device="cuda", generator=g)
    key = keys[0].clone()
    color = dict(brightness=0.4, contrast=0.4, saturation=0.4, hue=0.1, to_grayscale_prob=0.2, color_jitter_prob=1.0, apply_prob=1.0,
                 shuffle=True)
    cases = {
        "batched_random_crop u8": (lambda: DA.batched_random_crop(u8, key, padding=4), u8),
        "random_crop u8": (lambda: DA.random_crop(u8, keys, padding=4), u8),
        "random_crop f32": (lambda: DA.random_crop(f32, keys, padding=4), f32),
        "color_transform f32": (lambda: DA.color_transform(f32, keys, **color), f32),
        "gaussian_blur f32": (lambda: DA.gaussian_blur(f32, keys), f32),
        "random_flip f32": (lambda: DA.random_flip(f32, keys), f32),
        "solarize f32": (lambda: DA.solarize(f32, keys, threshold=0.5, apply_prob=1.0), f32),
    }
    rows = {}
    for name, (call, x) in cases.items():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(20):
                call()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(args.calls):
                call()
        graph.replay()
        torch.cuda.synchronize()
        times = []
        for _ in range(args.windows):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            graph.replay()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) * 1e3 / args.calls)
        del graph
        us = statistics.median(times)
        nbytes = 2 * x.numel() * x.element_size()
        rows[name] = dict(us_per_call=round(us, 2), spread_us=round(max(times) - min(times), 2), GB_per_s=round(nbytes / us / 1e3, 1),
                          MB_moved=round(nbytes / 1e6, 2))
    cond = gpu_conditions()
    print(f"{'function':<26}{'us/call':>10}{'spread':>9}{'GB/s':>9}{'MB r+w':>9}   on {cond}")
    for name, r in rows.items():
        print(f"{name:<26}{r['us_per_call']:>10.2f}{r['spread_us']:>9.2f}{r['GB_per_s']:>9.1f}{r['MB_moved']:>9.2f}")
    line = json.dumps(dict(shape=list(shape), calls=args.calls, windows=args.windows, gpu=cond, results=rows))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_augment.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
