"""Replay-ring save / load throughput on one GPU.

    python scripts/bench_replay_io.py [--slots 20000] [--chunk-mb 32] [--repeats 3] [--out result.json]

* fills a synthetic two-camera frame-dedup ring (128x128x3 frames; 20 k slots = 1.97 GB of frames) straight in HBM;
* saves it into a temporary directory and loads it into a second ring of the same shape, `--repeats` times; each direction is
  timed by a host clock around `save` / `load`, which return after the device synchronise and the file's close (and rename);
  the load reads a file the save just wrote, so it is usually served from the page cache;
* checks the loaded ring equals the saved one, deletes the directory, and reports GB/s (file bytes over the median time),
  the pinned staging the calls held, the host's zlib CRC-32 rate (the only compute on the path) and the card's name and
  power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def make_ring(cams, slots, seed):
    from helpers import fake_env
    from serl_b200.utils.launcher import make_replay_buffer
    return make_replay_buffer(fake_env(cams), capacity=slots, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=seed)


def fill(ring, seed):
    """Synthetic full ring written straight into HBM (inserting 20 k transitions through the host would time the staging)."""
    g = torch.Generator(device=ring.device).manual_seed(seed)
    for c in ring.cams:
        ring.frames[c].copy_(torch.randint(0, 256, ring.frames[c].shape, generator=g, device=ring.device, dtype=torch.uint8))
    for t in (ring.state, ring.next_state, ring.actions, ring.rewards):
        t.normal_(generator=g)
    ring.masks.fill_(1.0)
    ring.valid.copy_((torch.rand(ring.valid.shape, generator=g, device=ring.device) < 0.99).to(torch.uint8))
    ring._valid_host[:] = ring.valid.cpu().numpy().astype(bool)
    ring._size, ring._insert_index, ring._first = ring._capacity, 0, False
    ring.size_dev.fill_(ring._capacity)
    torch.cuda.synchronize()


def crc_rate(nbytes=256 << 20):
    buf = np.random.default_rng(0).integers(0, 256, nbytes, dtype=np.uint8)
    t0 = time.perf_counter()
    zlib.crc32(buf)
    return nbytes / (time.perf_counter() - t0) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=20_000)
    ap.add_argument("--chunk-mb", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_replay_io needs a CUDA device"
    torch.cuda.set_device(0)
    cams = ("front", "wrist")
    src, dst = make_ring(cams, args.slots, 1), make_ring(cams, args.slots, 2)
    fill(src, 0)
    chunk = args.chunk_mb << 20
    saves, loads = [], []
    with tempfile.TemporaryDirectory(prefix="bench_replay_io_") as d:
        path = os.path.join(d, "replay_buffer.npz")
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            nbytes = src.save(path, chunk_bytes=chunk)
            saves.append(time.perf_counter() - t0)
            pinned_save = src.io_pinned_bytes
            t0 = time.perf_counter()
            dst.load(path, chunk_bytes=chunk)
            loads.append(time.perf_counter() - t0)
            pinned_load = dst.io_pinned_bytes
    for c in cams:
        assert torch.equal(src.frames[c], dst.frames[c]), c
    for name in ("state", "next_state", "actions", "rewards", "masks", "dones", "valid"):
        assert torch.equal(getattr(src, name), getattr(dst, name)), name
    assert len(dst) == len(src) and dst._seed == src._seed
    res = {"bench": "replay_io", "card": card(), "slots": args.slots, "cams": len(cams), "file_bytes": nbytes,
           "chunk_bytes": chunk, "pinned_bytes_save": pinned_save, "pinned_bytes_load": pinned_load,
           "save_s": [round(t, 4) for t in saves], "load_s": [round(t, 4) for t in loads],
           "save_GBps": round(nbytes / statistics.median(saves) / 1e9, 3),
           "load_GBps": round(nbytes / statistics.median(loads) / 1e9, 3),
           "host_crc32_GBps": round(crc_rate(), 3)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
