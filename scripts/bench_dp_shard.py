"""Frame-sharded replay: what the owner lookup costs the sampler, measured at world size 1 on one GPU.

    python scripts/bench_dp_shard.py [--capacity 50000] [--batch 128] [--iters 200] [--windows 5] [--out DIR]

Two rings of bench.py's frames (two 128x128x3 cameras, T = 1) hold the same random contents: a replicated
MemoryEfficientReplayBuffer and one built with frame_shard=(0, 1), whose single shard is the whole ring plus its halo.  Each
timed window launches the sampler `--iters` times on one ring (serl_replay_sample_crop, or serl_replay_sample_crop_sharded
through the shard table), CUDA events around the window; windows alternate between the rings, and n_step = 3 windows follow
the same pattern.  Before timing, one launch per ring with the same draw is checked to give bitwise equal outputs.  Prints
one JSON line with the card's name and power limit; with --out, also writes it there.

Steps/s of sharded against replicated stores at 2 and 8 GPUs, and the largest ring each mode can hold per GPU, need a
multi-GPU node: this script does not measure them.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_conditions():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:                      # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")])) if "," in out else {"nvidia-smi": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacity", type=int, default=50_000)
    ap.add_argument("--batch", type=int, default=128, help="rows per launch (bench.py: 128 online rows of its batch of 256)")
    ap.add_argument("--iters", type=int, default=200, help="sampler launches per timed window")
    ap.add_argument("--windows", type=int, default=5, help="timed windows per ring and n_step")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_dp_shard.py measures on a CUDA device; none is available")
    from helpers import pixel_spaces
    from serl_b200 import _lib as L
    from serl_b200.data.memory_efficient_replay_buffer import MemoryEfficientReplayBuffer

    torch.cuda.set_device(0)
    cams, cap, B, T = ("front", "wrist"), args.capacity, args.batch, 1
    obs_space, act_space = pixel_spaces(cams, 128)
    rep = MemoryEfficientReplayBuffer(obs_space, act_space, cap, pixel_keys=cams, seed=5)
    sh = MemoryEfficientReplayBuffer(obs_space, act_space, cap, pixel_keys=cams, seed=5, frame_shard=(0, 1))
    g = torch.Generator(device="cuda").manual_seed(0)
    for c in cams:
        rep.frames[c].copy_(torch.randint(0, 256, rep.frames[c].shape, dtype=torch.uint8, device="cuda", generator=g))
        sh.frames[c][T:].copy_(rep.frames[c])                     # range: slot s at local s + T
        sh.frames[c][:T].copy_(rep.frames[c][cap - T:])           # rank 0's halo wraps to the last T slots
    rng = np.random.default_rng(0)
    valid = rng.random(cap) < 0.9
    for r in (rep, sh):
        r.state.normal_(generator=g)
        r.rewards.uniform_(generator=g)
        r.masks.fill_(1.0)
        r.valid.copy_(torch.from_numpy(valid.astype(np.uint8)))
        r._valid_host[:] = valid
        r._size = cap
        r.size_dev.fill_(cap)
    sh.state.copy_(rep.state); sh.rewards.copy_(rep.rewards)
    torch.cuda.synchronize()

    hw, key = 128, torch.tensor([3, 9], dtype=torch.int32, device="cuda")

    def outputs():
        o = {"pix": {c: torch.empty(2 * B, hw, hw, 3, dtype=torch.uint8, device="cuda") for c in cams},
             "f": torch.empty(6, B, 8, device="cuda"), "i": torch.empty(3, B, dtype=torch.int32, device="cuda")}
        out = L.BatchOut()
        for j, c in enumerate(cams):
            out.obs_pix[j], out.next_pix[j] = o["pix"][c].data_ptr(), o["pix"][c].data_ptr() + B * hw * hw * 3
        out.obs_state, out.next_state, out.actions = o["f"][0].data_ptr(), o["f"][1].data_ptr(), o["f"][2].data_ptr()
        out.rewards, out.masks, out.dones = o["f"][3].data_ptr(), o["f"][4].data_ptr(), o["i"][2].data_ptr()
        out.idx, out.status = o["i"][0].data_ptr(), o["i"][1].data_ptr()
        return o, out

    def launch(ring, out, n_step, step):
        part = dict(ring=ring, seed=ring._seed, step=step, batch=B, indx=None, n_step=n_step, discount=0.9 if n_step > 1 else None)
        ring.launch_sample(part, out, crop_total=B, out_row_offset=0, key_obs=key.data_ptr(), key_next=key.data_ptr(),
                           record_event=False)

    # the same draw from both rings gives the same bytes
    check = {}
    for name, ring in (("replicated", rep), ("sharded", sh)):
        o, out = outputs()
        o["i"].zero_()
        launch(ring, out, 1, 17)
        torch.cuda.synchronize()
        check[name] = o
    same = all(torch.equal(check["replicated"]["pix"][c], check["sharded"]["pix"][c]) for c in cams) and \
        torch.equal(check["replicated"]["i"], check["sharded"]["i"])
    if not same:
        raise SystemExit("sharded and replicated sampler outputs differ")

    o, out = outputs()
    times = {f"{n}_n{k}": [] for n in ("replicated", "sharded") for k in (1, 3)}
    for k in (1, 3):
        for ring in (rep, sh):
            for s in range(5):
                launch(ring, out, k, s)                               # warm-up (module load, shared-memory opt-in)
    torch.cuda.synchronize()
    for w in range(args.windows):
        for k in (1, 3):
            for name, ring in (("replicated", rep), ("sharded", sh)) if w % 2 == 0 else (("sharded", sh), ("replicated", rep)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for s in range(args.iters):
                    launch(ring, out, k, 100 + s)
                e1.record()
                e1.synchronize()
                times[f"{name}_n{k}"].append(e0.elapsed_time(e1) * 1e3 / args.iters)
    res = {k: {"median_us": float(np.median(v)), "min_us": float(np.min(v)), "max_us": float(np.max(v))} for k, v in times.items()}
    line = {"metric": "sampler_launch_us", "what": f"one sampler launch, {B} rows x 2 cameras 128x128x3, world size 1, "
                                                   f"{cap}-slot rings; device time per launch from CUDA events over {args.iters} launches",
            "results": res, "bitwise_equal": same, "gpu": gpu_conditions(),
            "multi_gpu": "not measured (steps/s at 2 and 8 GPUs and the largest ring per GPU need a multi-GPU node)"}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_dp_shard.json"), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
