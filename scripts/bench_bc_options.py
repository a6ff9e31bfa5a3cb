"""BCAgent.update steps/s for three network configurations on one GPU: the launcher's (make_bc_agent: tanh [256, 256], proprio,
"exp" std), the reference constructor's defaults (pixel-only, swish [256, 256]) and a large one ([512, 512, 512] + LayerNorm +
dropout 0.1 + tanh squash + "uniform" std).  fp16 build, two 128x128 cameras, batch 256; the configurations are timed in
alternating windows so that drift of a shared GPU falls on all of them.  Prints one JSON line with the card name and power limit.

    python scripts/bench_bc_options.py [--steps 50] [--windows 3] [--precision fp16]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = {
    "launcher": dict(network_kwargs={"activations": "tanh", "use_layer_norm": False, "hidden_dims": [256, 256]},
                     policy_kwargs={"std_parameterization": "exp", "std_max": 5}, use_proprio=True),
    "reference_defaults": dict(network_kwargs={"activations": "swish", "use_layer_norm": False, "hidden_dims": [256, 256]},
                               policy_kwargs={}, use_proprio=False),
    "large": dict(network_kwargs={"activations": "tanh", "use_layer_norm": True, "hidden_dims": [512, 512, 512], "dropout_rate": 0.1},
                  policy_kwargs={"std_parameterization": "uniform", "tanh_squash_distribution": True}, use_proprio=True),
}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--precision", default="fp16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bc_options: needs a CUDA device")
    from serl_b200.agents.continuous.bc import BCAgent
    cams, B, A, S, hw = ("front", "wrist"), args.batch, 7, 19, 128
    rng = np.random.default_rng(0)
    obs = {c: torch.as_tensor(rng.integers(0, 256, (B, 1, hw, hw, 3), dtype=np.uint8), device="cuda") for c in cams}
    obs["state"] = torch.as_tensor(rng.standard_normal((B, 1, S)).astype(np.float32), device="cuda")
    batch = {"observations": obs, "actions": torch.as_tensor(rng.uniform(-0.99, 0.99, (B, A)).astype(np.float32), device="cuda")}
    sample = {**{c: np.zeros((1, hw, hw, 3), np.uint8) for c in cams}, "state": np.zeros((1, S), np.float32)}
    agents = {k: BCAgent.create(0, sample, np.zeros(A, np.float32), encoder_type="resnet-pretrained", image_keys=cams,
                                precision=args.precision, **cfg) for k, cfg in CONFIGS.items()}
    for agent in agents.values():
        for _ in range(args.warmup):
            agent.update(batch)
    torch.cuda.synchronize()
    rates = {k: [] for k in agents}
    for _ in range(args.windows):
        for k, agent in agents.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                agent.update(batch)
            torch.cuda.synchronize()
            rates[k].append(args.steps / (time.perf_counter() - t0))
    name, power = _card()
    print(json.dumps({"metric": "bc_update_steps_per_s", "precision": args.precision, "batch": B, "cameras": len(cams), "steps": args.steps,
                      "windows": rates, "median": {k: statistics.median(v) for k, v in rates.items()}, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
