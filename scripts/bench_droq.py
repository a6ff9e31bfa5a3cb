"""Cost of dropout Q-functions (DroQ) next to the launcher's REDQ agent, on bench.py's DrQ workload: fp16 trunk, two 128x128
cameras, batch 256 drawn as RLPD halves (online + demo ring), cross-step pipeline and CUDA graphs.

Arms, run in alternating windows:
  launcher   E = 10, critic_subsample_size = 2, launcher MLPs (fused tgemm heads)
  droq       E = 2, no subsample, critic dropout_rate 0.01, launcher widths / LayerNorm / tanh (fused tgemm heads with masked
             LayerNorm epilogues)
  droq_perop the same DroQ agent with SERL_FUSED_HEADS=0 (per-op heads chain)

Prints one JSON line: per arm the median update_critics and update_high_utd(utd_ratio=1) steps/s over the windows, the kernel
launches per step, and the card's name, power limit and max SM clock read in the same run.

    python scripts/bench_droq.py --windows 3 --steps 200
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

DROQ = {"hidden_dims": [256, 256], "activations": "tanh", "use_layer_norm": True, "dropout_rate": 0.01}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                               # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


def _arm(name, B):
    import numpy as np
    from helpers import fake_env, random_transitions
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.utils.train_utils import concat_batches
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    cams = ("front", "wrist")
    os.environ["SERL_FUSED_HEADS"] = "0" if name == "droq_perop" else "1"
    rings = []
    for seed in (3, 4):
        rb = make_replay_buffer(fake_env(cams), capacity=4096, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=seed)
        for tr in random_transitions(np.random.default_rng(seed), 1200, cams):
            rb.insert(tr)
        rings.append(rb)
    trs = random_transitions(np.random.default_rng(0), 1, cams)
    if name == "launcher":
        agent = make_drq_agent(0, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained",
                               precision="fp16")
    else:                                                # make_drq_agent's settings with the DroQ ensemble and critic
        agent = DrQAgent.create_drq(0, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet-pretrained", use_proprio=True,
                                    image_keys=cams, policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "exp",
                                                                    "std_min": 1e-5, "std_max": 5},
                                    temperature_init=1e-2, discount=0.96, backup_entropy=False, critic_ensemble_size=2,
                                    critic_subsample_size=None, precision="fp16", critic_network_kwargs=DROQ)
    agent.pipeline_critic_steps = True
    its = [rb.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True}) for rb in rings]
    nxt = lambda: concat_batches(next(its[0]), next(its[1]), axis=0)
    return agent, nxt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_droq.py measures on the GPU"
    arms = {n: _arm(n, args.batch) for n in ("launcher", "droq", "droq_perop")}
    res = {n: {"update_critics": [], "update_high_utd": [], "launches_per_step": {}} for n in arms}
    for n, (agent, nxt) in arms.items():                  # warm-up: eager, capture, replay of both step kinds
        os.environ["SERL_FUSED_HEADS"] = "0" if n == "droq_perop" else "1"
        for _ in range(5):
            agent.update_critics(nxt())
            agent.update_high_utd(nxt(), utd_ratio=1)
        torch.cuda.synchronize()
    for _ in range(args.windows):
        for n, (agent, nxt) in arms.items():
            os.environ["SERL_FUSED_HEADS"] = "0" if n == "droq_perop" else "1"
            for kind in ("update_critics", "update_high_utd"):
                batches = [nxt() for _ in range(args.steps)]
                torch.cuda.synchronize()
                c0, t0 = agent.kernel_launches, time.perf_counter()
                for b in batches:
                    agent.update_critics(b) if kind == "update_critics" else agent.update_high_utd(b, utd_ratio=1)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                res[n][kind].append(args.steps / dt)
                res[n]["launches_per_step"][kind] = (agent.kernel_launches - c0) / args.steps
    for n, (agent, _) in arms.items():
        agent.check_status()
        assert all((e.fused is None) == (n == "droq_perop") for e in agent._engines.values()), n
    import statistics
    out = {"workload": f"fp16, 2 cams 128x128, batch {args.batch} RLPD, pipeline + CUDA graphs", **_card(), "windows": args.windows,
           "steps_per_window": args.steps}
    for n, r in res.items():
        out[n] = {k: {"median_steps_per_s": round(statistics.median(v), 1), "all": [round(x, 1) for x in v]}
                  for k, v in r.items() if k != "launches_per_step"}
        out[n]["launches_per_step"] = r["launches_per_step"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
