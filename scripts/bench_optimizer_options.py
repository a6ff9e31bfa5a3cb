"""What gradient clipping, or a network architecture other than the launcher's, costs in the DrQ critic step, on one GPU.

    python scripts/bench_optimizer_options.py [--arms default,clip] [--clip-grad-norm 1.0] [--steps 100] [--rounds 3]
                                              [--precision fp16] [--out result.json]

Arms: "default" (the launcher agent), "clip" (`clip_grad_norm` on every tx), "reference_defaults" (the reference
constructors' own networks: swish MLPs [256, 256] without LayerNorm, "uniform" std) and "512x3" (relu MLPs [512, 512, 512]
with LayerNorm, "softplus" std).  The non-launcher architectures run the per-op heads chain instead of the fused tgemm heads.

bench.py's workload (BASELINE configs[2]: two 128x128x3 cameras, batch 256 drawn 50/50 from the online and demo rings,
cross-step pipeline on, whole step replayed as a CUDA graph) with one agent per arm, all of the same seed on the same rings.  `clip_grad_norm`
adds the global-norm pass over the flat gradient buffer and the options variant of the fused Adam.  The arms are timed in
alternating windows of `--steps` steps (CUDA events,
closed by a device synchronise) after a warm-up that captures every graph variant.  The output is one JSON line with
steps/s per window and arm, the medians, each arm's overhead over the first, and the card's name, power limit and max SM clock read in the same run.
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


ARCHITECTURES = {
    "reference_defaults": ({"hidden_dims": [256, 256], "activations": "swish", "use_layer_norm": False}, "uniform"),
    "512x3": ({"hidden_dims": [512, 512, 512], "activations": "relu", "use_layer_norm": True}, "softplus"),
}


def make_arm(name, w, args):
    """The agent of one arm, with the launcher's hyper-parameters (utils/launcher.py:79-116) and the workload's seed."""
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.utils.launcher import make_drq_agent
    obs, act = w.transitions[0]["observations"], w.transitions[0]["actions"]
    if name == "clip":
        clip = {"clip_grad_norm": args.clip_grad_norm}
        return make_drq_agent(42, obs, act, image_keys=w.cams, encoder_type="resnet-pretrained", precision=args.precision,
                              **{f"{tx}_optimizer_kwargs": clip for tx in ("actor", "critic", "temperature")})
    nk, std = ARCHITECTURES[name]
    return DrQAgent.create_drq(42, obs, act, encoder_type="resnet-pretrained", use_proprio=True, image_keys=w.cams, temperature_init=1e-2,
                               discount=0.96, backup_entropy=False, critic_ensemble_size=10, critic_subsample_size=2, precision=args.precision,
                               critic_network_kwargs=nk, policy_network_kwargs=nk,
                               policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": std, "std_min": 1e-5, "std_max": 5})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arms", default="default,clip", help="comma-separated: default, clip, reference_defaults, 512x3")
    ap.add_argument("--clip-grad-norm", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", default="fp16", choices=["fp32", "bf16", "fp16"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    import bench
    w = bench.Workload(args, 2, True, 200_000, 256)
    arms = args.arms.split(",")
    agents = {name: w.agent if name == "default" else make_arm(name, w, args) for name in arms}
    for name, agent in agents.items():
        agent.pipeline_critic_steps = True
        w.agent = agent
        for _ in range(12):                      # serial, pipeline start and both steady-state variants: eager once, then captured
            agent.update_critics(w.next_batch())
    rates = {name: [] for name in agents}
    for r in range(args.rounds):
        for name in (arms if r % 2 == 0 else arms[::-1]):
            w.agent = agents[name]
            w.agent.update_critics(w.next_batch())           # each window starts the agent's pipeline afresh, untimed
            rates[name].append(1e3 * args.steps / w.timed_steps(args.steps))
    med = {name: statistics.median(v) for name, v in rates.items()}
    out = {"workload": "bench.py configs[2] critic step (2 cameras, batch 256, RLPD 50/50, pipeline, CUDA graph)",
           "precision": args.precision, "clip_grad_norm": args.clip_grad_norm, "card": card(), "steps_per_window": args.steps,
           "steps_per_s": rates, "median_steps_per_s": med,
           "overhead_pct": {name: 100.0 * (med[arms[0]] / med[name] - 1.0) for name in arms[1:]}}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    w.close()


if __name__ == "__main__":
    main()
