"""Runs the frozen trunk alone.

    python scripts/prof_trunk.py [fp16|bf16] [B] [reps]             # CUDA-event time of one one-camera pass (N = 2 B images)
    python scripts/prof_trunk.py [fp16|bf16] [B] [reps] --launches  # torch.profiler (CUDA activities): every kernel launch of
                                                                     # one pass, in launch order, with its device time
"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
from helpers import random_transitions
from serl_b200.utils.launcher import make_drq_agent

argv = [a for a in sys.argv[1:] if not a.startswith("--")]
prec = argv[0] if len(argv) > 0 else "fp16"
B = int(argv[1]) if len(argv) > 1 else 256
reps = int(argv[2]) if len(argv) > 2 else 3
cams = ("cam0",)
tr = random_transitions(np.random.default_rng(0), 1, cams)[0]
agent = make_drq_agent(42, tr["observations"], tr["actions"], image_keys=cams, encoder_type="resnet-pretrained", precision=prec)
eng = agent._engine(B)
eng.pix["cam0"].copy_(torch.randint(0, 256, eng.pix["cam0"].shape, dtype=torch.uint8, device="cuda"))
for _ in range(reps):
    eng.trunk_forward("cam0", eng.pix["cam0"], eng.feats["cam0"])
torch.cuda.synchronize()

if "--launches" in sys.argv:
    # One profiled run of its own (the profiler slows the host, so no end-to-end number is taken here).  Each pass's kernels
    # are listed in launch order; the per-launch time is the median over the reps.
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.trunk_forward("cam0", eng.pix["cam0"], eng.feats["cam0"])
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0
                 and not e.name.startswith(("Memset", "Memcpy"))), key=lambda e: e.time_range.start)
    per = len(ev) // reps
    assert per * reps == len(ev), f"{len(ev)} kernel records for {reps} passes"
    total = 0.0
    print(f"trunk {prec} N={2*B}: {per} kernel launches per pass (median of {reps} passes)")
    print(f"{'#':>3} {'us':>9}  kernel")
    for i in range(per):
        us = float(np.median([ev[r * per + i].device_time_total for r in range(reps)]))
        total += us
        print(f"{i:3d} {us:9.1f}  {ev[i].name[:150]}")
    print(f"sum of kernel times {total / 1e3:.3f} ms per pass")
    sys.exit(0)

a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(reps):
    eng.trunk_forward("cam0", eng.pix["cam0"], eng.feats["cam0"])
b.record(); torch.cuda.synchronize()
print(f"trunk {prec} N={2*B}: {a.elapsed_time(b)/reps:.3f} ms per pass -> {2*B*0.5804/1e3/(a.elapsed_time(b)/reps/1e3):.1f} TFLOP/s")
