"""CPU, world_size 2, gloo: the data-parallel host logic of `VICEAgent.update_vice` - ONE all-reduce per call over the vice
gradient AND its info scalars (which sit right behind it), the kernels asked to pre-scale both by 1/world (so the SUM is the
mean), and both ranks ending with identical buffers.  Kernels are replaced by a recorder (dry run)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from serl_b200 import _lib as L
    real = L.call
    scales = []

    def fake(name, *a):
        if name.startswith("serl_host_"):
            return real(name, *a)
        if name == "serl_vice_bce":
            scales.append(("bce", float(a[3])))                   # grad_scale: gradient and info[0]
        if name == "serl_vice_gp_rows":
            scales.append(("gp_rows", float(a[4])))               # coef = 10 * 2 / (ncams B) * grad_scale
        if name == "serl_vice_gp_finish":
            scales.append(("gp_finish", float(a[3])))            # info_scale
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    L.call, L.require_cuda, L.stream_ptr, L.new_event, L.pin = fake, (lambda d: None), (lambda: 0), (lambda: Ev()), (lambda t: t)
    from helpers import random_transitions
    from serl_b200.utils.launcher import make_vice_agent
    cams = ("front",)
    trs = random_transitions(np.random.default_rng(rank), 4, cams, 128)
    agent = make_vice_agent(7, trs[0]["observations"], trs[0]["actions"], image_keys=cams, vice_image_keys=cams,
                            encoder_type="resnet-pretrained", device="cpu")
    agent.data_parallel = True
    batch = {"observations": {c: np.stack([t["observations"][c] for t in trs]) for c in cams},
             "next_observations": {c: np.stack([t["next_observations"][c] for t in trs]) for c in cams},
             "actions": np.stack([t["actions"] for t in trs]), "rewards": np.zeros(4, np.float32), "masks": np.ones(4, np.float32)}
    for k in ("observations", "next_observations"):
        batch[k]["state"] = np.stack([t[k]["state"] for t in trs])
    vp = agent._vice
    n_coll = []
    real_ar = dist.all_reduce
    dist.all_reduce = lambda t, *a, **k: (n_coll.append(t.numel()), real_ar(t, *a, **k))[1]
    vp.grad_info.copy_(torch.arange(vp.n + 4, dtype=torch.float32) * (rank + 1))     # what the (no-op) kernels would have written
    agent.update_vice(batch)
    torch.save(dict(n=vp.n, n_coll=list(n_coll), g=vp.grad_info.clone(), scales=scales), out.format(rank))
    dist.destroy_process_group()


def test_one_collective_per_update_vice_with_mean_semantics(tmp_path):
    world, port = 2, 33000 + os.getpid() % 2000
    out = str(tmp_path / "rank{}.pt")
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    r0, r1 = torch.load(out.format(0)), torch.load(out.format(1))
    n = r0["n"]
    assert r0["n_coll"] == [n + 4] and r1["n_coll"] == [n + 4]          # gradient + bce, grad_norm, gp, total in ONE collective
    base = torch.arange(n + 4, dtype=torch.float32)
    torch.testing.assert_close(r0["g"], 3.0 * base)
    torch.testing.assert_close(r0["g"], r1["g"], rtol=0, atol=0)
    s = dict(r0["scales"])
    assert abs(s["bce"] - 0.5) < 1e-12 and abs(s["gp_finish"] - 0.5) < 1e-12
    assert abs(s["gp_rows"] - 10.0 * 2.0 / (1 * 4) * 0.5) < 1e-6
