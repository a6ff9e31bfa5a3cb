"""Times the two GEMM carriers (serl_gemm_f32 / serl_gemm_tf32x3) on the head shapes of the B=256 step and reports their
error against fp64.  GPU only:  python scripts/bench_gemm.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from serl_b200 import ops

SHAPES = [  # (name, M, K, N, Z)
    ("bottleneck 512x4096x256", 512, 4096, 256, 1),
    ("bottleneck 256x4096x256", 256, 4096, 256, 1),
    ("critic l1 256x327x256 E10", 256, 327, 256, 10),
    ("critic l2 256x256x256 E10", 256, 256, 256, 10),
    ("policy 256x320x256", 256, 320, 256, 1),
]


def timed(fn, iters=20, reps=5):
    """20 launches captured in one CUDA graph (no host launch overhead), replayed; operands stay L2-hot like in the step."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(iters):
                fn()
        g.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            g.replay()
        b.record()
        torch.cuda.synchronize()
    return a.elapsed_time(b) / (iters * reps) * 1e3


def main():
    rng = np.random.default_rng(0)
    for name, M, K, N, Z in SHAPES:
        x = torch.as_tensor(rng.standard_normal((Z, M, K)).astype(np.float32)).cuda()
        w = torch.as_tensor((rng.standard_normal((Z, K, N)) / np.sqrt(K)).astype(np.float32)).cuda()
        b = torch.zeros(Z, N, device="cuda")
        dz = torch.as_tensor(rng.standard_normal((Z, M, N)).astype(np.float32)).cuda()
        out, dw, dx = torch.empty(Z, M, N, device="cuda"), torch.empty(Z, K, N, device="cuda"), torch.empty(Z, M, K, device="cuda")
        ref = torch.bmm(x.double(), w.double())
        refdw = torch.bmm(x.double().transpose(1, 2), dz.double())
        refdx = torch.bmm(dz.double(), w.double().transpose(1, 2))
        for impl in ("f32", "tf32x3"):
            ws = ops.Workspace(64 << 20, "cuda", impl)
            f = lambda: ops.dense_fwd(ws, x.data_ptr(), K, w.data_ptr(), b.data_ptr(), out.data_ptr(), N, M, K, N, Z=Z, x_z=M * K, out_z=M * N)
            g = lambda: ops.dense_bwd_weight(ws, x.data_ptr(), K, dz.data_ptr(), N, dw.data_ptr(), M, K, N, Z=Z, x_z=M * K, dz_z=M * N)
            h = lambda: ops.dense_bwd_input(ws, dz.data_ptr(), N, w.data_ptr(), dx.data_ptr(), K, M, K, N, Z=Z, dz_z=M * N, dx_z=M * K)
            tf, tg, th = timed(f), timed(g), timed(h)
            ef = float((out.double() - ref).abs().max() / ref.abs().max())
            eg = float((dw.double() - refdw).abs().max() / refdw.abs().max())
            eh = float((dx.double() - refdx).abs().max() / refdx.abs().max())
            print(f"{name:28s} {impl:7s} fwd {tf:7.1f} us err {ef:.1e} | dW {tg:7.1f} us err {eg:.1e} | dX {th:7.1f} us err {eh:.1e}", flush=True)


if __name__ == "__main__":
    main()
