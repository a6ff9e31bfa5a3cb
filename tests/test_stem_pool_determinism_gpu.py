"""GPU: the fused stem (conv_init + GroupNorm sums + 3x3/2 max-pool) is deterministic.  A cluster of CTAs shares each
image's GroupNorm partial sums through distributed shared memory and rank 0 adds their rank-ordered total once (no float
atomics racing each other), so two runs on the same input give bit-identical statistics and pooled outputs."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_stem_pool_two_runs_bitwise_equal(prec):
    from serl_b200 import _lib as L
    from serl_b200 import trunk_bf16 as T
    N = 512
    rng = np.random.default_rng(5)
    pix = torch.as_tensor(rng.integers(0, 256, (N, 128, 128, 3), dtype=np.uint8)).cuda()
    w = torch.as_tensor((rng.standard_normal((7, 7, 3, 64)) * np.sqrt(2.0 / 147)).astype(np.float32)).cuda()
    gamma = torch.as_tensor((rng.standard_normal(64) + 0.3).astype(np.float32)).cuda()
    beta = torch.as_tensor((0.2 * rng.standard_normal(64)).astype(np.float32)).cuda()
    wp = T.pack_stem_weight(w, DT[prec])
    plan = T._Plan(N, 128, "cuda", prec)
    s = L.stream_ptr()
    L.call("serl_trunk_stem_prep_h16", pix.data_ptr(), plan.xs.data_ptr(), N, 128, 128, plan.fmt, s)
    runs = []
    for _ in range(2):
        st = torch.zeros(N, 4, 2, device="cuda")
        pooled = torch.full((N, 32, 32, 64), float("nan"), dtype=DT[prec], device="cuda")
        side = torch.full((N, 4, 32, 64), float("nan"), dtype=DT[prec], device="cuda")
        d = L.StemPoolDesc()
        d.xs, d.w, d.pooled, d.side, d.stats, d.error = plan.xs.data_ptr(), wp.data_ptr(), pooled.data_ptr(), side.data_ptr(), st.data_ptr(), plan.error.data_ptr()
        d.neg_mask = sum(1 << c for c, g in enumerate(gamma.cpu().tolist()) if g < 0)
        d.N, d.fmt = N, plan.fmt
        L.call("serl_stem_conv_pool_tc_h16", C.byref(d), s)
        out = torch.empty(N, 32, 32, 64, dtype=DT[prec], device="cuda")
        L.call("serl_pool_finish_gn_h16", pooled.data_ptr(), side.data_ptr(), st.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(),
               N, T.GN_EPS, plan.fmt, s)
        torch.cuda.synchronize()
        assert int(plan.error.item()) == 0, f"pipeline barrier timeout (flags {int(plan.error.item())})"
        runs.append((st.cpu(), out.view(torch.int16).cpu()))
    assert torch.isfinite(runs[0][0]).all() and (runs[0][0][:, :, 1] > 0).all()
    assert torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
    assert torch.equal(runs[0][1], runs[1][1])
