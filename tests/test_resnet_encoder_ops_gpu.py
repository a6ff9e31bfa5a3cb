"""GPU: the trainable ResNet-10's kernels op by op against float64 autograd, at every layer shape of a 128x128 image and batches
1, 3, 256 and 514, on the CUDA-core (fp32 build) and tensor-core (16-bit builds) convs: forward within 1e-5 / 1e-4 of the
output's max, input and weight gradients within 2e-4; the GroupNorm backward with and without ReLU / residual; the max-pool
backward's first-max rule on tied and all-zero windows; two launches bitwise equal."""
import numpy as np
import pytest
import torch

from oracle import drq
from resnet_encoder_oracle import max_pool_first_max

pytestmark = pytest.mark.gpu
BATCHES = (1, 3, 256, 514)


def _convs():
    from serl_b200.engine import resnet_convs
    return resnet_convs(128)


def _err(got, ref):
    ref = ref.detach().double()
    return float((got.double() - ref).abs().max() / max(float(ref.abs().max()), 1e-12))


@pytest.mark.parametrize("tc", [0, 1], ids=["cuda-cores", "tensor-cores"])
@pytest.mark.parametrize("N", BATCHES)
def test_convs_match_float64(N, tc):
    from serl_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N)
    for leaf, k, st, lo, hi, H, ci, co in _convs():
        c4 = 4 if ci == 3 else ci
        x = torch.randn(N, H, H, c4, device="cuda", generator=g)
        if ci == 3:
            x[..., 3] = 0
        w = torch.randn(k, k, ci, co, device="cuda", generator=g) / (k * k * ci) ** 0.5
        x64, w64 = x[..., :ci].double().requires_grad_(), w.double().requires_grad_()
        ref = drq.conv_nhwc(x64, w64, st, lo, hi)
        Ho = ref.shape[1]
        y = torch.empty(N, Ho, Ho, co, device="cuda")
        ops.rconv_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, H, c4, ci, co, k, st, lo, hi, tc)
        assert _err(y, ref) < (1e-4 if tc else 1e-5), (leaf, N, _err(y, ref))
        y2 = torch.empty_like(y)
        ops.rconv_fwd(x.data_ptr(), w.data_ptr(), y2.data_ptr(), N, H, H, c4, ci, co, k, st, lo, hi, tc)
        assert torch.equal(y, y2), leaf
        dz = torch.randn(N, Ho, Ho, co, device="cuda", generator=g)
        (ref * dz.double()).sum().backward()
        ws = torch.empty(ops.rconv_wgrad_workspace(N, H, H, c4, co, k, st, lo, hi), device="cuda")
        dw, dw2 = torch.empty_like(w), torch.empty_like(w)
        for out in (dw, dw2):
            ops.rconv_wgrad(x.data_ptr(), dz.data_ptr(), out.data_ptr(), ws, N, H, H, c4, ci, co, k, st, lo, hi, tc)
        assert _err(dw, w64.grad) < 2e-4 and torch.equal(dw, dw2), (leaf, N, _err(dw, w64.grad))
        if leaf == "conv_init":                       # the image needs no input gradient
            continue
        dx, dx2 = torch.empty_like(x), torch.empty_like(x)
        for out in (dx, dx2):
            ops.rconv_dgrad(dz.data_ptr(), w.data_ptr(), out.data_ptr(), N, H, H, ci, co, k, st, lo, hi, False, tc)
        assert _err(dx, x64.grad) < 2e-4 and torch.equal(dx, dx2), (leaf, N, _err(dx, x64.grad))
        base = torch.randn_like(x)                  # accumulate adds to what dx holds
        acc = base.clone()
        ops.rconv_dgrad(dz.data_ptr(), w.data_ptr(), acc.data_ptr(), N, H, H, ci, co, k, st, lo, hi, True, tc)
        assert _err(acc, base.double() + x64.grad) < 2e-4, leaf
    torch.cuda.synchronize()


GN_SHAPES = ((64, 64), (32, 64), (16, 128), (8, 256), (4, 512))


@pytest.mark.parametrize("N", BATCHES)
@pytest.mark.parametrize("mode", ["relu", "relu+residual", "plain"])
def test_groupnorm_backward_matches_float64(N, mode):
    from serl_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(7 * N)
    relu, res_on = mode != "plain", mode == "relu+residual"
    for H, C in GN_SHAPES:
        x = torch.randn(N, H, H, C, device="cuda", generator=g) * 2 + 0.5
        sc = 1 + 0.3 * torch.randn(C, device="cuda", generator=g)
        bi = 0.2 * torch.randn(C, device="cuda", generator=g)
        res = torch.randn_like(x) if res_on else None
        y = torch.empty_like(x)
        ops.groupnorm_nhwc(x, y, sc, bi, res, 4, 1e-5, relu)
        x64, s64, b64 = x.double().requires_grad_(), sc.double().requires_grad_(), bi.double().requires_grad_()
        r64 = res.double().requires_grad_() if res_on else None
        ref = drq.group_norm_nhwc(x64, s64, b64)
        if res_on:
            ref = ref + r64
        dy = torch.randn_like(x)
        if relu:                                    # the kernel's mask is the fp32 forward's output: gate the reference the same way
            ref = ref * (y > 0).double()
        (ref * dy.double()).sum().backward()
        ws = torch.empty(ops.groupnorm_bwd_workspace(N, C, 4), device="cuda")
        outs = []
        for _ in range(2):
            dx, dres, ds, db = torch.empty_like(x), torch.empty_like(x) if res_on else None, torch.empty_like(sc), torch.empty_like(bi)
            ops.groupnorm_bwd_nhwc(x.data_ptr(), y.data_ptr(), dy.data_ptr(), sc.data_ptr(), dx.data_ptr(),
                                   dres.data_ptr() if res_on else None, ds.data_ptr(), db.data_ptr(), ws, N, H * H, C, 4, 1e-5, relu)
            outs.append((dx, dres, ds, db))
        dx, dres, ds, db = outs[0]
        assert _err(dx, x64.grad) < 2e-4, (H, C, _err(dx, x64.grad))
        assert _err(ds, s64.grad) < 2e-4 and _err(db, b64.grad) < 2e-4, (H, C, _err(ds, s64.grad), _err(db, b64.grad))
        if res_on:
            assert _err(dres, r64.grad) < 2e-4
        for a, b in zip(outs[0], outs[1]):
            assert a is None or torch.equal(a, b)


@pytest.mark.parametrize("N", BATCHES)
def test_maxpool_backward_first_max(N):
    """Post-ReLU-like maps with many ties (values on a coarse grid, a block of all-zero windows): the gradient goes to each
    window's first maximal element; tied zero windows route it to their first element."""
    from serl_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3 * N)
    x = (torch.randint(0, 4, (N, 64, 64, 64), device="cuda", generator=g).float() * 0.5)
    x[:, :8, :8] = 0
    y = torch.empty(N, 32, 32, 64, device="cuda")
    ops.maxpool3x3s2_nhwc(x, y)
    x64 = x.double().requires_grad_()
    ref = max_pool_first_max(x64)
    assert torch.equal(y.double(), ref.detach())
    dy = torch.randn(N, 32, 32, 64, device="cuda", generator=g)
    (ref * dy.double()).sum().backward()
    dx, dx2 = torch.empty_like(x), torch.empty_like(x)
    for out in (dx, dx2):
        ops.maxpool3x3s2_bwd_nhwc(x.data_ptr(), dy.data_ptr(), out.data_ptr(), N, 64, 64, 64)
    assert _err(dx, x64.grad) < 1e-6 and torch.equal(dx, dx2)
    assert ((dx != 0) == (x64.grad != 0)).all()
