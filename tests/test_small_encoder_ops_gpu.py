"""GPU: the small encoder's kernels (serl_sconv_*) op by op against float64 torch at the four layer shapes of a 128x128 image,
batches 1, 3, 256 and 514, on both implementations: the CUDA-core kernels of the fp32 build and the tensor-core (3xTF32 wgmma)
kernels of the fp16 / bf16 builds.  Forward within 1e-5 of the output's max on the CUDA cores and 1e-4 on the tensor cores (well
inside the 16-bit builds' 1e-2 bar); input, weight and bias gradients within 2e-4 of each result's max; two launches bitwise
equal."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from small_encoder_oracle import SMALL_CONVS

pytestmark = pytest.mark.gpu
SIZES = (128, 63, 31, 15, 7)


def _conv64(x, w, b):
    """x (N,H,W,Ci) float64 -> conv3x3/2 VALID + b, NHWC, pre-activation."""
    return F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), stride=2).permute(0, 2, 3, 1) + b


def _inputs(layer, N, gen):
    ci, co = SMALL_CONVS[layer]
    H = SIZES[layer]
    if layer == 0:
        x = torch.randint(0, 256, (N, H, H, ci), dtype=torch.uint8, device="cuda", generator=gen)
        x64 = x.double() / 255.0
    else:                                       # a post-ReLU map: about half exact zeros
        x = torch.randn(N, H, H, ci, device="cuda", generator=gen).relu_()
        x64 = x.double()
    w = torch.randn(3, 3, ci, co, device="cuda", generator=gen) / (9 * ci) ** 0.5
    b = torch.randn(co, device="cuda", generator=gen) * 0.1
    return x, x64, w, b, H


def _rel(got, ref):
    return float((got.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


@pytest.mark.parametrize("tc", [False, True], ids=["cuda_cores", "tensor_cores"])
@pytest.mark.parametrize("N", [1, 3, 256, 514])
@pytest.mark.parametrize("layer", [0, 1, 2, 3])
def test_conv_forward_and_gradients_match_float64(layer, N, tc):
    from serl_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(100 * layer + N)
    ci, co = SMALL_CONVS[layer]
    x, x64, w, b, H = _inputs(layer, N, gen)
    Ho = SIZES[layer + 1]
    u8 = layer == 0
    # forward
    y = torch.full((N, Ho, Ho, co), float("nan"), device="cuda")
    ops.sconv_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), N, H, H, ci, co, u8, tc)
    ref = _conv64(x64, w.double(), b.double()).relu()
    assert _rel(y, ref) <= (1e-4 if tc else 1e-5), _rel(y, ref)
    y2 = torch.empty_like(y)
    ops.sconv_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), y2.data_ptr(), N, H, H, ci, co, u8, tc)
    assert torch.equal(y, y2)
    # weight + bias gradient from a pre-activation gradient dz
    dz = torch.randn(N, Ho, Ho, co, device="cuda", generator=gen) * (y > 0)
    w64 = w.double().requires_grad_(True)
    b64 = b.double().requires_grad_(True)
    xg = x64.clone().requires_grad_(layer > 0)
    out = _conv64(xg, w64, b64)
    grads = torch.autograd.grad(out, [w64, b64] + ([xg] if layer > 0 else []), dz.double())
    ws = torch.empty(ops.sconv_wgrad_workspace(N, H, H, ci, co), device="cuda")
    dw, db = torch.full_like(w, float("nan")), torch.full_like(b, float("nan"))
    ops.sconv_wgrad(x.data_ptr(), u8, dz.data_ptr(), dw.data_ptr(), db.data_ptr(), ws, N, H, H, ci, co, tc)
    assert _rel(dw, grads[0]) <= 2e-4, _rel(dw, grads[0])
    assert _rel(db, grads[1]) <= 2e-4, _rel(db, grads[1])
    dw2, db2 = torch.empty_like(dw), torch.empty_like(db)
    ops.sconv_wgrad(x.data_ptr(), u8, dz.data_ptr(), dw2.data_ptr(), db2.data_ptr(), ws, N, H, H, ci, co, tc)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)
    # input gradient through the previous layer's ReLU (its output x > 0)
    if layer > 0:
        dx = torch.full_like(x, float("nan"))
        ops.sconv_dgrad(dz.data_ptr(), w.data_ptr(), x.data_ptr(), dx.data_ptr(), N, H, H, ci, co, tc)
        ref_dx = grads[2] * (x64 > 0)
        assert _rel(dx, ref_dx) <= 2e-4, _rel(dx, ref_dx)
        assert bool((dx[x == 0] == 0).all())
        dx2 = torch.empty_like(dx)
        ops.sconv_dgrad(dz.data_ptr(), w.data_ptr(), x.data_ptr(), dx2.data_ptr(), N, H, H, ci, co, tc)
        assert torch.equal(dx, dx2)


@pytest.mark.parametrize("N", [1, 3, 256, 514])
def test_mean_pool_forward_and_backward(N):
    from serl_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(N)
    y = torch.randn(N, 7, 7, 256, device="cuda", generator=gen).relu_()
    out = torch.full((N, 256), float("nan"), device="cuda")
    ops.sconv_mean_fwd(y.data_ptr(), out.data_ptr(), N, 49, 256)
    assert _rel(out, y.double().mean(dim=(1, 2))) <= 1e-6
    # d(pooled) with a row stride wider than 256
    dpool = torch.randn(N, 300, device="cuda", generator=gen)
    dz = torch.full_like(y, float("nan"))
    ops.sconv_mean_bwd(dpool.data_ptr(), 300, y.data_ptr(), dz.data_ptr(), N, 49, 256)
    ref = (dpool[:, None, None, :256].double() / 49).expand(N, 7, 7, 256) * (y > 0)
    assert _rel(dz, ref) <= 1e-6


def test_wgrad_splits_depend_on_the_shape_only():
    from serl_b200 import ops
    for N in (1, 3, 256, 514):
        for layer, (ci, co) in enumerate(SMALL_CONVS):
            H = SIZES[layer]
            s = ops.sconv_wgrad_splits(N, H, H, ci, co)
            K = N * SIZES[layer + 1] ** 2
            assert 1 <= s <= max(1, -(-K // 256)) and ops.sconv_wgrad_workspace(N, H, H, ci, co) >= (9 * ci + 1) * co
