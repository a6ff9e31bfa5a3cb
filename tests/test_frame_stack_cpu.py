"""CPU: frame stacks (ChunkingWrapper(obs_horizon=T)) for the trainable encoders, without a GPU.

- The oracle's stacked encoders equal a direct numpy restatement of EncodingWrapper(enable_stacking=True) + the encoder's first
  layer ("B T H W C -> B H W (T C)", then SmallEncoder's Conv_0 3x3/2 VALID + ReLU, or ResNetEncoder's normalisation + conv_init
  7x7/2 + GroupNorm + ReLU) at T in {2, 3}; at T = 1 they are the existing oracles exactly.
- Parameter shapes and initial-value scale at T = 3: Conv_0 (3, 3, 9, 32) lecun_normal, conv_init (7, 7, 9, 64) kaiming_normal.
- The refusals that stay: "resnet-pretrained" DrQ and VICE agents and the reward classifier with T > 1.
"""
import numpy as np
import pytest
import torch

from frame_stack_oracle import resnet_stack_oracle, stack
from helpers import random_transitions
from oracle import drq as O


@pytest.fixture()
def dry(monkeypatch):
    """The library's calls recorded instead of launched: host logic only."""
    from serl_b200 import _lib as L
    calls = []
    real_call = L.call

    def fake_call(name, *args):
        if name.startswith("serl_host_"):
            return real_call(name, *args)
        calls.append(name)
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    monkeypatch.setattr(L, "call", fake_call)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(L, "new_event", lambda: Ev())
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: len(calls))
    return calls


def _params(rng, encoder, T):
    from serl_b200.params import camera_encoder_leaves, init_leaves, kaiming_in_resnet_encoder
    spec = camera_encoder_leaves(f"{O.ENC}/encoder_cam", encoder, in_channels=3 * T)
    vals = init_leaves(rng, spec, kaiming=kaiming_in_resnet_encoder)
    return {k: torch.as_tensor(v).double() for k, v in vals.items()}


def _conv_np(x, w, stride, pad):
    """NHWC x, HWIO w: a direct sum over the taps."""
    N, H, W, Ci = x.shape
    kh, kw, _, Co = w.shape
    xp = np.pad(x, ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    Ho, Wo = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
    out = np.zeros((N, Ho, Wo, Co))
    for i in range(kh):
        for j in range(kw):
            patch = xp[:, i:i + stride * Ho:stride, j:j + stride * Wo:stride, :]
            out += patch @ w[i, j]
    return out


def _frames(T, B=2, hw=32, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (B, T, hw, hw, 3), dtype=np.uint8)


@pytest.mark.parametrize("T", [2, 3])
def test_small_stacked_first_conv_matches_numpy(T):
    from small_encoder_oracle import conv_stack
    p = _params(np.random.default_rng(T), "small", T)
    imgs = _frames(T)
    x = np.concatenate([imgs[:, t] for t in range(T)], axis=-1).astype(np.float64) / 255.0   # channel t*3 + c = frame t, channel c
    k, b = p[f"{O.ENC}/encoder_cam/Conv_0/kernel"].numpy(), p[f"{O.ENC}/encoder_cam/Conv_0/bias"].numpy()
    ref = np.maximum(_conv_np(x, k, 2, 0) + b, 0)
    _, maps = conv_stack(p, "cam", stack(imgs), keep=True)
    np.testing.assert_allclose(maps[0].numpy(), ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("T", [2, 3])
def test_resnet_stacked_stem_matches_numpy(T):
    import resnet_encoder_oracle as R
    p = _params(np.random.default_rng(T), "resnet", T)
    imgs = _frames(T)
    mean, std = np.array(O.IMAGENET_MEAN), np.array(O.IMAGENET_STD)
    x = np.concatenate([(imgs[:, t].astype(np.float64) / 255.0 - mean) / std for t in range(T)], axis=-1)
    z = _conv_np(x, p[f"{O.ENC}/encoder_cam/conv_init/kernel"].numpy(), 2, 3)
    N, H, W, C = z.shape
    g = z.reshape(N, H * W, 4, C // 4)
    mu, var = g.mean(axis=(1, 3), keepdims=True), g.var(axis=(1, 3), keepdims=True)
    zn = ((g - mu) / np.sqrt(var + 1e-5)).reshape(N, H, W, C)
    ref = np.maximum(zn * p[f"{O.ENC}/encoder_cam/norm_init/scale"].numpy() + p[f"{O.ENC}/encoder_cam/norm_init/bias"].numpy(), 0)
    with resnet_stack_oracle(T):
        _, acts = R.trunk(p, "cam", stack(imgs), keep=True)
    np.testing.assert_allclose(acts["stem"].numpy(), ref, rtol=1e-9, atol=1e-9)


def test_stacked_oracles_at_one_frame_are_the_existing_oracles():
    import resnet_encoder_oracle as R
    from small_encoder_oracle import conv_stack
    imgs = _frames(1, hw=64)
    for encoder in ("small", "resnet"):
        p = _params(np.random.default_rng(5), encoder, 1)
        x = stack(imgs)
        assert np.array_equal(x, imgs[:, 0])
        if encoder == "small":
            assert torch.equal(conv_stack(p, "cam", x), conv_stack(p, "cam", imgs[:, 0]))
        else:
            with resnet_stack_oracle(1):
                a = R.trunk(p, "cam", x)
            assert torch.equal(a, R.trunk(p, "cam", imgs[:, 0]))


def test_parameter_shapes_and_fan_in_at_three_frames():
    from serl_b200.params import trainable_spec
    spec = {l.path: l.shape for l in trainable_spec(("cam",), 21, 4, 2, True, encoder="small", in_channels=9)}
    assert spec[f"{O.ENC}/encoder_cam/Conv_0/kernel"] == (3, 3, 9, 32)
    assert spec[f"{O.ENC}/encoder_cam/Conv_1/kernel"] == (3, 3, 32, 64)
    assert spec[f"{O.ENC}/Dense_0/kernel"] == (21, 64)                      # proprio Dense on T*S = 3*7 state values
    spec = {l.path: l.shape for l in trainable_spec(("cam",), 21, 4, 2, True, encoder="resnet", in_channels=9)}
    assert spec[f"{O.ENC}/encoder_cam/conv_init/kernel"] == (7, 7, 9, 64)
    assert spec[f"{O.ENC}/encoder_cam/ResNetBlock_0/Conv_0/kernel"] == (3, 3, 64, 64)
    # truncated normal of std sqrt(scale / fan_in): fan_in = kh * kw * 3T
    for encoder, leaf, scale, fan_in in (("small", "Conv_0", 1.0, 81), ("resnet", "conv_init", 2.0, 441)):
        w = _params(np.random.default_rng(0), encoder, 3)[f"{O.ENC}/encoder_cam/{leaf}/kernel"].numpy()
        # the truncated normal's std is its scale's; the sample std is within a few percent at these sizes
        assert abs(w.std() / np.sqrt(scale / fan_in) - 1) < 0.05, (encoder, w.std(), np.sqrt(scale / fan_in))


def test_stacked_agents_build_and_the_refusals_stay(dry):
    from serl_b200.agents.continuous.bc import BCAgent
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.networks.reward_classifier import create_classifier
    from serl_b200.utils.launcher import make_drq_agent, make_vice_agent
    t3 = random_transitions(np.random.default_rng(0), 1, ("front",), T=3)[0]
    for enc, leaf, shp in (("small", "Conv_0", (3, 3, 9, 32)), ("resnet", "conv_init", (7, 7, 9, 64))):
        agent = make_drq_agent(0, t3["observations"], t3["actions"], image_keys=("front",), encoder_type=enc, device="cpu")
        assert agent._cfg.obs_horizon == 3 and agent._cfg.state_in == 21
        assert agent._store.leaf[f"{O.ENC}/encoder_front/{leaf}/kernel"].shape == shp
        bc = BCAgent.create(0, t3["observations"], t3["actions"], encoder_type=enc, image_keys=("front",), use_proprio=True, device="cpu")
        assert bc._cfg.obs_horizon == 3 and bc._store.leaf[f"{O.ENC}/encoder_front/{leaf}/kernel"].shape == shp
    with pytest.raises(NotImplementedError, match="obs_horizon must be 1"):
        DrQAgent.create_drq(0, t3["observations"], t3["actions"], encoder_type="resnet-pretrained", image_keys=("front",), device="cpu")
    with pytest.raises(NotImplementedError):
        make_vice_agent(0, t3["observations"], t3["actions"], image_keys=("front",), device="cpu")
    with pytest.raises(NotImplementedError, match="obs_horizon 1"):
        create_classifier(np.random.default_rng(0), t3["observations"], ["front"])
    t9 = random_transitions(np.random.default_rng(0), 1, ("front",), T=9)[0]
    with pytest.raises(NotImplementedError, match="obs_horizon=9"):
        make_drq_agent(0, t9["observations"], t9["actions"], image_keys=("front",), encoder_type="small", device="cpu")
