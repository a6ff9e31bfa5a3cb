"""CPU: DrQ's trainable "resnet" encoder.  The float64 restatement (tests/resnet_encoder_oracle.py) against central finite
differences and its max-pool first-max rule, the parameter tree, groups and initialisation, the constructors that build it or
keep refusing, and the host call sequence of a step (kernel launches replaced by a recorder)."""
import math

import numpy as np
import pytest
import torch

from helpers import random_transitions
from resnet_encoder_oracle import image_embedding, max_pool_first_max
from test_small_encoder_cpu import _ring, dry  # noqa: F401

ENC = "modules_actor/encoder"


def _random_params(rng, cam="c"):
    from serl_b200.params import image_head_leaves, trunk_spec
    p = {}
    for k, shp in trunk_spec():
        if k.endswith("kernel"):
            v = rng.standard_normal(shp) * math.sqrt(2.0 / int(np.prod(shp[:-1])))
        elif k.endswith("scale"):
            v = 1 + 0.2 * rng.standard_normal(shp)
        else:
            v = 0.2 * rng.standard_normal(shp)
        p[f"{ENC}/encoder_{cam}/{k}"] = torch.as_tensor(v)
    for leaf in image_head_leaves(f"{ENC}/encoder_{cam}"):
        fan = leaf.shape[0] if len(leaf.shape) == 2 else 1
        p[leaf.path] = torch.as_tensor(rng.standard_normal(leaf.shape) / math.sqrt(fan) * (1 if "kernel" in leaf.path else 0.1))
    p[f"{ENC}/encoder_{cam}/SpatialLearnedEmbeddings_0/kernel"] = torch.as_tensor(rng.standard_normal((1, 1, 512, 8)) * 0.05)
    p[f"{ENC}/encoder_{cam}/Dense_0/kernel"] = torch.as_tensor(rng.standard_normal((4096, 256)) / 64)
    return p


def test_oracle_gradients_match_finite_differences():
    """d(w . embedding) / d(leaf) by autograd against central differences for sampled entries of every kind of leaf (conv,
    GroupNorm scale and bias, projection conv and norm, SLE kernel) on 32x32 images (16, 8, 8, 4, 2, 1 maps)."""
    rng = np.random.default_rng(0)
    params = _random_params(rng)
    imgs = torch.as_tensor(rng.integers(0, 256, (2, 32, 32, 3), dtype=np.uint8))
    wout = torch.as_tensor(rng.standard_normal((2, 256)))
    p = f"{ENC}/encoder_c"
    leaves = ["conv_init/kernel", "norm_init/scale", "norm_init/bias", "ResNetBlock_0/Conv_0/kernel", "ResNetBlock_0/MyGroupNorm_1/scale",
              "ResNetBlock_1/conv_proj/kernel", "ResNetBlock_1/norm_proj/scale", "ResNetBlock_1/norm_proj/bias",
              "ResNetBlock_2/Conv_1/kernel", "ResNetBlock_3/MyGroupNorm_0/bias", "SpatialLearnedEmbeddings_0/kernel"]
    f = lambda: float((image_embedding(params, "c", imgs) * wout).sum())
    for leaf in leaves:
        t = params[f"{p}/{leaf}"]
        t.requires_grad_(True)
        (image_embedding(params, "c", imgs) * wout).sum().backward()
        g = t.grad.clone()
        t.grad = None
        t.requires_grad_(False)
        flat = t.view(-1)
        for idx in rng.choice(flat.numel(), 3, replace=False):
            h = 1e-6
            old = float(flat[idx])
            flat[idx] = old + h
            up = f()
            flat[idx] = old - h
            dn = f()
            flat[idx] = old
            fd = (up - dn) / (2 * h)
            assert abs(fd - float(g.view(-1)[idx])) <= 1e-5 * max(1.0, abs(fd)), (leaf, idx, fd, float(g.view(-1)[idx]))


def test_maxpool_first_max_rule_on_ties():
    x = torch.zeros(1, 4, 4, 1, dtype=torch.float64)
    x[0, 0, 1, 0] = x[0, 1, 0, 0] = 2.0           # window (0, 0) covers rows / cols 0..2: tie between (0, 1) and (1, 0)
    x[0, 2, 2, 0] = x[0, 2, 3, 0] = 1.0           # window (1, 1): rows / cols 2..3 (+ padding): tie between (2, 2) and (2, 3)
    x.requires_grad_(True)
    y = max_pool_first_max(x)
    assert y.shape == (1, 2, 2, 1)
    y.sum().backward()
    gx = x.grad[0, :, :, 0]
    assert gx[0, 1] == 1 and gx[1, 0] == 0        # the first maximal element in row-major window order
    assert gx[2, 2] >= 1 and gx[2, 3] == 0
    z = torch.zeros(1, 4, 4, 1, dtype=torch.float64, requires_grad=True)      # all-zero windows: each window's first element
    max_pool_first_max(z).sum().backward()
    assert z.grad[0, 0, 0, 0] == 1 and z.grad[0, 0, 2, 0] == 1 and z.grad[0, 2, 0, 0] == 1 and z.grad[0, 2, 2, 0] == 1
    assert float(z.grad.sum()) == 4


def _agent(cams=("front", "wrist"), use_proprio=True):
    from serl_b200.agents.continuous.drq import DrQAgent
    tr = random_transitions(np.random.default_rng(0), 1, cams, 128)[0]
    obs = tr["observations"] if use_proprio else {c: tr["observations"][c] for c in cams}
    return DrQAgent.create_drq(0, obs, tr["actions"], encoder_type="resnet", use_proprio=use_proprio, image_keys=cams, device="cpu")


def test_leaves_groups_and_init(dry):
    from serl_b200.params import image_head_leaves, trunk_spec
    agent = _agent(cams=("front",))
    st = agent._store
    vals = st.dump(st.params)
    p = f"{ENC}/encoder_front"
    for k, shp in trunk_spec():
        leaf = st.leaf[f"{p}/{k}"]
        assert leaf.shape == shp and leaf.group == 0
        v = vals[leaf.path].astype(np.float64)
        if k.endswith("kernel"):                     # kaiming_normal: truncated normal, variance 2 / fan_in
            std = math.sqrt(2.0 / int(np.prod(shp[:-1])))
            assert abs(v.std() / std - 1) < 0.05, (k, v.std(), std)
            assert np.abs(v).max() <= 2 * std / 0.87962566103423978 + 1e-6
        elif k.endswith("scale"):
            assert (v == 1).all()
        else:
            assert not v.any()
    for leaf in image_head_leaves(p):
        assert st.leaf[leaf.path].group == 0
    sle = vals[f"{p}/SpatialLearnedEmbeddings_0/kernel"].astype(np.float64)
    assert abs(sle.std() / math.sqrt(1.0 / (4 * 4 * 512)) - 1) < 0.05          # lecun_normal over fan_in 4*4*512
    assert abs(vals[f"{p}/Dense_0/kernel"].std() * 64 - 1) < 0.05
    assert not any("pretrained_encoder" in l.path for l in st.spec)
    assert agent.state.trunk is None if hasattr(agent.state, "trunk") else True


def test_constructors_that_still_refuse(dry):
    from serl_b200.agents.continuous.bc import BCAgent
    from serl_b200.utils.launcher import make_drq_agent, make_vice_agent
    trs = random_transitions(np.random.default_rng(0), 1, ("front",), 16)
    for enc in ("small", "resnet"):
        with pytest.raises(NotImplementedError):
            BCAgent.create(0, trs[0]["observations"], trs[0]["actions"], encoder_type=enc, image_keys=("front",), device="cpu")
    with pytest.raises(NotImplementedError):
        make_vice_agent(0, trs[0]["observations"], trs[0]["actions"], image_keys=("front",), device="cpu")
    with pytest.raises(NotImplementedError):
        make_vice_agent(0, trs[0]["observations"], trs[0]["actions"], image_keys=("front",), encoder_type="resnet", device="cpu")
    t2 = random_transitions(np.random.default_rng(0), 1, ("front",), 16, T=2)
    from serl_b200.agents.continuous.drq import DrQAgent
    for enc in ("small", "resnet"):
        with pytest.raises(NotImplementedError):
            DrQAgent.create_drq(0, t2[0]["observations"], t2[0]["actions"], encoder_type=enc, image_keys=("front",), device="cpu")
    for hw in (16, 64):                             # the SLE head's (4, 4, 512, 8) kernel is that of 128x128 frames
        with pytest.raises(NotImplementedError):
            t = random_transitions(np.random.default_rng(0), 1, ("front",), hw)[0]
            DrQAgent.create_drq(0, t["observations"], t["actions"], encoder_type="resnet", image_keys=("front",), device="cpu")
    tr = random_transitions(np.random.default_rng(0), 1, ("front",), 128)[0]
    agent = make_drq_agent(0, tr["observations"], tr["actions"], image_keys=("front",), encoder_type="resnet", device="cpu")
    assert agent._cfg.resnet and agent._cfg.trainable_encoder


def test_step_call_sequence(dry):
    """update_high_utd(2): each minibatch's trunk convs run after the previous minibatch's Adam; the critic step's backward runs
    the stem's wgrad last; the pipeline / utd copy crops, not features; no frozen trunk and no fused heads."""
    cams = ("front", "wrist")
    agent = _agent(cams)
    rb = _ring(cams, 64)
    for tr in random_transitions(np.random.default_rng(1), 40, cams, 128):
        rb.insert(tr)
    it = rb.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    eng = agent._engine(4)
    assert eng.fused is None and not hasattr(eng, "feats") and not hasattr(eng, "trunk")
    del dry[:]
    agent.update_high_utd(next(it), utd_ratio=2)
    seq = [c for c in dry if c.startswith(("serl_rconv", "serl_conv2d", "serl_groupnorm_bwd", "serl_vice_sle_input_grad"))
           or c in ("serl_adam_polyak", "serl_critic_loss")]
    adams = [i for i, c in enumerate(seq) if c == "serl_adam_polyak"]
    assert len(adams) == 3
    n_fwd = 12                                      # fp32 build: 12 convs per pass on the CUDA-core forward kernel
    for lo, hi in ((-1, adams[0]), (adams[0], adams[1])):
        part = seq[lo + 1:hi]
        assert part.count("serl_conv2d_nhwc_f32") == 2 * 3 * n_fwd      # online obs (saved), target next, policy next
        assert part.count("serl_rconv_wgrad") == 2 * n_fwd and part.count("serl_rconv_dgrad") == 2 * (n_fwd - 1)
        assert part.count("serl_vice_sle_input_grad") == 2
        assert part.index("serl_critic_loss") < part.index("serl_vice_sle_input_grad")
    tail = seq[adams[1] + 1:adams[2]]
    assert tail.count("serl_conv2d_nhwc_f32") == 2 * 3 * n_fwd and "serl_rconv_wgrad" not in tail
