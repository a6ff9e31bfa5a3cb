"""CPU: DrQ's "small" encoder.  The float64 restatement (tests/small_encoder_oracle.py) against central finite differences, the
parameter tree and its initialisation, the optimizer group of the new leaves, the constructors that build it or keep refusing,
and the host call sequence of a step (kernel launches replaced by a recorder): the convs run inside each loss pass, after the
previous minibatch's Adam."""
import math

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions
from small_encoder_oracle import SMALL_CONVS, conv_stack, image_embedding

ENC = "modules_actor/encoder"


@pytest.fixture()
def dry(monkeypatch):
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


def _random_params(rng, cam="c"):
    p = {}
    for i, (ci, co) in enumerate(SMALL_CONVS):
        p[f"{ENC}/encoder_{cam}/Conv_{i}/kernel"] = torch.as_tensor(rng.standard_normal((3, 3, ci, co)) / math.sqrt(9 * ci))
        p[f"{ENC}/encoder_{cam}/Conv_{i}/bias"] = torch.as_tensor(rng.standard_normal(co) * 0.1)
    p[f"{ENC}/encoder_{cam}/Dense_0/kernel"] = torch.as_tensor(rng.standard_normal((256, 256)) / 16)
    p[f"{ENC}/encoder_{cam}/Dense_0/bias"] = torch.as_tensor(rng.standard_normal(256) * 0.1)
    p[f"{ENC}/encoder_{cam}/LayerNorm_0/scale"] = torch.as_tensor(1 + rng.standard_normal(256) * 0.1)
    p[f"{ENC}/encoder_{cam}/LayerNorm_0/bias"] = torch.as_tensor(rng.standard_normal(256) * 0.1)
    return p


def test_oracle_gradients_match_finite_differences():
    """d(w . embedding) / d(leaf) by autograd against central differences, for sampled entries of every leaf (31x31 images:
    15x15, 7x7, 3x3 and 1x1 maps)."""
    rng = np.random.default_rng(0)
    params = _random_params(rng)
    imgs = torch.as_tensor(rng.integers(0, 256, (2, 31, 31, 3), dtype=np.uint8))
    wsum = torch.as_tensor(rng.standard_normal((2, 256)))
    f = lambda p: (image_embedding(p, "c", imgs) * wsum).sum()
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    grads = dict(zip(leaves, torch.autograd.grad(f(leaves), list(leaves.values()))))
    h = 1e-6
    for k, v in params.items():
        for idx in rng.integers(0, v.numel(), 6):
            up, dn = dict(params), dict(params)
            up[k], dn[k] = v.clone(), v.clone()
            up[k].view(-1)[idx] += h
            dn[k].view(-1)[idx] -= h
            fd = float(f(up) - f(dn)) / (2 * h)
            got = float(grads[k].reshape(-1)[idx])
            assert abs(got - fd) <= 1e-6 * max(1.0, abs(fd)), (k, int(idx), got, fd)


def test_conv_stack_shapes_and_mean_pool():
    rng = np.random.default_rng(1)
    params = _random_params(rng)
    imgs = rng.integers(0, 256, (3, 128, 128, 3), dtype=np.uint8)
    pooled, maps = conv_stack(params, "c", imgs, keep=True)
    assert [tuple(m.shape[1:]) for m in maps] == [(63, 63, 32), (31, 31, 64), (15, 15, 128), (7, 7, 256)]
    torch.testing.assert_close(pooled, maps[-1].reshape(3, 49, 256).sum(1) / 49, rtol=1e-14, atol=0)


def _agent(cams=("front", "wrist"), hw=128, **kw):
    from serl_b200.utils.launcher import make_drq_agent
    trs = random_transitions(np.random.default_rng(0), 1, cams, hw)
    return make_drq_agent(3, trs[0]["observations"], trs[0]["actions"], image_keys=cams, device="cpu", **kw), trs


def test_default_make_drq_agent_builds_the_small_encoder(dry):
    agent, _ = _agent()
    assert agent._cfg.encoder == "small" and agent._cfg.small and agent._frozen_trunk is None and agent._trunk == {}
    enc = agent.state.params["modules_actor"]["encoder"]
    for cam in ("front", "wrist"):
        e = enc[f"encoder_{cam}"]
        assert sorted(e) == ["Conv_0", "Conv_1", "Conv_2", "Conv_3", "Dense_0", "LayerNorm_0"]
        for i, (ci, co) in enumerate(SMALL_CONVS):
            assert e[f"Conv_{i}"]["kernel"].shape == (3, 3, ci, co) and e[f"Conv_{i}"]["bias"].shape == (co,)
        assert e["Dense_0"]["kernel"].shape == (256, 256) and e["Dense_0"]["bias"].shape == (256,)
        assert e["LayerNorm_0"]["scale"].shape == (256,) and e["LayerNorm_0"]["bias"].shape == (256,)
    assert agent._cfg.enc_dim == 2 * 256 + 64
    assert agent.state.params["modules_critic"]["network"]["Dense_0"]["kernel"].shape == (10, 2 * 256 + 64 + 4, 256)


def test_small_leaves_are_critic_group_with_flax_default_init(dry):
    agent, _ = _agent(cams=("front",))
    st = agent._store
    vals = st.dump(st.params)
    p = f"{ENC}/encoder_front"
    for i, (ci, co) in enumerate(SMALL_CONVS):
        for leaf in ("kernel", "bias"):
            assert st.leaf[f"{p}/Conv_{i}/{leaf}"].group == 0
        k = vals[f"{p}/Conv_{i}/kernel"].astype(np.float64)
        std = math.sqrt(1.0 / (9 * ci))                         # lecun_normal: truncated normal, variance 1 / fan_in
        assert abs(k.std() / std - 1) < (0.2 if k.size < 1000 else 0.05), (i, k.std(), std)
        assert np.abs(k).max() <= 2 * std / 0.87962566103423978 + 1e-6
        assert not vals[f"{p}/Conv_{i}/bias"].any()
    d = vals[f"{p}/Dense_0/kernel"].astype(np.float64)
    assert abs(d.std() * 16 - 1) < 0.05 and not vals[f"{p}/Dense_0/bias"].any()
    assert (vals[f"{p}/LayerNorm_0/scale"] == 1).all() and not vals[f"{p}/LayerNorm_0/bias"].any()
    assert all(l.group == 0 for l in st.spec if l.path.startswith(p))


def test_other_encoders_and_horizons_still_raise(dry):
    from serl_b200.agents.continuous.bc import BCAgent
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.utils.launcher import make_vice_agent
    trs = random_transitions(np.random.default_rng(0), 1, ("front",), 16)
    with pytest.raises(NotImplementedError):
        DrQAgent.create_drq(0, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet", image_keys=("front",), device="cpu")
    with pytest.raises(NotImplementedError):
        BCAgent.create(0, trs[0]["observations"], trs[0]["actions"], encoder_type="small", image_keys=("front",), device="cpu")
    with pytest.raises(NotImplementedError):
        make_vice_agent(0, trs[0]["observations"], trs[0]["actions"], image_keys=("front",), device="cpu")
    t2 = random_transitions(np.random.default_rng(0), 1, ("front",), 16, T=2)
    with pytest.raises(NotImplementedError):
        DrQAgent.create_drq(0, t2[0]["observations"], t2[0]["actions"], encoder_type="small", image_keys=("front",), device="cpu")


def _ring(cams, cap, hw=128):
    from serl_b200.utils.launcher import make_replay_buffer
    return make_replay_buffer(fake_env(cams, hw), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams),
                              device="cpu", seed=5)


def _conv_calls(seq):
    return [c for c in seq if c.startswith("serl_sconv") or c in ("serl_adam_polyak", "serl_critic_loss")]


def test_step_call_sequences(dry):
    cams = ("front", "wrist")
    agent, _ = _agent(cams)
    rb = _ring(cams, 64)
    for tr in random_transitions(np.random.default_rng(1), 40, cams, 128):
        rb.insert(tr)
    it = rb.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    eng = agent._engine(4)
    assert eng.fused is None and not hasattr(eng, "feats") and not hasattr(eng, "trunk")
    # update_critics: per camera online obs (saved) + target next + online next (policy) = 3 conv passes of 4 convs, then the
    # backward of the obs rows: 4 wgrads, dgrads of layers 3..1
    del dry[:]
    agent.update_critics(next(it))
    assert "serl_conv2d_nhwc_f32" not in dry and "serl_sle_fwd" not in dry and "serl_dropout_mask_fill" not in dry
    assert dry.count("serl_sconv_fwd") == 2 * 3 * 4 and dry.count("serl_sconv_mean_fwd") == 2 * 3
    assert dry.count("serl_sconv_wgrad") == 2 * 4 and dry.count("serl_sconv_dgrad") == 2 * 3 and dry.count("serl_sconv_mean_bwd") == 2
    seq = _conv_calls(dry)
    assert seq.index("serl_critic_loss") < seq.index("serl_sconv_mean_bwd") and seq[-1] == "serl_adam_polyak"
    # update_high_utd(2): each minibatch's convs run after the previous minibatch's Adam; the actor / temperature passes after the
    # last critic Adam (actor pass + critic Q on obs, temperature pass on next obs: 3 forward passes per camera)
    del dry[:]
    agent.update_high_utd(next(it), utd_ratio=2)
    seq = _conv_calls(dry)
    adams = [i for i, c in enumerate(seq) if c == "serl_adam_polyak"]
    assert len(adams) == 3
    for lo, hi in ((-1, adams[0]), (adams[0], adams[1])):
        part = seq[lo + 1:hi]
        assert part.count("serl_sconv_fwd") == 2 * 3 * 4 and part.count("serl_sconv_wgrad") == 2 * 4
    tail = seq[adams[1] + 1:adams[2]]
    assert tail.count("serl_sconv_fwd") == 2 * 3 * 4 and "serl_sconv_wgrad" not in tail
    # sample_actions / forward passes: one conv pass per camera, no trunk
    del dry[:]
    obs = {c: np.zeros((2, 1, 128, 128, 3), np.uint8) for c in cams}
    obs["state"] = np.zeros((2, 1, 7), np.float32)
    agent.sample_actions(obs, argmax=True)
    assert dry.count("serl_sconv_fwd") == 2 * 4 and "serl_conv2d_nhwc_f32" not in dry
