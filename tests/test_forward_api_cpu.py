"""CPU: the agents' public forward passes (forward_critic / forward_target_critic / forward_policy / forward_temperature /
temperature_lagrange_penalty) with the kernel launches replaced by a recorder, as in test_dryrun_cpu.py: argument checks, result
shapes for batched and unbatched, pixel and state observations, which entry points run (the encoder once per state for
multi-action Q), and that the inference engines are not the training engines.  Plus the float64 oracle's log_prob."""
import numpy as np
import pytest
import torch

from helpers import random_transitions

A = 4


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

    monkeypatch.setattr(L, "call", fake_call)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: len(calls))
    return calls


def _pixel_agent():
    from serl_b200.utils.launcher import make_drq_agent
    cams = ("front", "wrist")
    trs = random_transitions(np.random.default_rng(0), 6, cams, 128)
    agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu")
    batch = {k: np.stack([t["observations"][k] for t in trs]) for k in (*cams, "state")}
    one = {k: v[0] for k, v in batch.items()}
    return agent, batch, one


def _state_agent():
    from serl_b200.utils.launcher import make_sac_agent
    rng = np.random.default_rng(0)
    agent = make_sac_agent(0, rng.standard_normal(10).astype(np.float32), np.zeros(A, np.float32), device="cpu")
    batch = rng.standard_normal((6, 10)).astype(np.float32)
    return agent, batch, batch[0]


@pytest.mark.parametrize("kind", ["pixel", "state"])
def test_result_shapes(dry, kind):
    agent, batch, one = (_pixel_agent if kind == "pixel" else _state_agent)()
    E, B, N, key = agent._cfg.ensemble, 6, 5, np.array([0, 3], np.uint32)
    assert agent.forward_critic(batch, np.zeros((B, A), np.float32), key).shape == (E, B)
    assert agent.forward_critic(batch, np.zeros((B, N, A), np.float32), key).shape == (E, B, N)
    assert agent.forward_critic(one, np.zeros(A, np.float32), None, train=False).shape == (E,)
    assert agent.forward_critic(one, np.zeros((N, A), np.float32), key).shape == (E, N)
    assert agent.forward_target_critic(batch, torch.zeros(B, 1, A), key).shape == (E, B, 1)
    d = agent.forward_policy(batch, key)
    assert d.loc.shape == d.scale_diag.shape == d.mode().shape == d.stddev().shape == d.sample(seed=key).shape == (B, A)
    act, logp = d.sample_and_log_prob(seed=key)
    assert act.shape == (B, A) and logp.shape == (B,) and d.log_prob(np.zeros((B, A), np.float32)).shape == (B,)
    d1 = agent.forward_policy(one, train=False)
    assert d1.mode().shape == d1.sample(seed=key).shape == (A,) and d1.log_prob(np.zeros(A)).shape == ()
    assert agent.forward_temperature().shape == () and agent.temperature_lagrange_penalty(1.5).shape == ()
    assert agent.temperature_lagrange_penalty(np.ones(3, np.float32)).shape == (3,)


def test_argument_checks(dry):
    agent, batch, one = _state_agent()
    key = np.array([0, 1], np.uint32)
    with pytest.raises(AssertionError, match="rng"):
        agent.forward_critic(batch, np.zeros((6, A), np.float32), None)
    with pytest.raises(AssertionError, match="rng"):
        agent.forward_policy(batch)
    with pytest.raises(AssertionError, match="rng"):
        agent.forward_target_critic(batch, np.zeros((6, A), np.float32), None)
    for call in (lambda g: agent.forward_critic(batch, np.zeros((6, A), np.float32), key, grad_params=g),
                 lambda g: agent.forward_policy(batch, key, grad_params=g),
                 lambda g: agent.forward_temperature(grad_params=g),
                 lambda g: agent.temperature_lagrange_penalty(1.0, grad_params=g)):
        with pytest.raises(NotImplementedError, match="grad_params"):
            call(agent.state.params)
    for bad in (np.zeros(A), np.zeros((6, 2, 3, A)), np.zeros((6, A + 1)), np.zeros((5, A)), np.zeros((6, 2, A - 1))):
        with pytest.raises(ValueError, match="actions of shape"):
            agent.forward_critic(batch, bad, key)
    for bad in (np.zeros((6, A + 1)), np.zeros((2, 3, A)), np.zeros(())):
        with pytest.raises(ValueError, match="actions of shape"):
            agent.forward_critic(one, bad, key)
    with pytest.raises(ValueError, match="log_prob"):
        agent.forward_policy(batch, train=False).log_prob(np.zeros((5, A)))


def test_call_sequences_and_separate_engines(dry):
    agent, batch, one = _pixel_agent()
    key = np.array([0, 3], np.uint32)
    del dry[:]
    agent.forward_critic(batch, np.zeros((6, 16, A), np.float32), key)
    # the trunk and encoder heads run once per state (2 cameras), not once per candidate action
    assert dry.count("serl_conv2d_nhwc_f32") == 2 * 12 and dry.count("serl_sle_fwd") == 2
    assert dry.count("serl_critic_multi_action_fwd") == 1 and dry.count("serl_copy2d_f32") == 0
    del dry[:]
    agent.forward_critic(batch, np.zeros((6, A), np.float32), key)
    assert dry.count("serl_critic_multi_action_fwd") == 0 and dry.count("serl_copy2d_f32") == 1
    del dry[:]
    agent.forward_policy(batch, key)                                   # train=True: one keep-mask per camera
    assert dry.count("serl_dropout_mask_fill") == 2 and dry.count("serl_tanh_gaussian_fwd") == 1
    del dry[:]
    agent.forward_policy(batch, key, train=False).log_prob(np.zeros((6, A), np.float32))
    assert dry.count("serl_dropout_mask_fill") == 0 and dry.count("serl_tanh_normal_log_prob") == 1
    agent.sample_actions(batch, seed=key)
    # inference never allocates or touches a training engine
    assert agent._engines == {} and set(agent._infer_engines) == {6}
    rng0, step0 = np.array(agent.state.rng), agent.state.step
    agent.forward_temperature()
    np.testing.assert_array_equal(agent.state.rng, rng0)
    assert agent.state.step == step0


def test_oracle_log_prob_matches_sample_and_log_prob():
    """float64: log_prob of the sample that tanh_normal_sample_logp drew gives its log-probability back."""
    from forward_oracle import tanh_normal_log_prob
    from oracle.drq import tanh_normal_sample_logp
    g = torch.Generator().manual_seed(0)
    means = torch.randn(64, 7, generator=g, dtype=torch.float64)
    stds = torch.rand(64, 7, generator=g, dtype=torch.float64) * 0.8 + 0.05
    eps = torch.randn(64, 7, generator=g, dtype=torch.float64)
    a, lp = tanh_normal_sample_logp(means, stds, eps)
    torch.testing.assert_close(tanh_normal_log_prob(means, stds, a), lp, rtol=1e-9, atol=1e-9)
    assert torch.isnan(tanh_normal_log_prob(means[:1], stds[:1], torch.ones(1, 7, dtype=torch.float64))).all()


def test_oracle_multi_action_critic_stacks_single_calls():
    import arch_oracle
    from forward_oracle import multi_action_critic
    from serl_b200.params import MlpArch
    arch = MlpArch((64, 64), "relu", False)
    g = torch.Generator().manual_seed(1)
    E, B, N, Fd = 3, 5, 4, 9
    p = {"modules_critic/network/Dense_0/kernel": torch.randn(E, Fd + A, 64, generator=g, dtype=torch.float64),
         "modules_critic/network/Dense_0/bias": torch.randn(E, 64, generator=g, dtype=torch.float64),
         "modules_critic/network/Dense_1/kernel": torch.randn(E, 64, 64, generator=g, dtype=torch.float64),
         "modules_critic/network/Dense_1/bias": torch.randn(E, 64, generator=g, dtype=torch.float64),
         "modules_critic/Dense_0/kernel": torch.randn(64, 1, generator=g, dtype=torch.float64),
         "modules_critic/Dense_0/bias": torch.randn(1, generator=g, dtype=torch.float64)}
    enc, acts = torch.randn(B, Fd, generator=g, dtype=torch.float64), torch.randn(B, N, A, generator=g, dtype=torch.float64)
    q = multi_action_critic(p, enc, acts, arch, True)
    assert q.shape == (E, B, N)
    for n in range(N):
        torch.testing.assert_close(q[:, :, n], arch_oracle.critic_forward(p, enc, acts[:, n], arch, True), rtol=0, atol=0)
