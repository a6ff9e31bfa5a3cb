"""GPU: the agents' public forward passes (forward_critic / forward_target_critic with single and multiple actions per state,
forward_policy's distribution, forward_temperature, temperature_lagrange_penalty) against the float64 oracle
(tests/forward_oracle.py) on the fp32 build at 1e-5 (the fp16 build at 1e-2); the distribution's mode and sample against
sample_actions bit for bit; the multi-action kernel against N single-action calls; and isolation: forward calls between
pipelined update_critics steps change no bit of what the steps compute."""
import numpy as np
import pytest
import torch

import forward_oracle as FO
from helpers import oracle_state_from_agent, random_transitions, rel_err
from test_agent_gpu import _perturb, _setup

pytestmark = pytest.mark.gpu
TOL, TOL16 = 1e-5, 1e-2
A = 4


def _obs(rng, cams, B):
    obs = {c: rng.integers(0, 256, (B, 1, 128, 128, 3), dtype=np.uint8) for c in cams}
    obs["state"] = rng.standard_normal((B, 1, 7)).astype(np.float32)
    return obs


def _np(t):
    return t.detach().cpu().numpy()


def _check_critics(agent, obs, one, tol, B, key):
    """Online and target critic, single and multiple actions per state, batched and unbatched, against the oracle."""
    o = oracle_state_from_agent(agent)
    rng = np.random.default_rng(5)
    E = agent._cfg.ensemble
    acts = rng.uniform(-1, 1, (B, A)).astype(np.float32)
    q = agent.forward_critic(obs, acts, key)
    qt = agent.forward_target_critic(obs, acts, key)
    assert q.shape == qt.shape == (E, B)
    assert rel_err(_np(q), FO.critic(agent, o.params, obs, acts).numpy()) < tol
    assert rel_err(_np(qt), FO.critic(agent, o.target_params, obs, acts).numpy()) < tol
    assert float((q - qt).abs().max()) > 1e-4 * float(q.abs().max()), "target critic gave the online values"
    torch.testing.assert_close(agent.forward_critic(obs, acts, None, train=False), q, rtol=0, atol=0)
    for N in (1, 7):
        multi = rng.uniform(-1, 1, (B, N, A)).astype(np.float32)
        for fwd, params in ((agent.forward_critic, o.params), (agent.forward_target_critic, o.target_params)):
            qm = fwd(obs, multi, key)
            assert qm.shape == (E, B, N)
            stacked = torch.stack([fwd(obs, multi[:, n], key) for n in range(N)], -1)
            assert rel_err(_np(qm), _np(stacked)) < tol, N
            assert rel_err(_np(qm), FO.critic(agent, params, obs, multi).numpy()) < tol, N
        q1 = agent.forward_critic(one, multi[0], key)
        assert q1.shape == (E, N) and rel_err(_np(q1), _np(agent.forward_critic(obs, multi, key)[:, 0])) < tol
    assert agent.forward_critic(one, acts[0], key).shape == (E,)


def _check_policy(agent, obs, one, tol, B):
    o = oracle_state_from_agent(agent)
    rng = np.random.default_rng(6)
    d = agent.forward_policy(obs, train=False)
    assert torch.equal(d.mode(), agent.sample_actions(obs, argmax=True, return_device=True))
    key = np.array([123, 456], np.uint32)
    assert torch.equal(d.sample(seed=key), agent.sample_actions(obs, seed=key, return_device=True))
    mu, sd = FO.policy(agent, o.params, obs)
    assert rel_err(_np(d.loc), mu.numpy()) < tol and rel_err(_np(d.scale_diag), sd.numpy()) < tol
    assert rel_err(_np(d.stddev()), torch.tanh(sd).numpy()) < tol
    a, lp = d.sample_and_log_prob(seed=key)
    ra, rlp = FO.sample_and_log_prob(mu, sd, key)
    assert torch.equal(a, d.sample(seed=key)) and rel_err(_np(a), ra.numpy()) < tol and rel_err(_np(lp), rlp.numpy()) < tol
    x = rng.uniform(-0.99, 0.99, (B, A)).astype(np.float32)
    assert rel_err(_np(d.log_prob(x)), FO.tanh_normal_log_prob(mu, sd, x).numpy()) < tol
    d1 = agent.forward_policy(one, train=False)
    assert torch.equal(d1.mode(), agent.sample_actions(one, argmax=True, return_device=True))
    assert torch.equal(d1.sample(seed=key), agent.sample_actions(one, seed=key, return_device=True))
    assert d1.log_prob(x[0]).shape == ()


def _check_temperature(agent):
    lam = float(agent._store.view(agent._store.params, "modules_temperature/lagrange"))
    alpha = float(torch.nn.functional.softplus(torch.tensor(lam, dtype=torch.float64)))
    assert abs(float(agent.forward_temperature()) - alpha) <= 1e-6 * alpha
    ent = np.array([0.3, -1.5, 2.0], np.float32)
    ref = alpha * (ent.astype(np.float64) - agent.config["target_entropy"])
    assert rel_err(_np(agent.temperature_lagrange_penalty(torch.as_tensor(ent, device="cuda"))), ref) < 1e-6


def test_pixel_agent_matches_oracle_after_updates():
    cams, B = ("front", "wrist"), 5
    agent, rb = _setup(cams, 8, seed=11)
    _perturb(agent, seed=2)
    it = rb.get_iterator(sample_args={"batch_size": 8, "pack_obs_and_next_obs": True})
    for _ in range(3):
        agent.update_critics(next(it))
    rng = np.random.default_rng(0)
    obs = _obs(rng, cams, B)
    one = {k: v[0] for k, v in obs.items()}
    rng0, step0, graphs0 = agent.state.rng.copy(), agent.state.step, len(agent._graphs)
    _check_critics(agent, obs, one, TOL, B, np.array([0, 9], np.uint32))
    _check_policy(agent, obs, one, TOL, B)
    _check_temperature(agent)
    np.testing.assert_array_equal(agent.state.rng, rng0)
    assert agent.state.step == step0 == 3 and len(agent._graphs) == graphs0


def test_pixel_policy_dropout_masks_match_oracle():
    """train=True: camera j's keep-mask is bernoulli(fold_in(rng, j), 0.9), bit for bit; the distribution follows it."""
    from oracle import drq as O
    cams, B = ("front", "wrist"), 6
    agent, _ = _setup(cams, 8, seed=12)
    _perturb(agent, seed=3)
    obs = _obs(np.random.default_rng(1), cams, B)
    key = np.array([7, 2024], np.uint32)
    d = agent.forward_policy(obs, key)
    masks = O._dropout_masks(key, cams, B)
    eng = agent._infer_engines[B]
    for cam in cams:
        np.testing.assert_array_equal(_np(eng.masks_u8[cam]).astype(bool), masks[cam])
    mu, sd = FO.policy(agent, oracle_state_from_agent(agent).params, obs, dropout_key=key)
    assert rel_err(_np(d.loc), mu.numpy()) < TOL and rel_err(_np(d.scale_diag), sd.numpy()) < TOL
    assert not torch.equal(d.loc, agent.forward_policy(obs, train=False).loc)


STATE_CASES = {
    "launcher": {},
    # a non-launcher architecture: relu without LayerNorm, "uniform" std, critic and policy of different widths and depths
    "relu_uniform": dict(critic_network_kwargs={"hidden_dims": [256, 128], "activations": "relu", "use_layer_norm": False},
                         policy_network_kwargs={"hidden_dims": [192], "activations": "relu", "use_layer_norm": False},
                         policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "uniform", "std_min": 1e-5, "std_max": 5}),
}


@pytest.mark.parametrize("case", sorted(STATE_CASES))
def test_state_agent_matches_oracle_after_updates(case):
    from serl_b200.agents.continuous.sac import SACAgent
    S, B = 10, 6
    rng = np.random.default_rng(0)
    agent = SACAgent.create_states(42, rng.standard_normal(S).astype(np.float32), rng.uniform(-1, 1, A).astype(np.float32),
                                   temperature_init=1e-2, discount=0.99, critic_ensemble_size=10, critic_subsample_size=2,
                                   **STATE_CASES[case])
    _perturb(agent, seed=4)
    agent._store.counts.fill_(700)                                   # inside the warm-up ramp: the updates move the parameters
    for _ in range(2):
        batch = dict(observations=rng.standard_normal((32, S)).astype(np.float32), next_observations=rng.standard_normal((32, S)).astype(np.float32),
                     actions=rng.uniform(-1, 1, (32, A)).astype(np.float32), rewards=rng.random(32).astype(np.float32),
                     masks=np.ones(32, np.float32), dones=np.zeros(32, bool))
        agent.update(batch)
    obs = rng.standard_normal((B, S)).astype(np.float32)
    rng0, step0 = agent.state.rng.copy(), agent.state.step
    _check_critics(agent, obs, obs[0], TOL, B, np.array([0, 9], np.uint32))
    _check_policy(agent, obs, obs[0], TOL, B)
    _check_temperature(agent)
    np.testing.assert_array_equal(agent.state.rng, rng0)
    assert agent.state.step == step0 == 2


def test_fp16_build_matches_oracle():
    from serl_b200.utils.launcher import make_drq_agent
    cams, B = ("front", "wrist"), 5
    trs = random_transitions(np.random.default_rng(2), 4, cams)
    agent = make_drq_agent(9, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", precision="fp16")
    _perturb(agent, seed=5)
    o = oracle_state_from_agent(agent)
    rng = np.random.default_rng(3)
    obs = _obs(rng, cams, B)
    key = np.array([1, 2], np.uint32)
    acts, multi = rng.uniform(-1, 1, (B, A)).astype(np.float32), rng.uniform(-1, 1, (B, 16, A)).astype(np.float32)
    assert rel_err(_np(agent.forward_critic(obs, acts, key)), FO.critic(agent, o.params, obs, acts).numpy()) < TOL16
    assert rel_err(_np(agent.forward_target_critic(obs, multi, key)), FO.critic(agent, o.target_params, obs, multi).numpy()) < TOL16
    d = agent.forward_policy(obs, train=False)
    mu, sd = FO.policy(agent, o.params, obs)
    assert rel_err(_np(d.loc), mu.numpy()) < TOL16 and rel_err(_np(d.scale_diag), sd.numpy()) < TOL16
    assert torch.equal(d.mode(), agent.sample_actions(obs, argmax=True, return_device=True))


def test_forward_calls_between_pipelined_steps_change_nothing():
    """Pipelined update_critics at batch B, with sample_actions and every forward method called at batch B between the steps:
    losses, infos, parameters, target parameters and the key chain are bitwise those of the same sequence without the calls."""
    cams, B = ("front", "wrist"), 8
    runs = []
    for with_calls in (False, True):
        agent, rb = _setup(cams, B, seed=21)
        agent.pipeline_critic_steps = True
        it = rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})
        rng = np.random.default_rng(4)
        obs = _obs(rng, cams, B)
        acts, multi = rng.uniform(-1, 1, (B, A)).astype(np.float32), rng.uniform(-1, 1, (B, 3, A)).astype(np.float32)
        key = np.array([5, 6], np.uint32)
        out = []
        for step in range(6):                                         # W eager, P eager, P capture, P replay ...
            agent, info = agent.update_critics(next(it))
            out.append(([float(info["critic"][k]) for k in ("critic_loss", "predicted_qs", "target_qs")], float(info["critic_lr"]),
                        agent._store.params.clone(), agent._store.target.clone(), agent.state.rng.copy()))
            if with_calls:
                rng0, step0, graphs0 = agent.state.rng.copy(), agent.state.step, len(agent._graphs)
                agent.sample_actions(obs, seed=key)
                agent.sample_actions(obs, argmax=True)
                agent.forward_critic(obs, acts, key)
                agent.forward_critic(obs, multi, key)
                agent.forward_target_critic(obs, acts, key)
                d = agent.forward_policy(obs, key)
                d.sample_and_log_prob(seed=key)
                d.log_prob(acts * 0.5)
                agent.forward_policy(obs, train=False).stddev()
                agent.forward_temperature()
                agent.temperature_lagrange_penalty(1.0)
                np.testing.assert_array_equal(agent.state.rng, rng0)
                assert agent.state.step == step0 and len(agent._graphs) == graphs0
        agent.check_status()
        runs.append(out)
    for step, (a, b) in enumerate(zip(*runs)):
        assert a[0] == b[0] and a[1] == b[1], step
        assert torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]), step
        np.testing.assert_array_equal(a[4], b[4])
