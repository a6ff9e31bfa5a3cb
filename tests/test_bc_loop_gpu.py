"""GPU: BCAgent's learner loop (reference examples/bc_policy.py).  The device key chain against the host derivation it replaced,
the captured step against the eager one and against the dict-batch path, and a run that is checkpointed, restored into a fresh
agent and continued against an uninterrupted one, with the restored policy's evaluation actions.  fp32 and fp16 builds."""
import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

pytestmark = pytest.mark.gpu

CAMS = ("front", "wrist")
LAUNCHER = None                                                      # make_bc_agent's MLP: [256, 256] tanh, no LayerNorm
DROPOUT = {"activations": "tanh", "use_layer_norm": True, "hidden_dims": [256, 256], "dropout_rate": 0.1}
TRS = random_transitions(np.random.default_rng(0), 60, CAMS)


def _agent(precision, seed=3, mlp=LAUNCHER, use_proprio=True):
    from serl_b200.agents.continuous.bc import BCAgent
    return BCAgent.create(seed, TRS[0]["observations"], TRS[0]["actions"], encoder_type="resnet-pretrained", image_keys=CAMS,
                          use_proprio=use_proprio, network_kwargs=mlp, precision=precision,
                          policy_kwargs={"tanh_squash_distribution": False, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5})


def _ring(seed=11):
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(CAMS), capacity=64, type="memory_efficient_replay_buffer", image_keys=list(CAMS), seed=seed)
    for tr in TRS:
        rb.insert(tr)
    return rb


def _iterator(rb, B):
    return rb.get_iterator(sample_args={"batch_size": B, "pack_obs_and_next_obs": True})      # bc_policy.py:158-164


def _host_chain(rng):
    """BCAgent.update's key chain as the host computed it before it moved to the device: new_rng, k = split(rng); key = split(k)[1]."""
    from serl_b200.agents.continuous.sac import _host_split
    new_rng, k = _host_split(rng, 2)
    return new_rng, _host_split(k, 2)[1]


def _assert_same_state(a, b):
    sa, sb = a._store, b._store
    for name in ("params", "target", "m", "v", "counts"):
        assert torch.equal(getattr(sa, name), getattr(sb, name)), name
    assert np.array_equal(a.state.rng, b.state.rng) and a.state.step == b.state.step


@pytest.mark.parametrize("mlp", [LAUNCHER, DROPOUT], ids=["launcher", "dropout"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_device_key_chain_matches_the_host_chain(precision, mlp):
    """Agent `dev` keys its masks on the device; agent `host` gets the masks of the host-derived key through explicit_dropout.
    Masks, infos, parameters, Adam state and rng: bitwise equal over 5 steps."""
    from serl_b200 import ops
    dev, host = _agent(precision, mlp=mlp), _agent(precision, mlp=mlp)
    rb = _ring()
    B = 32
    key = torch.zeros(2, dtype=torch.uint32, device="cuda")
    rng = host.state.rng
    for _ in range(5):
        batch = rb.sample(B, pack_obs_and_next_obs=True).to_dict()
        rng, drop = _host_chain(rng)
        key.copy_(torch.from_numpy(drop.view(np.int32)).view(torch.uint32))
        masks = {}
        for j, cam in enumerate(CAMS):
            masks[cam] = torch.empty(B, 4096, dtype=torch.uint8, device="cuda")
            ops.dropout_mask_fill(key.data_ptr(), j, 0.9, masks[cam], B * 4096)
        hidden = host.arch.hidden if host.arch.dropout else ()
        masks["mlp"] = [torch.empty(B, H, dtype=torch.uint8, device="cuda") for H in hidden]
        for i, m in enumerate(masks["mlp"]):
            ops.dropout_mask_fill(key.data_ptr(), len(CAMS) + i, 1.0 - host.arch.dropout, m, m.numel())
        host.explicit_dropout = {cam: masks[cam].cpu().numpy() for cam in CAMS} | {"mlp": [m.cpu().numpy() for m in masks["mlp"]]}
        _, ih = host.update(batch)
        _, idv = dev.update(batch)
        b = dev._bufs[B]
        for cam in CAMS:
            assert torch.equal(b["masks"][cam], masks[cam]), cam
        for got, want in zip(b.get("mlp_masks") or (), masks["mlp"]):
            assert torch.equal(got, want)
        assert all(torch.equal(idv[k], ih[k]) for k in ("actor_loss", "mse"))
        np.testing.assert_array_equal(dev.state.rng, rng)
        _assert_same_state(dev, host)


# batch 256 (bc_policy.py's default), and the sizes where serl_bc_loss / serl_bc_loss_std run one row per thread of their one
# 1024-thread CTA (2) or loop over rows (1100), as in test_bc_options_ops_gpu.py
CASES = [(256, True, LAUNCHER), (256, False, DROPOUT), (2, True, DROPOUT), (2, False, LAUNCHER), (1100, True, LAUNCHER),
         (1100, False, DROPOUT)]


@pytest.mark.parametrize("B,use_proprio,mlp", CASES, ids=[f"B{c[0]}-{'proprio' if c[1] else 'pixels'}-{'launcher' if c[2] is None else 'dropout'}"
                                                         for c in CASES])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_captured_step_equals_eager(precision, B, use_proprio, mlp):
    """Three agents, three identical rings: the dict batch of each handle (to_dict + ingest), the sampler-loaded eager step and the
    captured step (warm-up, capture, replays).  Infos every step and the whole state after 5 steps: bitwise equal."""
    agents = [_agent(precision, mlp=mlp, use_proprio=use_proprio) for _ in range(3)]
    agents[1].use_cuda_graphs = False
    its = [_iterator(_ring(), B) for _ in range(3)]
    for _ in range(5):
        batches = [next(it) for it in its]
        infos = [agents[0].update(batches[0].to_dict())[1], agents[1].update(batches[1])[1], agents[2].update(batches[2])[1]]
        for k in ("actor_loss", "mse"):
            assert infos[0][k].dim() == 0 and infos[0][k].is_cuda
            assert torch.equal(infos[1][k], infos[0][k]) and torch.equal(infos[2][k], infos[0][k]), k
    assert not agents[1]._graphs and len(agents[2]._graphs) == 1
    for a in agents[1:]:
        _assert_same_state(agents[0], a)
        a.check_status()


def _train(agent, it, steps, log):
    for _ in range(steps):                                           # bc_policy.py:166-169
        batch = next(it)
        agent, info = agent.update(batch)
        log.append({k: v.clone() for k, v in info.items()})
    return agent


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_checkpoint_restore_continues_the_run(tmp_path, precision):
    """bc_policy.py's training mode stopped after N steps (save_checkpoint), a fresh agent restoring it (restore_checkpoint +
    agent.replace(state=...)) and training M more, against N + M uninterrupted steps; and its evaluation mode: the restored
    agent's argmax actions against the trained agent's."""
    from serl_b200.utils import checkpoints
    N, M, B = 4, 4, 256
    log_a, log_b = [], []
    agent_a = _train(_agent(precision), _iterator(_ring(), B), N + M, log_a)
    it = _iterator(_ring(), B)
    agent = _train(_agent(precision), it, N, log_b)
    checkpoints.save_checkpoint(str(tmp_path), agent.state, step=N, keep=100, overwrite=True)
    # evaluation mode (bc_policy.py:204-225)
    obs = {**{c: np.stack([t["observations"][c] for t in TRS[:5]]) for c in CAMS}, "state": np.stack([t["observations"]["state"] for t in TRS[:5]])}
    evaluator = _agent(precision, seed=7)
    ckpt = checkpoints.restore_checkpoint(str(tmp_path), evaluator.state, step=N)
    evaluator = evaluator.replace(state=ckpt)
    one = {k: v[0] for k, v in obs.items()}
    np.testing.assert_array_equal(evaluator.sample_actions(obs, argmax=True), agent.sample_actions(obs, argmax=True))
    np.testing.assert_array_equal(evaluator.sample_actions(one, argmax=True), agent.sample_actions(one, argmax=True))
    # training resumes in a fresh agent with the same replay iterator
    del agent
    agent_b = _agent(precision, seed=7)
    agent_b = agent_b.replace(state=checkpoints.restore_checkpoint(str(tmp_path), None))
    agent_b = _train(agent_b, it, M, log_b)
    agent_a.check_status()
    agent_b.check_status()
    assert len(log_a) == len(log_b) == N + M
    if precision == "fp32":
        for x, y in zip(log_a, log_b):
            assert all(torch.equal(x[k], y[k]) for k in x), (x, y)
        _assert_same_state(agent_a, agent_b)
    else:                                                            # test_replay_persistence_gpu.py's 16-bit bar
        for x, y in zip(log_a, log_b):
            for k in x:
                assert abs(float(x[k]) - float(y[k])) <= 1e-2 * max(abs(float(x[k])), 1.0), (k, x[k], y[k])
        assert np.array_equal(agent_a.state.rng, agent_b.state.rng) and agent_a.state.step == agent_b.state.step
