"""CPU: the reference's network architecture options (MLP hidden_dims / activations / use_layer_norm, the policy's "exp",
"softplus" and "uniform" std parameterisations).  How the agents resolve the kwargs; the parameter tree against a literal list
written from the reference's module definitions; finite-difference gradients of the restated networks; and, on the dry
device, which launches a step makes."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "launcher_arch_launches.json")


# ---- dry device ----------------------------------------------------------------------------------------------------------
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


def _ring(cams, cap=64):
    from serl_b200.utils.launcher import make_replay_buffer
    rb = make_replay_buffer(fake_env(cams, 128), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams), device="cpu", seed=5)
    trs = random_transitions(np.random.default_rng(0), 40, cams, 128)
    for tr in trs:
        rb.insert(tr)
    return rb, trs


def launch_sequences(scenario, calls, **arch):
    """Launch names of update_critics, update, update_high_utd and sample_actions on the dry device.  `arch`: network kwargs."""
    from serl_b200.utils.launcher import make_drq_agent, make_sac_agent
    out = {}
    env = {"drq_fp16_fused": "force", "drq_fp16_perop": "0"}.get(scenario)
    old = os.environ.get("SERL_FUSED_HEADS")
    if env is not None:
        os.environ["SERL_FUSED_HEADS"] = env
    try:
        if scenario.startswith("drq"):
            cams = ("front", "wrist")
            rb, trs = _ring(cams)
            agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained",
                                   device="cpu", precision="fp32" if scenario == "drq_fp32" else "fp16", **arch)
            for name, fn in (("update_critics", lambda: agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))),
                             ("update", lambda: agent.update(rb.sample(4, pack_obs_and_next_obs=True))),
                             ("update_high_utd", lambda: agent.update_high_utd(rb.sample(4, pack_obs_and_next_obs=True), utd_ratio=1)),
                             ("sample_actions", lambda: agent.sample_actions({k: v for k, v in trs[0]["observations"].items()},
                                                                            seed=np.array([0, 3], np.uint32))),
                             ("sample_argmax", lambda: agent.sample_actions({k: v for k, v in trs[0]["observations"].items()}, argmax=True))):
                del calls[:]
                fn()
                out[name] = [c for c in calls if c not in ("serl_replay_scatter", "serl_replay_set_valid", "serl_replay_commit")]
        else:
            rng = np.random.default_rng(0)
            agent = make_sac_agent(0, rng.standard_normal(10).astype(np.float32), np.zeros(4, np.float32), device="cpu", **arch)
            B = 32
            batch = dict(observations=rng.standard_normal((B, 10)).astype(np.float32), next_observations=rng.standard_normal((B, 10)).astype(np.float32),
                         actions=np.zeros((B, 4), np.float32), rewards=np.zeros(B, np.float32), masks=np.ones(B, np.float32), dones=np.zeros(B, bool))
            for name, fn in (("update_high_utd", lambda: agent.update_high_utd(batch, utd_ratio=4)),
                             ("update", lambda: agent.update(batch)),
                             ("sample_actions", lambda: agent.sample_actions(batch["observations"][:3], seed=np.array([0, 7], np.uint32))),
                             ("sample_argmax", lambda: agent.sample_actions(batch["observations"][0], argmax=True))):
                del calls[:]
                fn()
                out[name] = list(calls)
    finally:
        if old is None:
            os.environ.pop("SERL_FUSED_HEADS", None)
        else:
            os.environ["SERL_FUSED_HEADS"] = old
    return out


# ---- kwargs resolution ----------------------------------------------------------------------------------------------------
def _arch(policy_kwargs=None, **nets):
    from serl_b200.agents.continuous.sac import architecture_settings
    return architecture_settings(policy_kwargs, dict(nets), pixel=True)


def test_omitted_or_launcher_valued_dicts_build_the_launcher_architecture():
    from serl_b200.params import LAUNCHER_MLP
    want = dict(critic_arch=LAUNCHER_MLP, policy_arch=LAUNCHER_MLP, std_parameterization="exp")
    assert _arch() == want
    assert _arch({"tanh_squash_distribution": True, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5}) == want
    assert _arch(critic_network_kwargs={"hidden_dims": [256, 256]}, policy_network_kwargs={}) == want
    assert _arch(critic_network_kwargs={"activations": torch.tanh, "use_layer_norm": True, "activate_final": False}) == want
    assert _arch(policy_network_kwargs={"hidden_dims": (256, 256), "activations": "tanh", "dropout_rate": None}) == want


class _Fn:                                    # a flax / jax activation function: matched by __name__
    def __init__(self, name):
        self.__name__ = name


@pytest.mark.parametrize("given,act", [("relu", "relu"), ("swish", "swish"), ("silu", "swish"), (_Fn("silu"), "swish"),
                                       ("leaky_relu", "leaky_relu"), (_Fn("gelu"), "gelu"), ("tanh", "tanh")])
@pytest.mark.parametrize("hidden,ln", [([64], False), ([512, 512, 512], True), ([1024, 128], False), ([256, 256], False)])
def test_accepted_architectures(given, act, hidden, ln):
    from serl_b200.params import MlpArch
    nk = {"hidden_dims": hidden, "activations": given, "use_layer_norm": ln, "activate_final": True}
    got = _arch(critic_network_kwargs=nk)
    assert got["critic_arch"] == MlpArch(tuple(hidden), act, ln)
    for std in ("exp", "softplus", "uniform"):
        got = _arch({"std_parameterization": std, "std_min": 1e-4}, policy_network_kwargs=nk)
        assert got["policy_arch"] == MlpArch(tuple(hidden), act, ln) and got["std_parameterization"] == std


@pytest.mark.parametrize("nk,missing", [({"hidden_dims": [512, 512]}, "activations"), ({"activations": "relu"}, "use_layer_norm"),
                                        ({"hidden_dims": [128], "use_layer_norm": True}, "activations"),
                                        ({"hidden_dims": [128], "activations": "relu"}, "use_layer_norm"),
                                        ({"use_layer_norm": False}, "activations")])
def test_non_launcher_dict_must_state_activations_and_layer_norm(nk, missing):
    for name in ("critic_network_kwargs", "policy_network_kwargs"):
        with pytest.raises(ValueError, match=f"{missing}.*nn.swish, use_layer_norm=False"):
            _arch(**{name: nk})


@pytest.mark.parametrize("policy_kwargs,nets,err", [
    ({"std_parameterization": "fixed", "fixed_std": [0.1] * 4}, {}, NotImplementedError),
    ({"fixed_std": [0.1] * 4}, {}, NotImplementedError),
    ({"tanh_squash_distribution": False}, {}, NotImplementedError),
    ({"std_parameterization": "cube"}, {}, NotImplementedError),
    (None, {"critic_network_kwargs": {"hidden_dims": [256, 256], "activations": "tanh", "use_layer_norm": True, "dropout_rate": 0.1}}, NotImplementedError),
    (None, {"policy_network_kwargs": {"hidden_dims": [256], "activations": "elu", "use_layer_norm": True}}, NotImplementedError),
    (None, {"policy_network_kwargs": {"hidden_dims": [256], "activations": _Fn("sigmoid"), "use_layer_norm": True}}, NotImplementedError),
    (None, {"shared_encoder": False}, NotImplementedError),
    (None, {"critic_network_kwargs": {"hidden_dims": [], "activations": "relu", "use_layer_norm": True}}, ValueError),
    (None, {"critic_network_kwargs": {"hidden_dims": [96], "activations": "relu", "use_layer_norm": True}}, ValueError),
    (None, {"critic_network_kwargs": {"hidden_dims": [2048], "activations": "relu", "use_layer_norm": True}}, ValueError),
    (None, {"critic_network_kwargs": {"hidden_dims": [32], "activations": "relu", "use_layer_norm": False}}, ValueError),
    (None, {"critic_network_kwargs": {"widths": [256]}}, TypeError),
])
def test_refused_architectures(policy_kwargs, nets, err):
    with pytest.raises(err):
        _arch(policy_kwargs, **nets)


def test_constructors_pass_the_architecture_through(dry):
    from serl_b200.agents.continuous.sac import SACAgent
    from serl_b200.params import MlpArch
    from serl_b200.utils.launcher import make_sac_agent
    rng = np.random.default_rng(0)
    obs, act = rng.standard_normal(10).astype(np.float32), np.zeros(4, np.float32)
    # the reference constructor's own defaults, stated explicitly
    nk = {"hidden_dims": [256, 256], "activations": "swish", "use_layer_norm": False}
    a = SACAgent.create_states(0, obs, act, critic_network_kwargs=nk, policy_network_kwargs=nk,
                               policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "uniform"}, device="cpu")
    assert a._cfg.critic_arch == a._cfg.policy_arch == MlpArch((256, 256), "swish", False) and a._cfg.std_parameterization == "uniform"
    assert a.state.params["modules_actor"]["log_stds"].shape == (4,) and "Dense_1" not in a.state.params["modules_actor"]
    b = make_sac_agent(0, obs, act, device="cpu", critic_network_kwargs={"hidden_dims": [128], "activations": "gelu", "use_layer_norm": True})
    assert b._cfg.critic_arch == MlpArch((128,), "gelu", True) and b._cfg.std_parameterization == "exp"
    assert b.state.params["modules_critic"]["Dense_0"]["kernel"].shape == (10, 128, 1)


# ---- parameter tree: literal lists written from the reference's module definitions -------------------------------------------
# state SAC, S = 10, A = 4, ensemble 2 (vmapped critic incl. head, sac.py:523-524); flat order = this project's layout
S, A, E = 10, 4, 2
REF_DEFAULTS = [        # hidden_dims [256, 256], swish, no LayerNorm, "uniform" (sac.py:486-504 defaults)
    ("modules_critic/network/Dense_0/kernel", (2, 14, 256)), ("modules_critic/network/Dense_0/bias", (2, 256)),
    ("modules_critic/network/Dense_1/kernel", (2, 256, 256)), ("modules_critic/network/Dense_1/bias", (2, 256)),
    ("modules_critic/Dense_0/kernel", (2, 256, 1)), ("modules_critic/Dense_0/bias", (2, 1)),
    ("modules_actor/network/Dense_0/kernel", (10, 256)), ("modules_actor/network/Dense_0/bias", (256,)),
    ("modules_actor/network/Dense_1/kernel", (256, 256)), ("modules_actor/network/Dense_1/bias", (256,)),
    ("modules_actor/Dense_0/kernel", (256, 4)), ("modules_actor/Dense_0/bias", (4,)),
    ("modules_actor/log_stds", (4,)),
    ("modules_temperature/lagrange", ()),
]
WIDE_RELU_LN_SOFTPLUS = [   # [512, 512, 512], relu, LayerNorm, "softplus"
    ("modules_critic/network/Dense_0/kernel", (2, 14, 512)), ("modules_critic/network/Dense_0/bias", (2, 512)),
    ("modules_critic/network/LayerNorm_0/scale", (2, 512)), ("modules_critic/network/LayerNorm_0/bias", (2, 512)),
    ("modules_critic/network/Dense_1/kernel", (2, 512, 512)), ("modules_critic/network/Dense_1/bias", (2, 512)),
    ("modules_critic/network/LayerNorm_1/scale", (2, 512)), ("modules_critic/network/LayerNorm_1/bias", (2, 512)),
    ("modules_critic/network/Dense_2/kernel", (2, 512, 512)), ("modules_critic/network/Dense_2/bias", (2, 512)),
    ("modules_critic/network/LayerNorm_2/scale", (2, 512)), ("modules_critic/network/LayerNorm_2/bias", (2, 512)),
    ("modules_critic/Dense_0/kernel", (2, 512, 1)), ("modules_critic/Dense_0/bias", (2, 1)),
    ("modules_actor/network/Dense_0/kernel", (10, 512)), ("modules_actor/network/Dense_0/bias", (512,)),
    ("modules_actor/network/LayerNorm_0/scale", (512,)), ("modules_actor/network/LayerNorm_0/bias", (512,)),
    ("modules_actor/network/Dense_1/kernel", (512, 512)), ("modules_actor/network/Dense_1/bias", (512,)),
    ("modules_actor/network/LayerNorm_1/scale", (512,)), ("modules_actor/network/LayerNorm_1/bias", (512,)),
    ("modules_actor/network/Dense_2/kernel", (512, 512)), ("modules_actor/network/Dense_2/bias", (512,)),
    ("modules_actor/network/LayerNorm_2/scale", (512,)), ("modules_actor/network/LayerNorm_2/bias", (512,)),
    ("modules_actor/Dense_0/kernel", (512, 4)), ("modules_actor/Dense_0/bias", (4,)),
    ("modules_actor/Dense_1/kernel", (512, 4)), ("modules_actor/Dense_1/bias", (4,)),
    ("modules_temperature/lagrange", ()),
]
NARROW_LEAKY_EXP = [        # [128], leaky_relu, no LayerNorm, "exp"
    ("modules_critic/network/Dense_0/kernel", (2, 14, 128)), ("modules_critic/network/Dense_0/bias", (2, 128)),
    ("modules_critic/Dense_0/kernel", (2, 128, 1)), ("modules_critic/Dense_0/bias", (2, 1)),
    ("modules_actor/network/Dense_0/kernel", (10, 128)), ("modules_actor/network/Dense_0/bias", (128,)),
    ("modules_actor/Dense_0/kernel", (128, 4)), ("modules_actor/Dense_0/bias", (4,)),
    ("modules_actor/Dense_1/kernel", (128, 4)), ("modules_actor/Dense_1/bias", (4,)),
    ("modules_temperature/lagrange", ()),
]


def _tree_case(case):
    from serl_b200.params import MlpArch
    return {"reference_defaults": (MlpArch((256, 256), "swish", False), "uniform", REF_DEFAULTS),
            "512x3_relu_ln_softplus": (MlpArch((512, 512, 512), "relu", True), "softplus", WIDE_RELU_LN_SOFTPLUS),
            "128_leaky_exp": (MlpArch((128,), "leaky_relu", False), "exp", NARROW_LEAKY_EXP)}[case]


@pytest.mark.parametrize("case", ["reference_defaults", "512x3_relu_ln_softplus", "128_leaky_exp"])
def test_parameter_tree_matches_the_reference_modules(case):
    from serl_b200.params import ParamStore, init_trainable, trainable_spec
    arch, std, literal = _tree_case(case)
    spec = trainable_spec((), S, A, E, False, arch, arch, std)
    assert [(l.path, l.shape) for l in spec] == literal
    assert [l.group for l in spec] == [0 if p.startswith("modules_critic") else 2 if "temperature" in p else 1 for p, _ in literal]
    vals = init_trainable(np.random.default_rng(0), spec, 1.0)
    for p, v in vals.items():                                       # xavier Dense, zero bias, ones / zeros LayerNorm, zero log_stds
        if p.endswith(("bias", "log_stds")):
            assert not v.any(), p
        elif p.endswith("scale"):
            assert (v == 1).all(), p
        elif p.endswith("kernel"):
            fi, fo = v.shape[-2], v.shape[-1]
            assert np.abs(v).max() <= np.sqrt(6.0 / (fi + fo)) and v.std() > 0, p
    st = ParamStore(spec, "cpu")                                    # log_stds sits in the actor tx's group, inside [seg_end[0]+gap, seg_end[1])
    if std == "uniform":
        off = st.leaf["modules_actor/log_stds"].offset
        assert st.info_off + 16 <= off < st.seg_end[1]


def test_pixel_agent_tree_has_shared_value_head_on_the_last_width():
    from serl_b200.params import MlpArch, trainable_spec
    arch = MlpArch((512, 128, 64), "gelu", True)
    spec = {l.path: l.shape for l in trainable_spec(("front", "wrist"), 7, 4, 10, True, arch, MlpArch((64,), "relu", False), "uniform")}
    F = 256 * 2 + 64
    assert spec["modules_critic/network/Dense_0/kernel"] == (10, F + 4, 512) and spec["modules_critic/network/Dense_2/kernel"] == (10, 128, 64)
    assert spec["modules_critic/Dense_0/kernel"] == (64, 1) and spec["modules_critic/Dense_0/bias"] == (1,)
    assert spec["modules_actor/network/Dense_0/kernel"] == (F, 64) and "modules_actor/network/LayerNorm_0/scale" not in spec
    assert spec["modules_actor/log_stds"] == (4,) and "modules_actor/Dense_1/kernel" not in spec


# ---- oracle: activations against torch's own functions, finite-difference gradients ----------------------------------------
def test_oracle_activations_match_torch():
    import torch.nn.functional as Fn
    from arch_oracle import ACTIVATIONS
    x = torch.linspace(-6, 6, 2001, dtype=torch.float64)
    ref = {"tanh": torch.tanh(x), "relu": Fn.relu(x), "swish": Fn.silu(x), "leaky_relu": Fn.leaky_relu(x, 0.01),
           "gelu": Fn.gelu(x, approximate="tanh")}
    for k, f in ACTIVATIONS.items():
        torch.testing.assert_close(f(x), ref[k], rtol=1e-14, atol=1e-15)


@pytest.mark.parametrize("act", ["tanh", "relu", "swish", "leaky_relu", "gelu"])
@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("std", ["exp", "softplus", "uniform"])
def test_oracle_gradients_match_finite_differences(act, ln, std):
    """The actor loss of a state agent (critic ensemble + policy + tanh-Gaussian) through the restated networks: autograd vs
    central differences in float64, w.r.t. every parameter leaf of the critic and the policy."""
    from arch_oracle import critic_forward, policy_forward
    from oracle.drq import tanh_normal_sample_logp
    from serl_b200.params import MlpArch, init_trainable, trainable_spec
    arch = MlpArch((8, 6), act, ln)
    Sd, Ad, Ed, B = 5, 3, 2, 7
    rng = np.random.default_rng(1)
    spec = trainable_spec((), Sd, Ad, Ed, False, arch, arch, std)
    params = {k: torch.as_tensor(v, dtype=torch.float64) + 0.1 * torch.as_tensor(rng.standard_normal(np.shape(v)))
              for k, v in init_trainable(rng, spec, 1.0).items()}
    obs = torch.as_tensor(rng.standard_normal((B, Sd)))
    eps = torch.as_tensor(rng.standard_normal((B, Ad)))
    names = [k for k in params if "temperature" not in k]

    def loss(*leaves):
        p = dict(params, **dict(zip(names, leaves)))
        mu, sd = policy_forward(p, obs, arch, std, 1e-3, 5.0)
        a, logp = tanh_normal_sample_logp(mu, sd, eps)
        return -(critic_forward(p, obs, a, arch, pixel_agent=False).mean(0) - 0.1 * logp).mean()

    leaves = [params[k].clone().requires_grad_(True) for k in names]
    assert torch.autograd.gradcheck(loss, leaves, eps=1e-6, atol=1e-6, rtol=1e-4)


# ---- dry device: launches ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scenario", ["drq_fp32", "drq_fp16_fused", "drq_fp16_perop", "sac_state"])
def test_launcher_architecture_launch_sequence_is_unchanged(dry, scenario):
    """Recorded from the commit before architecture options existed: omitted network dicts and launcher-valued ones launch the
    same kernels in the same order."""
    want = json.load(open(GOLDEN))[scenario]
    assert launch_sequences(scenario, dry) == want
    same = {"hidden_dims": [256, 256], "activations": "tanh", "use_layer_norm": True}
    assert launch_sequences(scenario, dry, critic_network_kwargs=same, policy_network_kwargs={"hidden_dims": [256, 256]}) == want


WIDE = {"hidden_dims": [512, 512, 512], "activations": "relu", "use_layer_norm": True}
REF_NET = {"hidden_dims": [256, 256], "activations": "swish", "use_layer_norm": False}


@pytest.mark.parametrize("nets", [dict(critic_network_kwargs=WIDE), dict(policy_network_kwargs=REF_NET),
                                  dict(critic_network_kwargs=REF_NET, policy_network_kwargs=REF_NET)], ids=["critic_wide", "policy_ref", "both_ref"])
def test_non_launcher_architecture_on_fp16_takes_the_per_op_chain(dry, nets):
    seqs = launch_sequences("drq_fp16_fused", dry, **nets)          # SERL_FUSED_HEADS=force: fused if the architecture allowed it
    for name, seq in seqs.items():
        assert "serl_tgemm_tf32" not in seq and "serl_enc_finish" not in seq, name
        assert "serl_gemm_f32" not in seq, name                     # 16-bit builds: 3xTF32 GEMMs
    assert "serl_gemm_tf32x3" in seqs["update_critics"]
    assert "serl_layernorm_act_fwd" in seqs["update_critics"] and "serl_layernorm_act_bwd" in seqs["update_high_utd"]
    assert seqs["update_high_utd"].count("serl_actor_loss") == 1


def test_std_heads_launch_their_kernels(dry):
    from serl_b200.agents.continuous.drq import DrQAgent
    cams = ("front",)
    rb, trs = _ring(cams)
    for std, head in (("softplus", "serl_actor_loss_std"), ("uniform", "serl_actor_loss_std"), ("exp", "serl_actor_loss")):
        agent = DrQAgent.create_drq(0, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet-pretrained", image_keys=cams,
                                    policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": std}, device="cpu",
                                    critic_network_kwargs=REF_NET, policy_network_kwargs=REF_NET)
        del dry[:]
        agent.update_high_utd(rb.sample(4, pack_obs_and_next_obs=True), utd_ratio=1)
        assert dry.count(head) == 1
        gauss = "serl_tanh_gaussian_fwd" + ("" if std == "exp" else "_std")
        assert dry.count(gauss) == 3                                # critic-next, actor, temperature passes
        del dry[:]
        agent.sample_actions({k: v for k, v in trs[0]["observations"].items()}, argmax=True)
        assert dry.count(gauss) == 1


# ---- data parallel (gloo, world 2): one collective per step, and it covers log_stds --------------------------------------------
def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from serl_b200 import _lib as L
    real = L.call
    events = []

    def fake(name, *a):
        if name.startswith("serl_host_"):
            return real(name, *a)
        events.append(name)
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    L.call, L.require_cuda, L.stream_ptr, L.new_event, L.pin = fake, (lambda d: None), (lambda: 0), (lambda: Ev()), (lambda t: t)
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.utils.launcher import make_replay_buffer
    cams = ("front",)
    rb = make_replay_buffer(fake_env(cams, 128), capacity=40, type="memory_efficient_replay_buffer", image_keys=list(cams), device="cpu",
                            seed=100 + rank)
    trs = random_transitions(np.random.default_rng(rank), 30, cams, 128)
    for tr in trs:
        rb.insert(tr)
    agent = DrQAgent.create_drq(7, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu",
                                policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "uniform"},
                                critic_network_kwargs=WIDE, policy_network_kwargs=REF_NET, actor_optimizer_kwargs={"clip_grad_norm": 1.0})
    agent.data_parallel = True
    agent.use_cuda_graphs = False
    spans = []
    real_ar = dist.all_reduce

    def ar(t, *a, **k):
        lo = (t.data_ptr() - agent._store.grad.data_ptr()) // 4
        spans.append((lo, lo + t.numel()))
        return real_ar(t, *a, **k)

    dist.all_reduce = ar
    seqs = []
    for call in (lambda b: agent.update_critics(b), lambda b: agent.update(b, pmap_axis="devices"),
                 lambda b: agent.update_high_utd(b, utd_ratio=1)):
        del spans[:]
        call(rb.sample(4, pack_obs_and_next_obs=True))
        seqs.append(list(spans))
    st = agent._store
    torch.save(dict(seqs=seqs, n=st.n, cut=st.info_off + 4, log_stds=st.leaf["modules_actor/log_stds"].offset,
                    norms=[e for e in events if e == "serl_grad_global_norms"]), out.format(rank))
    dist.destroy_process_group()


def test_data_parallel_keeps_one_collective_and_covers_log_stds(tmp_path):
    import torch.multiprocessing as mp
    world, port = 2, 35000 + os.getpid() % 2000
    out = str(tmp_path / "rank{}.pt")
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    r0 = torch.load(out.format(0))
    n, cut, ls = r0["n"], r0["cut"], r0["log_stds"]
    assert r0["seqs"] == [[(0, cut)], [(0, n)], [(0, cut), (cut, n)]]           # one collective per step
    assert cut <= ls < n                                                         # ... whose actor range holds log_stds
    assert torch.load(out.format(1))["seqs"] == r0["seqs"]
