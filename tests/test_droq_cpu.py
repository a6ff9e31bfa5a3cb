"""CPU: the critic and policy MLPs' dropout_rate for SACAgent / DrQAgent (dropout Q-functions).  Option resolution and refusals,
the parameter tree, the float64 oracle's gradients and key schedule, the device key derivation's host mirror, and on the dry device
the launches a dropout agent's step makes."""
import json

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions
from test_architecture_options_cpu import GOLDEN, _ring, dry, launch_sequences  # noqa: F401  (dry: fixture)

LAUNCHER = {"hidden_dims": [256, 256], "activations": "tanh", "use_layer_norm": True}


def _arch(**nets):
    from serl_b200.agents.continuous.sac import architecture_settings
    return architecture_settings(None, dict(nets), pixel=True, allow_dropout=True)


# ---- option resolution ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", [0.01, 0.1, 0.5, 0.99])
def test_rates_in_the_open_unit_interval_are_accepted(rate):
    from serl_b200.params import MlpArch
    for name in ("critic_network_kwargs", "policy_network_kwargs"):
        got = _arch(**{name: dict(LAUNCHER, dropout_rate=rate)})
        key = "critic_arch" if name.startswith("critic") else "policy_arch"
        assert got[key] == MlpArch((256, 256), "tanh", True, rate)
    got = _arch(critic_network_kwargs={"hidden_dims": [128], "activations": "relu", "use_layer_norm": False, "dropout_rate": rate})
    assert got["critic_arch"] == MlpArch((128,), "relu", False, rate)


@pytest.mark.parametrize("rate", [None, 0, 0.0])
def test_no_rate_is_the_launcher_architecture(rate):
    from serl_b200.params import LAUNCHER_MLP
    got = _arch(critic_network_kwargs=dict(LAUNCHER, dropout_rate=rate), policy_network_kwargs={"dropout_rate": rate})
    assert got["critic_arch"] is LAUNCHER_MLP and got["policy_arch"] is LAUNCHER_MLP


@pytest.mark.parametrize("rate", [1.0, 1.5, -0.1])
def test_rates_outside_the_unit_interval_raise(rate):
    with pytest.raises(ValueError, match=r"need None, 0 or a rate in \(0, 1\)"):
        _arch(critic_network_kwargs=dict(LAUNCHER, dropout_rate=rate))


def test_a_dropout_dict_must_still_state_activations_and_layer_norm():
    with pytest.raises(ValueError, match="use_layer_norm.*nn.swish, use_layer_norm=False"):
        _arch(critic_network_kwargs={"hidden_dims": [256, 256], "activations": "tanh", "dropout_rate": 0.01})
    with pytest.raises(ValueError, match="activations"):
        _arch(policy_network_kwargs={"dropout_rate": 0.01})


def test_helpers_refuse_dropout_unless_the_caller_trains_it():
    from serl_b200.agents.continuous.sac import _mlp_arch, architecture_settings
    with pytest.raises(NotImplementedError, match="dropout_rate"):
        _mlp_arch("critic_network_kwargs", dict(LAUNCHER, dropout_rate=0.01))
    with pytest.raises(NotImplementedError, match="dropout_rate"):
        architecture_settings(None, {"policy_network_kwargs": dict(LAUNCHER, dropout_rate=0.01)}, pixel=True)


@pytest.mark.parametrize("name", ["critic_network_kwargs", "policy_network_kwargs"])
def test_vice_keeps_refusing_mlp_dropout(name):
    from serl_b200.agents.continuous.vice import VICEAgent
    trs = random_transitions(np.random.default_rng(0), 1, ("front",))
    with pytest.raises(NotImplementedError, match="VICEAgent.*dropout_rate"):
        VICEAgent.create_vice(0, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet-pretrained", image_keys=("front",),
                              device="cpu", **{name: dict(LAUNCHER, dropout_rate=0.01)})


def test_constructors_pass_the_rate_through(dry):
    from serl_b200.agents.continuous.drq import DrQAgent
    from serl_b200.agents.continuous.sac import SACAgent
    from serl_b200.utils.launcher import make_drq_agent, make_sac_agent
    rng = np.random.default_rng(0)
    obs, act = rng.standard_normal(10).astype(np.float32), np.zeros(4, np.float32)
    nk = dict(LAUNCHER, dropout_rate=0.01)
    a = SACAgent.create_states(0, obs, act, critic_network_kwargs=nk, device="cpu")
    assert a._cfg.critic_arch.dropout == 0.01 and a._cfg.policy_arch.dropout == 0 and a._cfg.mlp_dropout
    a = make_sac_agent(0, obs, act, device="cpu", policy_network_kwargs=nk)
    assert a._cfg.policy_arch.dropout == 0.01 and a._cfg.mlp_dropout
    trs = random_transitions(np.random.default_rng(0), 1, ("front",))
    for make in (lambda **k: DrQAgent.create_drq(0, trs[0]["observations"], trs[0]["actions"], image_keys=("front",), **k),
                 lambda **k: make_drq_agent(0, trs[0]["observations"], trs[0]["actions"], image_keys=("front",), **k)):
        a = make(encoder_type="resnet-pretrained", device="cpu", critic_network_kwargs=nk, policy_network_kwargs=nk)
        assert a._cfg.critic_arch.dropout == a._cfg.policy_arch.dropout == 0.01
        assert a._keys.numel() == 24                       # NUM_KEYS_MLP slots for the critic-MLP keys


def test_parameter_trees_are_those_of_the_network_without_dropout(dry):
    from serl_b200.utils.launcher import make_drq_agent, make_sac_agent
    rng = np.random.default_rng(0)
    obs, act = rng.standard_normal(10).astype(np.float32), np.zeros(4, np.float32)
    trs = random_transitions(np.random.default_rng(0), 1, ("front", "wrist"))
    for nk in (LAUNCHER, {"hidden_dims": [512, 128], "activations": "relu", "use_layer_norm": False}):
        for make in (lambda **k: make_sac_agent(3, obs, act, device="cpu", **k),
                     lambda **k: make_drq_agent(3, trs[0]["observations"], trs[0]["actions"], image_keys=("front", "wrist"),
                                                encoder_type="resnet-pretrained", device="cpu", **k)):
            plain = make(critic_network_kwargs=nk, policy_network_kwargs=nk)
            drop = make(critic_network_kwargs=dict(nk, dropout_rate=0.2), policy_network_kwargs=dict(nk, dropout_rate=0.3))
            assert [(l.path, l.shape, l.group) for l in plain._store.spec] == [(l.path, l.shape, l.group) for l in drop._store.spec]
            assert torch.equal(plain._store.params, drop._store.params)            # same seed, same initial values


# ---- the float64 oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act,ln", [("tanh", True), ("relu", False)])
def test_oracle_gradients_match_finite_differences_with_fixed_masks(act, ln):
    from droq_oracle import critic_forward, mlp_masks, policy_forward
    from oracle import jax_prng as P
    from serl_b200.params import MlpArch
    arch = MlpArch((64, 64), act, ln, 0.25)
    E, B, F, A = 3, 5, 6, 2
    g = torch.Generator().manual_seed(0)
    r = lambda *s: (torch.randn(*s, generator=g, dtype=torch.float64) * 0.5)
    params = {"modules_critic/Dense_0/kernel": r(64, 1), "modules_critic/Dense_0/bias": r(1),
              "modules_actor/Dense_0/kernel": r(64, A), "modules_actor/Dense_0/bias": r(A),
              "modules_actor/Dense_1/kernel": r(64, A), "modules_actor/Dense_1/bias": r(A)}
    for net, rows, fin in (("modules_critic/network", E, F + A), ("modules_actor/network", None, F)):
        for i, (k, H) in enumerate(zip((fin, 64), arch.hidden)):
            params[f"{net}/Dense_{i}/kernel"] = r(rows, k, H) if rows else r(k, H)
            params[f"{net}/Dense_{i}/bias"] = r(rows, H) if rows else r(H)
            if ln:
                params[f"{net}/LayerNorm_{i}/scale"] = 1 + r(rows, H) if rows else 1 + r(H)
                params[f"{net}/LayerNorm_{i}/bias"] = r(rows, H) if rows else r(H)
    masks = mlp_masks(P.prng_key(5), 2, B, arch)
    assert all(0 < np.mean(m) < 1 for m in masks)
    enc, a = r(B, F), r(B, A)
    names = [k for k in params if "critic" in k]
    def q_of(*leaves):
        p = dict(params, **dict(zip(names, leaves)))
        return critic_forward(p, enc, a, arch, pixel_agent=True, masks=masks)
    assert torch.autograd.gradcheck(q_of, tuple(params[k].clone().requires_grad_(True) for k in names), eps=1e-6, atol=1e-5)
    q_a = lambda x: critic_forward(params, enc, x, arch, pixel_agent=True, masks=masks)
    assert torch.autograd.gradcheck(q_a, (a.clone().requires_grad_(True),), eps=1e-6, atol=1e-5)
    pnames = [k for k in params if k.startswith("modules_actor")]
    def pol(*leaves):
        p = dict(params, **dict(zip(pnames, leaves)))
        return policy_forward(p, enc, arch, "exp", 1e-5, 5.0, masks=masks)
    assert torch.autograd.gradcheck(pol, tuple(params[k].clone().requires_grad_(True) for k in pnames), eps=1e-6, atol=1e-5)


def test_oracle_key_schedule_online_and_target_masks():
    from droq_oracle import derive_mlp_masks, update_keys
    from oracle import jax_prng as P
    from serl_b200.params import MlpArch
    arch = MlpArch((256, 256), "tanh", True, 0.1)
    rng = P.prng_key(11)
    nets = ("critic", "actor", "temperature")
    for sub in (False, True):
        calls = derive_mlp_masks(rng, nets, 8, 2, arch, arch, sub)
        assert [n for n, _ in calls] == ["policy", "critic", "critic", "policy", "critic", "policy"]
        tgt, online = calls[1][1], calls[2][1]
        same = all(np.array_equal(x, y) for x, y in zip(tgt, online))
        assert same == (not sub)
    keys = [k for _, k in update_keys(rng, nets, True)]
    assert len({tuple(k) for k in keys}) == len(keys)                   # every other call has a key of its own


@pytest.mark.parametrize("do_aug", [0, 1])
def test_device_key_derivation_matches_the_oracle(do_aug):
    """serl_mlp_dropout_keys' host mirror (the device kernel's code) against the oracle's key chain."""
    from droq_oracle import update_keys
    from oracle import jax_prng as P
    from serl_b200 import _lib as L
    L.load()
    for seed in (0, 7, 123456):
        rng = P.prng_key(seed)
        keys = np.zeros(2 * L.NUM_KEYS_MLP, np.uint32)
        L.call("serl_host_mlp_dropout_keys", rng.ctypes.data, keys.ctypes.data, do_aug)
        r = P.split(rng, 3)[0] if do_aug else rng
        sub, nosub = update_keys(r, ("critic", "actor"), True), update_keys(r, ("critic",), False)
        np.testing.assert_array_equal(keys[2 * L.KEY_MLP_CRITIC_TARGET:][:2], nosub[1][1])
        np.testing.assert_array_equal(keys[2 * L.KEY_MLP_CRITIC_SUBSAMPLED:][:2], sub[2][1])
        np.testing.assert_array_equal(keys[2 * L.KEY_MLP_ACTOR_CRITIC:][:2], sub[4][1])
        host, state = np.zeros(2 * L.NUM_KEYS, np.uint32), rng.copy()    # the policy passes' keys are rng_schedule's
        L.call("serl_host_rng_schedule", state.ctypes.data, host.ctypes.data, do_aug, 1)
        np.testing.assert_array_equal(host[2 * L.KEY_CRITIC_NEXT:][:2], sub[0][1])
        np.testing.assert_array_equal(host[2 * L.KEY_ACTOR_DROPOUT:][:2], sub[3][1])


# ---- launches on the dry device --------------------------------------------------------------------------------------------
DROQ = dict(LAUNCHER, dropout_rate=0.01)


@pytest.mark.parametrize("scenario", ["drq_fp32", "drq_fp16_fused", "drq_fp16_perop", "sac_state"])
def test_rate_zero_reproduces_the_launcher_launches(dry, scenario):
    want = json.load(open(GOLDEN))[scenario]
    zero = dict(LAUNCHER, dropout_rate=0.0)
    assert launch_sequences(scenario, dry, critic_network_kwargs=zero, policy_network_kwargs=dict(zero, dropout_rate=None)) == want


@pytest.mark.parametrize("scenario", ["drq_fp32", "drq_fp16_perop", "sac_state"])
def test_dropout_agent_launches(dry, scenario):
    """A dropout agent on the per-op chain: the critic-MLP keys, one mask fill per (pass, layer), the masked LayerNorm / tanh
    forward and backward; inference passes draw none."""
    got = launch_sequences(scenario, dry, critic_network_kwargs=DROQ, policy_network_kwargs=DROQ)
    ncam = 2 if scenario.startswith("drq") else 0
    seq = got["update"]                                             # critic, actor and temperature losses
    assert "serl_tgemm_tf32" not in seq and seq.count("serl_mlp_dropout_keys") == 1
    assert seq.index("serl_mlp_dropout_keys") < seq.index("serl_rng_schedule")
    # three policy passes x (cams + 2 layers) + (online, target, actor-loss critic) x 2 layers
    assert seq.count("serl_dropout_mask_fill") == 3 * (ncam + 2) + 3 * 2
    # the critic's E*B rows read their (B, H) masks through the row period; the policy's B rows through the plain entry
    assert seq.count("serl_ln_act_dropout_rows_fwd") == 3 * 2 and seq.count("serl_ln_act_dropout_rows_bwd") == 2 * 2
    assert seq.count("serl_ln_act_dropout_fwd") == 3 * 2 and seq.count("serl_ln_act_dropout_bwd") == 2
    assert "serl_layernorm_tanh_fwd" in seq or not ncam                 # the encoder heads keep their unmasked LayerNorm
    for step in ("update_high_utd",) + (("update_critics",) if ncam else ()):
        s2 = got[step]
        assert "serl_mlp_dropout_keys" in s2 and "serl_tgemm_tf32" not in s2
    if ncam:
        assert got["update_critics"].count("serl_ln_act_dropout_rows_fwd") == 2 * 2
        assert got["update_critics"].count("serl_ln_act_dropout_rows_bwd") == 2
    for step in ("sample_actions", "sample_argmax"):
        assert not any("dropout" in c or "mlp" in c for c in got[step])


def _plain(seq):
    """A dropout agent's fused launch list with its Dropout launches taken out: masked launches under their plain names, no key
    derivation or MLP mask fill, and the policy backward's masked LayerNorm / tanh + parameter gradient as the launcher's one call."""
    out, i = [], 0
    while i < len(seq):
        c = seq[i]
        if c == "serl_mlp_dropout_keys":
            pass
        elif c == "serl_ln_act_dropout_bwd" and seq[i + 1] == "serl_layernorm_param_grad":
            out.append("serl_layernorm_tanh_bwd")
            i += 1
        else:
            out.append({"serl_tgemm_tf32_masked": "serl_tgemm_tf32",
                        "serl_layernorm_tanh_bwd_multi_masked": "serl_layernorm_tanh_bwd_multi"}.get(c, c))
        i += 1
    return out


def test_dropout_agent_on_fp16_takes_the_fused_heads(dry):
    """At the launcher widths / LayerNorm / tanh a dropout agent's 16-bit critic and actor steps run on the fused tgemm heads: every
    MLP layer launch is the masked variant of the launcher's, plus the key derivation and one mask fill per (pass, layer)."""
    want = json.load(open(GOLDEN))["drq_fp16_fused"]
    got = launch_sequences("drq_fp16_fused", dry, critic_network_kwargs=DROQ, policy_network_kwargs=DROQ)
    for step in ("update_critics", "update", "update_high_utd"):
        seq = got[step]
        assert "serl_ln_act_dropout_rows_fwd" not in seq and "serl_tgemm_tf32_masked" in seq
        fills = [c for c in seq if c == "serl_dropout_mask_fill"]
        nomlp = [c for c in want[step] if c == "serl_dropout_mask_fill"]
        mlp_fills = len(fills) - len(nomlp)
        assert mlp_fills == (3 * 2 if step == "update_critics" else 3 * 2 + 3 * 2)    # layers x (policy passes + critic passes)
        nofill = lambda q: [c for c in q if c != "serl_dropout_mask_fill"]
        assert nofill(_plain(seq)) == nofill(want[step]), step
    seq = got["update"]
    assert seq.count("serl_tgemm_tf32_masked") == 8 and seq.count("serl_layernorm_tanh_bwd_multi_masked") == 4
    for step in ("sample_actions", "sample_argmax"):
        assert got[step] == want[step]


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_data_parallel_step_keeps_one_collective(dry, monkeypatch, precision):
    """Under data parallelism a dropout agent's step all-reduces its gradients and infos in one collective, as the launcher
    agent's does: the masks are drawn from each rank's key chain on the device and add nothing to exchange."""
    from serl_b200.agents.continuous import sac
    from serl_b200.utils.launcher import make_drq_agent
    calls = []

    class FakeDist:
        class ReduceOp:
            SUM = "sum"

        def get_world_size(self):
            return 2

        def all_reduce(self, t, op=None):
            calls.append((t.numel(), op))

    monkeypatch.setattr(sac, "_dist", lambda: FakeDist())
    cams = ("front", "wrist")
    rb, trs = _ring(cams)
    counts = {}
    for name, nets in (("launcher", {}), ("droq", dict(critic_network_kwargs=DROQ, policy_network_kwargs=DROQ))):
        agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained",
                               device="cpu", precision=precision, **nets)
        agent.data_parallel = True
        per = []
        for fn in (lambda: agent.update(rb.sample(4, pack_obs_and_next_obs=True)),
                   lambda: agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))):
            del calls[:]
            fn()
            per.append(list(calls))
        counts[name] = per
    assert [len(c) for c in counts["droq"]] == [1, 1]
    assert counts["droq"] == counts["launcher"]
