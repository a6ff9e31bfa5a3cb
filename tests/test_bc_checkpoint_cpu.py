"""CPU: BCAgent's checkpoint state (kernel launches replaced by a recorder).  `agent.state.state_dict()` holds the
JaxRLTrainState fields of one optax.adam in the Flax tree layout, a checkpoint of it pickles NumPy arrays and plain Python values
only, and `agent.replace(state=...)` writes a restored state into the agent (reference examples/bc_policy.py:165-178, 204-209)."""
import pickle

import numpy as np
import pytest
import torch

from helpers import random_transitions

CAMS = ("front", "wrist")
FIELDS = {"step", "params", "target_params", "opt_states", "rng"}


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
    return calls


def _flat(tree, prefix=""):
    out = {}
    for k, v in tree.items():
        p = f"{prefix}/{k}" if prefix else k
        out.update(_flat(v, p)) if isinstance(v, dict) else out.__setitem__(p, v)
    return out


def _launcher_agent(seed):
    from serl_b200.utils.launcher import make_bc_agent
    trs = random_transitions(np.random.default_rng(0), 1, CAMS, 128)
    return make_bc_agent(seed, trs[0]["observations"], trs[0]["actions"], image_keys=CAMS, encoder_type="resnet-pretrained", device="cpu")


def _options_agent(seed):
    from serl_b200.agents.continuous.bc import BCAgent
    trs = random_transitions(np.random.default_rng(0), 1, CAMS, 128)
    return BCAgent.create(seed, trs[0]["observations"], trs[0]["actions"], encoder_type="resnet-pretrained", image_keys=CAMS,
                          use_proprio=False, device="cpu",
                          network_kwargs={"activations": "gelu", "use_layer_norm": True, "hidden_dims": [128, 64], "dropout_rate": 0.1},
                          policy_kwargs={"std_parameterization": "uniform"})


def _perturb(agent, seed):
    """Moves every buffer of the state off its initial value, as training would."""
    g = torch.Generator().manual_seed(seed)
    st = agent._store
    for buf in (st.params, st.target, st.m, st.v):
        buf.add_(torch.rand(buf.shape, generator=g))
    st.counts.fill_(17)
    agent.state.replace(rng=np.array([seed, 3 * seed + 1], np.uint32), step=17)


def _store_equal(a, b):
    sa, sb = a._store, b._store
    for name in ("params", "target", "m", "v", "counts"):
        assert torch.equal(getattr(sa, name), getattr(sb, name)), name
    for cam in CAMS:
        for k, v in a._frozen_trunk.leaves[cam].items():
            assert torch.equal(v, b._frozen_trunk.leaves[cam][k]), (cam, k)
    assert torch.equal(a._rng, b._rng) and a.state.step == b.state.step


@pytest.mark.parametrize("make", [_launcher_agent, _options_agent])
def test_state_dict_has_the_train_state_fields(dry, make):
    from serl_b200.agents.continuous.bc import bc_spec
    from serl_b200.params import TRUNK_PATH
    agent = make(1)
    cfg = agent._cfg
    spec, _ = bc_spec(cfg.cams, cfg.state_in, cfg.action_dim, agent.arch, agent.std_parameterization, cfg.use_proprio)
    d = agent.state.state_dict()
    assert set(d) == FIELDS
    assert d["step"] == 0 and isinstance(d["step"], int)
    assert d["rng"].dtype == np.uint32 and d["rng"].shape == (2,)
    trunk = {f"{TRUNK_PATH.format(cam)}/{k}": tuple(v.shape) for cam in CAMS for k, v in agent._frozen_trunk.leaves[cam].items()}
    assert trunk
    own = {l.path: tuple(l.shape) for l in spec}
    for key in ("params", "target_params"):
        flat = _flat(d[key])
        assert {k: v.shape for k, v in flat.items()} == {**own, **trunk}, key
    assert set(d["opt_states"]) == {"count", "mu", "nu"} and d["opt_states"]["count"] == 0
    for key in ("mu", "nu"):
        assert {k: v.shape for k, v in _flat(d["opt_states"][key]).items()} == own, key


@pytest.mark.parametrize("make", [_launcher_agent, _options_agent])
def test_checkpoint_round_trip_pickles_numpy_only(dry, tmp_path, make):
    from serl_b200.utils.checkpoints import restore_checkpoint, save_checkpoint
    a = make(1)
    _perturb(a, 5)
    path = save_checkpoint(str(tmp_path), a.state, step=17, keep=100, overwrite=True)

    class NumpyOnly(pickle.Unpickler):
        def find_class(self, module, name):
            assert module.split(".")[0] in ("numpy", "builtins"), (module, name)
            return super().find_class(module, name)

    with open(path, "rb") as f:
        payload = NumpyOnly(f).load()
    restored = restore_checkpoint(str(tmp_path), None)
    assert set(restored) == FIELDS
    want = _flat(a.state.state_dict())
    for got in (_flat(payload), _flat(restored)):
        assert got.keys() == want.keys()
        for k, v in want.items():
            np.testing.assert_array_equal(np.asarray(got[k]), np.asarray(v), err_msg=k)


@pytest.mark.parametrize("make", [_launcher_agent, _options_agent])
def test_replace_installs_a_restored_state(dry, tmp_path, make):
    from serl_b200.utils.checkpoints import restore_checkpoint, save_checkpoint
    a = make(1)
    _perturb(a, 5)
    save_checkpoint(str(tmp_path), a.state, step=17)
    # without a target: restore_checkpoint returns the state dict
    b = make(2)
    b._graphs["stale"] = "warm"
    assert not torch.equal(b._store.params, a._store.params)
    assert b.replace(state=restore_checkpoint(str(tmp_path), None)) is b
    _store_equal(a, b)
    assert not b._graphs
    # with the agent's state as the target (examples/bc_policy.py:204-209): restored in place, then installed
    c = make(3)
    ckpt = restore_checkpoint(str(tmp_path), c.state, step=17)
    assert ckpt is c.state
    c = c.replace(state=ckpt)
    _store_equal(a, c)
    # another agent's state object
    d = make(4)
    d.replace(state=a.state)
    _store_equal(a, d)


def test_replace_refuses_unknown_fields(dry):
    agent = _launcher_agent(1)
    with pytest.raises(TypeError):
        agent.replace(foo=1)
    with pytest.raises(TypeError):
        agent.replace(state=42)
    with pytest.raises(TypeError):
        agent.state.replace(foo=1)
