"""CPU (dry device): the agents' flat parameter stores against tests/golden/flat_store_golden.json, which was generated before
BC, the reward classifier and VICE shared `params.FlatParams`, `FrozenTrunk.dump / load` and the engine's policy-MLP loops
(tests/golden/make_flat_store_golden.py): layouts and initial values, the ORDER of the kernel launches of one training step and
one inference call, and the tree round trip through `replace`."""
import importlib.util
import json
import os

import numpy as np
import pytest

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_spec = importlib.util.spec_from_file_location("make_flat_store_golden", os.path.join(GOLDEN_DIR, "make_flat_store_golden.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

with open(G.GOLDEN) as f:
    GOLDEN = json.load(f)


@pytest.fixture()
def dry(monkeypatch):
    calls = []
    G.patch_dry(monkeypatch.setattr, calls)
    return calls


@pytest.mark.parametrize("kind", G.KINDS)
def test_layout_and_initial_values(dry, kind):
    """(path, shape, offset) of every leaf, and the digests of the seeded initial parameters, trunk leaves and rng."""
    got = G.layout(kind, G.build(kind))
    want = GOLDEN["layout"][kind]
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("kind", ["bc_launcher", "bc_options", "classifier", "vice"])
def test_ordered_launch_names(dry, kind, precision):
    got = G.launches(kind, precision, dry)
    want = GOLDEN["launches"][f"{kind}-{precision}"]
    assert sorted(got) == sorted(want)
    for call in want:
        assert got[call] == want[call], call


def _perturbed(tree, rng):
    return {k: _perturbed(v, rng) if isinstance(v, dict) else (np.asarray(v) + rng.standard_normal(np.shape(v)).astype(np.float32)) for k, v in tree.items()}


def _assert_trees_equal(a, b, path=""):
    assert sorted(a) == sorted(b), path
    for k in a:
        if isinstance(a[k], dict):
            _assert_trees_equal(a[k], b[k], f"{path}/{k}")
        else:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{path}/{k}")


@pytest.mark.parametrize("kind", ["bc_launcher", "classifier", "vice"])
def test_replace_writes_every_leaf_and_drops_the_trunk_packing(dry, kind):
    obj = G.build(kind, "fp16")
    state = obj if kind == "classifier" else obj.state
    trunk = obj._frozen_trunk
    for cam in G.CAMS:
        trunk.packed(cam)
    assert set(trunk._packed) == set(G.CAMS)
    tree = _perturbed(state.params, np.random.default_rng(0))
    if kind == "vice":                                            # the trunk copies under modules_vice are exports of the agent's trunk
        from serl_b200.agents.continuous.vice import trunk_clone_paths
        from serl_b200.params import flatten, nest
        flat, src = flatten(tree), "modules_actor/encoder/encoder_{}/pretrained_encoder"
        for pre, cam in zip(trunk_clone_paths(G.CAMS), (G.CAMS[0],) + G.CAMS):
            for k in [k for k in flat if k.startswith(pre + "/")]:
                flat[k] = flat[src.format(cam) + k[len(pre):]]
        tree = nest(flat)
    state.replace(params=tree)
    assert trunk._packed == {}
    _assert_trees_equal(state.params, tree)
    assert G.optimizer_shapes(kind, obj) == GOLDEN["trees"][kind]


def test_classifier_state_dict_round_trip(dry):
    a, b = G.build("classifier"), G.build("classifier")
    rng = np.random.default_rng(1)
    sd = a.state_dict()
    sd = {"step": 7, "params": _perturbed(sd["params"], rng),
          "opt_state": {"count": 3, "mu": _perturbed(sd["opt_state"]["mu"], rng), "nu": _perturbed(sd["opt_state"]["nu"], rng)}}
    b.load_state_dict(sd)
    got = b.state_dict()
    assert got["step"] == 7 and got["opt_state"]["count"] == 3
    _assert_trees_equal(got["params"], sd["params"])
    _assert_trees_equal(got["opt_state"]["mu"], sd["opt_state"]["mu"])
    _assert_trees_equal(got["opt_state"]["nu"], sd["opt_state"]["nu"])
