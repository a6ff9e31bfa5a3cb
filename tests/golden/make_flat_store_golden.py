"""Generates flat_store_golden.json: what the SAC / DrQ / BC / reward-classifier / VICE builders produce on the dry device (kernel
launches recorded, not run) - every spec's (path, shape, offset), SHA-256 digests of the initial parameters, trunk leaves and
rng, the ordered kernel names of one training step + one inference call, and the key -> shape lists of the optimizer trees.

The committed fixture was generated at the commit BEFORE the agents shared one flat parameter store; this script regenerates it
unchanged on every later commit (tests/test_flat_store_cpu.py compares against it):

    python tests/golden/make_flat_store_golden.py
"""
import contextlib
import hashlib
import json
import os
import sys
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "flat_store_golden.json")
CAMS = ("front", "wrist")
BC_OPTIONS = dict(use_proprio=False, policy_kwargs={"std_parameterization": "uniform", "tanh_squash_distribution": True},
                  network_kwargs={"activations": "gelu", "use_layer_norm": True, "hidden_dims": [128, 64, 64], "dropout_rate": 0.1})
KINDS = ("drq", "sac", "bc_launcher", "bc_options", "classifier", "vice")


def patch_dry(setattr_, calls):
    """Replaces the library's launch entry by a recorder of kernel names; setattr_(obj, name, value) as monkeypatch.setattr."""
    from serl_b200 import _lib as L
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

    setattr_(L, "call", fake_call)
    setattr_(L, "require_cuda", lambda d: None)
    setattr_(L, "stream_ptr", lambda: 0)
    setattr_(L, "new_event", lambda: Ev())
    setattr_(L, "pin", lambda t: t)
    setattr_(L, "launch_count", lambda: len(calls))


def transitions(n, seed=0):
    from helpers import random_transitions
    return random_transitions(np.random.default_rng(seed), n, CAMS, 128)


def stack(trs, key):
    return {**{c: np.stack([t[key][c] for t in trs]) for c in CAMS}, "state": np.stack([t[key]["state"] for t in trs])}


def sac_batch(trs):
    return {"observations": stack(trs, "observations"), "next_observations": stack(trs, "next_observations"),
            "actions": np.stack([t["actions"] for t in trs]), "rewards": np.array([t["rewards"] for t in trs], np.float32),
            "masks": np.array([t["masks"] for t in trs], np.float32), "dones": np.array([t["dones"] for t in trs])}


def build(kind, precision="fp32"):
    from serl_b200.agents.continuous.bc import BCAgent
    from serl_b200.networks.reward_classifier import create_classifier
    from serl_b200.utils import launcher
    tr = transitions(1)[0]
    obs, act = tr["observations"], tr["actions"]
    px = dict(image_keys=CAMS, encoder_type="resnet-pretrained", precision=precision, device="cpu")
    if kind == "drq":
        return launcher.make_drq_agent(3, obs, act, **px)
    if kind == "sac":
        return launcher.make_sac_agent(4, obs["state"][0], act, device="cpu")
    if kind == "bc_launcher":
        return launcher.make_bc_agent(5, obs, act, **px)
    if kind == "bc_options":
        return BCAgent.create(6, obs, act, **BC_OPTIONS, **px)
    if kind == "classifier":
        return create_classifier(np.array([0, 8], np.uint32), obs, CAMS, precision=precision, device="cpu")
    return launcher.make_vice_agent(7, obs, act, vice_image_keys=CAMS, **px)


def stores(kind, obj):
    """name -> every flat store the object owns."""
    return {"main": obj._store, "vice": obj._vice} if kind == "vice" else {"main": obj._store}


def _sha(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def layout(kind, obj):
    out = {}
    for name, st in stores(kind, obj).items():
        out[name] = {"spec": [[l.path, list(l.shape), l.offset] for l in st.spec], "n": int(st.params.numel()), "params": _sha([st.params.numpy()])}
    out["trunk"] = _sha([t.numpy() for cam in obj._trunk for t in obj._trunk[cam].values()])
    out["trunk_leaves"] = [f"{cam}/{k}" for cam in obj._trunk for k in obj._trunk[cam]]
    if kind != "classifier":
        out["rng"] = _sha([obj.state.rng])
    return out


def launches(kind, precision, calls):
    """Ordered kernel names of one training step and one inference call (VICE: update_vice, update_critics, vice_reward)."""
    obj = build(kind, precision)
    trs = transitions(4, seed=1)
    obs = stack(trs, "observations")
    out = {}

    def run(name, fn):
        del calls[:]
        fn()
        out[name] = list(calls)
    if kind.startswith("bc"):
        batch = {"observations": obs, "actions": np.stack([t["actions"] for t in trs]).astype(np.float32)}
        run("update", lambda: obj.update(batch))
        run("sample_actions", lambda: obj.sample_actions(obs, argmax=True))
        run("sample_actions_seeded", lambda: obj.sample_actions(obs, seed=np.array([1, 2], np.uint32)))
    elif kind == "classifier":
        data = {c: obs[c] for c in CAMS}
        labels = np.array([[1.0], [1.0], [0.0], [0.0]], np.float32)
        run("train_step", lambda: obj.train_step({"data": data, "labels": labels}, np.array([3, 4], np.uint32)))
        run("call", lambda: obj(data))
    else:
        batch = sac_batch(trs)
        run("update_vice", lambda: obj.update_vice(batch))
        run("update_critics", lambda: obj.update_critics(batch))
        run("vice_reward", lambda: obj.vice_reward(obs))
    return out


def shapes(tree, prefix=""):
    """Nested tree -> sorted [path, shape] list."""
    out = []
    for k in sorted(tree):
        p = f"{prefix}/{k}" if prefix else k
        out += shapes(tree[k], p) if isinstance(tree[k], dict) else [[p, list(np.shape(tree[k]))]]
    return out


def optimizer_shapes(kind, obj):
    if kind == "classifier":
        sd = obj.state_dict()
        return {"state_dict": sorted(sd), "params": shapes(sd["params"]), "opt_state": shapes(sd["opt_state"])}
    return {"opt_states": shapes(obj.state.opt_states)}


def generate(calls):
    out = {"layout": {}, "launches": {}, "trees": {}}
    for kind in KINDS:
        obj = build(kind)
        out["layout"][kind] = layout(kind, obj)
        if kind not in ("drq", "sac"):
            out["trees"][kind] = optimizer_shapes(kind, obj)
            for precision in ("fp32", "fp16"):
                out["launches"][f"{kind}-{precision}"] = launches(kind, precision, calls)
    return out


if __name__ == "__main__":
    sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
    calls = []
    with contextlib.ExitStack() as stack_:
        patch_dry(lambda o, n, v: stack_.enter_context(mock.patch.object(o, n, v)), calls)
        golden = generate(calls)
    with open(GOLDEN, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {GOLDEN}")
