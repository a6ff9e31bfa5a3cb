"""Train state of the H100 learner: the host-visible face of the flat HBM parameter buffers.

Mirrors `JaxRLTrainState` (reference common/common.py:81-245): fields `step, params, target_params,
opt_states, rng`, `.replace(...)`.  `params` / `target_params` are materialised on demand as nested
dicts of NumPy arrays in the Flax tree layout (SURVEY.md Appendix D) - the wire format
`TrainerServer.publish_network(agent.state.params)` ships to the untouched JAX actor
(examples/async_drq_sim/async_drq_sim.py:229,297) and what checkpoints store (:303-307).
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from ..params import TRUNK_PATH, ParamStore, flatten, nest
from ..trunk import FrozenTrunk


class TrainState:
    def __init__(self, store: ParamStore, trunk: Optional[FrozenTrunk], rng_dev: torch.Tensor, step: int = 0):
        self._store = store
        self._trunk = trunk            # None: the small encoder (no frozen leaves in the tree)
        self._rng = rng_dev            # device uint32[2]: JAX-style key, advanced by the key-schedule kernel
        self.step = step

    # -- trees ----------------------------------------------------------------------------------
    def _tree(self, buf) -> dict:
        flat = self._store.dump(buf)
        if self._trunk is not None:
            flat.update(self._trunk.dump(TRUNK_PATH.format))
        return nest(flat)

    @property
    def params(self) -> dict:
        return self._tree(self._store.params)

    @property
    def target_params(self) -> dict:
        return self._tree(self._store.target)

    @property
    def rng(self) -> np.ndarray:
        return self._rng.cpu().numpy().copy()

    @property
    def opt_states(self) -> dict:
        """Three full-tree Adam states like the reference's (common.py:243).  A leaf's moments under a tx that never sees
        a non-zero gradient for it are identically zero and are synthesised here; the proprio-encoder leaves are live under
        BOTH the critic tx (main buffer) and the actor tx (aux tail of the flat buffers, params.py)."""
        st = self._store
        counts = st.counts.cpu().numpy()
        mu, nu = st.dump(st.m), st.dump(st.v)
        mu_aux, nu_aux = st.dump_aux(st.m), st.dump_aux(st.v)
        out = {}
        for gid, name in ((1, "actor"), (0, "critic"), (2, "temperature")):
            own = {l.path for l in st.spec if l.group == gid}

            def z(d, aux):
                t = {k: (v if k in own else np.zeros_like(v)) for k, v in d.items()}
                if gid == 1:
                    t.update(aux)
                return nest(t)
            out[name] = {"count": int(counts[gid]), "mu": z(mu, mu_aux), "nu": z(nu, nu_aux)}
        return out

    # -- checkpoints (async_drq_sim.py:303-307 passes `agent.state` to flax.training.checkpoints) --------------
    def state_dict(self) -> dict:
        return {"step": int(self.step), "params": self.params, "target_params": self.target_params,
                "opt_states": self.opt_states, "rng": self.rng}

    def load_state_dict(self, d: dict) -> "TrainState":
        return self.replace(step=d["step"], params=d["params"], target_params=d["target_params"], opt_states=d["opt_states"],
                            rng=d["rng"])

    # -- functional-style updates ------------------------------------------------------------------
    def replace(self, **kw) -> "TrainState":
        st = self._store
        for key, buf in (("params", st.params), ("target_params", st.target)):
            if key in kw:
                flat = flatten(kw.pop(key))
                own = {l.path: np.asarray(flat[l.path], np.float32) for l in st.spec}
                st.load(buf, own)
                if key == "params" and self._trunk is not None:
                    self._trunk.load(flat, TRUNK_PATH.format)
        if "rng" in kw:
            key = np.ascontiguousarray(np.asarray(kw.pop("rng")), dtype=np.uint32).reshape(2)
            self._rng.copy_(torch.from_numpy(key.view(np.int32)).view(torch.uint32))
            st.version += 1               # the step pipeline's look-ahead key chain (and any prefetched batch) is stale: agents re-check the version
        if "step" in kw:
            self.step = int(kw.pop("step"))
        if "opt_states" in kw:
            os_ = kw.pop("opt_states")
            mu = {l.path: None for l in st.spec}
            nu = dict(mu)
            mu_aux, nu_aux = {}, {}
            counts = [0, 0, 0]
            for gid, name in ((1, "actor"), (0, "critic"), (2, "temperature")):
                fm, fn = flatten(os_[name]["mu"]), flatten(os_[name]["nu"])
                counts[gid] = int(os_[name]["count"])
                for l in st.spec:
                    if l.group == gid:
                        mu[l.path], nu[l.path] = fm[l.path], fn[l.path]
                    elif gid == 1 and st.two_tx(l.path):                  # actor-tx twin of the proprio encoder
                        mu_aux[l.path], nu_aux[l.path] = fm[l.path], fn[l.path]
            st.load(st.m, mu, mu_aux)
            st.load(st.v, nu, nu_aux)
            st.counts.copy_(torch.tensor(counts, dtype=torch.int32))
        if kw:
            raise TypeError(f"TrainState.replace: unknown fields {sorted(kw)}")
        return self


def _register_flax_serialization():
    try:
        from flax import serialization
    except Exception:                                   # noqa: BLE001
        return False
    try:
        serialization.register_serialization_state(TrainState, lambda s: s.state_dict(), lambda s, d: s.load_state_dict(d))
    except ValueError:
        pass
    return True


_register_flax_serialization()
