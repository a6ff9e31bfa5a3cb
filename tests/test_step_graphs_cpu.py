"""CPU: the agents' step-graph cache (serl_b200/step_graphs.py) with torch.cuda.CUDAGraph / torch.cuda.graph replaced by a
recorder, on real DeviceRings in host memory.  Pins the warm-up / capture / replay order, the state's step, the launch-counter
correction, the rings' draw counters for the serial and cross-step pipeline draw patterns, and what holds while a step is
captured: the rings' locks are held and the cyclic garbage collector is paused."""
import contextlib
import gc
import threading
import types

import pytest
import torch

from serl_b200 import _lib as L
from serl_b200.data.replay_buffer import DeviceRing
from serl_b200.step_graphs import StepGraphs

LAUNCHES = 5            # library launches one step enqueues
STEPS = 2               # state steps one step advances (update_high_utd's critic + actor update)


class Recorder:
    """Stands in for the CUDA runtime: a captured graph keeps the device work its body recorded and runs it on replay."""

    def __init__(self):
        self.log, self.launches, self.capturing = [], 0, None

    def graph_cls(self):
        rec = self

        class FakeGraph:
            def __init__(self):
                self.work = []

            def replay(self):
                rec.log.append(("replay", self))
                for w in self.work:
                    w()
        return FakeGraph

    @contextlib.contextmanager
    def graph(self, g, capture_error_mode=None):
        assert capture_error_mode == "thread_local"
        self.log.append(("capture", g))
        self.capturing = g
        try:
            yield
        finally:
            self.capturing = None


@pytest.fixture()
def rec(monkeypatch):
    r = Recorder()
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: r.launches)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", r.graph_cls())
    monkeypatch.setattr(torch.cuda, "graph", r.graph)
    return r


def _ring():
    """A host-memory ring whose counter fills are logged in `ring.fills`."""
    ring = DeviceRing(16, (), (1, 1, 1), 1, 3, 2, device="cpu", seed=0)
    ring.fills, fill = [], ring.step_dev.fill_
    ring.step_dev.fill_ = lambda v: (ring.fills.append(v), fill(v))[1]
    return ring


def _lock_free_elsewhere(ring) -> bool:
    """Whether another thread can take the ring's lock now (a DataStore insert thread would)."""
    got = []

    def try_lock():
        ok = ring._lock.acquire(blocking=False)
        if ok:
            ring._lock.release()
        got.append(ok)
    t = threading.Thread(target=try_lock)
    t.start()
    t.join()
    return got[0]


def _step(rec, state, draws, drawn, seen):
    """An agent step: `n` draws per ring from the handle's steps when eager; a captured step's draws read and advance the
    ring's device counter (the sampler's step_dev and ops.counter_add) at replay."""
    def body(graph_mode):
        seen.append((graph_mode, gc.isenabled(), [_lock_free_elsewhere(ring) for ring, _, _ in draws]))
        rec.log.append(("body", graph_mode))
        rec.launches += LAUNCHES
        state.step += STEPS
        for ring, first, n in draws:
            for i in range(n):
                if graph_mode:
                    def draw(ring=ring):
                        drawn[ring].append(int(ring.step_dev.item()))
                        ring.step_dev.add_(1)
                    rec.capturing.work.append(draw)
                else:
                    drawn[ring].append(first + i)
    return body


# first draw of a handle at `step` and the number of draws: the serial SAC / DrQ / BC step, the pipeline's cold start "W" (this
# step's batch, then the next one's) and its continuing step "P" (the next step's batch only)
PATTERNS = {"serial": (0, 1), "W": (0, 2), "P": (1, 1)}


@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_eager_warm_capture_replay(rec, pattern):
    off, n = PATTERNS[pattern]
    rings = [_ring(), _ring()]
    graphs, state = StepGraphs(), types.SimpleNamespace(step=0)
    drawn, seen = {r: [] for r in rings}, []
    # handles that continue each other, then a jump (another iterator's handle): the counter is re-armed
    handle_steps = [0, n, 2 * n, 3 * n, 10, 10 + n]
    for call, s in enumerate(handle_steps):
        draws = [(rings[0], s + off, n), (rings[1], 100 + s + off, n)]
        seen.clear()
        graphs.run(("key",), draws, _step(rec, state, draws, drawn, seen), state)
        assert state.step == STEPS * (call + 1)
        assert rec.launches + graphs.launch_adj == LAUNCHES * (call + 1)          # launches executed, not recorded
        assert gc.isenabled()
        if call == 0:
            assert graphs[("key",)] == "warm" and seen == [(False, True, [True, True])]
            continue
        g, steps, recorded = graphs[("key",)]
        assert (steps, recorded) == (STEPS, LAUNCHES)
        if call == 1:                                   # captured with the rings locked and the collector paused, then replayed
            assert seen == [(True, False, [False, False])]
            assert rec.log[-4:] == [("body", False), ("capture", g), ("body", True), ("replay", g)]
        else:
            assert seen == [] and rec.log[-1] == ("replay", g)
        for ring, first, k in draws:
            assert ring._dev_step_mirror == first + k and int(ring.step_dev.item()) == first + k
    for r, base in zip(rings, (0, 100)):
        assert drawn[r] == [base + s + off + i for s in handle_steps for i in range(n)]
        assert r.fills == [base + handle_steps[c] + off for c in (1, 4)]      # only where the sequence does not continue
    assert [e[0] for e in rec.log].count("capture") == 1


def test_no_key_runs_eagerly(rec):
    ring = _ring()
    graphs, state = StepGraphs(), types.SimpleNamespace(step=0)
    drawn, seen = {ring: []}, []
    for s in range(3):
        draws = [(ring, s, 1)]
        graphs.run(None, draws, _step(rec, state, draws, drawn, seen), state)
    assert not graphs and graphs.launch_adj == 0 and state.step == 3 * STEPS
    assert rec.log == [("body", False)] * 3 and drawn[ring] == [0, 1, 2]
    assert ring._dev_step_mirror == 0 and int(ring.step_dev.item()) == 0


def test_capture_that_raises_restores_the_collector_and_locks(rec):
    ring = _ring()
    graphs, state = StepGraphs(), types.SimpleNamespace(step=0)

    def body(graph_mode):
        if graph_mode:
            raise RuntimeError("capture failed")

    graphs.run(("key",), [(ring, 0, 1)], body, state)
    with pytest.raises(RuntimeError, match="capture failed"):
        graphs.run(("key",), [(ring, 1, 1)], body, state)
    assert gc.isenabled() and _lock_free_elsewhere(ring)
    gc.disable()                                        # a collector the caller turned off stays off
    try:
        with pytest.raises(RuntimeError, match="capture failed"):
            graphs.run(("key",), [(ring, 1, 1)], body, state)
        assert not gc.isenabled()
    finally:
        gc.enable()
