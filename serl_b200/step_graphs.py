"""The agents' step-graph cache: a training step is captured once as a CUDA graph and replayed after that."""
from __future__ import annotations

import contextlib
import gc

import torch

from . import _lib as L


class StepGraphs(dict):
    """Graph key -> "warm" (the key's first step ran eagerly) or (graph, state steps, recorded launches) once captured.

    `launch_adj` corrects the library's launch counter: the launches recorded by a capture did not execute, and every replay
    executes them."""

    def __init__(self):
        super().__init__()
        self.launch_adj = 0

    def run(self, key, draws, body, state):
        """body(graph_mode) enqueues one step that advances `state.step`.  key None: eager.  The 1st call with a key runs
        eagerly (warm-up: lazy allocations, function attributes), the 2nd captures and replays, later ones replay only.

        draws: (ring, first draw step, number of draws the step makes) per replay-ring part of the batch.  A captured
        sampler launch reads its draw step from the ring's device counter, which is armed here before every capture or replay."""
        if key is None:
            return body(False)
        entry = self.get(key)
        if entry is None:
            self[key] = "warm"
            return body(False)
        for ring, step, n in draws:
            ring.arm_draw_counter(step, n)
        if entry == "warm":
            entry = self[key] = self._capture(draws, body, state)
        graph, steps, recorded = entry
        graph.replay()
        self.launch_adj += recorded
        state.step += steps

    def _capture(self, draws, body, state):
        graph = torch.cuda.CUDAGraph()
        s0, c0 = state.step, L.launch_count()
        # An agent and its state refer to each other, so a dropped agent's graphs are freed by the cyclic collector; freeing a
        # graph inside a capture invalidates the capture, so the collector waits until it ends.
        gc_on = gc.isenabled()
        gc.disable()
        try:
            # the ring locks and thread-local capture mode: a DataStore insert thread must not enqueue its flush (an H2D copy on
            # another stream) into - or invalidate - this capture
            with contextlib.ExitStack() as stack:
                for ring, _, _ in draws:
                    stack.enter_context(ring._lock)
                with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                    body(True)
        finally:
            if gc_on:
                gc.enable()
        recorded = L.launch_count() - c0
        self.launch_adj -= recorded                     # recorded, not executed
        steps, state.step = state.step - s0, s0         # the capture only recorded the step
        return graph, steps, recorded
