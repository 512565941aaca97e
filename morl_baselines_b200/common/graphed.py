"""CUDA-graph capture of a device-only update step (replacement of the reference's eager op-by-op updates).

The small actor-critic updates of the reference (MOSAC: mosac_continuous_action.py:429-507; CAPQL: capql.py:321-362;
GPI-PD continuous: gpi_pd_continuous_action.py:373-452) are ~250 tiny tensor operations -- launch-bound on any GPU.  ``GraphedStep`` captures one whole update over
STATIC input buffers (replay indices, optional injected noise) once and replays it: one host call per update.

Warm-up iterations and the capture pass itself must leave no trace (the number of updates applied to the parameters has to match
the reference exactly), so the caller lists every tensor the step mutates and they are restored IN PLACE after capture.
"""

from __future__ import annotations

import contextlib
import gc
from typing import Callable, Iterable, List

import torch as th


@contextlib.contextmanager
def _gc_paused():
    """Collect cyclic garbage now and keep the collector off during a capture.  A dropped graph that sits in a reference cycle (a step
    closure that holds its own state dict) is otherwise destroyed by whichever collection happens to run inside a later capture; CUDA
    forbids that while a stream captures, and the capture is invalidated."""
    gc.collect()
    enabled = gc.isenabled()
    gc.disable()
    try:
        yield
    finally:
        if enabled:
            gc.enable()


class GraphedStep:
    def __init__(self, fn: Callable[[], None], mutated: Callable[[], Iterable[th.Tensor]], warmup: int = 3):
        self.fn = fn
        self.mutated = mutated
        self.warmup = warmup
        self.graph = None

    def capture(self):
        tensors: List[th.Tensor] = list(self.mutated())
        snap = [t.detach().clone() for t in tensors]
        rng = th.cuda.get_rng_state()
        side = th.cuda.Stream()
        side.wait_stream(th.cuda.current_stream())
        with th.cuda.stream(side):
            for _ in range(self.warmup):
                self.fn()
        th.cuda.current_stream().wait_stream(side)
        g = th.cuda.CUDAGraph()
        with _gc_paused(), th.cuda.graph(g):
            self.fn()
        with th.no_grad():
            for t, s in zip(tensors, snap):
                t.copy_(s)
        th.cuda.set_rng_state(rng)
        self.graph = g

    def __call__(self):
        if self.graph is None:
            self.capture()
        self.graph.replay()


class PopulationGraph:
    """ONE CUDA graph for the device halves of many independent learners (MORL/D ``__update_others``, reference morld.py:423-433, runs them
    strictly one after the other).  Inside the capture the steps are forked round-robin onto ``n_streams`` side streams and joined again,
    so the graph has that many parallel branches: the tiny kernels of a 2 x 256, batch-128 actor-critic update leave most of the GPU idle,
    and independent learners fill it.  The result per learner is bit-identical to replaying its own graph (no cross-learner data flow)."""

    def __init__(self, steps, mutated, n_streams: int = 8, warmup: int = 3):
        self.steps, self.mutated = list(steps), mutated
        self.n_streams = max(1, min(n_streams, len(self.steps)))
        self.warmup = warmup
        self.graph = None

    def _run_forked(self, streams):
        main = th.cuda.current_stream()
        for s in streams:
            s.wait_stream(main)
        for i, fn in enumerate(self.steps):
            with th.cuda.stream(streams[i % len(streams)]):
                fn()
        for s in streams:
            main.wait_stream(s)

    def capture(self):
        tensors: List[th.Tensor] = list(self.mutated())
        snap = [t.detach().clone() for t in tensors]
        rng = th.cuda.get_rng_state()
        streams = [th.cuda.Stream() for _ in range(self.n_streams)]
        side = th.cuda.Stream()
        side.wait_stream(th.cuda.current_stream())
        with th.cuda.stream(side):
            for _ in range(self.warmup):
                for fn in self.steps:
                    fn()
        th.cuda.current_stream().wait_stream(side)
        g = th.cuda.CUDAGraph()
        with _gc_paused(), th.cuda.graph(g):
            self._run_forked(streams)
        with th.no_grad():
            for t, s in zip(tensors, snap):
                t.copy_(s)
        th.cuda.set_rng_state(rng)
        self.graph = g

    def __call__(self):
        if self.graph is None:
            self.capture()
        self.graph.replay()


def optimizer_tensors(opt) -> List[th.Tensor]:
    """Every state tensor of a FusedClipAdam (created if the optimiser has not stepped yet, so that a snapshot exists)."""
    opt._ensure_state()
    out = []
    for st in opt.state.values():
        out += [st["step"], st["exp_avg"], st["exp_avg_sq"]]
    return out
