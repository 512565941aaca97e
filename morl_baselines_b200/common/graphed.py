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
from typing import Any, Callable, Hashable, Iterable, List, Optional

import numpy as np
import torch as th

from .. import ops


@contextlib.contextmanager
def _gc_paused():
    """Collect cyclic garbage now and keep the collector off during a capture.  A dropped graph that sits in a reference cycle (a step
    closure that reaches its own learner) is otherwise destroyed by whichever collection happens to run inside a later capture; CUDA
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
        self.launches = None

    def _record(self):
        """The work the graph records (the warm-up passes run ``fn``)."""
        self.fn()

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
        before = ops.launch_count
        with _gc_paused(), th.cuda.graph(g):
            self._record()
        self.launches = ops.launch_count - before  # the project's kernel launches one replay makes
        with th.no_grad():
            for t, s in zip(tensors, snap):
                t.copy_(s)
        th.cuda.set_rng_state(rng)
        self.graph = g

    def __call__(self):
        if self.graph is None:
            self.capture()
        self.graph.replay()


class PopulationGraph(GraphedStep):
    """ONE CUDA graph for the device halves of many independent learners (MORL/D ``__update_others``, reference morld.py:423-433, runs them
    strictly one after the other).  Inside the capture the steps are forked round-robin onto ``n_streams`` side streams and joined again,
    so the graph has that many parallel branches: the tiny kernels of a 2 x 256, batch-128 actor-critic update leave most of the GPU idle,
    and independent learners fill it.  The result per learner is bit-identical to replaying its own graph (no cross-learner data flow)."""

    def __init__(self, steps, mutated, n_streams: int = 8, warmup: int = 3):
        super().__init__(self._run_serial, mutated, warmup)
        self.steps = list(steps)
        self.streams = [th.cuda.Stream() for _ in range(max(1, min(n_streams, len(self.steps))))]

    def _run_serial(self):
        for fn in self.steps:
            fn()

    def _record(self):
        main = th.cuda.current_stream()
        for s in self.streams:
            s.wait_stream(main)
        for i, fn in enumerate(self.steps):
            with th.cuda.stream(self.streams[i % len(self.streams)]):
                fn()
        for s in self.streams:
            main.wait_stream(s)


class Staging:
    """A pinned host tensor, its device twin and the event of the last copy between them.

    The host may run more than one update ahead of the device (several replays queued, a population graph), so a pinned tensor must not
    be rewritten while an asynchronous copy that reads it is still queued: ``host()`` waits for the previous ``upload()`` before it hands
    out the writable view, and an update reads its own inputs."""

    def __init__(self, shape, dtype: th.dtype, device):
        self.pin = th.zeros(shape, dtype=dtype).pin_memory()
        self.dev = th.zeros(shape, dtype=dtype, device=device)
        self._copied = th.cuda.Event()

    def host(self) -> np.ndarray:
        """Writable numpy view of the pinned tensor, once the previous upload has read it."""
        self._copied.synchronize()
        return self.pin.numpy()

    def _rows(self, n: Optional[int]):
        # whole tensors unless n is given: a slice costs microseconds of host time, paid per learner and update
        return (self.pin, self.dev) if n is None else (self.pin[:n], self.dev[:n])

    def upload(self, n: Optional[int] = None):
        """Queue the copy of the first ``n`` rows (all by default) to the device on the current stream."""
        pin, dev = self._rows(n)
        dev.copy_(pin, non_blocking=True)
        self._copied.record()

    def fetch(self, n: Optional[int] = None) -> np.ndarray:
        """The first ``n`` rows of the device tensor on the host: queues the copy after the work that writes them and waits for it."""
        pin, dev = self._rows(n)
        pin.copy_(dev, non_blocking=True)
        self._copied.record()
        self._copied.synchronize()
        return pin.numpy().copy()


class Variant:
    """One captured update variant: its cache ``key``, the device half ``step`` (an argument-free closure over the static inputs), the
    ``graph`` that replays it for this learner alone, and the static inputs themselves as further attributes."""

    def __init__(self, key: Hashable, step: Callable[[], None], mutated: Callable[[], Iterable[th.Tensor]], **inputs):
        self.key, self.step, self.graph = key, step, GraphedStep(step, mutated)
        self.__dict__.update(inputs)

    def __getitem__(self, name: str):
        """``variant["graph"]`` is ``variant.graph``: code written against the earlier per-variant dicts keeps working."""
        return getattr(self, name)


class GraphCache(dict):
    """Captured update variants (or population graphs) by key, each built once.  A captured graph keeps reading the storage it saw at
    capture (the replay mirror, optimiser state, the support matrix), so the owner calls ``clear()`` whenever it replaces one of those."""

    def get_or_build(self, key: Hashable, build: Callable[[], Any]):
        v = super().get(key)
        if v is None:
            v = self[key] = build()
        return v


def optimizer_tensors(opt) -> List[th.Tensor]:
    """Every state tensor of a FusedClipAdam (created if the optimiser has not stepped yet, so that a snapshot exists)."""
    opt._ensure_state()
    out = []
    for st in opt.state.values():
        out += [st["step"], st["exp_avg"], st["exp_avg_sq"]]
    return out
