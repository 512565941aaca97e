"""Binding of Pareto Q-learning's set-table kernels (csrc/pql.cu: ``morl_pql_update_f64``, ``morl_pql_score_f64``).

The table is the caller's float64 / int32 CUDA tensors (:class:`PqlTable` allocates and initialises them as the reference does).  Every
tensor passes the argument contract of :mod:`ops` (``ops._Args``) and every launch goes through ``ops._launch``, so ``ops.launch_count``
counts it.  The reward and the reference point are passed to the kernel by value: a step makes no host-to-device copy.
"""

from __future__ import annotations

import ctypes
from typing import Optional

import numpy as np
import torch as th

from . import _lib
from .ops import _Args, _launch

HYPERVOLUME, CARDINALITY = 0, 1  # MORL_PQL_* of include/morl_b200.h
MODES = {"hypervolume": HYPERVOLUME, "pareto_cardinality": CARDINALITY}


def pql_supported(n_actions: int, cap: int, d: int, mode: int) -> bool:
    """Whether the kernels cover A actions, set capacity K and d objectives in scoring ``mode`` (:data:`HYPERVOLUME` or
    :data:`CARDINALITY`, whose range the update needs): 1 <= A <= 16, 1 <= K <= 256, A * K <= 2048, 1 <= d <= 8, and d <= 4 for
    hypervolume scores.  Needs no device."""
    return bool(_lib.load().morl_pql_supported(int(n_actions), int(cap), int(d), int(mode)))


def _host_vec(x, d: int, name: str, a: _Args):
    v = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1))
    if v.shape != (d,):
        a.fail(name, f"must hold {d} values, got {v.size}")
    return (ctypes.c_double * d)(*v.tolist())


def _index(a: _Args, name: str, v, n: int) -> int:
    i = int(v)
    if not 0 <= i < n:
        a.fail(name, f"= {i} is outside [0, {n})")
    return i


class PqlTable:
    """The device state of one agent: ``nd`` f64 [S, A, K, d], ``nd_count`` int32 [S, A], ``avg_reward`` f64 [S, A, d], ``counts`` f64
    [S, A] and ``status`` int32 [3] ({needed size, s, a} of the first overflow, zero while none).  Initial state as the reference's:
    every stored set is {0}, every count and average zero."""

    def __init__(self, S: int, A: int, K: int, d: int, device):
        if not pql_supported(A, K, d, CARDINALITY) or S < 1:
            raise _lib.MorlB200Error(f"PqlTable: S={S}, A={A}, K={K}, d={d} outside the kernels' range "
                                     "(S >= 1, 1 <= A <= 16, 1 <= K <= 256, A * K <= 2048, 1 <= d <= 8)")
        self.S, self.A, self.K, self.d = int(S), int(A), int(K), int(d)
        self.nd = th.zeros((S, A, K, d), dtype=th.float64, device=device)
        self.nd_count = th.ones((S, A), dtype=th.int32, device=device)
        self.avg_reward = th.zeros((S, A, d), dtype=th.float64, device=device)
        self.counts = th.zeros((S, A), dtype=th.float64, device=device)
        self.status = th.zeros(3, dtype=th.int32, device=device)

    def _args(self, binding: str, write: bool) -> _Args:
        a = _Args(binding)
        S, A, K, d = self.S, self.A, self.K, self.d
        a.inp(self.nd, "nd", (S, A, K, d), th.float64, inplace=write)
        a.inp(self.nd_count, "nd_count", (S, A), th.int32, inplace=write)
        a.inp(self.avg_reward, "avg_reward", (S, A, d), th.float64, inplace=write)
        if write:
            a.inp(self.counts, "counts", (S, A), th.float64, inplace=True)
            a.inp(self.status, "status", (3,), th.int32, inplace=True)
        return a


def pql_update(t: PqlTable, s: int, a: int, s_next: int, reward, gamma: float) -> None:
    """One reference step (pql.py:260-262) on the table: ``counts[s, a] += 1``, ``ND[s][a] = ND(U_a' Q-set(s_next, a'))``, ``avg_reward[s, a]
    += (reward - avg_reward[s, a]) / counts[s, a]``.  ``reward``: d host values.  On a set of more than K points nothing is written but
    ``status`` (read it with :func:`check_status`).  One launch, no host synchronisation."""
    args = t._args("pql_update", True)
    s = _index(args, "s", s, t.S)
    a = _index(args, "a", a, t.A)
    s_next = _index(args, "s_next", s_next, t.S)
    r = _host_vec(reward, t.d, "reward", args)
    _launch("morl_pql_update_f64", t.nd, t.nd_count, t.avg_reward, t.counts, t.status, t.S, t.A, t.K, t.d, s, a, s_next, float(gamma), r)


def pql_score(t: PqlTable, state: int, mode: int, gamma: float, ref=None, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Action scores f64 [A] of ``state`` on the device: exact hypervolume of each Q-set above ``ref`` (d host values) for
    :data:`HYPERVOLUME`, the pareto cardinality for :data:`CARDINALITY`.  One launch, no host synchronisation."""
    args = t._args("pql_score", False)
    state = _index(args, "state", state, t.S)
    if mode not in (HYPERVOLUME, CARDINALITY):
        args.fail("mode", f"= {mode} is neither HYPERVOLUME ({HYPERVOLUME}) nor CARDINALITY ({CARDINALITY})")
    if not pql_supported(t.A, t.K, t.d, mode):
        args.fail("mode", f"= {mode} does not support A={t.A}, K={t.K}, d={t.d}" + (" (hypervolume scores need d <= 4)" if t.d > 4 else ""))
    r = _host_vec(ref, t.d, "ref", args) if mode == HYPERVOLUME else None
    out = args.out(out, "out", (t.A,), th.float64)
    _launch("morl_pql_score_f64", t.nd, t.nd_count, t.avg_reward, t.S, t.A, t.K, t.d, state, float(gamma), int(mode), r, out)
    return out


def check_status(t: PqlTable, status=None) -> None:
    """Raise MorlB200Error if an update overflowed the set capacity.  ``status``: a host copy of ``t.status`` already made, else this
    copies it (one device-to-host synchronisation)."""
    st = t.status.cpu().numpy() if status is None else np.asarray(status)
    if int(st[0]) != 0:
        raise _lib.MorlB200Error(f"PQL: the Pareto set of state {int(st[1])}, action {int(st[2])} needs {int(st[0])} points, more than "
                                 f"max_set_size={t.K}: raise max_set_size to at least {int(st[0])}")
