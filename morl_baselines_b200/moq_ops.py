"""Binding of multi-policy scalarised Q-learning's table kernels (csrc/moq.cu: ``morl_moq_act_f64``, ``morl_moq_step_f64``).

:class:`MoqIndex` owns every key on the host: state tuples to dense ids (first seen, across all policies), ``(state, action)`` pairs to
model indices and each pair's outcomes ``(next state, reward, terminal)`` to outcome slots, in the reference TabularModel's dict order.
Real transitions are the only way a key enters, so the device never searches.  :class:`MoqTable` holds the device tensors and grows them
by doubling (torch copies, never inside a launch).  Every tensor passes the argument contract of :mod:`ops` (``ops._Args``) and every launch
goes through ``ops._launch``.  Weights, rewards and random draws reach the kernels by value: a step makes no host-to-device copy.
"""

from __future__ import annotations

import ctypes
import random
from typing import Optional, Sequence

import numpy as np
import torch as th

from . import _lib
from .ops import _Args, _launch

GPI, MODEL, PRIORITIZE = 1, 2, 4  # MORL_MOQ_* of include/morl_b200.h
N_LEVELS = 18                     # the reference's SumTree(max_size=1e5)
MAX_PAIRS = 1 << (N_LEVELS - 1)   # its leaves
DYNA_PER_LAUNCH = 64
ACT_ROWS = 32


def moq_supported(n_actions: int, d: int) -> bool:
    """Whether the kernels cover A actions and d objectives: 1 <= A <= 64, 1 <= d <= 8.  Needs no device."""
    return bool(_lib.load().morl_moq_supported(int(n_actions), int(d)))


def state_key(obs) -> tuple:
    """The reference's ``_state_to_tuple`` as a hashable key of python scalars (equal, and hash-equal, to the reference's key)."""
    return tuple(np.asarray(obs).reshape(-1).tolist())


class MoqIndex:
    """Host keys of one table: ``state_id`` (first-seen order), ``pairs`` [(state id, action)] with ``pair_of``, and per pair the outcome
    keys ``(next state id, reward tuple, terminal)`` in insertion order."""

    def __init__(self):
        self.state_id = {}
        self.states = []
        self.pair_of = {}
        self.pairs = []
        self.outcomes = []

    def find(self, obs) -> int:
        """Id of a state, -1 if never seen."""
        return self.state_id.get(state_key(obs), -1)

    def add_state(self, obs) -> int:
        key = state_key(obs)
        i = self.state_id.get(key)
        if i is None:
            i = self.state_id[key] = len(self.states)
            self.states.append(key)
        return i

    def add_outcome(self, s: int, a: int, s2: int, reward, terminal) -> tuple:
        """(pair, outcome) of a real transition, inserting either key as TabularModel.update does (tabular_model.py:29-49)."""
        m = self.pair_of.get((s, a))
        if m is None:
            if len(self.pairs) >= MAX_PAIRS:
                raise _lib.MorlB200Error(f"MoqIndex: more than {MAX_PAIRS} state-action pairs, the leaves of the model's SumTree(1e5)")
            m = self.pair_of[(s, a)] = len(self.pairs)
            self.pairs.append((s, a))
            self.outcomes.append({})
        out = self.outcomes[m]
        key = (s2, tuple(np.asarray(reward, dtype=np.float64).reshape(-1).tolist()), bool(terminal))
        o = out.get(key)
        if o is None:
            o = out[key] = len(out)
        return m, o


def dyna_draws(n_updates: int, n_pairs: int, prioritized: bool):
    """The host draws of ``n_updates`` TabularModel.random_transition calls (tabular_model.py:91-113), from the reference's generators in
    its order: per update the pair (``random.randint(0, n_pairs - 1)``, or the walk fraction ``u`` of ``np.random.uniform(0, root)`` ==
    ``root * np.random.random_sample()`` from numpy's legacy global generator), then ``random.random()`` of ``random.choices``.  Returns
    (pick, u, choice)."""
    pick, u, choice = [], [], []
    for _ in range(n_updates):
        if prioritized:
            u.append(np.random.random_sample())
        else:
            pick.append(random.randint(0, n_pairs - 1))
        choice.append(random.random())
    return pick, u, choice


def _grow(t: th.Tensor, shape) -> th.Tensor:
    if tuple(t.shape) == tuple(shape):
        return t
    new = th.zeros(shape, dtype=t.dtype, device=t.device)
    new[tuple(slice(0, n) for n in t.shape)] = t
    return new


def _cap(cap: int, need: int) -> int:
    while cap < need:
        cap *= 2
    return cap


class MoqTable:
    """Device state: ``q`` f64 [S, P, A, d] (zero where a policy never visited a state), ``visited`` u8 [S, P], and with ``model`` the Dyna
    model ``pairs`` int32 [M, 3], ``outcomes`` int32 [M, K, 2], ``counts`` int64 [M, K], ``out_reward`` f64 [M, K, d] and the sum tree
    ``tree`` f64 [2^18 - 1]; ``status`` int32 [2].  Capacities double when ``reserve`` asks for more."""

    def __init__(self, A: int, d: int, device, model: bool, S: int = 64, P: int = 4, M: int = 64, K: int = 2):
        if not moq_supported(A, d):
            raise _lib.MorlB200Error(f"MoqTable: A={A}, d={d} outside the kernels' range (1 <= A <= 64, 1 <= d <= 8)")
        self.A, self.d, self.model = int(A), int(d), bool(model)
        self.q = th.zeros((S, P, A, d), dtype=th.float64, device=device)
        self.visited = th.zeros((S, P), dtype=th.uint8, device=device)
        self.status = th.zeros(2, dtype=th.int32, device=device)
        if model:
            self.pairs = th.zeros((M, 3), dtype=th.int32, device=device)
            self.outcomes = th.zeros((M, K, 2), dtype=th.int32, device=device)
            self.counts = th.zeros((M, K), dtype=th.int64, device=device)
            self.out_reward = th.zeros((M, K, d), dtype=th.float64, device=device)
            self.tree = th.zeros((1 << N_LEVELS) - 1, dtype=th.float64, device=device)

    @property
    def S(self):
        return self.q.shape[0]

    @property
    def P(self):
        return self.q.shape[1]

    def reserve(self, S: int = 0, P: int = 0, M: int = 0, K: int = 0):
        """Grow (by doubling) so that S states, P policies, M pairs and K outcomes per pair fit; values are kept."""
        S2, P2 = _cap(self.S, S), _cap(self.P, P)
        if (S2, P2) != (self.S, self.P):
            self.q = _grow(self.q, (S2, P2, self.A, self.d))
            self.visited = _grow(self.visited, (S2, P2))
        if self.model:
            M2, K2 = _cap(self.pairs.shape[0], M), _cap(self.counts.shape[1], K)
            if (M2, K2) != tuple(self.counts.shape):
                self.pairs = _grow(self.pairs, (M2, 3))
                self.outcomes = _grow(self.outcomes, (M2, K2, 2))
                self.counts = _grow(self.counts, (M2, K2))
                self.out_reward = _grow(self.out_reward, (M2, K2, self.d))

    def clear_policy(self, p: int):
        self.q[:, p] = 0
        self.visited[:, p] = 0

    def copy_policy(self, src: int, dst: int):
        """Policy dst's table becomes a copy of policy src's (the reference's deepcopy(q_table))."""
        self.q[:, dst] = self.q[:, src]
        self.visited[:, dst] = self.visited[:, src]

    def keep_policies(self, keep: Sequence[int]):
        """Compact the policy axis to the slots ``keep``, in that order; the slots after them are cleared."""
        idx = th.as_tensor(list(keep), dtype=th.long, device=self.q.device)
        n = len(keep)
        q, vis = self.q.index_select(1, idx), self.visited.index_select(1, idx)
        self.q[:, n:] = 0
        self.visited[:, n:] = 0
        self.q[:, :n] = q
        self.visited[:, :n] = vis

    def _args(self, binding: str, step: bool) -> _Args:
        a = _Args(binding)
        S, P, A, d = self.S, self.P, self.A, self.d
        a.inp(self.q, "q", (S, P, A, d), th.float64, inplace=True)
        a.inp(self.visited, "visited", (S, P), th.uint8, inplace=True)
        if step:
            a.inp(self.status, "status", (2,), th.int32, inplace=True)
            if self.model:
                M, K = self.counts.shape
                a.inp(self.pairs, "pairs", (M, 3), th.int32, inplace=True)
                a.inp(self.outcomes, "outcomes", (M, K, 2), th.int32, inplace=True)
                a.inp(self.counts, "counts", (M, K), th.int64, inplace=True)
                a.inp(self.out_reward, "out_reward", (M, K, d), th.float64, inplace=True)
                a.inp(self.tree, "tree", ((1 << N_LEVELS) - 1,), th.float64, inplace=True)
        return a


def _host(x, ctype, n: int, name: str, a: _Args):
    v = np.ascontiguousarray(np.asarray(x, dtype=np.float64 if ctype is ctypes.c_double else np.int64).reshape(-1))
    if v.shape != (n,):
        a.fail(name, f"must hold {n} values, got {v.size}")
    return (ctype * max(1, n))(*v.tolist())


def _index(a: _Args, name: str, v, lo: int, n: int) -> int:
    i = int(v)
    if not lo <= i < n:
        a.fail(name, f"= {i} is outside [{lo}, {n})")
    return i


def moq_act(t: MoqTable, n_policies: int, states, policies, w, out: Optional[th.Tensor] = None, value: Optional[th.Tensor] = None):
    """Greedy rows on the device: row i is (state id or -1, policy slot or -1 for GPI over the first ``n_policies`` slots, weights
    w[i]).  Writes ``out`` int32 [n, 2] = (action, visited) and ``value`` f64 [n] = the winning scalarised value; returns both.  One
    launch per 32 rows, no host synchronisation."""
    args = t._args("moq_act", False)
    n_policies = _index(args, "n_policies", n_policies, 1, t.P + 1)
    st = np.asarray(states, dtype=np.int64).reshape(-1)
    pol = np.asarray(policies, dtype=np.int64).reshape(-1)
    n = st.size
    for i in range(n):
        _index(args, f"states[{i}]", st[i], -1, t.S)
        _index(args, f"policies[{i}]", pol[i], -1, n_policies)
    if pol.size != n:
        args.fail("policies", f"must hold {n} values, got {pol.size}")
    out = args.out(out, "out", (n, 2), th.int32)
    value = args.out(value, "value", (n,), th.float64)
    _launch("morl_moq_act_f64", t.q, t.visited, t.S, t.P, t.A, t.d, n_policies, _host(st, ctypes.c_int, n, "states", args),
            _host(pol, ctypes.c_int, n, "policies", args), _host(w, ctypes.c_double, n * t.d, "w", args), n, out, value,
            launches=max(1, -(-n // ACT_ROWS)) if n else 0)
    return out, value


def moq_step(t: MoqTable, n_policies: int, p: int, s: int, a: int, s_next: int, terminal: bool, w, reward, flags: int, gamma: float, lr: float,
             min_priority: float = 0.0001, alpha: float = 0.6, pair: int = 0, outcome: int = 0, n_pairs: int = 0, pick=None, u=None,
             choice=None) -> None:
    """One environment step of policy slot ``p`` (csrc/moq.cu) with, under :data:`MODEL`, the real transition entered as (``pair``,
    ``outcome``) and ``len(choice)`` Dyna updates drawn by ``pick`` (uniform pair indices) or ``u`` (:data:`PRIORITIZE` walk fractions).
    One launch per 64 Dyna updates (at least one), no host synchronisation."""
    args = t._args("moq_step", True)
    n_policies = _index(args, "n_policies", n_policies, 1, t.P + 1)
    p = _index(args, "p", p, 0, n_policies)
    s = _index(args, "s", s, 0, t.S)
    a = _index(args, "a", a, 0, t.A)
    s_next = _index(args, "s_next", s_next, 0, t.S)
    if flags & ~(GPI | MODEL | PRIORITIZE) or ((flags & PRIORITIZE) and not (flags & MODEL)) or (bool(flags & MODEL) != t.model):
        args.fail("flags", f"= {flags} is not a valid combination for this table (model={t.model})")
    n_upd, M, K = 0, 1, 1
    pk = uu = ch = None
    if flags & MODEL:
        M, K = t.counts.shape
        n_pairs = _index(args, "n_pairs", n_pairs, 1, M + 1)
        pair = _index(args, "pair", pair, 0, n_pairs)
        outcome = _index(args, "outcome", outcome, 0, K)
        n_upd = 0 if choice is None else len(choice)
        ch = _host(choice, ctypes.c_double, n_upd, "choice", args) if n_upd else None
        if n_upd and flags & PRIORITIZE:
            uu = _host(u, ctypes.c_double, n_upd, "u", args)
        elif n_upd:
            pk = np.asarray(pick, dtype=np.int64).reshape(-1)
            for j in range(pk.size):
                _index(args, f"pick[{j}]", pk[j], 0, n_pairs)
            pk = _host(pk, ctypes.c_int, n_upd, "pick", args)
    m = t if t.model else None
    _launch("morl_moq_step_f64", t.q, t.visited, m and m.pairs, m and m.outcomes, m and m.counts, m and m.out_reward, m and m.tree, t.status, t.S,
            t.P, t.A, t.d, M, K, n_policies, p, s, a, s_next, int(bool(terminal)), pair, outcome, n_pairs, _host(w, ctypes.c_double, t.d, "w", args),
            _host(reward, ctypes.c_double, t.d, "reward", args), int(flags), float(gamma), float(lr), float(min_priority), float(alpha), n_upd,
            pk, uu, ch, launches=max(1, -(-n_upd // DYNA_PER_LAUNCH)))


def check_status(t: MoqTable, status=None) -> None:
    """Raise MorlB200Error if a prioritised walk landed beyond the model's pairs (the reference raises IndexError there).  ``status``: a
    host copy of ``t.status`` already made, else this copies it (one device-to-host synchronisation)."""
    st = t.status.cpu().numpy() if status is None else np.asarray(status)
    if int(st[0]) != 0:
        raise _lib.MorlB200Error(f"MOQ Dyna model: a prioritised sample walked to leaf {int(st[1])}, beyond the model's state-action pairs "
                                 "(the reference raises IndexError here)")
