"""Float64 restatement of csrc/moq.cu (test infrastructure): the greedy / GPI rows and one environment step with its Dyna updates, on a host
copy of the device table (numpy arrays with the kernels' layout).  Python float operations are single IEEE float64 operations, so every
value but the priorities (libm's pow against the device's) is bit-identical to the kernels'."""

from __future__ import annotations

import math

import numpy as np

LEVELS = 18
GPI, MODEL, PRIORITIZE = 1, 2, 4


def new_table(S, P, A, d, M=0, K=0):
    return dict(q=np.zeros((S, P, A, d)), visited=np.zeros((S, P), dtype=np.uint8), pairs=np.zeros((M, 3), dtype=np.int32),
                outcomes=np.zeros((M, K, 2), dtype=np.int32), counts=np.zeros((M, K), dtype=np.int64), out_reward=np.zeros((M, K, d)),
                tree=np.zeros((1 << LEVELS) - 1), status=np.zeros(2, dtype=np.int32))


def dot(v, w) -> float:
    acc = float(v[0]) * float(w[0])
    for c in range(1, len(v)):
        acc = acc + float(v[c]) * float(w[c])
    return acc


def _better(v, i, bv, bi) -> bool:
    if math.isnan(v) or math.isnan(bv):
        return math.isnan(v) and (not math.isnan(bv) or i < bi)
    return v > bv or (v == bv and i < bi)


def greedy(T, s, p, n_pol, w):
    """(value, flat index) of the first maximum over policy p's actions (p >= 0) or every (policy, action) (p < 0)."""
    A = T["q"].shape[2]
    n = n_pol * A if p < 0 else A
    bv, bi = -math.inf, 1 << 31
    for k in range(n):
        pp, a = (k // A, k % A) if p < 0 else (p, k)
        x = dot(T["q"][s, pp, a], w) if s >= 0 and T["visited"][s, pp] else 0.0
        if _better(x, k, bv, bi):
            bv, bi = x, k
    return bv, bi


def act(T, n_pol, s, p, w):
    """(action, visited, value) of one row."""
    v, k = greedy(T, s, p, n_pol, w)
    return k % T["q"].shape[2], int(p >= 0 and s >= 0 and bool(T["visited"][s, p])), v


def _level(l):
    return (1 << l) - 1


def walk(tree, q) -> int:
    node = 0
    for l in range(1, LEVELS):
        left = tree[_level(l) + 2 * node]
        right = q > left
        node = 2 * node + int(right)
        q = q - left * (1.0 if right else 0.0)
    return node


def tree_set(tree, idx, p):
    diff = p - tree[_level(LEVELS - 1) + idx]
    for l in range(LEVELS):
        tree[_level(l) + (idx >> (LEVELS - 1 - l))] += diff


def _td(T, p, n_pol, s, a, r, s2, term, w, flags, gamma, lr, min_p, alpha, pair):
    A = T["q"].shape[2]
    T["visited"][s, p] = 1
    T["visited"][s2, p] = 1
    best, k = greedy(T, s2, -1 if flags & GPI else p, n_pol, w)
    cg = float(1 - term) * gamma
    q = T["q"]
    mq = q[s2, p, k % A].copy()
    for c in range(q.shape[3]):
        td = (float(r[c]) + cg * float(mq[c])) - float(q[s, p, a, c])
        q[s, p, a, c] = float(q[s, p, a, c]) + lr * td
    if flags & PRIORITIZE:
        best, _ = greedy(T, s2, -1, n_pol, w)
        x = abs((dot(r, w) + cg * best) - dot(q[s, p, a], w))
        tree_set(T["tree"], pair, (min_p if min_p > x else x) ** alpha)


def step(T, n_pol, p, s, a, s2, term, w, r, flags, gamma, lr, min_p=1e-4, alpha=0.6, pair=0, outcome=0, n_pairs=0, pick=(), u=(), choice=()):
    """One morl_moq_step_f64 call on the host table."""
    if T["status"][0]:
        return
    d = T["q"].shape[3]
    _td(T, p, n_pol, s, a, r, s2, term, w, flags, gamma, lr, min_p, alpha, pair)
    if not flags & MODEL:
        return
    T["pairs"][pair] = (s, a, max(int(T["pairs"][pair, 2]), outcome + 1))
    T["outcomes"][pair, outcome] = (s2, int(term))
    T["out_reward"][pair, outcome] = np.asarray(r, dtype=np.float64)[:d]
    T["counts"][pair, outcome] += 1
    for j in range(len(choice)):
        if flags & PRIORITIZE:
            m = walk(T["tree"], T["tree"][0] * u[j])
            if m >= n_pairs:
                T["status"][:] = (1, m)
                return
        else:
            m = int(pick[j])
        n = int(T["pairs"][m, 2])
        cnt = T["counts"][m, :n]
        probs = cnt / cnt.sum()
        cum, acc = [], None
        for x in probs:
            acc = float(x) if acc is None else acc + float(x)
            cum.append(acc)
        x = choice[j] * (cum[-1] + 0.0)
        o = next((i for i in range(n - 1) if cum[i] > x), n - 1)
        s_, a_ = int(T["pairs"][m, 0]), int(T["pairs"][m, 1])
        s2_, t_ = int(T["outcomes"][m, o, 0]), int(T["outcomes"][m, o, 1])
        _td(T, p, n_pol, s_, a_, T["out_reward"][m, o].copy(), s2_, t_, w, flags, gamma, lr, min_p, alpha, m)
