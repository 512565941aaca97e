"""Float64 numpy restatement of the reference PQL's per-step functions (multi_policy/pareto_q_learning/pql.py) on the device layout of
csrc/pql.cu: the oracle of the kernel tests.

A table is a dict of numpy arrays: ``nd`` [S, A, K, d], ``nd_count`` int32 [S, A], ``avg_reward`` [S, A, d], ``counts`` [S, A].  Every
operation is the reference's numpy expression, so the stored sets and averages are the reference's bit for bit; the sets are kept in the
canonical order (descending coordinate sum added left to right, ties lexicographically descending)."""

from __future__ import annotations

import numpy as np

from tests.hv_f64 import hv_max


def new_table(S, A, K, d):
    return dict(nd=np.zeros((S, A, K, d)), nd_count=np.ones((S, A), dtype=np.int32), avg_reward=np.zeros((S, A, d)), counts=np.zeros((S, A)))


def q_set(t, s, a, gamma) -> np.ndarray:
    """Q-set(s, a) rows in stored order: ``avg_reward[s, a] + gamma * ND[s][a]`` (pql.py:166-167)."""
    return t["avg_reward"][s, a] + gamma * t["nd"][s, a, : t["nd_count"][s, a]]


def prune(pts: np.ndarray) -> np.ndarray:
    """Keep mask: no distinct point is >= the point in every coordinate, and it is the first copy of its value."""
    ge = np.all(pts[None, :, :] >= pts[:, None, :], axis=-1)  # [i, j]: j >= i everywhere
    eq = np.all(pts[None, :, :] == pts[:, None, :], axis=-1)
    earlier = np.tril(np.ones((len(pts), len(pts)), dtype=bool), -1)  # j < i
    return ~np.any((ge & ~eq) | (eq & earlier), axis=1)


def coord_sum(pts: np.ndarray) -> np.ndarray:
    acc = pts[:, 0].copy()
    for c in range(1, pts.shape[1]):
        acc = acc + pts[:, c]
    return acc


def canonical(pts: np.ndarray) -> np.ndarray:
    """Distinct points in canonical order."""
    pts = np.asarray(pts, dtype=np.float64).reshape(len(pts), -1)
    keys = [tuple([float(sm)] + p) for sm, p in zip(coord_sum(pts), pts.tolist())]
    order = sorted(range(len(pts)), key=lambda i: keys[i], reverse=True)
    return pts[order]


def union(t, s, gamma) -> np.ndarray:
    return np.concatenate([q_set(t, s, a, gamma) for a in range(t["nd"].shape[1])])


def update(t, s, a, s_next, reward, gamma):
    """One reference step (pql.py:260-262) in place.  Returns None, or the needed size when more than K points survive (then nothing is
    written)."""
    u = union(t, s_next, gamma)
    front = canonical(u[prune(u)])
    K = t["nd"].shape[2]
    if len(front) > K:
        return len(front)
    t["counts"][s, a] += 1
    t["nd"][s, a, : len(front)] = front
    t["nd_count"][s, a] = len(front)
    t["avg_reward"][s, a] += (np.asarray(reward, dtype=np.float64) - t["avg_reward"][s, a]) / t["counts"][s, a]
    return None


def score_hypervolume(t, s, gamma, ref) -> np.ndarray:
    return np.array([hv_max(q_set(t, s, a, gamma), ref) for a in range(t["nd"].shape[1])])


def score_cardinality(t, s, gamma) -> np.ndarray:
    """pql.py:131-141: the points of ND(union) that are equal to a point of each action's Q-set."""
    A = t["nd"].shape[1]
    u = union(t, s, gamma)
    front = u[prune(u)]
    out = np.zeros(A)
    for a in range(A):
        qs = q_set(t, s, a, gamma)
        out[a] = sum(bool(np.any(np.all(qs == p, axis=1))) for p in front)
    return out


def as_sets(t) -> list:
    S, A = t["nd_count"].shape
    return [[{tuple(v) for v in t["nd"][s, a, : t["nd_count"][s, a]].tolist()} for a in range(A)] for s in range(S)]
