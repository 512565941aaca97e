"""Float64 numpy restatement of the corner-weight enumeration of csrc/linear_support.cu and of LinearSupport's optimistic-bound LP
(test and benchmark infrastructure; the product path runs the kernel and scipy's linprog).

corners_oracle(V) enumerates every d-subset S of the n value rows (v_i . w <= u) and d non-negativity rows (w_j >= 0) with itertools,
eliminates u through the first value row of S, solves the d x d system with np.linalg.solve (a batch per chunk), keeps the feasible
solutions with the kernel's tolerances, and merges solutions that agree to 1e-7 (a degenerate vertex is reached from several subsets).
It does not use the kernel's lexicographic-basis rule, so the two de-duplications are independent.  The output goes through the same
canonical post-processing (|w| / sum |w|, snap to 0 within 1e-9, lexicographic order on values rounded to 1e-9)."""

from __future__ import annotations

import itertools
from math import comb

import numpy as np

W_TOL, V_TOL, RANK_TOL = 1e-9, 1e-9, 1e-11


def canonical(w: np.ndarray) -> np.ndarray:
    w = np.abs(np.asarray(w, dtype=np.float64))
    if w.shape[0] == 0:
        return w.reshape(0, w.shape[1] if w.ndim == 2 else 0)
    w = w / w.sum(axis=1, keepdims=True)
    w[w <= 1e-9] = 0.0
    return w[np.lexsort(np.round(w, 9).T[::-1])]


def vertices_oracle(V, chunk: int = 200_000) -> np.ndarray:
    """All vertices (w, u) [K, d+1] of { V w <= u, w >= 0, sum w = 1 } for V [n, d] (already rounded), unordered, duplicates merged."""
    V = np.asarray(V, dtype=np.float64)
    n, d = V.shape
    scale = max(1.0, float(np.abs(V).max()))
    basis = np.vstack([V, np.eye(d)])  # row r < n: v_r (minus v_i0 below); row n + j: e_j
    out = []
    it = itertools.combinations(range(n + d), d)
    while True:
        S = np.array(list(itertools.islice(it, chunk)), dtype=np.int64).reshape(-1, d)
        if S.shape[0] == 0:
            break
        S = S[S[:, 0] < n]  # a subset without a value row leaves u free
        if S.shape[0] == 0:
            continue
        i0 = S[:, 0]
        A = np.empty((S.shape[0], d, d))
        A[:, 0, :] = 1.0
        rows = basis[S[:, 1:]]  # [C, d-1, d]
        rows = np.where((S[:, 1:] < n)[:, :, None], rows - V[i0][:, None, :], rows)
        A[:, 1:, :] = rows
        sv = np.linalg.svd(A, compute_uv=False)
        ok = sv[:, -1] > RANK_TOL * scale
        A, i0 = A[ok], i0[ok]
        if A.shape[0] == 0:
            continue
        rhs = np.zeros((A.shape[0], d, 1))
        rhs[:, 0, 0] = 1.0
        w = np.linalg.solve(A, rhs)[:, :, 0]
        u = np.einsum("cj,cj->c", V[i0], w)
        ok = (w >= -W_TOL).all(axis=1) & ((w @ V.T) <= u[:, None] + V_TOL * scale).all(axis=1)
        if ok.any():
            out.append(np.c_[w[ok], u[ok]])
    if not out:
        return np.zeros((0, d + 1))
    X = np.vstack(out)
    _, first = np.unique(np.round(X[:, :d], 7), axis=0, return_index=True)
    return X[np.sort(first)]


def corners_oracle(V) -> np.ndarray:
    """Corner weights of the value vectors V [n, d] as LinearSupport.compute_corner_weights returns them (rows of one array)."""
    V = np.round(np.asarray(V, dtype=np.float64), 4)
    return canonical(vertices_oracle(V)[:, :-1])


def candidate_count(n: int, d: int) -> int:
    return comb(n + d, d)


def max_value_lp_oracle(ccs, visited_weights, w_new) -> float:
    """OLS's optimistic bound: max w_new . v s.t. W v <= V (v free), V_i = max_{c in ccs} c . W_i; +inf when unbounded or ccs is empty."""
    from scipy.optimize import linprog

    if len(ccs) == 0:
        return float("inf")
    W = np.vstack(visited_weights).astype(np.float64)
    Vb = np.array([max(np.dot(c, w) for c in ccs) for w in visited_weights], dtype=np.float64)
    res = linprog(-np.asarray(w_new, dtype=np.float64), A_ub=W, b_ub=Vb, bounds=[(None, None)] * W.shape[1], method="highs")
    if res.status == 3:
        return float("inf")
    assert res.status == 0, res.message
    return float(-res.fun)
