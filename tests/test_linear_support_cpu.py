"""LinearSupport without a device: the float64 corner-weight oracle (tests/linear_support_oracle.py) against an independent Qhull
vertex enumeration and closed forms; the weight-selection bookkeeping against the unmodified reference class (cdd and cvxpy replaced by
the oracle); OLS's known answer; and the C ABI's argument errors."""

import random

import numpy as np
import pytest

from tests.linear_support_oracle import canonical, corners_oracle, max_value_lp_oracle


def _qhull_corners(V):
    """Vertices of the same polyhedron from scipy's HalfspaceIntersection (Qhull), in (w_1..w_{d-1}, u) with w_d = 1 - sum, capped at
    u <= U; the cap's vertices are dropped."""
    from scipy.optimize import linprog
    from scipy.spatial import HalfspaceIntersection

    V = np.round(np.asarray(V, float), 4)
    n, d = V.shape
    hs = [np.concatenate([v[:-1] - v[-1], [-1.0], [v[-1]]]) for v in V]  # v . w - u <= 0
    for j in range(d - 1):
        a = np.zeros(d + 1)
        a[j] = -1
        hs.append(a)  # w_j >= 0
    a = np.zeros(d + 1)
    a[:d - 1], a[-1] = 1, -1
    hs.append(a)  # w_d >= 0
    U = np.abs(V).max() * 10 + 10
    a = np.zeros(d + 1)
    a[d - 1], a[-1] = 1, -U
    hs.append(a)  # u <= U
    hs = np.array(hs)
    A, b = hs[:, :-1], -hs[:, -1]
    res = linprog(np.r_[np.zeros(d), -1], A_ub=np.c_[A, np.linalg.norm(A, axis=1)], b_ub=b, bounds=[(None, None)] * d + [(0, None)])
    P = HalfspaceIntersection(hs, res.x[:-1]).intersections
    P = P[P[:, -1] < U - 1e-6]
    W = np.c_[P[:, :-1], 1 - P[:, :-1].sum(1)]
    W = canonical(W)
    keep = [0] + [i for i in range(1, len(W)) if not np.allclose(W[i], W[i - 1], atol=1e-7)]
    return W[keep]


@pytest.mark.parametrize("d,n", [(2, 4), (3, 6), (3, 15), (4, 10), (5, 8)])
def test_oracle_matches_qhull(d, n):
    rng = np.random.default_rng(100 * d + n)
    for _ in range(3):
        V = rng.normal(size=(n, d)) * 10
        a, b = corners_oracle(V), _qhull_corners(V)
        assert a.shape == b.shape and np.allclose(a, b, atol=1e-7)


def test_oracle_two_objectives_is_the_line_intersections():
    """d = 2: corners are the extrema plus the crossing points of the upper envelope of the lines u = v_0 + (v_1 - v_0) t."""
    V = np.array([[0.0, 3.0], [1.0, 2.5], [2.0, 1.5], [3.0, 0.0], [0.5, 0.5]])
    got = corners_oracle(V)
    # crossings of consecutive envelope lines, as w = (1 - t, t) with t the weight on objective 1
    lines = V[:4]
    want = [np.array([0.0, 1.0]), np.array([1.0, 0.0])]
    for p, q in zip(lines[:-1], lines[1:]):
        # p . w = q . w  with w = (x, 1 - x)
        x = (q[1] - p[1]) / ((p[0] - p[1]) - (q[0] - q[1]))
        want.append(np.array([x, 1 - x]))
    assert np.allclose(got, canonical(np.array(want)), atol=1e-12)


@pytest.mark.parametrize("d", [2, 3, 5, 8])
def test_oracle_single_vector_gives_the_extrema(d):
    rng = np.random.default_rng(d)
    got = corners_oracle(rng.normal(size=(1, d)))
    assert np.array_equal(got, canonical(np.eye(d)))


def test_oracle_duplicate_and_dominated_vectors():
    """Repeated vectors and vectors that are dominated (or only weakly optimal somewhere) change nothing."""
    rng = np.random.default_rng(7)
    V = rng.normal(size=(6, 3)) * 5
    base = corners_oracle(V)
    dominated = V.min(axis=0, keepdims=True) - 1.0
    again = corners_oracle(np.vstack([V, V[:3], dominated, V[2:3]]))
    assert np.array_equal(base, again)
    ties = np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0], [0.5, 0.5, 0.0]])  # last: weakly optimal on an edge
    assert np.allclose(corners_oracle(ties), _qhull_corners(ties), atol=1e-9)


# ---------------------------------------------------------------------------------------------------- weight selection bookkeeping
class _OneStepEnv:
    """One-step environment: action a returns the value vector S[a] and terminates."""

    def __init__(self, S):
        self.S = np.asarray(S, dtype=np.float64)

    def reset(self, seed=None, options=None):
        return np.zeros(1, dtype=np.float32), {}

    def step(self, a):
        return np.zeros(1, dtype=np.float32), self.S[int(a)].copy(), True, False, {}


class _ArgmaxAgent:
    """GPI agent stand-in: picks argmax_a w . S[a] (first occurrence)."""

    gamma = 1.0

    def __init__(self, S):
        self.S = np.asarray(S, dtype=np.float64)

    def eval(self, obs, w):
        return int(np.argmax(self.S @ np.asarray(w)))

    def eval_batch(self, obs, w):
        return np.argmax(np.asarray(w) @ self.S.T, axis=1)


def _drive(ls, algo, S, iters, agent=None, env=None):
    """The weight-selection calls of GPIPD.train with an exact solver: returns the per-iteration record."""
    S = np.asarray(S, dtype=np.float64)
    solve = lambda w: S[int(np.argmax(S @ np.asarray(w)))].copy()  # noqa: E731
    trace = []
    for _ in range(iters):
        w = ls.next_weight(algo=algo, gpi_agent=agent, env=env, rep_eval=2) if algo == "gpi-ls" else ls.next_weight(algo="ols")
        trace.append((None if w is None else np.asarray(w).copy(), ls.ended()))
        if w is None:
            break
        if algo == "gpi-ls":
            M = ls.get_weight_support() + ls.get_corner_weights(top_k=4) + [w]
            for wcw in M:
                ls.add_solution(solve(wcw), wcw)
        else:
            ls.add_solution(solve(w), w)
    return trace


def _with_oracle(ls):
    ls.compute_corner_weights = lambda: list(corners_oracle(np.vstack(ls.ccs)))
    return ls


@pytest.mark.parametrize("algo", ["ols", "gpi-ls"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_weight_selection_matches_reference_class(algo, seed):
    from oracle.ref_harness import import_reference, reference_available

    if not reference_available():
        pytest.skip("reference sources not available")
    ref_mod = import_reference("morl_baselines.multi_policy.linear_support.linear_support")
    from morl_baselines_b200.multi_policy.linear_support.linear_support import LinearSupport

    rng = np.random.default_rng(seed)
    d = 2 + seed % 2
    S = np.round(rng.uniform(0, 10, size=(9, d)), 2)
    if seed == 2:
        S = np.vstack([S, S[:2], np.full((1, d), 5.0)])  # repeats and a tie-prone interior vector
    eps = 0.0 if algo == "ols" else None
    ref = ref_mod.LinearSupport(num_objectives=d, epsilon=eps, verbose=False)
    ref.compute_corner_weights = lambda: list(corners_oracle(np.vstack(ref.ccs)))
    ref.max_value_lp = lambda w_new: max_value_lp_oracle(ref.ccs, ref.visited_weights, w_new)
    mine = _with_oracle(LinearSupport(num_objectives=d, epsilon=eps, verbose=False))
    agent, env = _ArgmaxAgent(S), _OneStepEnv(S)
    random.seed(seed)
    t_ref = _drive(ref, algo, S, 12, agent, env)
    random.seed(seed)
    t_mine = _drive(mine, algo, S, 12, agent, env)
    assert len(t_ref) == len(t_mine)
    for (wr, er), (wm, em) in zip(t_ref, t_mine):
        assert er == em and (wr is None) == (wm is None)
        if wr is not None:
            assert np.array_equal(wr, wm)
    for a, b in [(ref.ccs, mine.ccs), (ref.weight_support, mine.weight_support), (ref.visited_weights, mine.visited_weights)]:
        assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
    assert ref.ended() == mine.ended()


def ccs_by_lp(S):
    """Indices of the points of S that are the unique maximiser of w . s for some w on the simplex (one LP per point)."""
    from scipy.optimize import linprog

    S = np.asarray(S, dtype=np.float64)
    n, d = S.shape
    keep = []
    for i in range(n):
        others = np.delete(S, i, axis=0)
        # max delta s.t. (others - s_i) . w + delta <= 0, sum w = 1, w >= 0
        A = np.c_[others - S[i], np.ones(n - 1)]
        res = linprog(np.r_[np.zeros(d), -1.0], A_ub=A, b_ub=np.zeros(n - 1), A_eq=np.r_[np.ones(d), 0.0][None], b_eq=[1.0],
                      bounds=[(0, None)] * d + [(None, None)], method="highs")
        if res.status == 0 and -res.fun > 1e-7:
            keep.append(i)
    return keep


def _ols_known_answer(LinearSupportCls, patch):
    for seed, (n, d) in enumerate([(8, 2), (10, 3), (12, 3), (8, 4)]):
        rng = np.random.default_rng(seed)
        S = np.round(rng.uniform(0, 10, size=(n, d)), 4)
        ls = LinearSupportCls(num_objectives=d, epsilon=0.0, verbose=False)
        if patch:
            _with_oracle(ls)
        _drive(ls, "ols", S, 200)
        assert ls.ended()
        got = np.array(sorted(map(tuple, np.asarray(ls.ccs))))
        want = np.array(sorted(map(tuple, S[ccs_by_lp(S)])))
        assert got.shape == want.shape and np.array_equal(got, want), (seed, got, want)


def test_ols_finds_the_convex_coverage_set():
    from morl_baselines_b200.multi_policy.linear_support.linear_support import LinearSupport

    _ols_known_answer(LinearSupport, patch=True)


def test_max_value_lp_unbounded_and_empty():
    from morl_baselines_b200.multi_policy.linear_support.linear_support import LinearSupport

    ls = LinearSupport(num_objectives=3, verbose=False)
    assert ls.max_value_lp(np.array([0.2, 0.3, 0.5])) == float("inf")
    ls.add_solution(np.array([1.0, 2.0, 3.0]), np.array([1.0, 0.0, 0.0]))
    assert ls.max_value_lp(np.array([0.2, 0.3, 0.5])) == float("inf")  # only one extremum visited: unbounded
    for w, v in [(np.array([0.0, 1.0, 0.0]), np.array([0.5, 4.0, 1.0])), (np.array([0.0, 0.0, 1.0]), np.array([0.0, 1.0, 5.0]))]:
        ls.add_solution(v, w)
    w = np.array([0.2, 0.3, 0.5])
    assert ls.max_value_lp(w) == pytest.approx(max_value_lp_oracle(ls.ccs, ls.visited_weights, w), rel=1e-9)
    assert ls.max_value_lp(w) == pytest.approx(0.2 * 1.0 + 0.3 * 4.0 + 0.5 * 5.0, rel=1e-9)


def test_corner_weights_argument_errors_need_no_device():
    import ctypes as C

    from morl_baselines_b200 import _lib

    lib = _lib.load()
    buf = (C.c_double * 64)()
    cnt = C.c_int(0)
    V = (C.c_double * 16)()
    assert lib.morl_corner_weights_f64(None, 4, 3, buf, 8, C.byref(cnt), None) == -1
    assert lib.morl_corner_weights_f64(V, 4, 3, None, 8, C.byref(cnt), None) == -1
    assert lib.morl_corner_weights_f64(V, 4, 3, buf, 8, None, None) == -1
    assert lib.morl_corner_weights_f64(V, 0, 3, buf, 8, C.byref(cnt), None) == -2
    assert lib.morl_corner_weights_f64(V, 4, 3, buf, -1, C.byref(cnt), None) == -2
    assert lib.morl_corner_weights_f64(V, 4, 1, buf, 8, C.byref(cnt), None) == -4
    assert lib.morl_corner_weights_f64(V, 4, 9, buf, 8, C.byref(cnt), None) == -4
    # candidate count above the documented bound 2^31: C(58, 8) = 1.9e9 is accepted by the checks, C(59, 8) = 2.5e9 is not
    assert lib.morl_corner_weights_f64(V, 51, 8, buf, 8, C.byref(cnt), None) == -4
    assert b"candidate" in lib.morl_last_error()
    assert lib.morl_corner_weights_f64(V, 105, 6, buf, 8, C.byref(cnt), None) == -4
    assert lib.morl_corner_weights_f64(V, 65535, 2, buf, 8, C.byref(cnt), None) == -4
