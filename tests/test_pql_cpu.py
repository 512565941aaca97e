"""CPU checks of Pareto Q-learning: the state index and space classification against the reference's, the float64 restatement of
tests/pql_f64.py against the reference's per-step functions, and the kernels' supported range (no device needed)."""

import numpy as np
import pytest

from morl_baselines_b200 import pql_ops
from morl_baselines_b200.multi_policy.pareto_q_learning.pql import PQL
from morl_baselines_b200.testing import Box, Discrete, MultiBinary, MultiDiscrete
from oracle import ref_harness as rh
from tests import pql_f64 as f64

needs_ref = pytest.mark.skipif(not rh.reference_available(), reason="reference not mounted")


class _Env:
    def __init__(self, obs, act=None, d=2):
        self.observation_space, self.action_space = obs, act or Discrete(4)
        self.reward_space = Box(-np.inf, np.inf, shape=(d,))
        self.unwrapped = self


def _bare(env):
    """A PQL with only the space classification of its constructor run (no device)."""
    agent = PQL.__new__(PQL)
    agent.env = env
    PQL._classify_spaces(agent)
    return agent


def _ref_pql():
    rh.install_stubs()
    import sys

    sys.modules["gymnasium.spaces"].MultiDiscrete = MultiDiscrete
    return rh.import_reference("morl_baselines.multi_policy.pareto_q_learning.pql").PQL


SPACES = {
    "discrete": (Discrete(9), [3, np.int64(7), np.int32(0)]),
    "multidiscrete": (MultiDiscrete([3, 4]), [np.array([2, 3]), np.array([0, 1])]),
    "box": (Box(low=np.zeros(2), high=np.array([5, 6]), dtype=np.dtype(np.int32)), [np.array([5, 6], dtype=np.int32), np.array([0, 3])]),
    "box_low1": (Box(low=np.ones(2), high=np.array([4, 4]), dtype=np.dtype(np.int64)), [np.array([1, 1]), np.array([3, 2])]),
}


@pytest.mark.parametrize("kind", list(SPACES))
def test_state_index_matches_reference(kind):
    space, states = SPACES[kind]
    mine = _bare(_Env(space))
    expect_shape = {"discrete": (9,), "multidiscrete": (3, 4), "box": (6, 7), "box_low1": (4, 4)}[kind]
    assert tuple(np.asarray(mine.env_shape).tolist()) == expect_shape
    assert mine.num_states == int(np.prod(expect_shape)) and mine.num_actions == 4
    if rh.reference_available():
        ref = _ref_pql().__new__(_ref_pql())
        ref.env_shape = mine.env_shape
        for st in states:
            assert mine._get_state_index(st) == ref._get_state_index(st)
    for st in states:
        idx = mine._get_state_index(st)
        assert isinstance(idx, int)
        assert idx == (int(st) if np.ndim(st) == 0 else int(np.ravel_multi_index(st, expect_shape)))


def test_multidiscrete_actions():
    assert _bare(_Env(Discrete(5), MultiDiscrete([2, 3]))).num_actions == 6


@pytest.mark.parametrize("obs,act", [(Box(-1.0, 1.0, shape=(2,)), None), (MultiBinary(3), None),
                                     (Discrete(4), Box(-1.0, 1.0, shape=(2,))), (Discrete(4), MultiBinary(3))])
def test_unsupported_spaces_raise(obs, act):
    with pytest.raises(Exception, match="PQL only supports"):
        _bare(_Env(obs, act))


def _random_table(rng, S, A, K, d, gamma):
    """A table reached by reference steps from the initial one, with rewards on a coarse grid so duplicates and cross-action dominance
    occur."""
    t = f64.new_table(S, A, K, d)
    for _ in range(3 * S * A):
        s, a, s2 = int(rng.integers(S)), int(rng.integers(A)), int(rng.integers(S))
        assert f64.update(t, s, a, s2, rng.integers(-3, 4, d) / 2, gamma) is None
    return t


@needs_ref
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("gamma", [1.0, 0.8])
def test_f64_restatement_matches_reference(d, gamma):
    """get_q_set, calc_non_dominated, both scores and the update of the reference, on the same random tables."""
    rng = np.random.default_rng(d * 10 + int(gamma * 10))
    S, A, K = 5, 3, 256
    t = _random_table(rng, S, A, K, d, gamma)
    Ref = _ref_pql()
    ref = Ref.__new__(Ref)
    ref.gamma, ref.num_actions, ref.ref_point = gamma, A, np.full(d, -4.0)
    ref.non_dominated, ref.avg_reward, ref.counts = f64.as_sets(t), t["avg_reward"].copy(), t["counts"].copy()
    for s in range(S):
        for a in range(A):
            assert ref.get_q_set(s, a) == {tuple(v) for v in f64.q_set(t, s, a, gamma).tolist()}
        u = f64.union(t, s, gamma)
        assert ref.calc_non_dominated(s) == {tuple(v) for v in u[f64.prune(u)].tolist()}
        np.testing.assert_array_equal(np.asarray(ref.score_pareto_cardinality(s)), f64.score_cardinality(t, s, gamma))
        np.testing.assert_allclose(np.asarray(ref.score_hypervolume(s)), f64.score_hypervolume(t, s, gamma, ref.ref_point), rtol=1e-12)
    for _ in range(20):  # the reference's update (pql.py:260-262) against f64.update, bit for bit
        s, a, s2 = int(rng.integers(S)), int(rng.integers(A)), int(rng.integers(S))
        r = rng.integers(-3, 4, d) / 2
        ref.counts[s, a] += 1
        ref.non_dominated[s][a] = ref.calc_non_dominated(s2)
        ref.avg_reward[s, a] += (r - ref.avg_reward[s, a]) / ref.counts[s, a]
        f64.update(t, s, a, s2, r, gamma)
        assert ref.non_dominated == f64.as_sets(t)
        assert np.array_equal(ref.avg_reward, t["avg_reward"]) and np.array_equal(ref.counts, t["counts"])


@pytest.mark.parametrize("A,K,d,mode,ok", [
    (8, 256, 4, pql_ops.HYPERVOLUME, True), (16, 64, 4, pql_ops.HYPERVOLUME, True), (16, 128, 4, pql_ops.HYPERVOLUME, True),
    (1, 1, 1, pql_ops.HYPERVOLUME, True), (4, 64, 5, pql_ops.HYPERVOLUME, False), (4, 64, 8, pql_ops.CARDINALITY, True),
    (4, 64, 9, pql_ops.CARDINALITY, False), (17, 64, 2, pql_ops.CARDINALITY, False), (8, 257, 2, pql_ops.CARDINALITY, False),
    (16, 256, 2, pql_ops.CARDINALITY, False), (0, 64, 2, pql_ops.CARDINALITY, False), (4, 0, 2, pql_ops.HYPERVOLUME, False),
    (4, 64, 0, pql_ops.CARDINALITY, False), (4, 64, 2, 2, False),
])
def test_supported_range(A, K, d, mode, ok):
    assert pql_ops.pql_supported(A, K, d, mode) is ok
