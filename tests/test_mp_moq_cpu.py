"""Host side of multi-policy MO Q-learning: the Dyna draw plan against the reference's TabularModel, the walk's uniform draw, the
random.choices restatement of csrc/moq.cu and tests/moq_f64.py, the host index and the construction refusals.  No GPU needed."""

import itertools
import random
from bisect import bisect_right

import numpy as np
import pytest

from morl_baselines_b200 import moq_ops
from tests import moq_f64 as f64


def test_uniform_walk_draw_is_root_times_random_sample():
    for seed in range(20):
        root = float(np.random.default_rng(seed).random() * 1e3)
        np.random.seed(seed)
        a = np.random.uniform(0, root, size=1)[0]
        np.random.seed(seed)
        b = root * np.random.random_sample()
        assert a.tobytes() == np.float64(b).tobytes()
        assert np.random.random_sample() == (np.random.seed(seed), np.random.uniform(0, root, size=1), np.random.random_sample())[2]


def _choice_index(counts, r):
    """The kernels' outcome choice: weights counts / counts.sum(), accumulate, then the first cum > r * total among the first n - 1."""
    probs = np.asarray(counts, dtype=np.int64) / np.asarray(counts, dtype=np.int64).sum()
    cum = list(itertools.accumulate(probs))
    x = r * (cum[-1] + 0.0)
    return next((i for i in range(len(cum) - 1) if cum[i] > x), len(cum) - 1)


def test_outcome_choice_equals_random_choices():
    rng = np.random.default_rng(0)
    for trial in range(2000):
        counts = rng.integers(1, 9, int(rng.integers(1, 7)))
        random.seed(trial)
        want = random.choices(range(len(counts)), weights=counts / counts.sum(), k=1)[0]
        random.seed(trial)
        assert _choice_index(counts, random.random()) == want
        probs = counts / counts.sum()
        cum = list(itertools.accumulate(probs))
        random.seed(trial)
        assert bisect_right(cum, random.random() * (cum[-1] + 0.0), 0, len(cum) - 1) == want


@pytest.mark.parametrize("prioritized", [False, True])
def test_draw_plan_consumes_the_reference_generators(prioritized):
    from oracle.ref_harness import import_reference, reference_available

    if not reference_available():
        pytest.skip("reference sources not available")
    tm = import_reference("morl_baselines.common.model_based.tabular_model")
    model = tm.TabularModel(prioritize=prioritized)
    rng = np.random.default_rng(1)
    for i in range(7):
        for k in range(int(rng.integers(1, 4))):
            model.update((i, 0), 1, np.array([float(k), 1.0]), (i + 1, 0), False, float(rng.random() + 0.1) if prioritized else None)
    n = len(model.state_actions_pairs)
    random.seed(5)
    np.random.seed(5)
    want = []
    for _ in range(9):
        t = model.random_transition()
        want.append((model.state_actions_pairs.index((t[0], t[1])) if not prioritized else t[5], t[3]))
    st_py, st_np = random.getstate(), np.random.get_state()[1].copy()
    random.seed(5)
    np.random.seed(5)
    pick, u, choice = moq_ops.dyna_draws(9, n, prioritized)
    assert random.getstate() == st_py and np.array_equal(np.random.get_state()[1], st_np)
    leaves = model.priorities.nodes if prioritized else None
    for j, (m_want, s2_want) in enumerate(want):
        if prioritized:
            tree = np.concatenate(leaves)
            m = f64.walk(tree, tree[0] * u[j])
        else:
            m = pick[j]
        assert m == m_want
        outs = list(model.model[model.state_actions_pairs[m]].items())
        o = _choice_index([c for _, c in outs], choice[j])
        assert outs[o][0][0] == s2_want


def test_index_keys_in_reference_order():
    idx = moq_ops.MoqIndex()
    s0, s1 = idx.add_state(np.array([0, 0], dtype=np.int32)), idx.add_state(np.array([0, 1], dtype=np.int32))
    assert (s0, s1) == (0, 1) and idx.add_state((0, 0)) == 0 and idx.find(np.array([3, 3])) == -1
    assert idx.add_outcome(0, 2, 1, np.array([1.5, -1.0], dtype=np.float32), False) == (0, 0)
    assert idx.add_outcome(0, 2, 1, np.array([1.5, -1.0], dtype=np.float32), np.bool_(False)) == (0, 0)
    assert idx.add_outcome(0, 2, 1, np.array([1.5, -1.0], dtype=np.float32), True) == (0, 1)
    assert idx.add_outcome(1, 2, 1, np.array([1.5, -1.0]), True) == (1, 0)
    assert idx.pairs == [(0, 2), (1, 2)] and moq_ops.state_key(np.int64(4)) == (4,)


def test_refusals_without_cuda():
    import torch as th

    from morl_baselines_b200._lib import MorlB200Error
    from morl_baselines_b200.multi_policy.multi_policy_moqlearning.mp_mo_q_learning import MPMOQLearning
    from tests.pql_standin import TreasureGrid

    if th.cuda.is_available():
        pytest.skip("checks the CPU-only refusal")
    with pytest.raises(MorlB200Error, match="needs a CUDA device"):
        MPMOQLearning(TreasureGrid(d=2), log=False)
