"""Pareto Q-learning on the device (csrc/pql.cu, pql_ops, multi_policy/pareto_q_learning): the reference's golden runs reproduced, the
kernels against the float64 restatement of tests/pql_f64.py, the overflow rule, the argument checks and the reference's test scenario.

Stored sets, counts and averages must match bit for bit.  Hypervolume scores may differ from the host sweep in the last bits (the slabs are
added in another order): relative 1e-12.  Cardinality scores are exact."""

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import _lib, ops, pql_ops
from morl_baselines_b200.multi_policy.pareto_q_learning.pql import PQL
from tests import pql_f64 as f64
from tests.pql_standin import CASES, TreasureGrid, run_case

pytestmark = pytest.mark.gpu
REL = 1e-12


def _golden():
    import os

    return np.load(os.path.join(os.path.dirname(__file__), "golden", "pql.npz"), allow_pickle=False)


def _scores_close(got, want):
    np.testing.assert_allclose(got, want, rtol=REL, atol=0.0)


@pytest.mark.parametrize("name", list(CASES))
def test_golden_case(cuda, name):
    g = {k.split("/", 1)[1]: g_ for k, g_ in _golden().items() if k.startswith(name + "/")}
    _, rec = run_case(name, PQL, int(g["seed"][0]))
    np.testing.assert_array_equal(rec["actions"], g["actions"])
    np.testing.assert_array_equal(rec["greedy_step"], g["greedy_step"])
    np.testing.assert_array_equal(rec["greedy_state"], g["greedy_state"])
    if CASES[name]["action_eval"] == "hypervolume":
        _scores_close(rec["greedy_scores"], g["greedy_scores"])
    else:
        np.testing.assert_array_equal(rec["greedy_scores"], g["greedy_scores"])
    np.testing.assert_array_equal(rec["epsilon"], g["epsilon"])
    assert rec["counts"].tobytes() == g["counts"].tobytes()
    assert rec["avg_reward"].tobytes() == g["avg_reward"].tobytes()
    np.testing.assert_array_equal(rec["nd_count"], g["nd_count"])
    S, A = g["nd_count"].shape
    for s in range(S):
        for a in range(A):
            n = g["nd_count"][s, a]
            assert {tuple(v) for v in rec["nd"][s, a, :n].tolist()} == {tuple(v) for v in g["nd"][s, a, :n].tolist()}, (s, a)
    np.testing.assert_array_equal(rec["pcs"], g["pcs"])
    np.testing.assert_array_equal(rec["tracked"], g["tracked"])


# ---- kernels against tests/pql_f64.py ------------------------------------------------------------------------------------------------------
def _upload(t, host, dev):
    for k in ("nd", "nd_count", "avg_reward", "counts"):
        getattr(t, k).copy_(th.from_numpy(host[k]).to(dev))


def _assert_table(t, host):
    cnt = t.nd_count.cpu().numpy()
    np.testing.assert_array_equal(cnt, host["nd_count"])
    nd = t.nd.cpu().numpy()
    S, A = cnt.shape
    for s in range(S):
        for a in range(A):  # canonical order on both sides: the valid rows are equal bytes
            assert nd[s, a, : cnt[s, a]].tobytes() == host["nd"][s, a, : cnt[s, a]].tobytes(), (s, a)
    assert t.avg_reward.cpu().numpy().tobytes() == host["avg_reward"].tobytes()
    assert t.counts.cpu().numpy().tobytes() == host["counts"].tobytes()


def _check_scores(t, host, s, gamma, ref, hv: bool):
    card = pql_ops.pql_score(t, s, pql_ops.CARDINALITY, gamma).cpu().numpy()
    np.testing.assert_array_equal(card, f64.score_cardinality(host, s, gamma))
    if hv:
        _scores_close(pql_ops.pql_score(t, s, pql_ops.HYPERVOLUME, gamma, ref).cpu().numpy(), f64.score_hypervolume(host, s, gamma, ref))


@pytest.mark.parametrize("gamma", [1.0, 0.99, 0.8])
@pytest.mark.parametrize("d", [1, 2, 3, 4, 6, 8])
@pytest.mark.parametrize("A", [1, 2, 4, 8, 16])
def test_kernels_match_f64(cuda, A, d, gamma):
    """Random steps on a small table, rewards on a coarse grid (duplicates within and across actions, points dominated only by another
    action's, points at and below ref), s' == s every few steps, each step's written state and next state scored.  A step whose set
    overflows must set status and leave the table as it was, on both sides."""
    rng = np.random.default_rng(1000 * A + 10 * d + int(100 * gamma))
    S, K = 4, 64 if A == 16 else 128
    dev = th.device("cuda")
    host = f64.new_table(S, A, K, d)
    t = pql_ops.PqlTable(S, A, K, d, dev)
    ref = np.full(d, -0.5)
    hv = d <= 4
    for step in range(40):
        s, a = int(rng.integers(S)), int(rng.integers(A))
        s2 = s if step % 4 == 0 else int(rng.integers(S))
        r = rng.integers(-2, 3, d) / 2
        need = f64.update(host, s, a, s2, r, gamma)
        pql_ops.pql_update(t, s, a, s2, r, gamma)
        st = t.status.cpu().numpy()
        if need is None:
            assert st[0] == 0
        else:
            assert list(st) == [need, s, a]
            with pytest.raises(_lib.MorlB200Error, match=f"state {s}, action {a} needs {need} points"):
                pql_ops.check_status(t)
            t.status.zero_()
        _assert_table(t, host)
        _check_scores(t, host, s, gamma, ref, hv)
        _check_scores(t, host, s2, gamma, ref, hv)


def _front(n, d, shift=0.0):
    """n distinct mutually non-dominated points (on the plane x0 + x1 = n - 1)."""
    p = np.zeros((n, d))
    p[:, 0] = np.arange(n) + shift
    if d > 1:
        p[:, 1] = n - 1 - np.arange(n) - shift
    return p


@pytest.mark.parametrize("A,K,d", [(8, 256, 4), (16, 64, 4), (16, 128, 2), (2, 64, 8)])
def test_exactly_K_points_pass_and_K_plus_1_overflow(cuda, A, K, d):
    dev = th.device("cuda")
    S = 3
    host = f64.new_table(S, A, K, d)
    # state 1: action 0 stores K non-dominated points; state 2: the same K plus one more in action A - 1
    host["nd"][1, 0, :K] = _front(K, d)
    host["nd_count"][1, 0] = K
    host["nd"][2, 0, :K] = _front(K, d)
    host["nd_count"][2, 0] = K
    host["nd"][2, A - 1, 0] = _front(1, d, shift=K)[0]  # (K, -K, 0, ...): beyond the plane's end, non-dominated
    host["nd_count"][2, A - 1] = 1
    t = pql_ops.PqlTable(S, A, K, d, dev)
    _upload(t, host, dev)
    r = np.ones(d) * 0.25
    assert f64.update(host, 0, 1, 1, r, 1.0) is None
    pql_ops.pql_update(t, 0, 1, 1, r, 1.0)
    pql_ops.check_status(t)
    assert int(t.nd_count[0, 1]) == K
    _assert_table(t, host)
    before = {k: getattr(t, k).clone() for k in ("nd", "nd_count", "avg_reward", "counts")}
    assert f64.update(host, 0, 1, 2, r, 1.0) == K + 1
    pql_ops.pql_update(t, 0, 1, 2, r, 1.0)
    assert t.status.cpu().tolist() == [K + 1, 0, 1]
    for k, v in before.items():
        assert th.equal(getattr(t, k), v), k
    with pytest.raises(_lib.MorlB200Error, match=f"max_set_size={K}: raise max_set_size to at least {K + 1}"):
        pql_ops.check_status(t)


def test_agent_raises_on_overflow(cuda):
    env = TreasureGrid(d=2, seed=0)
    agent = PQL(env, np.array([0.0, -25.0]), gamma=1.0, seed=3, log=False, epsilon_decay_steps=500, max_set_size=1)
    with pytest.raises(_lib.MorlB200Error, match="raise max_set_size to at least"):
        agent.train(total_timesteps=3000, eval_env=TreasureGrid(d=2, seed=1), action_eval="hypervolume")


@pytest.mark.parametrize("d", [2, 3, 4])
def test_equal_sets_give_equal_scores(cuda, d):
    rng = np.random.default_rng(d)
    A, K, S = 6, 64, 2
    dev = th.device("cuda")
    host = f64.new_table(S, A, K, d)
    pts = f64.canonical(rng.standard_normal((40, d)) + 3.0)
    pts = pts[f64.prune(pts)]
    for a in (1, 4):
        host["nd"][0, a, : len(pts)] = pts
        host["nd_count"][0, a] = len(pts)
        host["avg_reward"][0, a] = np.linspace(0.1, 0.7, d)
    t = pql_ops.PqlTable(S, A, K, d, dev)
    _upload(t, host, dev)
    for gamma in (1.0, 0.99, 0.8):
        sc = pql_ops.pql_score(t, 0, pql_ops.HYPERVOLUME, gamma, np.zeros(d)).cpu().numpy()
        assert sc[1].tobytes() == sc[4].tobytes() and sc[1] > 0
        _scores_close(sc, f64.score_hypervolume(host, 0, gamma, np.zeros(d)))


def test_argument_errors_raise_before_launch(cuda):
    dev = th.device("cuda")
    t = pql_ops.PqlTable(5, 4, 16, 2, dev)
    n0 = ops.launch_count
    for args, name in [((5, 0, 0), "s"), ((-1, 0, 0), "s"), ((0, 4, 0), "a"), ((0, -1, 0), "a"), ((0, 0, 5), "s_next")]:
        with pytest.raises(_lib.MorlB200Error, match=f"pql_update: {name} = "):
            pql_ops.pql_update(t, *args, np.zeros(2), 0.9)
    with pytest.raises(_lib.MorlB200Error, match="reward must hold 2 values"):
        pql_ops.pql_update(t, 0, 0, 0, np.zeros(3), 0.9)
    with pytest.raises(_lib.MorlB200Error, match="pql_score: state = 5"):
        pql_ops.pql_score(t, 5, pql_ops.CARDINALITY, 0.9)
    with pytest.raises(_lib.MorlB200Error, match="pql_score: mode"):
        pql_ops.pql_score(t, 0, 7, 0.9)
    t5 = pql_ops.PqlTable(2, 4, 16, 5, dev)
    with pytest.raises(_lib.MorlB200Error, match="hypervolume scores need d <= 4"):
        pql_ops.pql_score(t5, 0, pql_ops.HYPERVOLUME, 0.9, np.zeros(5))
    for S, A, K, d in [(2, 17, 16, 2), (2, 16, 256, 2), (2, 4, 257, 2), (2, 4, 16, 9), (0, 4, 16, 2)]:
        with pytest.raises(_lib.MorlB200Error, match="outside the kernels' range"):
            pql_ops.PqlTable(S, A, K, d, dev)
    assert ops.launch_count == n0
    env = TreasureGrid(d=2)
    agent = PQL(env, np.zeros(2), log=False, seed=0)
    with pytest.raises(_lib.MorlB200Error, match="pql_score: state = 42"):
        agent.score_hypervolume(42)
    assert ops.launch_count == n0


def test_reference_test_pql_scenario(cuda):
    """The reference's test_pql (tests/test_algos.py) on the stand-in: gamma 1, 1,000 steps, hypervolume scores."""
    env = TreasureGrid(d=2, seed=0)
    ref_point = np.array([0, -25])
    agent = PQL(env, ref_point, gamma=1.0, initial_epsilon=1.0, epsilon_decay_steps=5000, final_epsilon=0.2, seed=1, log=False)
    pf = agent.train(total_timesteps=1000, log_every=100, action_eval="hypervolume", ref_point=ref_point, eval_env=env)
    assert len(pf) > 0
    target = np.array(pf.pop())
    tracked = agent.track_policy(target, env=env)
    assert np.all(tracked == target)
