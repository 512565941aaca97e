"""Multi-policy MO Q-learning on the device (csrc/moq.cu, moq_ops, multi_policy/multi_policy_moqlearning): the reference's golden runs
reproduced, both kernels against the float64 restatement of tests/moq_f64.py, eval_batch, growth, policy deletion and the launch budget.

Actions, Q tables, ε, policy counts, the CCS and the model's keys and counts must match exactly.  Tree leaves carry priorities raised to
alpha by the device's pow, not glibc's: relative 1e-12.  Against the reference, a leaf's priority r.w + γ max - q.w also inherits numpy's
dot rounding (not the device's left-to-right adds), which the subtraction can magnify: a few ulps of terms of magnitude <= 20 times the
slope 0.6 x^-0.4 <= 24 of x^0.6 above min_priority = 1e-4, so absolute 1e-13 on top."""

import os

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import _lib, moq_ops, ops
from morl_baselines_b200.multi_policy.multi_policy_moqlearning.mp_mo_q_learning import MPMOQLearning
from tests import moq_f64 as f64
from tests.mp_moq_cases import CASES, device_model_view, run_case
from tests.pql_standin import TreasureGrid

pytestmark = pytest.mark.gpu
REL = 1e-12


def _golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "mp_moq.npz"), allow_pickle=False)


@pytest.mark.parametrize("name", list(CASES))
def test_golden_case(cuda, name):
    g = {k.split("/", 1)[1]: v for k, v in _golden().items() if k.startswith(name + "/")}
    _, rec = run_case(name, MPMOQLearning, int(g["seed"][0]), device_model_view)
    assert sorted(rec) == sorted(g)
    for k in sorted(g):
        if k.endswith("/leaves"):
            np.testing.assert_allclose(rec[k], g[k], rtol=REL, atol=1e-13, err_msg=k)
        else:
            assert rec[k].shape == g[k].shape and rec[k].tobytes() == g[k].astype(rec[k].dtype).tobytes(), k


# ---- kernels against tests/moq_f64.py --------------------------------------------------------------------------------------------------
def _upload(t, T):
    for k in ("q", "visited", "status") + (("pairs", "outcomes", "counts", "out_reward", "tree") if t.model else ()):
        getattr(t, k).copy_(th.from_numpy(T[k]))


def _assert_equal(t, T, tree_rel=False):
    for k in ("q", "visited", "status") + (("pairs", "outcomes", "counts", "out_reward") if t.model else ()):
        assert getattr(t, k).cpu().numpy().tobytes() == T[k].tobytes(), k
    if t.model:
        np.testing.assert_allclose(t.tree.cpu().numpy(), T["tree"], rtol=REL, atol=0.0)


def _random_table(rng, S, P, A, d, M, K, ties):
    T = f64.new_table(S, P, A, d, M, K)
    T["visited"][:] = rng.random((S, P)) < 0.6
    vals = rng.integers(-3, 4, (S, P, A, d)) / 4 if ties else rng.standard_normal((S, P, A, d))
    T["q"][:] = vals * T["visited"][:, :, None, None]
    return T


def _random_model(rng, T, n_pairs, A, d, K, prioritized):
    S = T["q"].shape[0]
    for m in range(n_pairs):
        n = int(rng.integers(1, K + 1))
        T["pairs"][m] = (int(rng.integers(S)), int(rng.integers(A)), n)
        for o in range(n):
            T["outcomes"][m, o] = (int(rng.integers(S)), int(rng.random() < 0.2))
            T["out_reward"][m, o] = rng.standard_normal(d)
            T["counts"][m, o] = int(rng.integers(1, 5))
        if prioritized:
            f64.tree_set(T["tree"], m, float(rng.random() + 0.01))


AXES = [  # P, A, d, dyna, prioritised, gpi, ties
    (1, 1, 1, 0, False, False, False), (1, 4, 2, 5, False, False, True), (3, 4, 3, 5, True, True, False), (8, 16, 8, 64, True, True, True),
    (64, 16, 4, 7, False, True, False), (64, 2, 1, 0, False, True, True), (17, 5, 8, 65, True, False, False), (5, 16, 6, 130, False, True, True),
]


@pytest.mark.parametrize("P,A,d,dyna,prio,gpi,ties", AXES)
def test_kernels_match_f64(cuda, P, A, d, dyna, prio, gpi, ties):
    rng = np.random.default_rng(P * 1000 + A * 10 + d)
    S, M, K = 9, 12, 3
    model = dyna > 0 or prio
    T = _random_table(rng, S, P, A, d, M if model else 0, K, ties)
    t = moq_ops.MoqTable(A, d, "cuda", model, S=S, P=P, M=max(M, 1), K=K)
    n_pairs = M - 2 if model else 0
    if model:
        _random_model(rng, T, n_pairs, A, d, K, prio)
    _upload(t, T)
    flags = (moq_ops.GPI if gpi else 0) | (moq_ops.MODEL if model else 0) | (moq_ops.PRIORITIZE if prio else 0)
    for it in range(6):
        n_pol = int(rng.integers(1, P + 1))
        p = int(rng.integers(n_pol))
        s = int(rng.integers(S))
        s2 = s if it % 3 == 0 else int(rng.integers(S))
        a, term = int(rng.integers(A)), bool(it % 4 == 1)
        w = rng.dirichlet(np.ones(d)) if not ties else rng.integers(0, 3, d) / 2
        r = rng.integers(-2, 3, d) / 2
        kw = {}
        if model:
            pair = int(rng.integers(n_pairs + 1)) if n_pairs < M else int(rng.integers(n_pairs))
            n_pairs = max(n_pairs, pair + 1)
            outcome = int(rng.integers(min(K, int(T["pairs"][pair, 2]) + 1)))
            kw = dict(pair=pair, outcome=outcome, n_pairs=n_pairs, pick=rng.integers(0, n_pairs, dyna).tolist(), u=rng.random(dyna).tolist(),
                      choice=rng.random(dyna).tolist())
        f64.step(T, n_pol, p, s, a, s2, term, w, r, flags, 0.9, 0.3, **kw)
        moq_ops.moq_step(t, n_pol, p, s, a, s2, term, w, r, flags, 0.9, 0.3, **kw)
        _assert_equal(t, T)
        states = [int(x) for x in rng.integers(-1, S, 40)]
        pols = [int(x) for x in rng.integers(-1, n_pol, 40)]
        ws = rng.dirichlet(np.ones(d), 40) if not ties else rng.integers(0, 3, (40, d)) / 2
        out, val = moq_ops.moq_act(t, n_pol, states, pols, ws)
        want = [f64.act(T, n_pol, states[i], pols[i], ws[i]) for i in range(40)]
        np.testing.assert_array_equal(out.cpu().numpy(), np.array([[x[0], x[1]] for x in want], dtype=np.int32))
        assert val.cpu().numpy().tobytes() == np.array([x[2] for x in want]).tobytes()


def test_exact_ties_resolve_to_first_policy_action(cuda):
    S, P, A, d = 2, 4, 3, 2
    T = f64.new_table(S, P, A, d)
    T["visited"][0] = 1
    T["q"][0, 1, 2] = (1.0, 0.0)
    T["q"][0, 2, 0] = (0.0, 1.0)
    T["q"][0, 3, 1] = (0.5, 0.5)
    t = moq_ops.MoqTable(A, d, "cuda", False, S=S, P=P)
    _upload(t, T)
    out, val = moq_ops.moq_act(t, 4, [0, 0, 1, -1], [-1, 3, -1, 0], np.array([[0.5, 0.5]] * 4))
    assert out.cpu().tolist() == [[2, 0], [1, 1], [0, 0], [0, 0]]  # GPI: (1, 2) first of three equal values
    assert val.cpu().tolist() == [0.5, 0.5, 0.0, 0.0]


def test_walk_beyond_pairs_sets_status(cuda):
    S, P, A, d, M, K = 4, 1, 2, 2, 8, 2
    T = f64.new_table(S, P, A, d, M, K)
    T["pairs"][0] = (0, 0, 1)
    T["counts"][0, 0] = 1
    f64.tree_set(T["tree"], 5, 100.0)  # mass on a leaf no pair owns
    t = moq_ops.MoqTable(A, d, "cuda", True, S=S, P=P, M=M, K=K)
    _upload(t, T)
    kw = dict(pair=0, outcome=0, n_pairs=1, u=[0.9, 0.5], choice=[0.5, 0.5])
    flags = moq_ops.MODEL | moq_ops.PRIORITIZE
    f64.step(T, 1, 0, 0, 0, 1, False, np.ones(d) / d, np.ones(d), flags, 0.9, 0.1, **kw)
    moq_ops.moq_step(t, 1, 0, 0, 0, 1, False, np.ones(d) / d, np.ones(d), flags, 0.9, 0.1, **kw)
    assert t.status.cpu().tolist() == [1, 5] == T["status"].tolist()
    _assert_equal(t, T)
    before = t.q.clone()
    moq_ops.moq_step(t, 1, 0, 2, 1, 3, False, np.ones(d) / d, np.ones(d), flags, 0.9, 0.1, **kw)
    assert th.equal(t.q, before)
    with pytest.raises(_lib.MorlB200Error, match="walked to leaf 5"):
        moq_ops.check_status(t)


def _trained(use_gpi=True, iters=3, steps=300, **kw):
    import random

    random.seed(0)  # Dyna's draws come from python's and numpy's global generators
    np.random.seed(0)
    env = TreasureGrid(d=2, seed=0)
    env.action_space.seed(1)
    agent = MPMOQLearning(env, use_gpi_policy=use_gpi, seed=3, log=False, initial_epsilon=0.3, final_epsilon=0.3, **kw)
    agent.linear_support.verbose = False
    agent.train(total_timesteps=iters * steps, eval_env=TreasureGrid(d=2, seed=2), ref_point=np.array([0.0, -25.0]),
                timesteps_per_iteration=steps, num_eval_episodes_for_front=1)
    return agent


def test_eval_batch_equals_serial_eval(cuda):
    agent = _trained(iters=4)
    rng = np.random.default_rng(0)
    obs = np.stack([rng.integers(0, 6, 100), rng.integers(0, 7, 100)], axis=1).astype(np.int32)
    w = rng.dirichlet(np.ones(2), 100)
    got = agent.eval_batch(obs, w)
    assert got.tolist() == [agent.eval(o, wi) for o, wi in zip(obs, w)]
    vals = [agent.max_scalar_q_value(o, wi) for o, wi in zip(obs[:10], w[:10])]
    assert all(np.isfinite(vals))
    with pytest.raises(AttributeError):
        _trained(use_gpi=False, iters=1, steps=10).eval_batch


def test_growth_keeps_values(cuda):
    a = _trained(dyna=True, gpi_pd=True, iters=3, steps=400)
    # the same run on a store that starts at capacity 1 everywhere grows through every axis and must end with the same values
    import morl_baselines_b200.multi_policy.multi_policy_moqlearning.mp_mo_q_learning as mod

    orig = mod.MoqStore.__init__

    def tiny(self, A, d, model):
        orig(self, A, d, model)
        self.table = moq_ops.MoqTable(A, d, th.device("cuda"), model, S=1, P=1, M=1, K=1)

    mod.MoqStore.__init__ = tiny
    try:
        b = _trained(dyna=True, gpi_pd=True, iters=3, steps=400)
    finally:
        mod.MoqStore.__init__ = orig
    n = len(a._store.index.states)
    P = len(a.policies)
    ta, tb = a._store.table, b._store.table
    assert ta.q[:n, :P].cpu().numpy().tobytes() == tb.q[:n, :P].cpu().numpy().tobytes()
    M = len(a._store.index.pairs)
    K = min(ta.counts.shape[1], tb.counts.shape[1])
    assert th.equal(ta.counts[:M, :K].cpu(), tb.counts[:M, :K].cpu())
    np.testing.assert_allclose(ta.tree.cpu().numpy(), tb.tree.cpu().numpy(), rtol=0, atol=0)


def test_delete_policies_keeps_surviving_tables(cuda):
    agent = _trained(iters=5, steps=200)
    tabs = [p.q_table for p in agent.policies]
    agent.delete_policies([1, 3])
    assert len(agent.policies) == 3 and agent._store.n_policies == 3
    for p, want in zip(agent.policies, [tabs[0], tabs[2], tabs[4]]):
        got = p.q_table
        assert list(got) == list(want) and all(got[k].tobytes() == want[k].tobytes() for k in want)
    assert not agent._store.table.visited[:, 3:].any() and not agent._store.table.q[:, 3:].any()


@pytest.mark.parametrize("kw", [dict(), dict(dyna=True, dyna_updates=5), dict(dyna=True, dyna_updates=100, gpi_pd=True)])
def test_at_most_two_launches_per_step_and_no_upload(cuda, kw):
    env = TreasureGrid(d=3, slip=0.2, seed=0)
    agent = MPMOQLearning(env, use_gpi_policy=True, seed=3, log=False, **kw)
    agent.linear_support.verbose = False
    agent.train(total_timesteps=200, eval_env=TreasureGrid(d=3, seed=2), ref_point=np.zeros(3), timesteps_per_iteration=200,
                num_eval_episodes_for_front=1)
    learner = agent.policies[0]
    learner.obs, _ = env.reset()
    n_upd = kw.get("dyna_updates", 0) if kw.get("dyna") else 0
    per_step = 2 + max(0, -(-n_upd // moq_ops.DYNA_PER_LAUNCH) - 1)
    from torch.profiler import ProfilerActivity, profile

    th.cuda.synchronize()
    n0 = ops.launch_count
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        learner.train(start_time=0.0, total_timesteps=100, reset_num_timesteps=False)
        th.cuda.synchronize()
    assert ops.launch_count - n0 <= per_step * 100
    assert not [e for e in prof.events() if "HtoD" in e.name], "a step copied host data to the device"


def test_refusals(cuda):
    from morl_baselines_b200.common.scalarization import tchebicheff
    from morl_baselines_b200.multi_policy.multi_policy_moqlearning.mp_mo_q_learning import DeviceMOQLearning

    env = TreasureGrid(d=2)
    with pytest.raises(NotImplementedError):
        MPMOQLearning(env, scalarization=tchebicheff(0.1, 2), log=False)
    with pytest.raises(ValueError):
        DeviceMOQLearning(env, gpi_pd=True, dyna=True, log=False)
    with pytest.raises(_lib.MorlB200Error):
        moq_ops.MoqTable(65, 2, "cuda", False)
