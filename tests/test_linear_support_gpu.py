"""LinearSupport on the device: the corner-weight kernel (csrc/linear_support.cu) against the float64 oracle over d x n x input kinds,
the buffer-growth protocol, OLS's known answer through the device path, the batched GPI evaluation (``eval_batch`` of both GPI-PD
classes) against ``eval``, and GPI-LS / OLS training end to end without a caller-supplied selector."""

import numpy as np
import pytest
import torch as th

from tests.golden.standin_env import HV_REF_POINT, TreasureChain
from tests.linear_support_oracle import candidate_count, canonical, corners_oracle

pytestmark = pytest.mark.gpu
ORACLE_MAX_CANDIDATES = 300_000  # the numpy oracle's enumeration stays within a few seconds


def _inputs(kind, n, d, rng):
    if kind == "random":
        return rng.normal(size=(n, d)) * 10
    if kind == "integer":  # many ties and degenerate vertices
        return rng.integers(0, 4, size=(n, d)).astype(np.float64)
    if kind == "repeated":
        X = rng.uniform(0, 5, size=(max(1, (n + 1) // 2), d))
        return np.vstack([X, X])[:n]
    # "extremum_tie": two vectors share the maximum of objective 0
    X = rng.uniform(0, 5, size=(n, d))
    if n >= 2:
        X[1, 0] = X[0, 0] = X[:, 0].max() + 1.0
    return X


def _device_vertices(V):
    from morl_baselines_b200 import ops

    return ops.corner_weights(th.from_numpy(V).cuda()).cpu().numpy()


GRID = [(d, n) for d in (2, 3, 4, 6, 8) for n in (1, 2, 4, 7, 12, 20, 35, 60) if candidate_count(n, d) <= ORACLE_MAX_CANDIDATES]


@pytest.mark.parametrize("d,n", GRID)
@pytest.mark.parametrize("kind", ["random", "integer", "repeated", "extremum_tie"])
def test_corner_kernel_matches_oracle(cuda, d, n, kind):
    rng = np.random.default_rng(1000 * d + n + 100_000 * ["random", "integer", "repeated", "extremum_tie"].index(kind))
    V = np.round(_inputs(kind, n, d, rng), 4)
    verts = _device_vertices(V)
    want = corners_oracle(V)
    got = canonical(verts[:, :d])
    assert got.shape == want.shape, (got, want)
    assert np.abs(got - want).max(initial=0.0) <= 1e-9
    # raw vertices: on the simplex, u = max_k v_k . w, and no two within tolerance
    assert (verts[:, :d] >= -1e-9).all() and np.allclose(verts[:, :d].sum(1), 1.0, atol=1e-12)
    assert np.allclose(verts[:, d], (verts[:, :d] @ V.T).max(1), atol=1e-9 * max(1.0, np.abs(V).max()))
    gap = np.abs(verts[:, None, :d] - verts[None, :, :d]).max(-1) + np.eye(len(verts)) * 1e9
    assert gap.min(initial=1e9) > 1e-9


def test_corner_count_beyond_cap_then_regrow(cuda):
    from morl_baselines_b200 import _lib, ops

    rng = np.random.default_rng(5)
    V = th.from_numpy(np.round(rng.uniform(0, 10, size=(30, 4)), 4)).cuda()
    lib = _lib.load()
    count = th.zeros(1, dtype=th.int32, device=cuda)
    small = th.empty((2, 5), dtype=th.float64, device=cuda)
    ops._lib.check(lib.morl_corner_weights_f64(V.data_ptr(), 30, 4, small.data_ptr(), 2, count.data_ptr(), ops._stream()), "corner")
    k = int(count.item())
    assert k > 2  # count is not clipped to cap
    full = th.empty((k, 5), dtype=th.float64, device=cuda)
    ops._lib.check(lib.morl_corner_weights_f64(V.data_ptr(), 30, 4, full.data_ptr(), k, count.data_ptr(), ops._stream()), "corner")
    assert int(count.item()) == k
    want = corners_oracle(V.cpu().numpy())
    for got in (canonical(full.cpu().numpy()[:, :4]), canonical(ops.corner_weights(V, cap=1).cpu().numpy()[:, :4])):
        assert got.shape == want.shape and np.abs(got - want).max() <= 1e-9
    # the query-only form: cap 0 with no buffer
    ops._lib.check(lib.morl_corner_weights_f64(V.data_ptr(), 30, 4, None, 0, count.data_ptr(), ops._stream()), "corner")
    assert int(count.item()) == k
    rc = lib.morl_corner_weights_f64(V.data_ptr(), 59, 8, None, 0, count.data_ptr(), ops._stream())
    assert rc == -4  # C(67, 8) is above the bound


def test_ols_finds_the_convex_coverage_set_on_device(cuda):
    from morl_baselines_b200.multi_policy.linear_support.linear_support import LinearSupport
    from tests.test_linear_support_cpu import _ols_known_answer

    _ols_known_answer(LinearSupport, patch=False)


def _gpils(cuda, **kw):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPILS

    th.manual_seed(0)
    return GPILS(TreasureChain(seed=0), net_arch=[32, 32], batch_size=16, buffer_size=512, learning_starts=10, gradient_updates=1, log=False,
                 seed=0, device=cuda, **kw)


@pytest.mark.parametrize("use_gpi", [True, False])
def test_gpipd_eval_batch_equals_eval(cuda, use_gpi):
    agent = _gpils(cuda)
    agent.train_iteration(total_timesteps=60, weight=np.array([0.2, 0.5, 0.3], np.float32),
                          weight_support=[np.eye(3, dtype=np.float32)[i] for i in range(3)] + [np.array([0.2, 0.5, 0.3], np.float32)])
    agent.use_gpi = use_gpi
    rng = np.random.default_rng(0)
    obs = rng.uniform(0, 1, size=(37, 4)).astype(np.float32)
    w = rng.dirichlet(np.ones(3), size=37).astype(np.float32)
    batched = agent.eval_batch(obs, w)
    serial = np.array([agent.eval(o, x) for o, x in zip(obs, w)])
    assert np.array_equal(batched, serial)
    assert all(n.training for n in agent.q_nets)


@pytest.mark.parametrize("use_gpi", [True, False])
def test_gpipd_continuous_eval_batch_equals_eval(cuda, use_gpi):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import GPILSContinuousAction
    from morl_baselines_b200.testing import FakeEnv

    agent = GPILSContinuousAction(FakeEnv(obs_dim=5, continuous_action_dim=2, reward_dim=3), net_arch=[32, 32], batch_size=16, buffer_size=256,
                                  log=False, seed=0, device=cuda, use_gpi=use_gpi)
    for net in agent.q_nets:
        for m in net.modules():
            if isinstance(m, th.nn.Dropout):
                m.p = 0.0
    agent.set_weight_support([np.eye(3, dtype=np.float32)[i] for i in range(3)] + [np.array([0.3, 0.3, 0.4], np.float32)])
    rng = np.random.default_rng(1)
    obs = rng.normal(size=(23, 5)).astype(np.float32)
    w = rng.dirichlet(np.ones(3), size=23).astype(np.float32)
    batched = agent.eval_batch(obs, w)
    serial = np.stack([agent.eval(o, x) for o, x in zip(obs, w)])
    assert batched.shape == serial.shape == (23, 2)
    np.testing.assert_allclose(batched, serial, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_batched_gpi_evaluation_equals_serial(cuda, dtype):
    from morl_baselines_b200.common.evaluation import policy_evaluation_mo, policy_evaluation_mo_batched

    agent = _gpils(cuda)
    support = [np.eye(3, dtype=np.float32)[i] for i in range(3)] + [np.array([0.4, 0.4, 0.2], np.float32)]
    agent.train_iteration(total_timesteps=80, weight=support[3], weight_support=support)
    weights = [np.asarray(w, dtype=dtype) for w in np.random.default_rng(2).dirichlet(np.ones(3), size=9)]
    serial = [policy_evaluation_mo(agent, TreasureChain(seed=123), w, rep=2) for w in weights]
    batched = policy_evaluation_mo_batched(agent, TreasureChain(seed=123), weights, rep=2, weight_dtype=dtype)
    for s_, b_ in zip(serial, batched):
        for x, y in zip(s_, b_):
            assert np.array_equal(np.asarray(x), np.asarray(y))
            assert np.asarray(x).dtype == np.asarray(y).dtype


def _record_linear_support(monkeypatch):
    from morl_baselines_b200.multi_policy.linear_support import linear_support as mod

    made = []

    class Recording(mod.LinearSupport):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    monkeypatch.setattr(mod, "LinearSupport", Recording)
    return made


def _check_selection(ls, agent, algo, d):
    assert ls.epsilon == (0.0 if algo == "ols" else None)
    assert len(ls.visited_weights) >= 2
    for w in ls.visited_weights + ls.get_weight_support() + ls.get_corner_weights():
        w = np.asarray(w, dtype=np.float64)
        assert w.shape == (d,) and (w >= 0).all() and abs(w.sum() - 1.0) < 1e-6
    ccs = np.array(ls.ccs)
    assert len(ccs) > 0 and len(ls.weight_support) == len(ccs)
    for i in range(len(ccs)):
        for j in range(len(ccs)):
            assert i == j or not ((ccs[j] >= ccs[i]).all() and (ccs[j] > ccs[i]).any()), "CCS holds a dominated vector"
    assert len(agent.weight_support) >= 1


@pytest.mark.parametrize("algo", ["gpi-ls", "ols"])
def test_gpils_trains_without_a_supplied_selector(cuda, algo, monkeypatch):
    made = _record_linear_support(monkeypatch)
    agent = _gpils(cuda)
    w_calls = []
    orig = agent.train_iteration

    def spy(**kw):
        w_calls.append((np.asarray(kw["weight"]).copy(), [np.asarray(x).copy() for x in kw["weight_support"]]))
        return orig(**kw)

    agent.train_iteration = spy
    agent.train(total_timesteps=400, eval_env=TreasureChain(seed=9), ref_point=HV_REF_POINT, timesteps_per_iter=100,
                weight_selection_algo=algo, num_eval_episodes_for_front=1, checkpoints=False)
    assert len(made) == 1
    ls = made[0]
    _check_selection(ls, agent, algo, 3)
    assert len(w_calls) >= 3
    for w, M in w_calls:
        assert (w >= 0).all() and abs(w.sum() - 1) < 1e-6
        assert np.array_equal(M[-1], w)  # M = support (+ top-4 corner weights for GPI-LS) + [w], as in the reference
        if algo == "ols":
            assert len(M) <= len(ls.visited_weights) + 1


@pytest.mark.parametrize("algo", ["gpi-ls", "ols"])
def test_gpils_continuous_trains_without_a_supplied_selector(cuda, algo, monkeypatch):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import GPILSContinuousAction
    from morl_baselines_b200.testing import FakeEnv

    made = _record_linear_support(monkeypatch)
    env = FakeEnv(obs_dim=5, continuous_action_dim=2, reward_dim=2, horizon=8, seed=0)
    agent = GPILSContinuousAction(env, net_arch=[32, 32], batch_size=16, buffer_size=512, learning_starts=10, gradient_updates=1, log=False,
                                  seed=0, device=cuda)
    agent.train(total_timesteps=150, eval_env=FakeEnv(obs_dim=5, continuous_action_dim=2, reward_dim=2, horizon=8, seed=1),
                ref_point=np.zeros(2), timesteps_per_iter=50, weight_selection_algo=algo, num_eval_episodes_for_front=1, checkpoints=False)
    assert len(made) == 1
    _check_selection(made[0], agent, algo, 2)
