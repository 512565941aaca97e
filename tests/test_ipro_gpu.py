"""IPRO and IPRO-2D on the device: every golden case of tests/golden/ipro.npz (made by the reference with the scripted oracle of
tests/ipro_standin.py) reproduced exactly, the hypervolume improvements of the batched kernel against the host sweep, and short end-to-end
runs with the real NLMOPPO learner on the ring environment."""

import os

import numpy as np
import pytest
import torch as th

from morl_baselines_b200.multi_policy.ipro import outer_loop
from morl_baselines_b200.multi_policy.ipro.ipro import IPRO
from morl_baselines_b200.multi_policy.ipro.ipro_2d import IPRO2D
from tests.ipro_standin import CASES, IproEnv, run_case

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ipro.npz")
CLASSES = {"IPRO": IPRO, "IPRO2D": IPRO2D}


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", list(CASES))
def test_golden_case_reproduced_exactly(cuda, golden, name):
    got = run_case(name, CLASSES, device=str(cuda))
    want = {k[len(name) + 1:]: golden[k] for k in golden.files if k.startswith(name + "/")}
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].shape == want[k].shape, k
        assert got[k].tobytes() == want[k].tobytes(), k


@pytest.mark.parametrize("d,n_front", [(3, 32), (3, 300), (4, 64), (4, 200)])
def test_hvis_kernel_equals_host_sweep(cuda, d, n_front):
    """compute_hvis's volumes through the kernel equal the host sweep's on dyadic fronts (exact), and the resulting order is the same."""
    rng = np.random.default_rng(d * n_front)
    agent = IPRO.__new__(IPRO)
    agent.ideal = np.full(d, 40.0)
    agent.pf = rng.integers(0, 300, (n_front, d)) / 8
    agent.completed = rng.integers(0, 300, (n_front // 4, d)) / 8
    lowers = rng.integers(-8, 300, (50, d)) / 8
    lowers[0] = 45.0  # not dominated by the ideal: pf U completed alone
    dev = agent._improvement_volumes(lowers, device=True)
    host = agent._improvement_volumes(lowers, device=False)
    np.testing.assert_array_equal(dev, host)
    assert (np.argsort(dev)[::-1] == np.argsort(host)[::-1]).all()


def _learner_kwargs():
    return dict(tolerance=0.0, gamma=1.0, num_steps=16, anneal_lr=False, iter_total_timesteps=2 * 16 * 4, num_minibatches=2, update_epochs=1,
                log=False, seed=3)


def _run(cls, d, reset_agent, extrema=None, **kw):
    env = IproEnv(num_envs=4, obs_dim=2, n_actions=4, d=d)
    eval_env = IproEnv(num_envs=1, obs_dim=2, n_actions=4, d=d).envs[0]
    seen = []
    th.manual_seed(7)  # the Agent's initial parameters and the learner's action sampling
    agent = cls(env, reset_agent=reset_agent, max_iterations=3, **_learner_kwargs(), **kw)
    ps = agent.train(eval_env=eval_env, ref_point=None, deterministic=True, extrema=extrema, callback=lambda *args: seen.append(args))
    return agent, ps, seen


# The d = 3 run starts from wide extrema: a learner trained for two updates can report an "ideal" below the "nadir" of the linear phase,
# and from such a box the outer loop runs out of lower points before it covers it (as the reference's does).
WIDE3 = (np.full(3, -50.0), np.full(3, 50.0))


@pytest.mark.parametrize("cls,d,reset_agent,extrema", [(IPRO, 2, True, None), (IPRO, 3, False, WIDE3), (IPRO, 3, True, WIDE3),
                                                       (IPRO2D, 2, True, None), (IPRO2D, 2, False, None)])
def test_end_to_end_with_nlmoppo(cuda, cls, d, reset_agent, extrema):
    agent, ps, seen = _run(cls, d, reset_agent, extrema)
    pf = agent.pf
    assert all(not (np.all(pf[j] >= pf[i]) and np.any(pf[j] > pf[i])) for i in range(len(pf)) for j in range(len(pf)) if i != j)
    assert 0.0 <= agent.coverage <= 1.0
    assert all(0.0 <= s[4] <= 1.0 for s in seen)
    assert all(np.any(np.all(np.isclose(v, pf), axis=1)) for v, _ in ps)
    again, ps2, _ = _run(cls, d, reset_agent, extrema)
    assert again.pf.tobytes() == pf.tobytes()
    assert [v.tobytes() for v, _ in ps2] == [v.tobytes() for v, _ in ps]


def test_utility_handed_to_learner_is_aasf_and_linear(cuda):
    """The utilities the outer loop gives the learner equal aasf / linear_scalarization, evaluated on random batches."""
    env = IproEnv(num_envs=4, obs_dim=2, n_actions=4, d=3)
    agent = IPRO(env, **_learner_kwargs())
    captured = []

    class Capture:
        agent = "captured"

        def reset_agent(self, pref_dim):
            pass

        def train(self, eval_env, u_func, pref=None, deterministic=False):
            captured.append((u_func, pref))
            return np.array([1.0, 2.0, 3.0])

    agent.agent = Capture()
    agent.nadir, agent.ideal = np.array([-2.0, -1.0, 0.0]), np.array([4.0, 5.0, 6.0])
    referent = np.array([0.5, 1.5, 2.5])
    for sign in (1, -1):
        agent.sign = sign
        agent.oracle_train(referent, deterministic=True, eval_env=None)
        agent.linear_train(np.array([0.2, 0.3, 0.5]), deterministic=True, eval_env=None)
    g = th.Generator(device=cuda).manual_seed(0)
    for k, sign in ((0, 1), (2, -1)):
        batch = th.randn(256, 3, device=cuda, generator=g)
        u, pref = captured[k]
        t = lambda v: sign * th.tensor(v, device=cuda, dtype=th.float32)  # noqa: E731
        want = outer_loop.aasf(batch, t(referent), t(agent.nadir), t(agent.ideal), aug=0.1, scale=100)
        assert th.equal(u(batch), want) and th.equal(pref, t(referent))
        u, pref = captured[k + 1]
        w = th.tensor([0.2, 0.3, 0.5], device=cuda, dtype=th.float32)
        assert th.equal(u(batch), (batch * w).sum(-1)) and th.equal(pref, w)
