"""PGMORL (multi_policy/pgmorl/pgmorl.py) end to end on the stand-in vector env of tests/ppo_standin.py (mo-gymnasium is not installed;
the module's ``mo_make`` / ``make_env`` / ``make_vector_env`` helpers are replaced).

Population of 4 (the predictor needs 4 distinct samples before the first task selection, so a population of 3 cannot reach it, in the
reference as here), 16 steps x 2 envs, 2 warm-up iterations, 1 evolutionary iteration per generation, 2 generations."""

import numpy as np
import pytest
import torch as th

from morl_baselines_b200.multi_policy.pgmorl import pgmorl as pg
from tests.ppo_standin import FakeVecEnv, fake_env

pytestmark = pytest.mark.gpu

POP, STEPS, ENVS, WARMUP, EVO = 4, 16, 2, 2, 1
ITERS = WARMUP + 2 * EVO


@pytest.fixture
def standin(monkeypatch):
    monkeypatch.setattr(pg, "mo_make", lambda env_id, **kw: fake_env())
    monkeypatch.setattr(pg, "make_env", lambda env_id, seed, idx, run_name, gamma: (lambda: fake_env(seed=seed)))
    monkeypatch.setattr(pg, "make_vector_env", lambda fns: FakeVecEnv([f() for f in fns]))


def _pgmorl(cuda, **kw):
    th.manual_seed(0)
    return pg.PGMORL("fake-v0", origin=np.array([-100.0, -100.0]), num_envs=ENVS, pop_size=POP, warmup_iterations=WARMUP,
                     steps_per_iteration=STEPS, evolutionary_iterations=EVO, num_performance_buffer=10, net_arch=[16, 16], num_minibatches=4,
                     update_epochs=2, seed=3, log=False, device=cuda, **kw)


def _train(agent):
    th.manual_seed(1)
    agent.train(total_timesteps=STEPS * ENVS * POP * ITERS, eval_env=fake_env(seed=9, horizon=10), ref_point=np.array([-100.0, -100.0]))


def test_train_end_to_end(cuda, standin):
    agent = _pgmorl(cuda)
    _train(agent)
    assert agent.global_step == ITERS * POP * STEPS * ENVS  # the reference's accounting: steps x envs per agent per iteration
    assert len(agent.archive.evaluations) > 0
    assert agent._population_graph is not None
    assert sorted(a.id for a in agent.agents) == list(range(POP))
    # snapshots never alias live parameters
    live = {p.data_ptr() for a in agent.agents for p in a.networks.parameters()}
    for ind in agent.population.individuals + agent.archive.individuals:
        assert not live & {p.data_ptr() for p in ind.networks.parameters()}


def test_population_graph_equals_sequential_updates(cuda, standin):
    """Rollouts, then one population replay per iteration, against each agent's own update right after the rollouts (two task
    selections included): the parameters end bit-identical."""
    a, b = _pgmorl(cuda), _pgmorl(cuda)
    b._update_all_agents = lambda: [x.update() for x in b.agents]
    _train(a)
    _train(b)
    for x, y in zip(a.agents, b.agents):
        for p, q in zip(x.networks.parameters(), y.networks.parameters()):
            assert th.equal(p, q)
        assert np.array_equal(x.weights.cpu().numpy(), y.weights.cpu().numpy())
    assert a.global_step == b.global_step
