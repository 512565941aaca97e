"""MOSACDiscrete (single_policy/ser/mosac_discrete_action.py) on the CUDA update engine, and MORL/D with it as the inner learner.

Whole-update parity against golden vectors of the UNMODIFIED reference on CPU (tests/golden/make_golden_mosac_discrete.py ->
tests/golden/mosac_discrete.npz): same initial parameters, same replay contents, same numpy stream for the replay indices; tolerance
1e-4 relative / 2e-6 absolute on parameters, log_alpha and the logged losses (the MOSAC test's tolerance), eager and graphed."""

import copy
import os

import numpy as np
import pytest
import torch as th

from oracle.ref_harness import Box, FakeEnv

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBS, A, D, B, N = 8, 4, 4, 16, 128
STEPS = (100, 200, 300)


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "mosac_discrete.npz"))


def _load_sd(module, gold, prefix, dev):
    module.load_state_dict({k[len(prefix) + 1:]: th.from_numpy(gold[k]).to(dev) for k in gold.files if k.startswith(prefix + "/")})


def _cmp_sd(module, gold, prefix, rtol=1e-4, atol=2e-6):
    for k, v in module.state_dict().items():
        np.testing.assert_allclose(v.detach().cpu().numpy(), gold[f"{prefix}/{k}"], rtol=rtol, atol=atol, err_msg=f"{prefix}/{k}")


def _make(cuda, graph, autotune, **kw):
    from morl_baselines_b200.single_policy.ser.mosac_discrete_action import MOSACDiscrete

    w = np.array([0.1, 0.4, 0.3, 0.2], dtype=np.float32)
    return MOSACDiscrete(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), weights=w, batch_size=B, net_arch=[32, 32], log=False, seed=4,
                         device=cuda, buffer_size=N, tau=0.5, update_frequency=1, target_net_freq=200, autotune=autotune, alpha=0.3,
                         use_cuda_graph=graph, **kw)


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("autotune", [True, False])
def test_update_matches_reference(cuda, gold, graph, autotune):
    tag = f"autotune{int(autotune)}"
    agent = _make(cuda, graph, autotune)
    for name in ("actor", "qf1", "qf2"):
        _load_sd(getattr(agent, name), gold, f"{tag}/init_{name}", cuda)
    agent.qf1_target.load_state_dict(agent.qf1.state_dict())
    agent.qf2_target.load_state_dict(agent.qf2.state_dict())
    buf = agent.buffer
    for k in ("obs", "next_obs", "actions", "rewards", "dones"):
        getattr(buf, k)[:] = gold[f"{tag}/rb_{k}"]
    buf.size, buf.ptr = N, 0
    buf.mark_all_dirty()
    np.random.seed(12)
    losses = {k: [] for k in ("qf", "actor", "alpha")}
    for step in STEPS:
        agent.global_step = step
        agent.update()
        losses["qf"].append(float(agent._last_qf_loss))
        losses["actor"].append(float(agent._last_actor_loss))
        if autotune:
            losses["alpha"].append(float(agent._last_alpha_loss))
    assert agent.graph_update_ready() == graph and len(agent._graphs) == (2 if graph else 0)  # with and without the target sync
    for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
        _cmp_sd(getattr(agent, name), gold, f"{tag}/final_{name}")
    np.testing.assert_allclose(losses["qf"], gold[f"{tag}/qf1_loss"] + gold[f"{tag}/qf2_loss"], rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(losses["actor"], gold[f"{tag}/actor_loss"], rtol=1e-4, atol=2e-6)
    if autotune:
        np.testing.assert_allclose(losses["alpha"], gold[f"{tag}/alpha_loss"], rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(agent.log_alpha.detach().cpu().numpy(), gold[f"{tag}/final_log_alpha"], rtol=1e-4, atol=2e-6)
    assert agent.alpha == pytest.approx(float(gold[f"{tag}/final_alpha"]), rel=1e-4, abs=2e-6)


def test_save_load_round_trip_and_deepcopy(cuda, tmp_path):
    agent = _make(cuda, True, True)
    rng = np.random.default_rng(2)
    for _ in range(64):
        agent.buffer.add(rng.standard_normal(OBS).astype(np.float32), int(rng.integers(A)), rng.standard_normal(D).astype(np.float32),
                         rng.standard_normal(OBS).astype(np.float32), False)
    for step in range(1, 4):
        agent.global_step = step
        agent.update()
    d = agent.get_save_dict(save_replay_buffer=True)
    assert {"actor_state_dict", "qf1_state_dict", "qf2_state_dict", "qf1_target_state_dict", "qf2_target_state_dict", "actor_optimizer_state_dict",
            "q_optimizer_state_dict", "weights", "alpha", "buffer", "log_alpha", "a_optimizer_state_dict", "target_entropy_scale"} == set(d)
    th.save(d, str(tmp_path / "ck.tar"))
    other = _make(cuda, True, True)
    other.load(path=str(tmp_path / "ck.tar"))
    for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
        for (k, va), (_, vb) in zip(getattr(agent, name).state_dict().items(), getattr(other, name).state_dict().items()):
            assert th.equal(va, vb), (name, k)
    assert th.equal(agent.log_alpha, other.log_alpha) and other.alpha == agent.alpha and len(other.buffer) == 64
    # both continue identically from the same state
    for a in (agent, other):
        np.random.seed(8)
        a.global_step = 4
        a.update()
    for (k, va), (_, vb) in zip(agent.actor.state_dict().items(), other.actor.state_dict().items()):
        assert th.equal(va, vb), k
    # the reference's deepcopy: networks and step copied, fresh optimisers, log_alpha NOT copied (alpha back to 1)
    c = copy.deepcopy(agent)
    for (k, va), (_, vb) in zip(agent.qf1.state_dict().items(), c.qf1.state_dict().items()):
        assert th.equal(va, vb), k
    assert c.global_step == agent.global_step and float(c.log_alpha.detach()) == 0.0 and c.alpha == 1.0
    assert len(c.actor_optimizer.state) == 0 and c.actor_optimizer.defaults["eps"] == 1e-4 and len(c.buffer) == 64
    assert isinstance(int(c.eval(np.zeros(OBS, np.float32))), int)


def test_update_with_image_observations(cuda):
    """Image observations take NatureCNN feature extractors; the kernels only see Q and the logits."""
    from morl_baselines_b200.single_policy.ser.mosac_discrete_action import MOSACDiscrete

    env = FakeEnv(obs_dim=4, n_actions=3, reward_dim=2)
    env.observation_space = Box(-np.inf, np.inf, shape=(2, 84, 84))
    rng = np.random.default_rng(4)
    for graph in (False, True):
        agent = MOSACDiscrete(env, weights=np.array([0.5, 0.5], np.float32), batch_size=8, net_arch=[64, 32], log=False, device=cuda,
                              buffer_size=32, use_cuda_graph=graph, update_frequency=1, target_net_freq=2)
        for _ in range(16):
            agent.buffer.add(rng.random((2, 84, 84)).astype(np.float32), int(rng.integers(3)), rng.standard_normal(2).astype(np.float32),
                             rng.random((2, 84, 84)).astype(np.float32), False)
        before = [p.detach().clone() for p in agent.actor.parameters()]
        for step in (1, 2):
            agent.global_step = step
            agent.update()
        assert all(bool(th.isfinite(p).all()) for p in agent.actor.parameters())
        assert any(not th.equal(a, b) for a, b in zip(before, agent.actor.parameters()))
        assert np.isfinite(float(agent._last_qf_loss)) and np.isfinite(float(agent._last_actor_loss))


def _discrete_morld(cuda, **kw):
    from morl_baselines_b200.multi_policy.morld.morld import MORLD

    env = FakeEnv(obs_dim=6, n_actions=4, reward_dim=2, horizon=20)
    args = dict(pop_size=3, exchange_every=60, update_passes=2, log=False, device=cuda, seed=0, weight_init_method="random",
                policy_name="MOSACDiscrete", neighborhood_size=1,
                policy_args={"learning_starts": 20, "batch_size": 16, "net_arch": [32, 32], "buffer_size": 512, "update_frequency": 1,
                             "target_net_freq": 10})
    args.update(kw)
    return MORLD(env, **args), FakeEnv(obs_dim=6, n_actions=4, reward_dim=2, horizon=20, seed=1)


def test_morld_discrete_population_smoke(cuda):
    """MORL/D with MOSACDiscrete learners on the stand-in MOMDP: one outer iteration (train, update the others, evaluate, archive)."""
    from morl_baselines_b200.common.performance_indicators import hypervolume

    algo, eval_env = _discrete_morld(cuda)
    algo.train(total_timesteps=60, eval_env=eval_env, ref_point=np.array([-100.0, -100.0]), num_eval_episodes_for_front=1, checkpoints=False)
    assert len(algo.archive.evaluations) >= 1 and algo.global_front.shape[1] == 2
    assert hypervolume(np.array([-100.0, -100.0]), list(algo.global_front)) > 0
    with pytest.raises(NotImplementedError, match="EUPG"):
        _discrete_morld(cuda, policy_name="EUPG")


def test_morld_discrete_population_graph_equals_per_learner_graphs(cuda):
    """One multi-branch population graph over MOSACDiscrete learners leaves every learner bit-identical to replaying each learner's own
    graph in the reference's policy order."""
    def build():
        th.manual_seed(0)
        algo, _ = _discrete_morld(cuda, pop_size=5, update_passes=3,
                                  policy_args={"learning_starts": 0, "batch_size": 16, "net_arch": [32, 32], "buffer_size": 256,
                                               "update_frequency": 1, "target_net_freq": 2})
        rng = np.random.default_rng(5)
        for p in algo.population:
            buf = p.wrapped.get_buffer()
            for _ in range(64):
                buf.add(rng.standard_normal(6).astype(np.float32), int(rng.integers(4)), rng.standard_normal(2).astype(np.float32),
                        rng.standard_normal(6).astype(np.float32), bool(rng.random() < 0.1))
            p.wrapped.global_step = 4
        return algo

    a, b = build(), build()
    b.population_graph = False
    for algo in (a, b):
        np.random.seed(3)
        algo._update_others(algo.population[1])
    assert len(a._pop_graphs) == 1 and len(b._pop_graphs) == 0
    assert all(len(p.wrapped._graphs) == 1 for i, p in enumerate(b.population) if i != 1)
    for pa, pb in zip(a.population, b.population):
        for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
            for (k, va), (_, vb) in zip(getattr(pa.wrapped, name).state_dict().items(), getattr(pb.wrapped, name).state_dict().items()):
                assert th.equal(va, vb), (pa.id, name, k)
        assert th.equal(pa.wrapped.log_alpha, pb.wrapped.log_alpha)


def test_morld_lunar_lander_example_arguments(cuda):
    """The reference's examples/morld_lunar_lander.py arguments (4 actions, 4 objectives, net_arch [256] * 4, batch 128, pop_size 6) on a
    stand-in with lunar-lander's shapes: constructs, and trains a few steps including the improvement passes."""
    from morl_baselines_b200.multi_policy.morld.morld import MORLD

    env = FakeEnv(obs_dim=8, n_actions=4, reward_dim=4, horizon=30)
    eval_env = FakeEnv(obs_dim=8, n_actions=4, reward_dim=4, horizon=30, seed=1)
    algo = MORLD(env=env, exchange_every=200, pop_size=6, policy_name="MOSACDiscrete", scalarization_method="ws", evaluation_mode="ser", gamma=0.99,
                 log=False, neighborhood_size=1, update_passes=10, shared_buffer=True, sharing_mechanism=[], weight_adaptation_method="PSA", seed=0,
                 device=cuda, policy_args={"target_net_freq": 200, "batch_size": 128, "buffer_size": 100000, "net_arch": [256, 256, 256, 256],
                                            "update_frequency": 1, "target_entropy_scale": 0.3, "learning_starts": 100})
    assert algo.population[0].wrapped.get_buffer() is algo.population[5].wrapped.get_buffer()
    algo.train(eval_env=eval_env, total_timesteps=200, ref_point=np.array([-101, -1001, -101, -101]), num_eval_episodes_for_front=1,
               num_eval_weights_for_eval=5, checkpoints=False)
    assert algo.global_step == 200
    assert all(bool(th.isfinite(p).all()) for pol in algo.population for p in pol.wrapped.actor.parameters())
