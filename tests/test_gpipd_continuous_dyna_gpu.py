"""The Dyna half of GPIPDContinuousAction against the unmodified reference (tests/golden/gpipd_continuous_dyna.npz, frozen on CPU by
tests/golden/make_golden_gpipd_continuous_dyna.py from gpi_pd_continuous_action.py:216-235, :311-371, :373-452), and its training loop.

Tolerances as tests/test_dyna_gpu.py: buffer values 1e-5 relative; kept / terminal rows, buffer positions and counts identical (the golden
threshold sits in a gap ~2,600x wider than the arithmetic noise); parameters after the updates 1e-4 relative; after three fit epochs 1e-3."""

import os
import random

import numpy as np
import pytest
import torch as th

from morl_baselines_b200.testing import FakeEnv, _Spec

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(OBS=11, ACT=3, D=3, B=16, N=256, ENV_ID="mo-hopper-standin-v4", ROLLOUT_B=300, ROLLOUT_LEN=3, DYN_BUF=200, REAL_RATIO=0.25,
           ARCH=[32, 32], DYN_ARCH=[32, 32], SEED_ROLLOUT=7, POLICY_NOISE_SEED=51, MODEL_NOISE_SEED=52, ELITES=[4, 2])


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "gpipd_continuous_dyna.npz"))


class _Noise:
    def __init__(self, seed, dev):
        self.rng, self.dev = np.random.default_rng(seed), dev

    def __call__(self, shape, dev=None):
        return th.from_numpy(self.rng.standard_normal(tuple(shape)).astype(np.float32)).to(self.dev)


def _sd(gold, prefix, dev):
    return {k[len(prefix) + 1:]: th.from_numpy(gold[k]).to(dev) for k in gold.files if k.startswith(prefix + "/")}


def _cmp_sd(module, gold, prefix, rtol, atol):
    for k, v in module.state_dict().items():
        np.testing.assert_allclose(v.detach().cpu().numpy(), gold[f"{prefix}/{k}"], rtol=rtol, atol=atol, err_msg=f"{prefix}/{k}")


def _agent(gold, dev, use_cuda_graph=True):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import GPIPDContinuousAction

    c = CFG
    env = FakeEnv(obs_dim=c["OBS"], continuous_action_dim=c["ACT"], reward_dim=c["D"])
    env.spec = _Spec(c["ENV_ID"])
    agent = GPIPDContinuousAction(env, batch_size=c["B"], net_arch=c["ARCH"], num_q_nets=2, gradient_updates=3, per=True, buffer_size=c["N"], dyna=True,
                                  dynamics_net_arch=c["DYN_ARCH"], dynamics_rollout_len=c["ROLLOUT_LEN"], dynamics_rollout_starts=0,
                                  dynamics_rollout_batch_size=c["ROLLOUT_B"], dynamics_buffer_size=c["DYN_BUF"], dynamics_min_uncertainty=float(gold["threshold"]),
                                  dynamics_real_ratio=c["REAL_RATIO"], log=False, seed=3, device=dev, use_cuda_graph=use_cuda_graph)
    for net in agent.q_nets + agent.target_q_nets:
        for m in net.modules():
            if isinstance(m, th.nn.Dropout):
                m.p = 0.0
    agent.policy.load_state_dict(_sd(gold, "init_policy", dev))
    agent.target_policy.load_state_dict(_sd(gold, "init_policy", dev))
    for i, (q, tq) in enumerate(zip(agent.q_nets, agent.target_q_nets)):
        q.load_state_dict(_sd(gold, f"init_q{i}", dev))
        tq.load_state_dict(_sd(gold, f"init_q{i}", dev))
    agent.dynamics.load_state_dict(_sd(gold, "init_dynamics", dev))
    agent.dynamics.elites = list(c["ELITES"])
    rb = agent.replay_buffer
    for k in ("obs", "next_obs", "actions", "rewards", "dones"):
        getattr(rb, k)[:] = gold[f"rb_{k}"]
    rb.size, rb.ptr = c["N"], 0
    rb.mark_all_dirty()
    rb.tree.batch_set(np.arange(c["N"]), gold["tree_leaves0"][:c["N"]])
    agent.set_weight_support(list(gold["support"]))
    agent._gold_support = gold["support"]
    return agent


def _rollout(agent, dev):
    c = CFG
    agent._noise_hook = _Noise(c["POLICY_NOISE_SEED"], dev)
    agent.dynamics.noise_fn = _Noise(c["MODEL_NOISE_SEED"], dev)
    np.random.seed(c["SEED_ROLLOUT"])
    agent._rollout_dynamics(th.tensor(agent._gold_support[2]).to(dev))
    agent._noise_hook, agent.dynamics.noise_fn = None, None


@pytest.mark.parametrize("use_cuda_graph", [True, False])
def test_rollout_and_update_match_reference(cuda, gold, use_cuda_graph):
    c = CFG
    agent = _agent(gold, cuda, use_cuda_graph)
    _rollout(agent, cuda)
    db = agent.dynamics_buffer
    assert [db.ptr, db.size] == gold["db_ptr_size"].tolist()
    assert np.array_equal(db.dones, gold["db_dones"])
    np.testing.assert_allclose(db.obs, gold["db_obs"], rtol=1e-5, atol=2e-6)
    np.testing.assert_allclose(db.actions, gold["db_actions"], rtol=1e-5, atol=2e-6)
    np.testing.assert_allclose(db.next_obs, gold["db_next_obs"], rtol=1e-5, atol=5e-6)
    np.testing.assert_allclose(db.rewards, gold["db_rewards"], rtol=1e-5, atol=5e-6)
    for h, d in zip(db._host_tensors(), db._dev):  # the numpy arrays are the device store
        assert th.equal(h.to(cuda), d)
    # three whole updates on mixed minibatches: PER real rows (their priorities written back) + model rows, support of five weights
    agent._noise_hook = _Noise(99, cuda)
    random.seed(15)
    np.random.seed(16)
    agent.global_step = 5
    agent.update(th.tensor(gold["support"][2]).to(cuda))
    assert any(k[5] for k in agent._graphs) == use_cuda_graph
    _cmp_sd(agent.policy, gold, "final_policy", 1e-4, 2e-6)
    for i, (q, tq) in enumerate(zip(agent.q_nets, agent.target_q_nets)):
        _cmp_sd(q, gold, f"final_q{i}", 1e-4, 2e-6)
        _cmp_sd(tq, gold, f"final_tq{i}", 1e-4, 2e-6)
    np.testing.assert_allclose(agent.replay_buffer.tree.nodes[-1][:c["N"]], gold["tree_leaves1"][:c["N"]], rtol=2e-4, atol=1e-7)
    assert agent.replay_buffer.min_priority == pytest.approx(float(gold["min_priority1"]), rel=2e-4)


def test_fit_with_normalized_inputs_matches_reference(cuda, gold):
    agent = _agent(gold, cuda)
    ens = agent.dynamics
    ens.load_state_dict(_sd(gold, "fit_init", cuda))
    rb = agent.replay_buffer
    m_obs, m_actions, m_rewards, m_next_obs, _ = rb.get_all_data()
    np.random.seed(5)
    mean_holdout = ens.fit(np.hstack((m_obs, m_actions)), np.hstack((m_rewards, m_next_obs - m_obs)), batch_size=64, max_epochs=3)
    assert mean_holdout == pytest.approx(float(gold["fit_mean_holdout"]), rel=1e-3)
    assert list(ens.elites) == gold["fit_elites"].tolist()
    _cmp_sd(ens, gold, "fit_final", 1e-3, 1e-5)


def test_real_ratio_zero_writes_no_priorities(cuda, gold):
    for use_cuda_graph in (True, False):
        agent = _agent(gold, cuda, use_cuda_graph)
        agent.dynamics_real_ratio = 0.0
        _rollout(agent, cuda)
        leaves = agent.replay_buffer.tree.nodes[-1].copy()
        agent.global_step = 5
        agent.update(th.tensor(gold["support"][2]).to(cuda))
        assert np.array_equal(agent.replay_buffer.tree.nodes[-1], leaves)
        assert all(bool(th.isfinite(p).all()) for q in agent.q_nets for p in q.parameters())


def test_train_iteration_fits_rolls_out_and_mixes(cuda, tmp_path):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import GPIPDContinuousAction

    env = FakeEnv(obs_dim=11, continuous_action_dim=3, reward_dim=3, horizon=20)
    env.spec = _Spec("mo-hopper-v4")
    agent = GPIPDContinuousAction(env, batch_size=16, net_arch=[32, 32], gradient_updates=1, learning_starts=20, buffer_size=512, dynamics_net_arch=[32, 32],
                                  dynamics_train_freq=25, dynamics_rollout_starts=50, dynamics_rollout_freq=25, dynamics_rollout_batch_size=200,
                                  dynamics_rollout_len=2, dynamics_buffer_size=1000, dynamics_min_uncertainty=1e9, log=False, seed=0, device=cuda)
    assert agent.get_config()["dyna"] is True
    fits, rollouts, mixed = [], [], []
    train, roll, upd = agent._train_dynamics, agent._rollout_dynamics, agent.update

    def spy_update(w):
        mixed.append((agent.global_step, agent._uses_model_samples()))
        upd(w)

    agent._train_dynamics = lambda: (fits.append(agent.global_step), train())[1]
    agent._rollout_dynamics = lambda w: (rollouts.append(agent.global_step), roll(w))[1]
    agent.update = spy_update
    M = [np.array([1.0, 0.0, 0.0], np.float32), np.array([0.0, 1.0, 0.0], np.float32), np.array([0.3, 0.3, 0.4], np.float32)]
    agent.train_iteration(total_timesteps=100, weight=M[2], weight_support=M, change_weight_every_episode=True)
    assert fits == [25, 50, 75, 100] and rollouts == [50, 75, 100]
    assert len(agent.dynamics_buffer) > 0
    assert [s for s, m in mixed if m] == list(range(50, 101))
    assert any(k[5] for k in agent._graphs)  # the graph path replayed mixed minibatches
    obs, act, rew, nobs, done, idx = agent._sample_batch_experiences()
    assert obs.shape[0] == 16 and len(idx) == int(16 * agent.dynamics_real_ratio)
    db = agent.dynamics_buffer
    stored = th.from_numpy(db.obs[:db.size]).to(cuda)
    assert all(bool((stored == o).all(-1).any()) for o in obs[len(idx):])  # the imagined rows come from the model buffer
    for m in (agent.policy, agent.dynamics, *agent.q_nets):
        assert all(bool(th.isfinite(p).all()) for p in m.parameters())

    # checkpoint round trip with the reference's keys
    agent.save(save_dir=str(tmp_path), filename="ckpt", save_replay_buffer=False)
    params = th.load(str(tmp_path / "ckpt.tar"), map_location="cpu", weights_only=False)
    assert "dynamics_state_dict" in params
    other = GPIPDContinuousAction(env, batch_size=16, net_arch=[32, 32], buffer_size=512, dynamics_net_arch=[32, 32], log=False, seed=1, device=cuda)
    other.load(str(tmp_path / "ckpt.tar"))
    for k, v in agent.dynamics.state_dict().items():
        assert th.equal(other.dynamics.state_dict()[k], v), k


def test_reference_defaults_construct_and_unknown_env_raises(cuda):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import GPIPDContinuousAction, GPILSContinuousAction

    env = FakeEnv(obs_dim=11, continuous_action_dim=3, reward_dim=3)
    with pytest.raises(NotImplementedError, match="fake-momdp-v0"):
        GPIPDContinuousAction(env, log=False, device=cuda)
    env.spec = _Spec("mo-hopper-v4")
    # the constructor arguments of the reference's examples/gpi_pd_hopper.py
    agent = GPIPDContinuousAction(env, gradient_updates=1, min_priority=0.1, batch_size=128, buffer_size=int(4e5), dynamics_rollout_starts=1000,
                                  dynamics_rollout_len=5, dynamics_rollout_freq=250, dynamics_rollout_batch_size=50000, dynamics_train_freq=250,
                                  dynamics_buffer_size=200000, dynamics_real_ratio=0.1, dynamics_min_uncertainty=2.0, dyna=True, per=True,
                                  project_name="MORL-Baselines", experiment_name="GPI-PD", log=False, device=cuda)
    assert agent.dyna and agent.dynamics.ensemble_size == 5 and agent.dynamics.num_elites == 2 and agent.dynamics.normalize_inputs
    assert agent.dynamics.arch == [200, 200, 200, 200] and agent.dynamics_buffer.max_size == 200000
    ls = GPILSContinuousAction(env, log=False, device=cuda)
    assert not ls.dyna and ls.dynamics is None and ls.dynamics_buffer is None and ls.get_config()["dyna"] is False
