"""Whole-update parity of morl_baselines_b200.Envelope (CUDA: device replay gather, Q on B*|W| rows, fused envelope-TD, fused
loss, CUDA-graph replay, optional tensor-core dense layers) against the PyTorch-CPU port of the reference update
(oracle/envelope_update_port.py, itself pinned bit-for-bit to the unmodified reference in tests/test_port_vs_reference.py).

Tolerance (BASELINE.json north_star): losses and parameters within 1e-5 relative; priorities within 1e-5 relative (they are
|w . td| of fp32 Q-values computed by a different fp32 GEMM than MKL)."""

import numpy as np
import pytest
import torch as th

from oracle.envelope_update_port import EnvelopeUpdatePort, synthetic_store
from oracle.ref_harness import FakeEnv

pytestmark = pytest.mark.gpu


def _run(cuda, per, tc, graph, lam=0.0, envelope=True, steps=3, W=8, net=(64, 64, 64), param_atol=2e-6, replay_on_device=True):
    from morl_baselines_b200.common.weights import random_weights
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    OBS, A, D, B, N = 12, 4, 3, 32, 2048
    net = list(net)
    th.manual_seed(0)
    agent = Envelope(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), batch_size=B, num_sample_w=W, per=per, buffer_size=N, net_arch=net,
                     log=False, seed=3, device=cuda, use_cuda_graph=graph, use_tensor_cores=tc, initial_homotopy_lambda=lam, envelope=envelope,
                     replay_on_device=replay_on_device)
    assert agent.use_tensor_cores == tc
    store = synthetic_store(N, OBS, A, D, seed=1)
    rb = agent.replay_buffer
    rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
    rb.size, rb.ptr = N, 0
    rb.mark_all_dirty()
    if per:
        rb.tree.batch_set(np.arange(N), np.full(N, rb.min_priority))
    sd = {k: v.detach().cpu().clone() for k, v in agent.q_net.state_dict().items()}
    port = EnvelopeUpdatePort(OBS, A, D, net, seed=0, state_dict=sd)
    rng = np.random.default_rng(3)
    agent.global_step = 1
    losses = []
    for step in range(steps):
        np.random.seed(50 + step)
        state = np.random.get_state()
        idx = rb.tree.sample(B) if per else np.random.choice(N, B, replace=True)
        np.random.set_state(state)
        wset = th.tensor(random_weights(D, W, dist="gaussian", rng=rng)).float()
        min_p = rb.min_priority if per else None
        agent.update()
        if envelope:
            loss, prio = port.update(th.from_numpy(store["obs"][idx]), th.from_numpy(store["actions"][idx]), th.from_numpy(store["rewards"][idx]),
                                     th.from_numpy(store["next_obs"][idx]), th.from_numpy(store["dones"][idx]), wset, homotopy_lambda=lam)
            got = float(agent._last_loss)
            assert abs(got - loss) <= 1e-5 * abs(loss), (step, got, loss)
            if per:
                exp_p = (prio + min_p) ** agent.per_alpha
                np.testing.assert_allclose(agent._last_priority, exp_p, rtol=2e-5, atol=1e-7)
        losses.append(float(agent._last_loss))
    if envelope:
        for (k, v), (_, v2) in zip(agent.q_net.state_dict().items(), port.q_net.state_dict().items()):
            np.testing.assert_allclose(v.cpu().numpy(), v2.numpy(), rtol=1e-4, atol=param_atol, err_msg=k)
    return losses, agent


@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("graph", [False, True])
def test_envelope_update_matches_reference_port(cuda, per, tc, graph):
    _run(cuda, per, tc, graph)


@pytest.mark.parametrize("graph", [False, True])
def test_envelope_update_single_tile_shape(cuda, graph):
    """B * |W| = 128 rows: exactly one 128-row tile, a one-CTA launch of the GEMM kernel with every epilogue flavour
    of the update -- hidden layers, ReLU mask, fp32 output -- on a 4 x 256 net (the hypervolume-parity training configuration)."""
    # (4 x 256 net: 140k parameters; Adam's first steps turn the ~1e-8 rounding noise of the smallest gradient elements into ~1e-5 parameter
    # differences on a handful of them -- tests/test_envelope_update_golden_gpu.py states the full bound)
    _run(cuda, per=True, tc=True, graph=graph, W=4, net=(256, 256, 256, 256), param_atol=3e-5)


def test_envelope_update_homotopy_and_ddqn(cuda):
    _run(cuda, per=True, tc=True, graph=True, lam=0.3)
    losses, _ = _run(cuda, per=False, tc=False, graph=False, envelope=False)  # ddqn_target ablation runs and stays finite
    assert all(np.isfinite(losses))


# the graph's mode: sum tree in HBM ("device_per"), HBM replay mirror without PER ("device"), host-resident buffer with PER ("host")
MODES = {"device_per": dict(per=True), "device": dict(per=False), "host": dict(per=True, replay_on_device=False)}


def _graph_equals_eager(cuda, mode):
    l_graph, a_g = _run(cuda, tc=True, graph=True, **MODES[mode])
    assert list(a_g._graphs) == [mode]
    l_eager, a_e = _run(cuda, tc=True, graph=False, **MODES[mode])
    assert l_graph == l_eager
    for v, v2 in zip(a_g.q_net.state_dict().values(), a_e.q_net.state_dict().values()):
        assert th.equal(v, v2)


def test_graph_and_eager_paths_agree_bitwise(cuda):
    _graph_equals_eager(cuda, "device_per")


@pytest.mark.parametrize("mode", ["device", "host"])
def test_graph_and_eager_paths_agree_bitwise_in_other_modes(cuda, mode):
    _graph_equals_eager(cuda, mode)


def test_envelope_api_surface(cuda):
    """eval / act / max_action / envelope_target / save / load keep the reference's calling conventions."""
    import os
    import tempfile

    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    env = FakeEnv(obs_dim=6, n_actions=3, reward_dim=2)
    agent = Envelope(env, batch_size=16, num_sample_w=4, buffer_size=256, net_arch=[64, 64], log=False, seed=0, device=cuda)
    obs, _ = env.reset(seed=0)
    w = np.array([0.3, 0.7], dtype=np.float32)
    a = agent.eval(obs, w)
    assert isinstance(a, int) and 0 <= a < 3
    with th.no_grad():  # (a grad-tracking forward kept alive on the default stream would pin AccumulateGrad nodes to it)
        q = agent.q_net(th.as_tensor(obs).float().to(cuda), th.as_tensor(w).to(cuda))
    assert a == int(th.argmax(th.einsum("r,bar->ba", th.as_tensor(w).to(cuda), q), dim=1).item())
    # reference calling convention of envelope_target: tiled obs [W*B, ...], repeat_interleaved weights
    B, W = 5, 4
    nobs = th.randn(B, 6, device=cuda)
    sw = th.rand(W, 2, device=cuda)
    t = agent.envelope_target(nobs.repeat(W, 1), sw.repeat_interleave(B, 0), sw)
    assert t.shape == (W * B, 2)
    for _ in range(40):
        agent.replay_buffer.add(env.observation_space.sample(), 1, np.zeros(2), env.observation_space.sample(), False)
    agent.global_step = 1
    agent.update()
    with tempfile.TemporaryDirectory() as d:
        agent.save(save_dir=d, filename="ckpt")
        sd = th.load(os.path.join(d, "ckpt.tar"), weights_only=False)
        assert {"q_net_state_dict", "q_net_optimizer_state_dict", "replay_buffer"} <= set(sd)
        before = {k: v.clone() for k, v in agent.q_net.state_dict().items()}
        agent.update()
        agent.load(os.path.join(d, "ckpt.tar"))
        for k, v in agent.q_net.state_dict().items():
            assert th.equal(v, before[k])
        agent.update()  # the captured graph is still valid after an in-place load
    assert np.isfinite(float(agent._last_loss))


def test_device_per_equals_host_per(cuda):
    """Device-resident PER (sum tree, sampling, priority power + ratchet + write-back inside the captured step) against the host-tree path
    of the same engine on the same RNG streams: identical sampled indices and losses every step, identical parameters; priorities equal up
    to numpy's float32 power (<= 1 ulp)."""
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    def build(per_dev):
        th.manual_seed(0)
        agent = Envelope(FakeEnv(obs_dim=12, n_actions=4, reward_dim=3), batch_size=32, num_sample_w=8, per=True, buffer_size=2048,
                         net_arch=[64, 64, 64], log=False, seed=3, device=cuda, per_on_device=per_dev)
        assert agent.replay_buffer.tree_on_device == per_dev
        store = synthetic_store(2048, 12, 4, 3, seed=1)
        rb = agent.replay_buffer
        rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
        rb.size, rb.ptr = 2048, 0
        rb.mark_all_dirty()
        rb.tree.batch_set(np.arange(2048), np.random.default_rng(2).random(2048) + 0.01)
        agent.global_step = 1
        return agent

    a, b = build(True), build(False)
    for step in range(6):
        rec = []
        for agent in (a, b):
            np.random.seed(70 + step)
            agent.update()
            rec.append((agent._last_inds.copy(), float(agent._last_loss), np.asarray(agent._last_priority).copy(), agent.replay_buffer.min_priority))
        (ia, la, pa, ma), (ib, lb, pb, mb) = rec
        assert np.array_equal(ia, ib), step
        assert la == lb, (step, la, lb)
        assert np.all(np.abs(pa.view(np.int32) - pb.view(np.int32)) <= 1), step
        assert abs(ma - mb) <= 1e-6 * mb
    for va, vb in zip(a.q_net.state_dict().values(), b.q_net.state_dict().values()):
        assert th.equal(va, vb)
    ta, tb = np.concatenate(a.replay_buffer.tree.nodes), np.concatenate(b.replay_buffer.tree.nodes)
    np.testing.assert_allclose(ta, tb, rtol=1e-6)


def test_envelope_checkpoint_resume(cuda, tmp_path):
    """ADVICE r1: train -> save -> load into a fresh agent -> train must continue exactly like the uninterrupted agent: the loaded replay
    buffer gets a new HBM mirror (and a new device sum tree), so captured graphs must be re-captured against it, and the optimiser's
    pointer tables must follow the re-created state tensors."""
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    def build():
        th.manual_seed(0)
        agent = Envelope(FakeEnv(obs_dim=12, n_actions=4, reward_dim=3), batch_size=32, num_sample_w=8, per=True, buffer_size=1024,
                         net_arch=[64, 64, 64], log=False, seed=3, device=cuda, target_net_update_freq=1)  # (load() sets target := online, as the reference)
        store = synthetic_store(1024, 12, 4, 3, seed=1)
        rb = agent.replay_buffer
        rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
        rb.size, rb.ptr = 1024, 0
        rb.mark_all_dirty()
        rb.tree.batch_set(np.arange(1024), np.random.default_rng(2).random(1024) + 0.01)
        agent.global_step = 1
        return agent

    a = build()
    for step in range(3):
        np.random.seed(10 + step)
        a.global_step += 1
        a.update()
    a.save(save_dir=str(tmp_path), filename="ckpt")
    b = build()
    np.random.seed(99)
    b.update()  # b has its own captured graph and optimiser state before loading
    b.load(str(tmp_path / "ckpt.tar"))
    b.np_random = np.random.default_rng(5)
    a.np_random = np.random.default_rng(5)
    b.global_step = a.global_step
    assert np.array_equal(np.concatenate(a.replay_buffer.tree.nodes), np.concatenate(b.replay_buffer.tree.nodes))
    for step in range(3):
        la = []
        for agent in (a, b):
            np.random.seed(40 + step)
            agent.global_step += 1
            agent.update()
            la.append((float(agent._last_loss), agent._last_inds.copy()))
        assert la[0][0] == la[1][0] and np.array_equal(la[0][1], la[1][1]), step
    for va, vb in zip(a.q_net.state_dict().values(), b.q_net.state_dict().values()):
        assert th.equal(va, vb)
