"""EUPG on the GPU: the returns kernel bit for bit against the reference's loop, the fused update and probabilities kernels against the
float64 restatement (tests/eupg_f64.py) and torch, determinism, refusals, and the learner against the reference's golden vectors
(tests/golden/eupg.npz) on both the kernel path and the eager path."""

import copy
import ctypes
import os
import tempfile

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import _lib, ops
from morl_baselines_b200.common.evaluation import eval_mo_reward_conditioned
from morl_baselines_b200.single_policy.esr.eupg import EUPG, PolicyNet, policy_tensors
from tests import eupg_f64
from tests.eupg_standin import EupgEnv, RecordingScalarization, fixed_episode, pack_calls, weighted_sum_scalarization
from tests.golden import make_golden_eupg as mg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "eupg.npz"))
RTOL, ATOL = 1e-4, 2e-6  # on parameters, as the PCN tests
DEV = th.device("cuda")


def _reference_returns(r: np.ndarray, gamma: float) -> np.ndarray:
    """eupg.py:263-270 verbatim in float32 torch."""
    rewards = th.from_numpy(r.copy())
    flip_rewards = rewards.flip(dims=[0])
    cumulative_rewards = th.zeros(r.shape[1])
    for i in range(len(rewards)):
        cumulative_rewards = gamma * cumulative_rewards + flip_rewards[i]
        flip_rewards[i] = cumulative_rewards
    return flip_rewards.flip(dims=[0]).numpy()


@pytest.mark.parametrize("T", [1, 2, 31, 32, 33, 200, 4097])
@pytest.mark.parametrize("d", [1, 2, 3, 8])
def test_returns_bit_identical_to_reference_loop(T, d):
    rng = np.random.default_rng(T * 10 + d)
    block = (rng.standard_normal((T, d + 3)) * 5).astype(np.float32)  # rewards are columns 2..2+d of a wider staged block
    dev = th.from_numpy(block).to(DEV)
    for gamma in (0.0, 0.5, 0.99, 1.0):
        out = ops.eupg_returns(dev[:, 2:2 + d], gamma).cpu().numpy()
        np.testing.assert_array_equal(out, _reference_returns(block[:, 2:2 + d], gamma), err_msg=f"gamma={gamma}")


def _stage(obs, acc, actions, rewards=None):
    """One interleaved device block like the learner's: obs int32 bits | acc | action int32 bits | rewards."""
    T, S = obs.shape
    d = acc.shape[1]
    host = np.zeros((T, S + 2 * d + 1), np.float32)
    host.view(np.int32)[:, :S] = obs
    host[:, S:S + d] = acc
    host.view(np.int32)[:, S + d] = actions
    if rewards is not None:
        host[:, S + d + 1:] = rewards
    rows = th.from_numpy(host).to(DEV)
    return rows[:, :S].view(th.int32), rows[:, S:S + d], rows[:, S + d].view(th.int32)


def _net(arch, S, d, A, seed):
    th.manual_seed(seed)
    net = PolicyNet((S,), A, d, arch).to(DEV)
    with th.no_grad():  # wider logits than the orthogonal init gives, so p spans a useful range
        net.net[-1].weight.mul_(3.0)
        net.net[-1].bias.uniform_(-1, 1)
    return net


def _kernel_update(net, arch, S, d, A, obs, acc, actions, v):
    params = policy_tensors(net)
    grads = [th.full_like(p, float("nan")) for p in params]  # overwritten, never accumulated
    knet = ops.EupgNet(S, d, arch, A, params, grads)
    loss = th.zeros(1, device=DEV)
    ops.eupg_update(knet, *_stage(obs, acc, actions), th.from_numpy(np.asarray(v, np.float32)).to(DEV), loss, knet.workspace(DEV))
    return loss.item(), [g.cpu().numpy() for g in grads]


UPDATE_CASES = [  # (net_arch, S, d, A, T)
    *[([50], 1, 2, 2, T) for T in (1, 15, 16, 17, 200, 5000, 100000)],
    ([64, 64], 8, 3, 5, 200),
    ([256], 250, 6, 32, 517),
    ([17, 5, 33], 4, 2, 1, 33),
    ([17, 5, 33], 4, 2, 5, 1000),
    ([32, 48, 20, 256], 10, 8, 32, 1000),
    ([256, 256], 8, 3, 4, 5000),
    ([1], 1, 1, 2, 40),
]


@pytest.mark.parametrize("arch,S,d,A,T", UPDATE_CASES)
def test_update_matches_f64(arch, S, d, A, T):
    rng = np.random.default_rng(T + S)
    net = _net(arch, S, d, A, seed=S + A)
    obs = rng.integers(-3, 4, (T, S)).astype(np.int32)
    acc = (rng.standard_normal((T, d)) * 2).astype(np.float32)
    actions = rng.integers(0, A, T).astype(np.int32)
    v = rng.standard_normal(T).astype(np.float32)
    v[::7] = 0.0
    loss, grads = _kernel_update(net, arch, S, d, A, obs, acc, actions, v)
    params = [p.detach().cpu().numpy().astype(np.float64) for p in policy_tensors(net)]
    x = np.concatenate([obs.astype(np.float64), acc.astype(np.float64)], axis=1)
    ref_loss, ref_grads = eupg_f64.update(params, x, actions, v.astype(np.float64))
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-4, atol=1e-6)
    for k, (g, r) in enumerate(zip(grads, ref_grads)):
        np.testing.assert_allclose(g, r, rtol=1e-4, atol=1e-5 * max(1e-3, np.abs(r).max()), err_msg=f"tensor {k}")
    if A == 1:
        assert all(np.all(g == 0) for g in grads)


def test_update_scalar_v_and_clamped_rows():
    arch, S, d, A, T = [50], 3, 2, 4, 300
    rng = np.random.default_rng(5)
    net = _net(arch, S, d, A, seed=1)
    with th.no_grad():
        net.net[-1].bias[0] = -40.0  # action 0 has p < 2^-23 on every row: its log-probability is clamped
    obs = rng.integers(-2, 3, (T, S)).astype(np.int32)
    acc = rng.standard_normal((T, d)).astype(np.float32)
    params = [p.detach().cpu().numpy().astype(np.float64) for p in policy_tensors(net)]
    x = np.concatenate([obs, acc], axis=1).astype(np.float64)
    # every row takes the clamped action: every gradient is exactly zero, the loss is -log(eps) * mean(v)
    zero_acts = np.zeros(T, np.int32)
    v = rng.standard_normal(T).astype(np.float32)
    loss, grads = _kernel_update(net, arch, S, d, A, obs, acc, zero_acts, v)
    assert all(np.all(g == 0) for g in grads)
    np.testing.assert_allclose(loss, -np.log(np.float32(eupg_f64.EPS)) * v.astype(np.float64).mean(), rtol=1e-5)
    # mixed rows and a scalar v broadcast over T
    actions = rng.integers(0, A, T).astype(np.int32)
    params_t = policy_tensors(net)
    grads_t = [th.zeros_like(p) for p in params_t]
    knet = ops.EupgNet(S, d, arch, A, params_t, grads_t)
    loss_t = th.zeros(1, device=DEV)
    ops.eupg_update(knet, *_stage(obs, acc, actions), th.tensor(-0.75, device=DEV), loss_t, knet.workspace(DEV))
    ref_loss, ref_grads = eupg_f64.update(params, x, actions, -0.75)
    np.testing.assert_allclose(loss_t.item(), ref_loss, rtol=1e-4)
    for g, r in zip(grads_t, ref_grads):
        np.testing.assert_allclose(g.cpu().numpy(), r, rtol=1e-4, atol=1e-5 * max(1e-3, np.abs(r).max()))


@pytest.mark.parametrize("T", [17, 100000])
def test_update_is_deterministic_and_workspace_does_not_grow(T):
    arch, S, d, A = [256, 256], 8, 3, 4
    rng = np.random.default_rng(T)
    net = _net(arch, S, d, A, seed=2)
    obs = rng.integers(-3, 4, (T, S)).astype(np.int32)
    acc = rng.standard_normal((T, d)).astype(np.float32)
    actions = rng.integers(0, A, T).astype(np.int32)
    v = rng.standard_normal(T).astype(np.float32)
    a = _kernel_update(net, arch, S, d, A, obs, acc, actions, v)
    b = _kernel_update(net, arch, S, d, A, obs, acc, actions, v)
    assert a[0] == b[0]
    for x, y in zip(a[1], b[1]):
        np.testing.assert_array_equal(x, y)
    per_cta = sum(p.numel() for p in policy_tensors(net)) * 4 + 8
    assert ops.eupg_workspace_bytes(S, d, arch, A) == 128 * per_cta


@pytest.mark.parametrize("N", [1, 7, 1000])
@pytest.mark.parametrize("pinned", [False, True])
def test_probs_match_torch(N, pinned):
    arch, S, d, A = [50], 5, 3, 6
    net = _net(arch, S, d, A, seed=N)
    rng = np.random.default_rng(N)
    x = rng.standard_normal((N, S + d)).astype(np.float32)
    knet = ops.EupgNet(S, d, arch, A, policy_tensors(net))
    if pinned:
        xin, out = th.from_numpy(x).pin_memory(), th.zeros((N, A)).pin_memory()
    else:
        xin, out = th.from_numpy(x).to(DEV), th.zeros((N, A), device=DEV)
    ops.eupg_probs(knet, xin, out)
    th.cuda.synchronize()
    with th.no_grad():
        ref = th.distributions.Categorical(net(th.from_numpy(x[:, :S]).to(DEV), th.from_numpy(x[:, S:]).to(DEV))).probs.cpu().numpy()
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(out.cpu().numpy(), eupg_f64.probs([p.detach().cpu().numpy() for p in policy_tensors(net)], x), rtol=1e-5,
                               atol=1e-7)


def test_unsupported_shapes_are_refused_and_the_learner_falls_back():
    lib = _lib.load()
    hidden = (ctypes.c_int * 1)(50)
    dummy = th.zeros(64, device=DEV)
    table = (ctypes.c_void_p * 4)(*([dummy.data_ptr()] * 4))
    p = dummy.data_ptr()
    # 33 actions, then S + d = 257: MORL_ERR_UNSUPPORTED, no launch; bad shapes and NULL pointers: their own codes
    assert lib.morl_eupg_update_f32(table, table, p, p, p, 300, p, 1, 4, 4, 2, hidden, 1, 33, p, p, None) == -4
    assert lib.morl_eupg_update_f32(table, table, p, p, p, 300, p, 1, 4, 255, 2, hidden, 1, 2, p, p, None) == -4
    assert lib.morl_eupg_probs_f32(table, p, 1, 4, 2, hidden, 1, 33, p, None) == -4
    assert lib.morl_eupg_returns_f32(p, 9, 4, 0, 0.5, p, None) == -2  # no objectives (any d >= 1 is taken)
    assert lib.morl_eupg_update_f32(table, table, None, p, p, 300, p, 1, 4, 4, 2, hidden, 1, 2, p, p, None) == -1
    th.cuda.synchronize()
    # a 300-wide hidden layer is outside the kernels' range: the learner runs the reference's expression through autograd
    env = EupgEnv(obs_dim=3, n_actions=3, reward_dim=2, seed=9)
    th.manual_seed(0)
    agent = EUPG(env, weighted_sum_scalarization([0.5, 0.5]), weights=np.array([0.5, 0.5]), net_arch=[300], log=False, device=DEV)
    assert not agent.fused
    assert agent.device == th.device("cuda", th.cuda.current_device())
    th.manual_seed(0)
    ref = PolicyNet((3,), 3, 2, [300]).to(DEV)
    opt = th.optim.Adam(ref.parameters(), lr=agent.learning_rate)
    for tr in fixed_episode(env, np.random.default_rng(3), 25):
        agent.buffer.add(*tr)
    obs, acc, act, rew, _, _ = agent.buffer.get_all_data(to_tensor=True, device=DEV)
    fwd = th.from_numpy(eupg_f64.returns(rew.cpu().numpy(), agent.gamma)).to(DEV)
    loss = -th.mean(ref.distribution(obs, acc).log_prob(act.squeeze()) * (fwd @ th.tensor([0.5, 0.5], device=DEV)))
    opt.zero_grad()
    loss.backward()
    opt.step()
    agent.update()
    for a, b in zip(agent.net.parameters(), ref.parameters()):
        np.testing.assert_allclose(a.detach().cpu().numpy(), b.detach().cpu().numpy(), rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(agent._loss.item(), loss.item(), rtol=1e-5)


def test_other_scalarisation_outputs_take_the_eager_path():
    env = EupgEnv(obs_dim=3, n_actions=3, reward_dim=2, seed=9)
    for out, fused in ((lambda c: c.sum(1), True), (lambda c: c.sum(), True), (lambda c: c.sum(1, keepdim=True), False),
                       (lambda c: c.sum(1).double(), False)):
        agent = EUPG(env, lambda r, w=None, out=out: out(r) if isinstance(r, th.Tensor) else float(np.sum(r)), log=False, device=DEV)
        for tr in fixed_episode(env, np.random.default_rng(3), 12):
            agent.buffer.add(*tr)
        before = [p.detach().clone() for p in agent.net.parameters()]
        agent.update()
        assert agent.last_update_fused == fused
        assert np.isfinite(agent._loss.item())
        assert any(not th.equal(a, b) for a, b in zip(before, agent.net.parameters()))


def _assert_params(net, prefix):
    for k, v in net.state_dict().items():
        np.testing.assert_allclose(v.cpu().numpy(), GOLDEN[f"{prefix}/{k}"], rtol=RTOL, atol=ATOL, err_msg=f"{prefix}/{k}")


@pytest.mark.parametrize("name", list(mg.UPDATE_CASES))
@pytest.mark.parametrize("fused", [True, False])
def test_update_matches_golden(name, fused):
    c = mg.UPDATE_CASES[name]
    env = EupgEnv(**c["env"], seed=c["seed"])
    th.manual_seed(c["seed"])
    agent = EUPG(env, weighted_sum_scalarization(c["weights"]), weights=np.array(c["weights"]), log=False, device=DEV, **c["ctor"])
    for k, v in agent.net.state_dict().items():
        np.testing.assert_array_equal(v.cpu().numpy(), GOLDEN[f"update_{name}/init/{k}"])
    assert agent.fused
    agent.fused = fused
    losses = []
    for k, T in enumerate(c["lengths"]):
        for tr in fixed_episode(env, np.random.default_rng(1000 * c["seed"] + k), T):
            agent.buffer.add(*tr)
        agent.update()
        assert agent.last_update_fused == fused
        losses.append(agent._loss.item())
        agent.buffer.cleanup()
        _assert_params(agent.net, f"update_{name}/after{k}")
    np.testing.assert_allclose(losses, GOLDEN[f"update_{name}/loss"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("name", list(mg.TRAIN_CASES))
@pytest.mark.parametrize("fused", [True, False])
def test_train_matches_golden(name, fused):
    c = mg.TRAIN_CASES[name]
    env = EupgEnv(**c["env"])
    scal = RecordingScalarization(env.reward_dim)
    th.manual_seed(c["seed"])
    agent = EUPG(env, scal, weights=np.array(c["weights"]), log=False, device=DEV, **c["ctor"])
    agent.fused = fused
    actions = []
    step = env.step

    def recording(a):
        actions.append(a)
        return step(a)

    env.step = recording
    agent.train(total_timesteps=c["steps"])
    assert agent.last_update_fused == fused
    np.testing.assert_array_equal(np.array(actions), GOLDEN[f"train_{name}/actions"])
    kinds, rets, ws, fwd, lens = pack_calls(scal.calls)
    np.testing.assert_array_equal(kinds, GOLDEN[f"train_{name}/call_kinds"])
    np.testing.assert_array_equal(rets, GOLDEN[f"train_{name}/call_returns"])
    np.testing.assert_array_equal(ws, GOLDEN[f"train_{name}/call_weights"])
    np.testing.assert_array_equal(lens, GOLDEN[f"train_{name}/call_forward_len"])
    np.testing.assert_array_equal(fwd, GOLDEN[f"train_{name}/call_forward"])
    assert agent.num_episodes == int(GOLDEN[f"train_{name}/num_episodes"])
    _assert_params(agent.net, f"train_{name}/final")


def _trained_agent(seed=3):
    env = EupgEnv(obs_dim=3, n_actions=3, reward_dim=2, seed=seed)
    th.manual_seed(seed)
    agent = EUPG(env, RecordingScalarization(2), weights=np.array([0.5, 0.5]), log=False, device=DEV, buffer_size=64)
    agent.train(total_timesteps=150)
    return agent


def test_save_load_round_trip():
    agent = _trained_agent()
    d = agent.get_save_dict(save_replay_buffer=True)
    assert set(d) == {"policy_net_state_dict", "optimizer_state_dict", "policy_weights", "replay_buffer"}
    assert set(agent.get_save_dict(save_replay_buffer=False)) == {"policy_net_state_dict", "optimizer_state_dict", "policy_weights"}
    with tempfile.TemporaryDirectory() as tmp:
        agent.save(save_dir=tmp, filename="eupg.pth", save_replay_buffer=True)
        th.manual_seed(99)
        other = EUPG(EupgEnv(obs_dim=3, n_actions=3, reward_dim=2, seed=5), RecordingScalarization(2), weights=np.ones(2), log=False,
                     device=DEV, buffer_size=64)
        other.load(path=os.path.join(tmp, "eupg.pth"))
    for a, b in zip(agent.net.parameters(), other.net.parameters()):
        assert th.equal(a, b)
    for sa, sb in zip(agent.optimizer.state.values(), other.optimizer.state.values()):
        for k in sa:
            assert th.equal(sa[k].cpu(), sb[k].cpu()), k
    np.testing.assert_array_equal(other.weights, agent.weights)
    np.testing.assert_array_equal(other.buffer.obs, agent.buffer.obs)
    # both keep training identically on the kernel path after the load
    for ag in (agent, other):
        for tr in fixed_episode(EupgEnv(obs_dim=3, n_actions=3, reward_dim=2, seed=1), np.random.default_rng(0), 30):
            ag.buffer.add(*tr)
        ag.scalarization = weighted_sum_scalarization([0.5, 0.5])
        ag.update()
    for a, b in zip(agent.net.parameters(), other.net.parameters()):
        assert th.equal(a, b)


def test_deepcopy_consumes_rng_like_the_reference_and_copies_parameters():
    agent = _trained_agent(seed=4)
    state = th.get_rng_state()
    copied = copy.deepcopy(agent)
    after = th.get_rng_state()
    th.set_rng_state(state)
    PolicyNet(agent.observation_shape, agent.action_dim, agent.reward_dim, agent.net_arch)  # what the copy's constructor draws
    assert th.equal(th.get_rng_state(), after)
    for a, b in zip(agent.net.parameters(), copied.net.parameters()):
        assert th.equal(a, b) and a.data_ptr() != b.data_ptr()
    assert [p for g in copied.optimizer.param_groups for p in g["params"]] == list(copied.net.parameters())
    assert copied.global_step == agent.global_step
    assert copied.buffer is not agent.buffer
    np.testing.assert_array_equal(copied.buffer.obs, agent.buffer.obs)
    copied.train(total_timesteps=40)  # the copy trains on its own kernels
    assert not all(th.equal(a, b) for a, b in zip(agent.net.parameters(), copied.net.parameters()))


def test_esr_evaluation_runs_with_the_agent():
    agent = _trained_agent(seed=6)
    env = EupgEnv(obs_dim=3, n_actions=3, reward_dim=2, seed=11)
    scal, disc_scal, vec, disc_vec = eval_mo_reward_conditioned(agent, env, scalarization=np.dot, w=np.array([0.5, 0.5]))
    assert vec.shape == (2,) and np.isfinite(scal) and np.isfinite(disc_scal)
    res = agent.policy_eval_esr(env, scalarization=np.dot, weights=np.array([0.5, 0.5]), log=False)
    assert len(res) == 4
    dagent = EUPG(EupgEnv(n_actions=2, reward_dim=2, discrete_obs=5, seed=2), RecordingScalarization(2), weights=np.ones(2), log=False,
                  device=DEV)
    assert dagent.eval(3, np.zeros(2)) in (0, 1)


@pytest.mark.parametrize("T,d", [(1, 9), (300, 9), (2049, 17), (40, 300)])
def test_returns_cover_any_number_of_objectives(T, d):
    rng = np.random.default_rng(T + d)
    block = rng.standard_normal((T, d + 1)).astype(np.float32)
    out = ops.eupg_returns(th.from_numpy(block).to(DEV)[:, 1:], 0.97).cpu().numpy()
    np.testing.assert_array_equal(out, _reference_returns(block[:, 1:], 0.97))


def test_learner_with_more_objectives_than_the_kernels_take():
    # reward_dim 9 > MORL_MAX_D: the update runs through autograd, the returns still on the kernel, and match the reference's expression
    env = EupgEnv(obs_dim=3, n_actions=3, reward_dim=9, seed=4)
    w = np.linspace(0.1, 0.9, 9)
    th.manual_seed(2)
    agent = EUPG(env, weighted_sum_scalarization(w), weights=w, log=False, device=DEV)
    assert not agent.fused
    th.manual_seed(2)
    ref = PolicyNet((3,), 3, 9, [50]).to(DEV)
    opt = th.optim.Adam(ref.parameters(), lr=agent.learning_rate)
    for k, T in enumerate((30, 1, 17)):
        for tr in fixed_episode(env, np.random.default_rng(k), T):
            agent.buffer.add(*tr)
        obs, acc, act, rew, _, _ = agent.buffer.get_all_data(to_tensor=True, device=DEV)
        fwd = th.from_numpy(_reference_returns(rew.cpu().numpy(), agent.gamma)).to(DEV)
        loss = -th.mean(ref.distribution(obs, acc).log_prob(act.squeeze()) * (fwd @ th.as_tensor(w, dtype=th.float32, device=DEV)))
        opt.zero_grad()
        loss.backward()
        opt.step()
        agent.update()
        agent.buffer.cleanup()
        assert not agent.last_update_fused
        np.testing.assert_allclose(agent._loss.item(), loss.item(), rtol=1e-5, atol=1e-7)
        for a, b in zip(agent.net.parameters(), ref.parameters()):
            np.testing.assert_allclose(a.detach().cpu().numpy(), b.detach().cpu().numpy(), rtol=RTOL, atol=ATOL)
    agent.train(total_timesteps=60)  # acting and training end to end at d = 9


def test_update_reads_the_staged_views_in_place_and_checks_shapes():
    arch, S, d, A, T = [50], 3, 2, 4, 64
    rng = np.random.default_rng(0)
    net = _net(arch, S, d, A, seed=0)
    params = policy_tensors(net)
    grads = [th.zeros_like(p) for p in params]
    knet = ops.EupgNet(S, d, arch, A, params, grads)
    ws, loss = knet.workspace(DEV), th.zeros(1, device=DEV)
    obs, acc, act = _stage(rng.integers(-2, 3, (T, S)).astype(np.int32), rng.standard_normal((T, d)).astype(np.float32),
                           rng.integers(0, A, T).astype(np.int32), rng.standard_normal((T, d)).astype(np.float32))
    v = th.randn(T, device=DEV)
    th.cuda.synchronize()
    before = th.cuda.memory_stats()["allocation.all.allocated"]
    ops.eupg_update(knet, obs, acc, act, v, loss, ws)  # strided views of one block: no copy is made
    assert th.cuda.memory_stats()["allocation.all.allocated"] == before
    bad = [
        lambda: ops.eupg_update(knet, obs[:, :2], acc, act, v, loss, ws),  # S mismatch
        lambda: ops.eupg_update(knet, obs, acc[:, :1], act, v, loss, ws),  # d mismatch
        lambda: ops.eupg_update(knet, obs, acc.t().contiguous().t(), act, v, loss, ws),  # not rows of the same block
        lambda: ops.eupg_update(knet, obs, acc, act, v, th.zeros(1, device=DEV, dtype=th.float64), ws),
        lambda: ops.eupg_update(knet, obs, acc, act, v, th.zeros(0, device=DEV), ws),
        lambda: ops.eupg_update(knet, obs, acc, act, v, loss, ws[:1]),  # workspace too small
        lambda: ops.eupg_update(knet, obs, acc, act, v[:5], loss, ws),
        lambda: ops.eupg_update(ops.EupgNet(S, d, arch, A, params), obs, acc, act, v, loss, ws),  # no gradient tables
        lambda: ops.eupg_probs(knet, th.zeros(2, S + d + 1, device=DEV), th.zeros(2, A, device=DEV)),
        lambda: ops.eupg_probs(knet, th.zeros(2, S + d, device=DEV), th.zeros(3, A, device=DEV)),
        lambda: ops.eupg_probs(knet, th.zeros(2, S + d, device=DEV), th.zeros(2, A + 1, device=DEV)),
        lambda: ops.eupg_returns(th.zeros(4, 2, device=DEV), 0.9, out=th.zeros(4, 3, device=DEV)),
        lambda: ops.eupg_returns(th.zeros(4, 2, device=DEV), 0.9, out=th.zeros(2, 4, device=DEV).t()),
        lambda: ops.eupg_returns(th.zeros(2, 4, device=DEV).t(), 0.9),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(_lib.MorlB200Error):
            call()
    th.cuda.synchronize()
