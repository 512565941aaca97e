"""EUPG without a device: the accrued-reward buffer against the reference's golden vectors (tests/golden/eupg.npz), the accrued-reward
promotion rule, the float64 restatement of the update (tests/eupg_f64.py) against torch autograd in float64, and the range of the fused
kernels (``ops.eupg_supported``)."""

import os

import numpy as np
import pytest
import torch as th
from torch.distributions import Categorical

from morl_baselines_b200 import ops
from morl_baselines_b200.common.accrued_reward_buffer import AccruedRewardReplayBuffer
from morl_baselines_b200.single_policy.esr.eupg import PolicyNet, accrue, kernel_takes
from tests import eupg_f64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "eupg.npz"))


def test_buffer_matches_reference():
    buf = AccruedRewardReplayBuffer((3,), (1,), rew_dim=2, max_size=5, obs_dtype=np.int32, action_dtype=np.int32)
    rng = np.random.default_rng(12)
    for i in range(8):
        obs = rng.uniform(-4, 4, 3)
        buf.add(obs, rng.standard_normal(2).astype(np.float32), i % 3, rng.standard_normal(2), obs + 0.5, i == 7)
    for k in ("obs", "next_obs", "actions", "rewards", "accrued_rewards", "dones"):
        a = getattr(buf, k)
        assert a.dtype == GOLDEN[f"buffer/{k}"].dtype, k
        np.testing.assert_array_equal(a, GOLDEN[f"buffer/{k}"], err_msg=k)
    assert [buf.ptr, buf.size] == list(GOLDEN["buffer/ptr_size"])
    np.random.seed(5)
    for k, v in zip(("obs", "accrued_rewards", "actions", "rewards", "next_obs", "dones"), buf.sample(4, use_cer=True)):
        np.testing.assert_array_equal(v, GOLDEN[f"buffer/sample_{k}"], err_msg=k)
    buf.cleanup()
    assert [buf.ptr, buf.size, len(buf)] == list(GOLDEN["buffer/after_cleanup"])


def test_buffer_truncates_float_observations_and_pickles():
    import pickle

    buf = AccruedRewardReplayBuffer((2,), (1,), rew_dim=1, max_size=3, obs_dtype=np.int32, action_dtype=np.int32)
    buf.add(np.array([1.9, -1.9]), np.zeros(1, np.float32), 2, np.ones(1), np.array([2.5, -0.5]), False)
    np.testing.assert_array_equal(buf.obs[0], [1, -1])
    np.testing.assert_array_equal(buf.next_obs[0], [2, 0])
    obs, acc, act, rew, nxt, done = buf.get_all_data(to_tensor=True, device="cpu")
    assert obs.dtype == th.int32 and act.dtype == th.int32 and obs.shape == (1, 2)
    clone = pickle.loads(pickle.dumps(buf))
    np.testing.assert_array_equal(clone.obs, buf.obs)
    assert (clone.ptr, clone.size) == (buf.ptr, buf.size)


def test_accrued_reward_follows_torch_promotion():
    # float64 rewards are added in float64 and rounded once: 1 + (2^-24 + 2^-50) rounds up to 1 + 2^-23, while a float32 add of the
    # reward rounded to float32 (2^-24) ties to even and stays at 1
    r64 = np.array([2.0 ** -24 + 2.0 ** -50], np.float64)
    acc = th.ones(1, dtype=th.float32)
    accrue(acc, r64)
    assert acc.dtype == th.float32
    assert acc.item() == np.float32(1.0 + 2.0 ** -23)
    acc32 = th.ones(1, dtype=th.float32)
    accrue(acc32, r64.astype(np.float32))
    assert acc32.item() == 1.0
    # the reference's own rule, for a sequence of rewards
    rng = np.random.default_rng(0)
    ref = th.zeros(3, dtype=th.float32)
    mine = th.zeros(3, dtype=th.float32)
    for _ in range(50):
        r = rng.standard_normal(3) * 1e3
        ref += th.from_numpy(r)
        accrue(mine, r)
    assert th.equal(ref, mine)


def _params(arch, S, d, A, seed):
    th.manual_seed(seed)
    net = PolicyNet((S,), A, d, arch).double()
    return net, [p.detach().numpy().copy() for p in net.parameters()]


@pytest.mark.parametrize("arch,S,d,A,T", [([50], 1, 2, 2, 9), ([17, 5], 4, 3, 5, 1), ([8, 8, 8, 8], 6, 2, 32, 30), ([4], 3, 2, 1, 7)])
def test_f64_restatement_matches_autograd(arch, S, d, A, T):
    net, params = _params(arch, S, d, A, 3)
    rng = np.random.default_rng(1)
    obs = th.from_numpy(rng.integers(-3, 4, (T, S)).astype(np.int32))
    acc = th.from_numpy(rng.standard_normal((T, d)))
    actions = th.from_numpy(rng.integers(0, A, (T, 1)).astype(np.int32))
    v = th.from_numpy(rng.standard_normal(T))
    v[0] = 0.0
    dist = Categorical(net(obs, acc))
    loss = -th.mean(dist.log_prob(actions.squeeze()) * v)
    grads = th.autograd.grad(loss, list(net.parameters()))
    x = np.concatenate([obs.numpy().astype(np.float64), acc.numpy()], axis=1)
    ref_loss, ref_grads = eupg_f64.update(params, x, actions.numpy(), v.numpy(), eps=float(np.finfo(np.float64).eps))
    np.testing.assert_allclose(ref_loss, loss.item(), rtol=1e-10, atol=1e-12)
    for g, r in zip(grads, ref_grads):
        np.testing.assert_allclose(r, g.numpy(), rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(eupg_f64.probs(params, x), Categorical(net(obs, acc)).probs.detach().numpy(), rtol=1e-10, atol=1e-14)


def test_f64_clamp_passes_no_gradient():
    # a row whose taken action has p < eps: its log-probability is log(eps) and contributes no gradient; A = 1 has p = 1, clamped too
    params = [np.zeros((2, 2)), np.array([0.0, -40.0])]
    x = np.zeros((2, 2))
    loss, grads = eupg_f64.update(params, x, [1, 1], [1.0, 2.0])
    assert all(np.all(g == 0) for g in grads)
    np.testing.assert_allclose(loss, -np.log(eupg_f64.EPS) * 1.5)
    loss1, grads1 = eupg_f64.update([np.ones((1, 3)), np.ones(1)], np.ones((4, 3)), [0] * 4, np.ones(4))
    assert all(np.all(g == 0) for g in grads1)
    # the same through torch autograd in float32
    net = PolicyNet((1,), 2, 1, [3])
    with th.no_grad():
        net.net[2].bias.copy_(th.tensor([0.0, -40.0]))
    loss_t = -th.mean(Categorical(net(th.zeros(2, 1), th.zeros(2, 1))).log_prob(th.tensor([1, 1])) * th.ones(2))
    assert all(th.all(g == 0) for g in th.autograd.grad(loss_t, list(net.parameters())))


def test_returns_restatement_is_the_reference_loop():
    rng = np.random.default_rng(2)
    r = rng.standard_normal((37, 3)).astype(np.float32)
    flip = th.from_numpy(r.copy()).flip(dims=[0])
    c = th.zeros(3)
    for i in range(len(r)):
        c = 0.99 * c + flip[i]
        flip[i] = c
    np.testing.assert_array_equal(eupg_f64.returns(r, 0.99), flip.flip(dims=[0]).numpy())


def test_supported_range_needs_no_device():
    assert ops.eupg_supported(1, 2, [50], 2)
    assert ops.eupg_supported(255, 1, [256, 256, 256, 256], 32)
    assert ops.eupg_supported(1, 8, [1], 1)
    assert ops.eupg_supported(248, 8, [17, 5, 33], 5)
    assert not ops.eupg_supported(256, 1, [50], 2)  # S + d = 257
    assert not ops.eupg_supported(4, 9, [50], 2)  # d > MORL_MAX_D
    assert not ops.eupg_supported(4, 2, [257], 2)
    assert not ops.eupg_supported(4, 2, [0], 2)
    assert not ops.eupg_supported(4, 2, [50] * 5, 2)
    assert not ops.eupg_supported(4, 2, [], 2)
    assert not ops.eupg_supported(4, 2, [50], 33)
    assert not ops.eupg_supported(4, 2, [50], 0)
    assert ops.eupg_workspace_bytes(1, 2, [50], 2) == ops.eupg_workspace_bytes(1, 2, [50], 2) > 0
    assert ops.eupg_workspace_bytes(4, 2, [50], 33) == 0


def test_kernel_takes_only_device_float32_rows():
    cpu = th.device("cpu")
    assert kernel_takes(th.zeros(5), 5, cpu)
    assert kernel_takes(th.tensor(1.0), 5, cpu)
    assert not kernel_takes(th.zeros(5, 1), 5, cpu)
    assert not kernel_takes(th.zeros(5, dtype=th.float64), 5, cpu)
    assert not kernel_takes(th.zeros(4), 5, cpu)
    assert not kernel_takes(1.5, 5, cpu)
    assert not kernel_takes(th.zeros(5), 5, th.device("cuda", 0))


def test_learner_needs_a_device():
    from morl_baselines_b200._lib import MorlB200Error
    from morl_baselines_b200.single_policy.esr.eupg import EUPG
    from tests.eupg_standin import EupgEnv

    with pytest.raises(MorlB200Error):
        EUPG(EupgEnv(), lambda r, w=None: r, log=False, device="cpu")
