"""The MO-PPO kernels of csrc/ppo.cu on the device.

morl_vector_gae_f32 against the unmodified reference's ``_MOPPO__compute_advantages`` (tests/golden/mo_ppo.npz) and against an eager torch
restatement of the reference's loop on the device: returns bit-exact, scalarised advantages within 2 ulp of the magnitude of their
terms (the kernel sums the d products in double and rounds once; torch's matmul rounds its own way).
morl_ppo_loss_f32 against the float64 restatement of tests/ppo_f64.py, including the exact-tie first minibatch (ratio == 1) and ratios
pushed outside the clip band."""

import os

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import _lib, ops
from tests.golden.make_golden_mo_ppo import NEXT_DONE, WEIGHTS, cases, split_gae, synthetic_batch, tag
from tests.ppo_f64 import ppo_loss_f64

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mo_ppo.npz"))
CASES = list(enumerate(cases()))


def _ulp_close(a, b, scale, n=2):
    ulp = np.spacing(np.abs(scale).astype(np.float32)).astype(np.float64)
    return np.all(np.abs(a.astype(np.float64) - b.astype(np.float64)) <= n * ulp)


def eager_gae(rewards, values, dones, next_value, next_done, w, gamma, lam, gae):
    """The reference's Python loop (mo_ppo.py:439-476), op by op, on the device."""
    T, E, d = rewards.shape
    ext = lambda x: x.unsqueeze(1).repeat(1, d)  # noqa: E731
    if gae:
        adv = th.zeros_like(rewards)
        last = 0
        for t in reversed(range(T)):
            if t == T - 1:
                nnt, nv = 1.0 - next_done, next_value
            else:
                nnt, nv = 1.0 - dones[t + 1], values[t + 1]
            nnt = ext(nnt)
            delta = rewards[t] + gamma * nv * nnt - values[t]
            adv[t] = last = delta + gamma * lam * nnt * last
        ret = adv + values
    else:
        ret = th.zeros_like(rewards)
        for t in reversed(range(T)):
            if t == T - 1:
                nnt, nr = 1.0 - next_done, next_value
            else:
                nnt, nr = 1.0 - dones[t + 1], ret[t + 1]
            ret[t] = rewards[t] + gamma * ext(nnt) * nr
        adv = ret - values
    return ret, adv @ w, adv


@pytest.mark.parametrize("k,c", CASES, ids=[tag(c) for _, c in CASES])
def test_gae_matches_reference_golden(cuda, k, c):
    d = c["d"]
    sb, ref = synthetic_batch(k, d), split_gae(G[f"{tag(c)}/gae"], d)
    t = lambda x: th.from_numpy(x).to(cuda)  # noqa: E731
    w = t(WEIGHTS[d])
    ret, adv = ops.vector_gae(t(sb["rewards"]), t(sb["values"]), t(sb["dones"]), t(ref["next_value"]), t(NEXT_DONE), w, 0.995, 0.95, bool(c["gae"]))
    assert np.array_equal(ret.cpu().numpy(), ref["returns"])
    scale = np.abs((ref["returns"] - sb["values"]) * WEIGHTS[d]).sum(-1)
    assert _ulp_close(adv.cpu().numpy(), ref["advantages"], scale)


@pytest.mark.parametrize("T", [1, 7, 2048])
@pytest.mark.parametrize("E", [1, 4])
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("gae", [True, False])
def test_gae_matches_eager_restatement(cuda, T, E, d, gae):
    gen = th.Generator(device="cuda").manual_seed(T * 100 + E * 10 + d)
    rewards = th.randn(T, E, d, device=cuda, generator=gen)
    values = th.randn(T, E, d, device=cuda, generator=gen)
    dones = (th.rand(T, E, device=cuda, generator=gen) < 0.1).float()
    next_value = th.randn(E, d, device=cuda, generator=gen)
    next_done = th.zeros(E, device=cuda)
    next_done[0] = 1.0
    w = th.rand(d, device=cuda, generator=gen)
    ret, adv = ops.vector_gae(rewards, values, dones, next_value, next_done, w, 0.995, 0.95, gae)
    r_ref, a_ref, vec = eager_gae(rewards, values, dones, next_value, next_done, w, 0.995, 0.95, gae)
    assert th.equal(ret, r_ref)
    scale = (vec.abs() * w).sum(-1).cpu().numpy()
    assert _ulp_close(adv.cpu().numpy(), a_ref.cpu().numpy(), scale)


def _loss_inputs(cuda, M, A, d, seed, tie=False, far=False):
    g = np.random.default_rng(seed)
    mean = g.standard_normal((M, A)).astype(np.float32)
    logstd = (g.standard_normal(A) * 0.3).astype(np.float32)
    actions = (mean + np.exp(logstd) * g.standard_normal((M, A))).astype(np.float32)
    value = g.standard_normal((M, d)).astype(np.float32)
    returns = (value + g.standard_normal((M, d)) * 0.5).astype(np.float32)
    old_values = (value + g.standard_normal((M, d)) * 0.3).astype(np.float32)
    adv = g.standard_normal(M).astype(np.float32)
    t = lambda x: th.from_numpy(x).to(cuda)  # noqa: E731
    # old log-probs: the kernel's own new log-probs when tied (ratio == 1 exactly, the first minibatch of an update)
    stats = th.zeros(6, device=cuda)
    if tie:
        # a zero advantage gives a zero policy gradient, so the kernel's log-prob can be read back from old_approx_kl
        lp = np.zeros(M, np.float32)
        for i in range(M):
            r = ops.ppo_loss(t(mean[i:i + 1].repeat(2, 0)), t(logstd), t(value[i:i + 1].repeat(2, 0)), t(actions[i:i + 1].repeat(2, 0)),
                             th.zeros(2, device=cuda), th.zeros(2, device=cuda), t(returns[i:i + 1].repeat(2, 0)), None, 0.2, 0.0, 0.5, False,
                             False, stats)
            lp[i] = -float(stats[3])
        old_lp = lp
    else:
        pert = g.standard_normal(M).astype(np.float32) * 0.05
        if far:
            pert[::3] = g.choice([-1.0, 1.0], len(pert[::3])) * g.uniform(0.3, 2.0, len(pert[::3]))
        lp = (-((actions - mean) ** 2) / (2 * np.exp(logstd) ** 2) - logstd - 0.5 * np.log(2 * np.pi)).sum(1)
        old_lp = (lp + pert).astype(np.float32)
    return dict(mean=mean, logstd=logstd, value=value, actions=actions, old_logprob=old_lp, advantages=adv, returns=returns, old_values=old_values)


@pytest.mark.parametrize("M,A,d", [(32, 3, 2), (256, 6, 2), (300, 17, 3), (2, 1, 1)])
@pytest.mark.parametrize("norm_adv", [True, False])
@pytest.mark.parametrize("clip_vloss", [True, False])
@pytest.mark.parametrize("case", ["tie", "near", "far"])
def test_ppo_loss_matches_f64(cuda, M, A, d, norm_adv, clip_vloss, case):
    x = _loss_inputs(cuda, M, A, d, seed=M * 7 + A + d, tie=case == "tie", far=case == "far")
    t = {k: th.from_numpy(v).to(cuda) for k, v in x.items()}
    stats = th.zeros(6, device=cuda)
    ent_coef = 0.01
    loss, dmean, dlogstd, dvalue = ops.ppo_loss(t["mean"], t["logstd"], t["value"], t["actions"], t["old_logprob"], t["advantages"], t["returns"],
                                                t["old_values"], 0.2, ent_coef, 0.5, norm_adv, clip_vloss, stats)
    ref = ppo_loss_f64(**x, clip_coef=0.2, ent_coef=ent_coef, vf_coef=0.5, norm_adv=norm_adv, clip_vloss=clip_vloss)

    def close(a, b, rel=2e-4):
        b = np.asarray(b, np.float64)
        return np.all(np.abs(np.asarray(a, np.float64) - b) <= rel * max(np.abs(b).max(), 1e-3))

    assert close(loss.item(), ref["loss"])
    assert close(dmean.cpu().numpy(), ref["dmean"])
    assert close(dlogstd.cpu().numpy(), ref["dlogstd"])
    assert close(dvalue.cpu().numpy(), ref["dvalue"])
    s = stats.cpu().numpy()
    for k, name in enumerate(("pg_loss", "v_loss", "entropy")):
        assert close(s[k], ref[name]), name
    assert abs(s[3] - ref["old_approx_kl"]) <= 1e-5 and abs(s[4] - ref["approx_kl"]) <= 1e-5
    assert abs(s[5] - ref["clipfrac"]) <= 1.0 / M + 1e-7  # a ratio within rounding of the band edge may count on either side
    if case == "tie":
        assert s[5] == 0.0 and abs(s[4]) < 1e-7
    if case == "far":
        assert s[5] > 0.2


def test_ppo_loss_clipfrac_accumulates(cuda):
    x = _loss_inputs(cuda, 64, 3, 2, seed=3, far=True)
    t = {k: th.from_numpy(v).to(cuda) for k, v in x.items()}
    stats = th.zeros(6, device=cuda)
    for _ in range(3):
        ops.ppo_loss(t["mean"], t["logstd"], t["value"], t["actions"], t["old_logprob"], t["advantages"], t["returns"], t["old_values"], 0.2, 0.0,
                     0.5, True, True, stats)
    one = th.zeros(6, device=cuda)
    ops.ppo_loss(t["mean"], t["logstd"], t["value"], t["actions"], t["old_logprob"], t["advantages"], t["returns"], t["old_values"], 0.2, 0.0, 0.5,
                 True, True, one)
    assert float(stats[5]) == pytest.approx(3 * float(one[5]), rel=1e-6) and th.equal(stats[:5], one[:5])


def test_ppo_loss_refuses_one_row_normalisation(cuda):
    z = lambda *s: th.zeros(*s, device=cuda)  # noqa: E731
    with pytest.raises(_lib.MorlB200Error, match="M >= 2"):
        ops.ppo_loss(z(1, 3), z(3), z(1, 2), z(1, 3), z(1), z(1), z(1, 2), z(1, 2), 0.2, 0.0, 0.5, True, True, z(6))
