"""NLMOPPO's kernels and learner on the GPU: the objective GAE bit for bit, the fused minibatch update against a float64 restatement,
the forward and commit kernels against torch, the bindings' argument contract, and the learner's graph, determinism, early-stopping,
schedule, utility, reset and fallback behaviour."""

import numpy as np
import pytest
import torch as th
from torch.distributions import Categorical

from morl_baselines_b200 import _lib, nl_ppo_ops, ops
from morl_baselines_b200.single_policy.ser.nl_mo_ppo import NLMOPPO, Agent
from tests import nl_ppo_f64
from tests.nl_ppo_standin import RingEnv, RingVecEnv

pytestmark = pytest.mark.gpu
DEV = th.device("cuda")


def _agent(S, d, Dp, A, seed=0, head_scale=1.0):
    th.manual_seed(seed)
    ag = Agent(RingVecEnv(1, obs_dim=S, n_actions=A, d=d), d, Dp).to(DEV)
    with th.no_grad():
        ag.actor[4].weight.mul_(head_scale * 100)  # logits of order one, so ratios leave the clip band
    return ag


def _net(ag, S, d, Dp, A, pref=None):
    params = list(ag.parameters())
    grads = [th.zeros_like(p) for p in params]
    pref = th.randn(Dp, device=DEV) if Dp and pref is None else pref
    return nl_ppo_ops.NlPpoNet(S, d, Dp, A, params, grads, pref), params, grads, pref


# ---- objective GAE ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,E,D", [(1, 1, 1), (37, 5, 3), (130, 9, 8), (16, 64, 2)])
def test_gae_objectives_bit_exact_and_scalarised_gae_unchanged(T, E, D):
    g = th.Generator(device="cpu").manual_seed(T * 100 + E)
    r = th.randn(T, E, D, generator=g).to(DEV)
    v = th.randn(T, E, D, generator=g).to(DEV)
    dones = (th.rand(T, E, generator=g) < 0.2).float().to(DEV)
    nv, nd = th.randn(E, D, generator=g).to(DEV), (th.rand(E, generator=g) < 0.3).float().to(DEV)
    gamma, lam = 0.99, 0.95
    # the reference's loop (nl_mo_ppo.py:295-307) on the device in float32
    adv = th.zeros_like(r)
    last = th.zeros(E, D, device=DEV)
    for t in reversed(range(T)):
        nnt, nxt = ((1.0 - nd).unsqueeze(-1), nv) if t == T - 1 else ((1.0 - dones[t + 1]).unsqueeze(-1), v[t + 1])
        delta = r[t] + gamma * nxt * nnt - v[t]
        last = delta + gamma * lam * nnt * last
        adv[t] = last
    ret = adv + v
    k_ret, k_adv = nl_ppo_ops.vector_gae_objectives(r, v, dones, nv, nd, gamma, lam)
    assert th.equal(k_ret, ret) and th.equal(k_adv, adv)
    w = th.rand(D, generator=g).to(DEV)
    s_ret, s_adv = ops.vector_gae(r, v, dones, nv, nd, w, gamma, lam)
    expect = sum(adv[..., o].double() * w[o].double() for o in range(D)).float()  # products exact in double, summed in objective order
    assert th.equal(s_ret, ret) and th.equal(s_adv, expect)


# ---- the fused minibatch update ------------------------------------------------------------------------------------------------------
# Gradient error relative to the largest gradient element of its tensor, and statistics relative to max(1, |value|), over CASES and the
# unequal-tiles case.  Measured worst on one H100 80GB HBM3 (700 W power limit): gradients 7.7e-7, statistics 6.5e-8.
GRAD_TOL = 1e-5
STAT_TOL = 1e-6

CASES = [  # M, B, S, d, Dp, A, norm_adv, clip_vloss, ent_coef
    (2, 9, 2, 2, 2, 4, True, True, 0.01),
    (33, 70, 2, 2, 0, 2, True, False, 0.0),
    (250, 300, 7, 3, 3, 6, True, True, 0.01),
    (1000, 1024, 2, 1, 0, 32, False, True, 0.01),
    (4096, 5000, 5, 8, 8, 9, True, True, 0.05),
    (517, 600, 240, 8, 8, 3, True, False, 0.01),
]


def _batch(B, S, d, A, seed):
    g = th.Generator(device="cpu").manual_seed(seed)
    obs, acc = th.randn(B, S, generator=g), th.randn(B, d, generator=g)
    actions = th.randint(0, A, (B,), generator=g)
    adv, ret, ov = th.randn(B, d, generator=g), th.randn(B, d, generator=g), th.randn(B, d, generator=g)
    return [t.to(DEV) for t in (obs, acc, actions, adv, ret, ov)]


def _check_update(case, zero_head=False):
    """The update pair against the float64 restatement; returns (worst relative gradient error, worst statistics error)."""
    M, B, S, d, Dp, A, norm_adv, clip_vloss, ent = case
    ag = _agent(S, d, Dp, A, seed=M)
    if zero_head:  # logits exactly 0: the kernel's log-probability is -logf(A), the same bits as torch's float32 log-softmax on the device
        with th.no_grad():
            ag.actor[4].weight.zero_()
            ag.actor[4].bias.zero_()
    net, params, grads, pref = _net(ag, S, d, Dp, A)
    obs, acc, actions, adv, ret, ov = _batch(B, S, d, A, M)
    perm = th.randperm(B, device=DEV)[:M].contiguous()
    w = th.randn(d, device=DEV)
    # old log-probabilities: the current ones moved by noise, so ratios fall inside and outside the clip band
    with th.no_grad():
        _, logits = nl_ppo_f64.agent_forward([p.double() for p in params],
                                             th.cat([obs, acc] + ([pref.expand(B, -1)] if Dp else []), 1).double())
        logp = (logits - th.logsumexp(logits, 1, keepdim=True)).gather(1, actions.view(-1, 1)).squeeze(1).float()
    old_logp = logp + 0.3 * th.randn(B, device=DEV)
    if zero_head:  # every third row: old log-probability equal to the new one, a ratio of exactly 1
        z = th.zeros(B, A, device=DEV)
        exact = (z - th.logsumexp(z, 1, keepdim=True))[:, 0]
        old_logp[::3] = exact[::3]
    stats, loss = th.zeros(6, device=DEV), th.zeros(1, device=DEV)
    ws = net.workspace(DEV)
    nl_ppo_ops.nl_ppo_update(net, obs, acc, actions, old_logp, adv, ret, ov, perm, w, 0.2, ent, 0.5, norm_adv, clip_vloss, stats, ws, loss_out=loss)
    ref_loss, ref_grads, ref_stats = nl_ppo_f64.minibatch(params, obs, acc, actions, old_logp, adv, ret, ov, perm, pref, w, 0.2, ent, 0.5,
                                                          norm_adv, clip_vloss)
    g_err = 0.0
    for i, (g, rg) in enumerate(zip(grads, ref_grads)):
        err = (g.double() - rg).abs().max().item() / max(rg.abs().max().item(), 1e-12)
        g_err = max(g_err, err)
        assert err < GRAD_TOL, (i, err)
    s_err = abs(loss.item() - ref_loss.item()) / max(1.0, abs(ref_loss.item()))
    for k, name in enumerate(("pg", "v", "ent", "okl", "kl", "clip")):
        s_err = max(s_err, abs(stats[k].item() - ref_stats[name]) / max(1.0, abs(ref_stats[name])))
    assert s_err <= STAT_TOL, s_err
    # both sides of the clip band were exercised, and the result repeats bit for bit
    assert 0.0 < ref_stats["clip"] < 1.0 or M < 8
    first = [g.clone() for g in grads]
    stats2 = th.zeros(6, device=DEV)
    nl_ppo_ops.nl_ppo_update(net, obs, acc, actions, old_logp, adv, ret, ov, perm, w, 0.2, ent, 0.5, norm_adv, clip_vloss, stats2, ws)
    assert all(th.equal(a, b) for a, b in zip(first, grads)) and th.equal(stats, stats2)
    return g_err, s_err


@pytest.mark.parametrize("case", CASES)
def test_update_matches_float64(case):
    _check_update(case)


def test_update_unequal_tile_shares_and_ratios_of_exactly_one():
    """M = 2100 rows are 132 tiles: the first 4 CTAs take two tiles, the other 124 one.  Every third row has a ratio of exactly 1."""
    _check_update((2100, 2200, 3, 2, 2, 4, True, True, 0.01), zero_head=True)


def test_update_refuses_single_row_with_norm_adv():
    S, d, Dp, A = 2, 2, 2, 4
    net, params, grads, pref = _net(_agent(S, d, Dp, A), S, d, Dp, A)
    obs, acc, actions, adv, ret, ov = _batch(8, S, d, A, 0)
    perm = th.zeros(1, dtype=th.int64, device=DEV)
    with pytest.raises(_lib.MorlB200Error, match="M >= 2"):
        nl_ppo_ops.nl_ppo_update(net, obs, acc, actions, th.zeros(8, device=DEV), adv, ret, ov, perm, th.ones(d, device=DEV), 0.2, 0.0, 0.5, True,
                                 True, th.zeros(6, device=DEV), net.workspace(DEV))


# ---- forward and commit ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,d,Dp,A,N", [(2, 2, 2, 4, 1), (7, 3, 0, 6, 64), (240, 8, 8, 32, 100)])
def test_forward_matches_torch(S, d, Dp, A, N):
    ag = _agent(S, d, Dp, A)
    net, params, _, pref = _net(ag, S, d, Dp, A)
    obs, acc = th.randn(N, S, device=DEV), th.randn(N, d, device=DEV)
    logits, values, arg = th.empty(N, A, device=DEV), th.empty(N, d, device=DEV), th.empty(N, dtype=th.int32, device=DEV)
    nl_ppo_ops.nl_ppo_forward(net, obs, acc, logits, values, arg)
    with th.no_grad():
        rv, rl = ag.get_value(obs, acc, pref), ag.actor(ag._build_aug_obs(obs, acc, pref))
    th.testing.assert_close(values, rv, rtol=1e-5, atol=1e-5)
    th.testing.assert_close(logits, rl, rtol=1e-5, atol=1e-6)
    assert th.equal(arg.long(), th.argmax(logits, 1))
    # one pinned row, and first-occurrence argmax on tied logits
    with th.no_grad():
        ag.actor[4].weight.zero_()
        ag.actor[4].bias.copy_(th.tensor([0.5 if a in (1, A - 1) else 0.0 for a in range(A)]))
    row_o, row_a = obs[:1].cpu().pin_memory(), acc[:1].cpu().pin_memory()
    pin_arg, pin_log = th.zeros(1, dtype=th.int32).pin_memory(), th.zeros(1, A).pin_memory()
    nl_ppo_ops.nl_ppo_forward(net, row_o, row_a, logits_out=pin_log, argmax_out=pin_arg)
    th.cuda.synchronize()
    assert int(pin_arg[0]) == (1 if A > 1 else 0)
    assert th.equal(pin_log, ag.actor[4].bias.detach().cpu().view(1, A))


def test_commit_matches_device_expression():
    T, E, S, d, A, gamma = 3, 37, 4, 3, 5, 0.97
    g = th.Generator(device="cpu").manual_seed(3)
    stores = dict(obs_store=th.zeros(T, E, S, device=DEV), acc_store=th.zeros(T, E, d, device=DEV), done_store=th.zeros(T, E, device=DEV),
                  rew_store=th.zeros(T, E, d, device=DEV), act_store=th.zeros(T, E, dtype=th.int64, device=DEV),
                  logp_store=th.zeros(T, E, device=DEV))
    nobs, nacc = th.randn(E, S, generator=g).to(DEV), th.randn(E, d, generator=g).to(DEV) * 10
    ndone = (th.rand(E, generator=g) < 0.2).float().to(DEV)
    ts = th.randint(0, 400, (E,), generator=g, dtype=th.int32).to(DEV)
    staged = th.randn(E, S + d + 2, generator=g).to(DEV)
    staged[:, S + d] = (th.rand(E, generator=g) < 0.2).float().to(DEV)
    staged[:, S + d + 1] = (th.rand(E, generator=g) < 0.2).float().to(DEV)
    logits, action = th.randn(E, A, device=DEV), th.randint(0, A, (E,), device=DEV)
    before = (nobs.clone(), nacc.clone(), ndone.clone(), ts.clone())
    nl_ppo_ops.nl_ppo_commit(staged, logits, action, 1, gamma, **stores, next_obs=nobs, next_acc=nacc, next_done=ndone, timestep=ts)
    done = th.logical_or(staged[:, S + d] != 0, staged[:, S + d + 1] != 0).float()
    r = staged[:, S:S + d]
    # the reference's expression (nl_mo_ppo.py:274-275) evaluated on the device
    exp_acc = (before[1] + (gamma ** before[3].unsqueeze(-1)) * r) * (1.0 - done.unsqueeze(-1))
    exp_ts = (before[3].unsqueeze(-1) + 1) * (1 - done.int().unsqueeze(-1))
    assert th.equal(nacc, exp_acc) and th.equal(ts, exp_ts.view(-1))
    assert th.equal(nobs, staged[:, :S]) and th.equal(ndone, done)
    assert th.equal(stores["obs_store"][1], before[0]) and th.equal(stores["acc_store"][1], before[1])
    assert th.equal(stores["done_store"][1], before[2]) and th.equal(stores["rew_store"][1], r) and th.equal(stores["act_store"][1], action)
    th.testing.assert_close(stores["logp_store"][1], Categorical(logits=logits).log_prob(action), rtol=0, atol=1e-6)
    assert stores["obs_store"][0].abs().sum() == 0 and stores["obs_store"][2].abs().sum() == 0


# ---- argument contract of nl_ppo_ops -------------------------------------------------------------------------------------------------
def _rows():
    """binding -> (call(**kw), kw of one valid call): every tensor argument of every binding in nl_ppo_ops."""
    S, d, Dp, A, B, M, T, E = 2, 2, 2, 4, 20, 8, 3, 5
    net, params, grads, pref = _net(_agent(S, d, Dp, A), S, d, Dp, A)
    obs, acc, actions, adv, ret, ov = _batch(B, S, d, A, 1)
    z = lambda *s, dt=th.float32: th.zeros(*s, device=DEV, dtype=dt)  # noqa: E731
    return {
        "vector_gae_objectives": (nl_ppo_ops.vector_gae_objectives,
                                  dict(rewards=z(T, E, d), values=z(T, E, d), dones=z(T, E), next_value=z(E, d), next_done=z(E), gamma=0.9,
                                       gae_lambda=0.9, returns_out=z(T, E, d), adv_out=z(T, E, d))),
        "nl_ppo_update": (lambda **k: nl_ppo_ops.nl_ppo_update(net, **k),
                          dict(obs=obs, acc=acc, actions=actions, old_logprob=z(B), advantages=adv, returns=ret, old_values=ov,
                               perm=th.arange(M, device=DEV), loss_weights=z(d), clip_coef=0.2, ent_coef=0.0, vf_coef=0.5, norm_adv=True,
                               clip_vloss=True, stats=z(6), workspace=net.workspace(DEV), loss_out=z(1))),
        "nl_ppo_forward": (lambda **k: nl_ppo_ops.nl_ppo_forward(net, **k),
                           dict(obs=z(E, S), acc=z(E, d), logits_out=z(E, A), values_out=z(E, d), argmax_out=z(E, dt=th.int32))),
        "nl_ppo_commit": (nl_ppo_ops.nl_ppo_commit,
                          dict(staged=z(E, S + d + 2), logits=z(E, A), action=z(E, dt=th.int64), step=0, gamma=0.9, obs_store=z(T, E, S),
                               acc_store=z(T, E, d), done_store=z(T, E), rew_store=z(T, E, d), act_store=z(T, E, dt=th.int64),
                               logp_store=z(T, E), next_obs=z(E, S), next_acc=z(E, d), next_done=z(E), timestep=z(E, dt=th.int32))),
    }


def test_every_launch_of_nl_ppo_ops_has_a_row():
    import inspect

    chunks = inspect.getsource(nl_ppo_ops).split("\ndef ")[1:]
    launched = {c.split("(", 1)[0] for c in chunks if "_launch(" in c}
    assert launched == set(_rows())


@pytest.mark.parametrize("binding", ["vector_gae_objectives", "nl_ppo_update", "nl_ppo_forward", "nl_ppo_commit"])
def test_bindings_refuse_bad_tensors_by_name(binding):
    call, kw = _rows()[binding]
    call(**kw)  # the valid call runs
    th.cuda.synchronize()
    for name, t in kw.items():
        if not isinstance(t, th.Tensor):
            continue
        bad_dtype = th.float64 if t.dtype != th.float64 else th.float32
        bads = [t.cpu(), t.to(bad_dtype)]
        if name != "perm":  # a minibatch of any length is valid
            bads.append(t.reshape(-1)[:-1] if t.numel() > 1 else t.reshape(1, 1, 1))
        for bad in bads:
            before = ops.launch_count
            with pytest.raises(_lib.MorlB200Error, match=name):
                call(**{**kw, name: bad})
            assert ops.launch_count == before, name


# ---- the learner -----------------------------------------------------------------------------------------------------------------------
def u_lin(v):
    return (v * th.tensor([0.7, 0.3], device=v.device)).sum()


def u_cheb(v):  # smooth Chebyshev-like utility
    return -th.logsumexp(-8.0 * (v - th.tensor([-1.0, -2.0], device=v.device)), 0) / 8.0


def _learner(seed=3, num_envs=8, num_steps=16, **kw):
    th.manual_seed(seed)
    np.random.seed(seed)
    kw = {"num_minibatches": 4, "update_epochs": 4, "total_timesteps": 3 * num_envs * num_steps, "seed": seed, **kw}
    return NLMOPPO(0, RingVecEnv(num_envs), num_steps=num_steps, device=DEV, **kw)


def _train(agent, u=u_lin, pref=None, seed=11, n_actions=4):
    th.manual_seed(seed)
    th.cuda.manual_seed(seed)
    return agent.train(RingEnv(n_actions=n_actions), u, pref, deterministic=True)


def _params(agent):
    return [p.detach().clone() for p in agent.agent.parameters()]


def test_learner_graph_and_eager_identical_and_runs_repeat():
    runs = []
    for graph in (True, False, True):
        ag = _learner(use_cuda_graph=graph, anneal_lr=True)
        assert ag.fused
        res = _train(ag, u_cheb, pref=[0.4, 0.6])
        runs.append((res, _params(ag), ag.values.clone(), ag.acc_rewards.clone()))
    for other in runs[1:]:
        assert np.array_equal(runs[0][0], other[0])
        assert all(th.equal(a, b) for a, b in zip(runs[0][1], other[1]))
        assert th.equal(runs[0][2], other[2]) and th.equal(runs[0][3], other[3])


def test_learner_matches_reference_expressions():
    """One update of the kernels against the reference's update expression (the fallback) from the same rollout and shuffles."""
    for kw in ({}, {"norm_adv": False, "clip_vloss": False, "ent_coef": 0.0}, {"num_minibatches": 3}):
        a, b = _learner(**kw), _learner(**kw)
        for ag in (a, b):
            ag.num_iterations = 1
        _train(a, u_cheb)
        _train(b, u_cheb)
        for name in ("obs", "acc_rewards", "actions", "rewards", "dones"):
            assert th.equal(getattr(a, name), getattr(b, name)), name
        with th.no_grad():
            for p, q in zip(b.agent.parameters(), a.agent.parameters()):
                q.copy_(p)
        a._compute_advantages_and_returns()
        b._compute_advantages_and_returns()
        b.fused = False
        ra, rb = a.update(), b.update()
        for p, q in zip(a.agent.parameters(), b.agent.parameters()):
            th.testing.assert_close(p, q, rtol=1e-4, atol=2e-5)
        assert abs(ra[5] - rb[5]) < 1e-6 and abs(float(ra[0]) - float(rb[0])) < 1e-4 * max(1.0, abs(float(rb[0])))
        assert a.rng.bit_generator.state == b.rng.bit_generator.state


def test_target_kl_stops_after_the_reference_number_of_shuffles():
    ag = _learner(target_kl=1e-12)
    _train(ag)
    B = ag.batch_size
    rng = np.random.default_rng(ag.seed)
    inds = np.arange(B)
    for _ in range(ag.num_iterations):  # one epoch per update: approx_kl of the first epoch already exceeds 1e-12
        inds = np.arange(B)
        rng.shuffle(inds)
    assert rng.bit_generator.state == ag.rng.bit_generator.state
    assert set(ag._graphs) == {"epoch"}


def test_schedule_utility_and_pref_change_without_recapture():
    ag = _learner(anneal_lr=True)
    _train(ag, u_lin)
    graph = ag._graphs["all"].graph.graph
    assert graph is not None
    w1 = ag._w.clone()
    _train(ag, u_cheb, pref=[0.2, 0.8])
    assert ag._graphs["all"].graph.graph is graph
    assert not th.equal(w1, ag._w)
    assert th.equal(ag._pref, th.tensor([0.2, 0.8], device=DEV))
    assert ag._lr.item() == pytest.approx(ag.learning_rate / ag.num_iterations)


def test_reset_agent_in_place_matches_a_fresh_agent():
    ag = _learner()
    _train(ag)
    graph = ag._graphs["all"].graph.graph
    storages = [p.data_ptr() for p in ag.agent.parameters()]
    th.manual_seed(123)
    ag.reset_agent(ag.num_objectives)
    th.manual_seed(123)
    fresh = Agent(ag.envs, ag.num_objectives, ag.num_objectives)
    assert [p.data_ptr() for p in ag.agent.parameters()] == storages
    assert all(th.equal(p.cpu(), q) for p, q in zip(ag.agent.parameters(), fresh.parameters()))
    assert all(float(st["step"]) == 0 for st in ag.optimizer.state.values())
    assert ag.u_func is None and ag.pref is None
    _train(ag)
    assert ag._graphs["all"].graph.graph is graph
    ag.reset_agent(0)  # another input width: a new Agent, graphs dropped
    assert ag.agent.pref_dim == 0 and len(ag._graphs) == 0
    _train(ag)


def test_unsupported_shape_takes_the_reference_expressions():
    big = NLMOPPO(0, RingVecEnv(2, n_actions=40), num_steps=8, num_minibatches=2, total_timesteps=32, device=DEV, seed=1)
    assert not big.fused and not nl_ppo_ops.nl_ppo_supported(2, 2, 2, 40, 8)
    with pytest.raises(_lib.MorlB200Error):
        nl_ppo_ops.NlPpoNet(2, 2, 2, 40, list(big.agent.parameters()))
    res = _train(big, n_actions=40)
    assert np.all(np.isfinite(res))


def test_policy_evaluate_paths_agree():
    ag = _learner()
    _train(ag)
    det = ag.policy_evaluate(RingEnv(), eval_episodes=2, deterministic=True)
    ag.fused = False
    assert np.array_equal(det, ag.policy_evaluate(RingEnv(), eval_episodes=2, deterministic=True))
    ag.fused = True
    th.cuda.manual_seed(5)
    s1 = ag.policy_evaluate(RingEnv(), eval_episodes=2)
    th.cuda.manual_seed(5)
    assert np.array_equal(s1, ag.policy_evaluate(RingEnv(), eval_episodes=2))
