"""CPU pinning of the oracle on the axes the per-row TD kernels are swept over (tests/test_td_kernels_sweep_gpu.py trusts the oracle bit
for bit): D = 1, 5, 8, three nets, the row-map combinations the algorithms pass, and exactly tied inputs.  Each test restates the cited
reference lines in PyTorch on CPU (the arithmetic the reference executes) and compares with oracle/morl_oracle.c.  Targets and indices:
bit-exact; reduced loss scalars: 1e-6 relative (summation order); gradients and einsum-scalarised priorities: the tolerances of
tests/test_oracle_restatements.py, stated at the assert."""

import numpy as np
import pytest
import torch as th
import torch.nn.functional as F

from oracle import oracle as orc

N_NETS = 3
EPS = np.finfo(np.float32).eps


def _q(r, shape, ties):
    """ties: small integers with weights in multiples of 1/8, so every score is exact and equal scores are common."""
    if ties:
        return r.integers(-2, 3, size=shape).astype(np.float32)
    return r.standard_normal(shape).astype(np.float32)


def _w(r, n, D, ties):
    if ties:
        return (r.integers(1, 4, size=(n, D)) / 8.0).astype(np.float32)
    return r.dirichlet(np.ones(D), n).astype(np.float32)


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("D", [1, 5, 8])
def test_critic_min_target_doubled_batch_restates_gpi_pd_445_463(D, ties):
    """gpi_pd.py:425-432 doubles the batch (rewards and dones .repeat(2, 1): the TILE map over B0 rows) with a weight per row; :445-463
    stack the target nets, argmin over nets of the scalarised values, gather, argmax over actions, gather, Bellman."""
    r = np.random.default_rng(D + 10 * ties)
    B0, A = 48, 6
    N = 2 * B0
    q = _q(r, (N_NETS, N, A, D), ties)
    w = _w(r, N, D, ties)
    rew, done = r.standard_normal((B0, D)).astype(np.float32), (r.random(B0) < 0.3).astype(np.float32)
    tq, tw = th.from_numpy(q), th.from_numpy(w)
    s_rewards, s_dones = th.from_numpy(rew).repeat(2, 1), th.from_numpy(done).reshape(-1, 1).repeat(2, 1)
    scal = th.einsum("nbar,br->nba", tq, tw)
    min_inds = th.argmin(scal, dim=0).reshape(1, N, A, 1).expand(1, N, A, D)
    next_q = tq.gather(0, min_inds).squeeze(0)
    max_acts = th.argmax(th.einsum("br,bar->ba", tw, next_q), dim=1)
    target = next_q.gather(1, max_acts.long().reshape(-1, 1, 1).expand(N, 1, D)).reshape(-1, D)
    target = s_rewards + (1 - s_dones) * 0.99 * target
    out, act = orc.critic_min_td(q, w, rew, done, 0.99, orc.DOT_UNFUSED, orc.MAP_BLOCK, orc.MAP_TILE)
    assert np.array_equal(act, max_acts.numpy().astype(np.int32))
    assert np.array_equal(out, target.numpy())
    if ties:  # equal scores from different nets / actions really occur
        assert int((scal[0] == scal[1]).sum()) > 0


@pytest.mark.parametrize("gpi", [False, True])
@pytest.mark.parametrize("D", [1, 5, 8])
def test_td_huber_doubled_batch_restates_gpi_pd_469_487_507_520(D, gpi):
    """gpi_pd.py:469-487 per net on the doubled batch (actions .repeat(2, 1): a_rows = B0, TILE), :507-520 priorities of the first
    len(idxes) = B0 rows from the element-wise max over nets of |td| (or |gtd|), scalarised with the row's weight."""
    r = np.random.default_rng(7 * D + gpi)
    B0, A, mp = 40, 5, 0.01
    N = 2 * B0
    q = (r.standard_normal((N_NETS, N, A, D)) * 0.03).astype(np.float32)
    t = (r.standard_normal((N, D)) * 0.03).astype(np.float32)
    tg = (t + 0.02 * r.standard_normal((N, D))).astype(np.float32) if gpi else None
    act = r.integers(0, A, B0)
    w = r.dirichlet(np.ones(D), N).astype(np.float32)

    def huber(x, min_priority):  # common/networks.py:90-100
        return th.where(x < min_priority, 0.5 * x.pow(2), min_priority * x).mean()

    tq = th.from_numpy(q).requires_grad_(True)
    s_actions = th.from_numpy(act).reshape(-1, 1).repeat(2, 1)
    losses, errs = [], []
    for k in range(N_NETS):
        psi = tq[k].gather(1, s_actions.long().reshape(-1, 1, 1).expand(N, 1, D)).reshape(-1, D)
        td = psi - th.from_numpy(t)
        losses.append(huber(td.abs(), mp))
        errs.append((psi - th.from_numpy(tg)).abs() if gpi else td.abs())
    loss = (1 / N_NETS) * sum(losses)
    loss.backward()
    per = th.einsum("br,br->b", th.from_numpy(w)[:B0], th.max(th.stack(errs), dim=0)[0][:B0].detach()).abs().numpy()
    got_loss, got_grad, got_prio = orc.td_huber(q, act, t, tg, w, mp, B0)
    assert abs(got_loss - float(loss.detach())) <= 1e-6 * abs(float(loss.detach()))
    # the reference's (1 / n) * sum(mean) chain vs the oracle's single double division: 2e-6 relative, as test_oracle_restatements
    np.testing.assert_allclose(got_grad, tq.grad.numpy(), rtol=2e-6, atol=1e-12)
    # einsum on [B0, D] may sum in another order than the oracle's left-to-right dot: 4 eps of the magnitude
    np.testing.assert_allclose(got_prio, per, rtol=0, atol=4 * EPS * float(np.abs(per).max() + 1))


@pytest.mark.parametrize("lam", [0.0, 0.35])
@pytest.mark.parametrize("order", [orc.ROWS_REFERENCE, orc.ROWS_BMAJOR])
@pytest.mark.parametrize("D", [1, 5, 8])
def test_td_mse_restates_envelope_301_313(D, order, lam):
    """envelope.py:301-313 (gather the taken action, MSE, homotopy term on the scalarised values) and :329-331 (priorities of weight 0) in
    both row orders."""
    r = np.random.default_rng(D * 10 + order + int(lam * 100))
    B, W, A = 20, 6, 4
    q = r.standard_normal((W * B, A, D)).astype(np.float32)
    t = r.standard_normal((W * B, D)).astype(np.float32)
    act = r.integers(0, A, B)
    wset = r.dirichlet(np.ones(D), W).astype(np.float32)
    rows = [(i, b) for i in range(W) for b in range(B)] if order == orc.ROWS_REFERENCE else [(i, b) for b in range(B) for i in range(W)]
    w_rows = th.from_numpy(np.stack([wset[i] for i, _ in rows]))
    a_rows = th.from_numpy(np.array([act[b] for _, b in rows]))
    tq = th.from_numpy(q).requires_grad_(True)
    q_value = tq.gather(1, a_rows.long().reshape(-1, 1, 1).expand(W * B, 1, D)).reshape(-1, D)
    loss = F.mse_loss(q_value, th.from_numpy(t))
    if lam > 0:
        loss = (1 - lam) * loss + lam * F.mse_loss(th.einsum("br,br->b", q_value, w_rows), th.einsum("br,br->b", th.from_numpy(t), w_rows))
    loss.backward()
    got_loss, got_grad, got_q, got_prio = orc.td_mse(q, act, t, wset, lam, B, W, order)
    assert abs(got_loss - float(loss.detach())) <= 1e-6 * abs(float(loss.detach()))
    assert np.array_equal(got_q, q_value.detach().numpy())
    np.testing.assert_allclose(got_grad, tq.grad.numpy(), rtol=2e-6, atol=1e-9)  # float autograd chain vs double-then-rounded
    first = [k for k, (i, _) in enumerate(rows) if i == 0]
    per = th.einsum("br,br->b", (q_value.detach() - th.from_numpy(t))[first], w_rows[first]).abs().numpy()
    np.testing.assert_allclose(got_prio, per, rtol=0, atol=4 * EPS * float(np.abs(per).max() + 1))


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("D", [1, 5, 8])
def test_ddqn_target_restates_envelope_442_463(D, ties):
    """envelope.py:442-463 + the Bellman line :298 on the b-major effective batch the Envelope passes (envelope.py:471 of this
    project): row k = b W + i, the weight TILE over the W sampled weights, reward and done BLOCK over the B transitions."""
    r = np.random.default_rng(3 * D + ties)
    B, W, A = 24, 5, 7
    N = B * W
    q_sel, q_eval = _q(r, (N, A, D), ties), r.standard_normal((N, A, D)).astype(np.float32)
    wset = _w(r, W, D, ties)
    rew, done = r.standard_normal((B, D)).astype(np.float32), (r.random(B) < 0.3).astype(np.float32)
    w = th.from_numpy(wset).repeat(B, 1)  # row b W + i -> wset[i]
    s_rew = th.from_numpy(rew).repeat_interleave(W, 0)  # row b W + i -> rew[b]
    s_done = th.from_numpy(done).reshape(-1, 1).repeat_interleave(W, 0)
    max_acts = th.argmax(th.einsum("br,bar->ba", w, th.from_numpy(q_sel)), dim=1)
    tgt = th.from_numpy(q_eval).gather(1, max_acts.long().reshape(-1, 1, 1).expand(N, 1, D)).reshape(-1, D)
    tgt = s_rew + (1 - s_done) * 0.99 * tgt
    out, act = orc.greedy_td(q_sel, q_eval, wset, rew, done, 0.99, orc.DOT_UNFUSED, orc.MAP_TILE, orc.MAP_BLOCK)
    assert np.array_equal(act, max_acts.numpy().astype(np.int32))
    assert np.array_equal(out, tgt.numpy())


@pytest.mark.parametrize("w_rows", ["one", "per_row"])
@pytest.mark.parametrize("D", [1, 5, 8])
def test_actor_critic_targets_restate_capql_gpi_pd_continuous_mosac(D, w_rows):
    """capql.py:329-331, gpi_pd_continuous_action.py:397-403 and mosac_continuous_action.py:438-442 with three critics; the weight is one
    shared row (MOSAC's fixed weight, TILE/BLOCK are the same map there) or one per row (CAPQL / GPI-PD continuous)."""
    r = np.random.default_rng(D + 50 * (w_rows == "one"))
    N = 96
    q = r.standard_normal((N_NETS, N, D)).astype(np.float32)
    q[:, ::5] = r.integers(-2, 3, size=(N_NETS, len(q[0, ::5]), D))  # exact ties between critics
    w = r.dirichlet(np.ones(D), 1 if w_rows == "one" else N).astype(np.float32)
    wf = np.broadcast_to(w, (N, D)).copy()
    rew, done = r.standard_normal((N, D)).astype(np.float32), (r.random(N) < 0.2).astype(np.float32)
    logp = r.standard_normal(N).astype(np.float32)
    tq, tw, tr, td, tl = map(th.from_numpy, (q, wf, rew, done, logp))
    soft = th.min(tq, dim=0)[0] - (0.2 * tl).reshape(-1, 1)
    ref = (tr + (1 - td).reshape(-1, 1) * 0.99 * soft).numpy()
    assert np.array_equal(orc.actor_critic_td(q, None, rew, done, logp, 0.2, 0.99, orc.AC_ELEMENTWISE_MIN), ref)
    inds = th.argmin(th.einsum("nbr,br->nb", tq, tw), dim=0, keepdim=True).reshape(1, -1, 1).expand(1, N, D)
    ref = (tr + (1 - td).reshape(-1, 1) * 0.99 * tq.gather(0, inds).squeeze(0)).numpy()
    assert np.array_equal(orc.actor_critic_td(q, w, rew, done, None, 0.0, 0.99, orc.AC_ARGMIN_GATHER), ref)
    if w_rows == "one":
        w1 = th.from_numpy(w[0])
        mn = th.min(th.stack([th.matmul(tq[n], w1) for n in range(N_NETS)]), dim=0)[0] - (0.2 * tl)
        ref = (th.matmul(tr, w1) + (1 - td) * 0.99 * mn).numpy()
        got = orc.actor_critic_td(q, w, rew, done, logp, 0.2, 0.99, orc.AC_SCALAR_MIN)
        # th.matmul may sum in another order than the oracle's left-to-right dot: 4 eps of the magnitude (test_oracle_restatements)
        np.testing.assert_allclose(got, ref, rtol=0, atol=4 * EPS * float(np.abs(ref).max() + 1))


@pytest.mark.parametrize("D", [1, 5, 8])
def test_oracle_nan_and_neg_inf_rule(D):
    """The rule the kernels follow and the oracle pins (include/morl_b200.h): a NaN score never wins and a row whose scores are all -inf or
    NaN takes candidate 0.  th.argmax would pick the NaN; this is the documented deviation."""
    r = np.random.default_rng(D)
    N, A = 6, 4
    q = r.standard_normal((N, A, D)).astype(np.float32)
    q[0, 0] = np.nan  # NaN first: the best finite action wins
    q[1, 2] = np.nan
    q[2] = -np.inf  # all -inf: action 0
    q[3] = np.nan  # all NaN: action 0
    q[4, 0], q[4, 1:] = -np.inf, np.nan  # -inf then NaN: action 0
    q[5, 3] = np.inf  # +inf wins
    w = r.dirichlet(np.ones(D), N).astype(np.float32)
    s = (q.astype(np.float64) * w[:, None, :]).sum(-1)
    fin = np.where(np.isnan(s), -np.inf, s)
    exp = np.where(fin.max(1) == -np.inf, 0, fin.argmax(1))
    _, act = orc.greedy_td(q, q, w, None, None, 0.0)
    assert np.array_equal(act, exp)
    _, act = orc.critic_min_td(np.stack([q, q + 1]), w, None, None, 0.0)
    assert np.array_equal(act, exp)
    _, pol, act = orc.gpi_envelope(np.stack([q, q + 1]).reshape(2, N, 2, 2, D), w)
    assert np.array_equal(pol * 2 + act, exp)
