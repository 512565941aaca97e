"""Float64 restatement of the discrete-action MOSAC update lines (reference single_policy/ser/mosac_discrete_action.py:452-498) and
the first-order error bound of the fp32 kernels against it.  Shared by tests/test_discrete_sac_oracle_cpu.py (the C oracle) and
tests/test_discrete_sac_gpu.py (the kernels, which equal the oracle bit for bit).

Derivation (u = 2^-24, per row, actions a in ascending order; see include/morl_b200.h for the exact fp32 operations):
  z_a = x_a - mx is one rounding; e^ and log are the library's own routines, <= 1 ulp and <= 1.5 ulp (checked on CPU), so
    e_a = e^z_a carries a relative error <= (2 + |z_a|) u,  s = sum e_a  <= (A + 2 + max|z|) u,
    lse = log s an absolute error <= 2u max(1, |lse|) + rel(s),  logp_a = z_a - lse an absolute error
    zeta_a <= u (|z_a| + |logp_a|) + err(lse),  and p_a = e_a / s a relative error rho_a <= rel(e_a) + rel(s) + u.
  A scalarised critic value w.q (D products, D - 1 sums) is off by <= (D + 1) u sum_r |w_r q_r| =: mu_a; the NaN-propagating
    min over critics adds nothing.
  A weighted row sum S = sum_a p_a y_a, with y_a computed with an absolute error delta_a, is then off by
    <= sum_a p_a (rho_a |y_a| + delta_a) + (A + 1) u sum_a p_a |y_a|.
  target: y_a = m_a - alpha logp_a, delta_a = mu_a + alpha zeta_a + 2u |y_a|; then w.r (mu over the reward) and the three-op Bellman
    line add (D + 4) u (|w.r| + gamma |v|).
  actor loss: y_a = f_a = alpha logp_a - m_a, same delta_a; the 256-row float block partials and the double final sum add
    <= 10 u sum_k |l_k| before the division by N*A.
  dL/dlogits: the closed form p_j (f_j - l) / (N A) drops autograd's alpha p_j (1 - sum_a p_a) / (N A), which is O(A u alpha p_j);
    its error is p_j (rho_j |f_j - l| + delta_j + err(l) + 3u |f_j - l| + A u alpha) / (N A).
  temperature loss: y_a = t (logp_a + H), t = -e^log_alpha (relative error 1u), delta_a = |t| (zeta_a + u |logp_a + H|) + 3u |y_a|.
A -inf logit is left out of every sum (p = 0, gradient 0); the float64 restatement applies the same rule.
"""

from __future__ import annotations

import numpy as np
import torch as th

U = 2.0**-24


def _softmax64(logits):
    x = th.as_tensor(np.asarray(logits, np.float64))
    logp = th.log_softmax(x, dim=1)
    p = th.softmax(x, dim=1)
    return x, p, logp


def _scal(q_nets, w, w_map, N):
    """[n_nets, N, A] scalarised critics and [n, N, A] sums of |w_r q_r| in float64"""
    q = th.as_tensor(np.asarray(q_nets, np.float64))
    D = q.shape[-1]
    w = th.as_tensor(np.asarray(w, np.float64)).reshape(-1, D)
    rows = w.shape[0]
    if rows == N:
        wk = w
    elif rows == 1:
        wk = w.expand(N, D)
    elif w_map == 0:
        wk = w[th.arange(N) % rows]
    else:
        wk = w[th.arange(N) // (N // rows)]
    s = (q * wk[None, :, None, :]).sum(-1)
    mag = (q * wk[None, :, None, :]).abs().sum(-1)
    return s, mag, wk


def _nanmin(s):
    m = s[0]
    for n in range(1, s.shape[0]):
        m = th.where(th.isnan(m) | th.isnan(s[n]), th.full_like(m, float("nan")), th.minimum(m, s[n]))
    return m


def _row_terms(logits, D):
    x, p, logp = _softmax64(logits)
    A = x.shape[1]
    mx = x.max(1, keepdim=True).values
    z = (x - mx).abs()
    lse = th.logsumexp(x - mx, 1, keepdim=True)
    excl = th.isneginf(logp)
    zf = th.where(excl, th.zeros_like(z), z)
    rel_s = (A + 2 + zf.max(1, keepdim=True).values) * U
    err_lse = 2 * U * th.clamp(lse.abs(), min=1.0) + rel_s
    zeta = U * (zf + th.where(excl, th.zeros_like(logp), logp).abs()) + err_lse
    rho = (2 + zf) * U + rel_s + U
    p = th.where(excl, th.zeros_like(p), p)
    logp_safe = th.where(excl, th.zeros_like(logp), logp)
    return p, logp_safe, excl, zeta, rho, A


def _wsum(p, rho, y, delta, A):
    s = (p * y).sum(1)
    err = (p * (rho * y.abs() + delta)).sum(1) + (A + 1) * U * (p * y.abs()).sum(1)
    return s, err


def target(q_nets, logits, w, reward, done, alpha, gamma, w_map=1):
    """(target [N], bound [N]) in float64"""
    n_nets, N, A, D = np.shape(q_nets)
    p, logp, excl, zeta, rho, A = _row_terms(logits, D)
    s, mag, wk = _scal(q_nets, w, w_map, N)
    m = _nanmin(s)
    mu = (D + 1) * U * mag.max(0).values
    y = m - alpha * logp
    y = th.where(excl, th.zeros_like(y), y)
    v, ev = _wsum(p, rho, y, mu + alpha * zeta + 2 * U * y.abs(), A)
    r = th.as_tensor(np.asarray(reward, np.float64)).reshape(N, D)
    d = th.as_tensor(np.asarray(done, np.float64)).reshape(N)
    wr = (wk * r).sum(1)
    t = wr + (1 - d) * gamma * v
    bound = (1 - d) * gamma * ev + (D + 4) * U * ((wk * r).abs().sum(1) + gamma * v.abs()) + U * t.abs() + 1e-37
    return t.numpy(), bound.numpy()


def actor_loss(logits, q_nets, w, alpha, log_alpha=None, target_entropy=0.0, w_map=1):
    """float64 values and bounds: (loss, loss_bound, dlogits [N, A], dlogits_bound, alpha_loss, alpha_loss_bound, dlog_alpha, dlog_alpha_bound);
    dlogits (and d alpha_loss / d log_alpha) come from float64 autograd of the reference expression, with the -inf rule."""
    n_nets, N, A, D = np.shape(q_nets)
    p_, logp_, excl, zeta, rho, A = _row_terms(logits, D)
    s, mag, _ = _scal(q_nets, w, w_map, N)
    m = _nanmin(s)
    mu = (D + 1) * U * mag.max(0).values
    # autograd of (probs * (alpha * log_pi - min_q)).mean() (:478-484), the -inf actions masked out of the product
    x = th.as_tensor(np.asarray(logits, np.float64)).clone().requires_grad_(True)
    logp = th.log_softmax(x, 1)
    p = th.softmax(x, 1)
    f = alpha * logp - m
    keep = ~excl
    terms = th.where(keep, p * th.where(keep, f, th.zeros_like(f)), th.zeros_like(f))
    loss = terms.mean()
    (g,) = th.autograd.grad(loss, x)
    f_d = th.where(excl, th.zeros_like(f), f.detach())
    lrow, el = _wsum(p_, rho, f_d, mu + alpha * zeta + 2 * U * f_d.abs(), A)
    NA = N * A
    loss_bound = (el.sum() + 10 * U * lrow.abs().sum()) / NA + U * abs(float(loss.detach()))
    diff = (f_d - lrow[:, None]).abs()
    g_bound = p_ * (rho * diff + mu + alpha * zeta + 2 * U * f_d.abs() + el[:, None] + 3 * U * diff + A * U * alpha) / NA + 1e-37
    out = [float(loss.detach()), float(loss_bound), g.numpy(), g_bound.numpy()]
    if log_alpha is None:
        return out + [None, None, None, None]
    la = th.tensor([float(log_alpha)], dtype=th.float64, requires_grad=True)
    uu = th.where(excl, th.zeros_like(logp_), logp_ + target_entropy)
    aterms = p_ * (-la.exp() * uu)
    aloss = aterms.mean()
    (dla,) = th.autograd.grad(aloss, la)
    t = float(np.exp(np.float64(log_alpha)))
    y = -t * uu
    arow, ea = _wsum(p_, rho, y, t * (zeta + U * uu.abs()) + 3 * U * y.abs(), A)
    a_bound = (ea.sum() + 10 * U * arow.abs().sum()) / NA + U * abs(float(aloss.detach())) + 1e-37
    return out + [float(aloss.detach()), float(a_bound), float(dla[0]), float(a_bound + 2 * U * abs(float(dla[0])))]
