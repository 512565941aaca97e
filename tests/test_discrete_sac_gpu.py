"""Discrete-action MOSAC kernels (csrc/discrete_sac.cu): morl_discrete_sac_target_f32 and morl_discrete_sac_actor_loss_f32 equal the
plain-C restatement tests/discrete_sac_oracle.c bit for bit, and lie within the float64 bound derived in tests/discrete_sac_f64.py of the
reference lines mosac_discrete_action.py:452-498 (dL/dlogits and d alpha_loss / d log_alpha against float64 autograd of the
reference expression).

Error bound, in brief (the derivation is the docstring of tests/discrete_sac_f64.py): with u = 2^-24, the portable e^ and log at <= 1
and <= 1.5 ulp, p_a carries a relative error rho_a <= (A + 5 + 2 |x_a - max x|) u and logp_a an absolute error
zeta_a <= u (|x_a - max x| + |logp_a| + 2 max(1, |log s|) + A + 2); a row sum sum_a p_a y_a with y_a off by delta_a is then off by
sum_a p_a (rho_a |y_a| + delta_a) + (A + 1) u sum_a p_a |y_a|, where delta_a collects the scalarisation ((D + 1) u sum |w q|),
alpha zeta_a and the two roundings of y_a.  The loss adds 10 u sum_k |l_k| for the block partials; the closed-form gradient drops
alpha p_j (1 - sum p) (<= A u alpha p_j).  Every comparison below uses that bound per element.
"""

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import ops
from tests import discrete_sac_oracle as orc
from tests import discrete_sac_f64 as f64

pytestmark = pytest.mark.gpu


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32).reshape(-1), np.asarray(b, np.float32).reshape(-1)
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb)
    assert np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _inputs(rng, N, A, D, n_nets, w_rows, scale=2.0):
    q = (rng.standard_normal((n_nets, N, A, D)) * scale).astype(np.float32)
    logits = (rng.standard_normal((N, A)) * scale).astype(np.float32)
    w = rng.dirichlet(np.ones(D), w_rows).astype(np.float32)
    r = rng.standard_normal((N, D)).astype(np.float32)
    d = (rng.random(N) < 0.5).astype(np.float32)
    return q, logits, w, r, d


def _check(cuda, q, logits, w, r, d, alpha, w_map, gamma=0.99, la=-0.4, H=0.7, f64_check=True):
    T = lambda x: th.from_numpy(np.ascontiguousarray(x)).to(cuda)  # noqa: E731
    a_dev = th.tensor([alpha], dtype=th.float32, device=cuda)
    t = ops.discrete_sac_target(T(q), T(logits), T(w), T(r), T(d), a_dev, gamma, w_map=w_map).cpu().numpy()
    _bits_equal(t, orc.discrete_sac_target(q, logits, w, r, d, alpha, gamma, w_map))
    la_dev = th.tensor([la], dtype=th.float32, device=cuda)
    loss, g, aloss, dla = ops.discrete_sac_actor_loss(T(logits), T(q), T(w), a_dev, la_dev, H, w_map=w_map)
    ol, og, oal, odla = orc.discrete_sac_actor_loss(logits, q, w, alpha, la, H, w_map)
    _bits_equal(loss.cpu().numpy(), [ol])
    _bits_equal(g.cpu().numpy(), og)
    _bits_equal(aloss.cpu().numpy(), [oal])
    _bits_equal(dla.cpu().numpy(), [odla])
    if f64_check:
        t64, tb = f64.target(q, logits, w, r, d, alpha, float(np.float32(gamma)), w_map)
        assert np.all(np.abs(t - t64) <= tb)
        l64, lb, g64, gb, a64, ab, d64, db = f64.actor_loss(logits, q, w, alpha, float(np.float32(la)), float(np.float32(H)), w_map)
        assert abs(float(loss) - l64) <= lb and abs(float(aloss) - a64) <= ab and abs(float(dla) - d64) <= db
        assert np.all(np.abs(g.cpu().numpy() - g64) <= gb)


# (N, A): every N and every A of the sweep; the largest products are kept to sizes the float64 restatement handles
SHAPES = [(1, 1), (1, 256), (127, 2), (127, 33), (128, 4), (128, 256), (4097, 6), (4097, 18), (4097, 1), (65536, 4), (65536, 2)]


@pytest.mark.parametrize("N,A", SHAPES)
def test_kernels_equal_oracle_and_float64(cuda, N, A):
    rng = np.random.default_rng(N * 7 + A)
    for D in range(1, 9):
        n_nets = 1 + (D + A) % 3
        w_map = D % 2
        w_rows = 1 if D % 3 == 0 else (N if D % 3 == 1 else (N if N < 4 else 4 if N % 4 == 0 else 1))
        alpha = (0.0, 0.2, 1.3)[D % 3]
        q, logits, w, r, d = _inputs(rng, N, A, D, n_nets, w_rows)
        _check(cuda, q, logits, w, r, d, float(np.float32(alpha)), w_map, f64_check=N * A <= 300000 or D <= 2)


def test_done_and_alpha_device_update_inside_a_graph(cuda):
    """alpha is read from device memory at run time: a captured graph replayed after an in-place update uses the new value."""
    rng = np.random.default_rng(3)
    N, A, D = 256, 6, 4
    q, logits, w, r, _ = _inputs(rng, N, A, D, 2, 1)
    T = lambda x: th.from_numpy(np.ascontiguousarray(x)).to(cuda)  # noqa: E731
    qd, ld, wd, rd = T(q), T(logits), T(w), T(r)
    for done_v in (0.0, 1.0):
        d = np.full(N, done_v, np.float32)
        dd = T(d)
        a_dev = th.tensor([0.2], dtype=th.float32, device=cuda)
        out = th.empty(N, device=cuda)
        s = th.cuda.Stream()
        s.wait_stream(th.cuda.current_stream())
        with th.cuda.stream(s):
            ops.discrete_sac_target(qd, ld, wd, rd, dd, a_dev, 0.9, out=out)
        th.cuda.current_stream().wait_stream(s)
        g = th.cuda.CUDAGraph()
        with th.cuda.graph(g):
            ops.discrete_sac_target(qd, ld, wd, rd, dd, a_dev, 0.9, out=out)
        for alpha in (0.2, 0.05, 0.0):
            a_dev.fill_(alpha)
            g.replay()
            th.cuda.synchronize()
            _bits_equal(out.cpu().numpy(), orc.discrete_sac_target(q, logits, w, r, d, float(np.float32(alpha)), 0.9))


def test_extreme_logits_ties_nan_and_neg_inf(cuda):
    rng = np.random.default_rng(9)
    N, A, D = 64, 6, 3
    q, logits, w, r, d = _inputs(rng, N, A, D, 2, 1)
    q[1] = q[0]  # exact ties between the critics everywhere
    logits[:16] = np.where(rng.random((16, A)) < 0.5, 80.0, -80.0)
    logits[16:32] = np.where(rng.random((16, A)) < 0.5, 1e30, -1e30)
    logits[32:40, 2] = -np.inf  # -inf rule: the action leaves the expectation, its gradient is 0
    _check(cuda, q, logits, w, r, d, 0.2, orc.MAP_BLOCK, f64_check=False)
    T = lambda x: th.from_numpy(np.ascontiguousarray(x)).to(cuda)  # noqa: E731
    a_dev = th.tensor([0.2], dtype=th.float32, device=cuda)
    t = ops.discrete_sac_target(T(q), T(logits), T(w), T(r), T(d), a_dev, 0.99).cpu().numpy()
    assert np.all(np.isfinite(t))
    _, g, _, _ = ops.discrete_sac_actor_loss(T(logits), T(q), T(w), a_dev)
    assert np.all(g.cpu().numpy()[32:40, 2] == 0.0)
    # bounds hold on the finite-logit rows (the float64 side evaluates the same -inf rule)
    keep = slice(0, 32)
    t64, tb = f64.target(q[:, keep], logits[keep], w, r[keep], d[keep], float(np.float32(0.2)), float(np.float32(0.99)))
    assert np.all(np.abs(t[keep] - t64) <= tb)
    # NaN in Q propagates through the min (th.min semantics) into exactly the rows that hold it (with p > 0)
    q[1, 40, 1, 0] = np.nan
    logits[40] = 0.0
    t = ops.discrete_sac_target(T(q), T(logits), T(w), T(r), T(d), a_dev, 0.99).cpu().numpy()
    assert np.isnan(t[40]) and np.all(np.isfinite(np.delete(t, 40)))
    _bits_equal(t, orc.discrete_sac_target(q, logits, w, r, d, float(np.float32(0.2)), 0.99))
