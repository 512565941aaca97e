"""CPU checks of the plain-C restatement of the discrete-action MOSAC kernels (tests/discrete_sac_oracle.c, the checker the kernels equal bit
for bit): its portable e^x / log x against float64, and both entry points against the float64 restatement of the reference lines
mosac_discrete_action.py:452-498 within the bound derived in tests/discrete_sac_f64.py."""

import numpy as np
import pytest

from tests import discrete_sac_oracle as orc
from tests import discrete_sac_f64 as f64


def test_portable_exp_and_log_within_two_ulp():
    rng = np.random.default_rng(0)
    xs = np.concatenate([-rng.random(20000) * 104, rng.uniform(-5, 5, 5000), [0.0, -87.3, -103.9]]).astype(np.float32)
    e = orc.ds_exp(xs)
    ref = np.exp(xs.astype(np.float64))
    normal = ref > 1.2e-38
    ulp = np.spacing(ref.astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(e - ref)[normal] <= 2 * ulp[normal])
    assert np.all(np.abs(e - ref)[~normal] <= 2 * 1.4e-45)
    ys = np.concatenate([rng.uniform(1, 256, 20000), np.exp(rng.uniform(-80, 80, 5000)), [1.0, 2.0, 0.5]]).astype(np.float32)
    lg = orc.ds_log(ys)
    ref = np.log(ys.astype(np.float64))
    assert np.all(np.abs(lg - ref) <= 2 * np.spacing(np.abs(ref).astype(np.float32)) + 1e-45)
    assert orc.ds_exp(np.float32([0.0]))[0] == 1.0 and orc.ds_log(np.float32([1.0]))[0] == 0.0
    assert orc.ds_exp(np.float32([-np.inf]))[0] == 0.0 and orc.ds_log(np.float32([0.0]))[0] == -np.inf


def _case(rng, N, A, D, n_nets, scale=3.0):
    q = (rng.standard_normal((n_nets, N, A, D)) * scale).astype(np.float32)
    logits = (rng.standard_normal((N, A)) * scale).astype(np.float32)
    w = rng.dirichlet(np.ones(D), 1 if N % 4 else 4).astype(np.float32)
    r = rng.standard_normal((N, D)).astype(np.float32)
    d = (rng.random(N) < 0.3).astype(np.float32)
    return q, logits, w, r, d


@pytest.mark.parametrize("N,A,D,n_nets", [(1, 1, 1, 1), (16, 4, 4, 2), (33, 18, 3, 3), (300, 6, 8, 2), (64, 256, 2, 1), (520, 33, 5, 2)])
@pytest.mark.parametrize("w_map", [orc.MAP_TILE, orc.MAP_BLOCK])
def test_oracle_within_float64_bound(N, A, D, n_nets, w_map):
    rng = np.random.default_rng(N * 1000 + A * 10 + D)
    q, logits, w, r, d = _case(rng, N, A, D, n_nets)
    logits[0, -1] = -np.inf if A > 1 else logits[0, -1]
    for alpha in (0.0, 0.2, 1.7):
        alpha = float(np.float32(alpha))
        t = orc.discrete_sac_target(q, logits, w, r, d, alpha, 0.99, w_map)
        t64, tb = f64.target(q, logits, w, r, d, alpha, float(np.float32(0.99)), w_map)
        assert np.all(np.abs(t - t64) <= tb), np.max(np.abs(t - t64) / tb)
        H = float(np.float32(-0.89 * np.log(1.0 / A)))
        loss, g, aloss, dla = orc.discrete_sac_actor_loss(logits, q, w, alpha, -0.3, H, w_map)
        l64, lb, g64, gb, a64, ab, d64, db = f64.actor_loss(logits, q, w, alpha, float(np.float32(-0.3)), H, w_map)
        assert abs(loss - l64) <= lb
        assert np.all(np.abs(g - g64) <= gb), np.max(np.abs(g - g64) / gb)
        assert abs(aloss - a64) <= ab and abs(dla - d64) <= db


def test_oracle_rules():
    """-inf logits leave the expectation (the reference's 0 * -inf = NaN is not reproduced), NaN in Q propagates through th.min,
    ties between critics are exact, and a row of equal logits is exactly uniform."""
    q = np.zeros((2, 1, 3, 2), np.float32)
    q[0, 0] = [[1, 2], [3, 4], [5, 6]]
    q[1, 0] = [[1, 2], [3, 4], [5, 6]]
    w = np.float32([[0.5, 0.5]])
    r, d = np.float32([[1, 1]]), np.float32([0])
    logits = np.float32([[0.0, 0.0, -np.inf]])
    t = orc.discrete_sac_target(q, logits, w, r, d, 0.0, 1.0)
    assert t[0] == np.float32(1.0) + np.float32(0.5 * 1.5 + 0.5 * 3.5)
    loss, g, _, _ = orc.discrete_sac_actor_loss(logits, q, w, 0.2, None, 0.0)
    assert np.isfinite(loss) and g[0, 2] == 0.0
    q[1, 0, 1, 0] = np.nan
    t = orc.discrete_sac_target(q, logits, w, r, d, 0.2, 1.0)
    assert np.isnan(t[0])
    q[1, 0, 1, 0] = 3.0
    q[1, 0, 0] = [0.5, 1.0]  # critic 1 is the min on action 0 only
    t = orc.discrete_sac_target(q, np.float32([[7.0, 7.0, 7.0]]), w, r, d, 0.0, 1.0)
    third = np.float32(1.0) / np.float32(3.0)
    v = np.float32(0.0) + third * np.float32(0.75)
    v = v + third * np.float32(3.5)
    v = v + third * np.float32(5.5)
    assert t[0] == np.float32(1.0) + v


def test_c_abi_rejects_null_and_oversize_arguments():
    """Argument errors come back from the C ABI before any device work: NULL pointers, A > 256, D > 8, bad w_rows."""
    import ctypes as C

    from morl_baselines_b200 import _lib

    lib = _lib.load()
    buf = (C.c_float * 16)()
    p = C.cast(buf, C.c_void_p)
    tgt, act = lib.morl_discrete_sac_target_f32, lib.morl_discrete_sac_actor_loss_f32
    assert tgt(None, 2, p, p, 1, 1, p, p, p, 0.99, 4, 4, 4, p, None) == -1
    assert tgt(p, 2, p, p, 1, 1, p, p, None, 0.99, 4, 4, 4, p, None) == -1
    assert tgt(p, 2, p, p, 1, 1, p, p, p, 0.99, 4, 257, 4, p, None) == -4
    assert tgt(p, 2, p, p, 1, 1, p, p, p, 0.99, 4, 4, 9, p, None) == -4
    assert tgt(p, 2, p, p, 3, 1, p, p, p, 0.99, 4, 4, 4, p, None) == -2
    assert tgt(p, 0, p, p, 1, 1, p, p, p, 0.99, 4, 4, 4, p, None) == -2
    assert act(p, p, 2, p, 1, 1, p, None, 0.0, 4, 4, 4, None, None, None, None, p, None) == -1
    assert act(p, p, 2, p, 1, 1, p, p, 0.0, 4, 4, 4, p, None, None, None, p, None) == -1
    assert act(p, p, 2, p, 1, 1, p, None, 0.0, 4, 300, 4, p, None, None, None, p, None) == -4
    assert act(p, p, 2, p, 1, 1, p, None, 0.0, 4, 4, 12, p, None, None, None, p, None) == -4
    assert b"D=12 > 8" in lib.morl_last_error()
    assert lib.morl_discrete_sac_workspace_bytes(257) == 2 * 3 * 4
