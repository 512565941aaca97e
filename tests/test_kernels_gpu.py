"""GPU parity tests: every CUDA operator, called through the C-ABI (morl_baselines_b200.ops -> ctypes -> libmorl_b200.so),
against (1) the committed golden vectors of the unmodified reference and (2) the CPU oracle on the same seeded inputs.

Bar: bit-exact (np.array_equal / SHA-256) for targets, indices and masks -- the kernels use explicit round-to-nearest
intrinsics in the documented order; 1e-6 relative for the reduced loss scalars (summation order differs), tolerance
stated at the assert."""

import numpy as np
import pytest
import torch as th

from oracle import oracle as orc
from tests.golden import cases

pytestmark = pytest.mark.gpu


def _t(x, dev, dtype=None):
    t = th.from_numpy(np.ascontiguousarray(x)).to(dev)
    return t if dtype is None else t.to(dtype)


# ------------------------------------------------------------------------------------------------ envelope TD
@pytest.mark.parametrize("name", [c[0] for c in cases.ENVELOPE_CASES])
def test_envelope_td_golden_and_oracle(cuda, golden, name):
    from morl_baselines_b200 import ops

    x = cases.envelope_inputs(name)
    args = [_t(x[k], cuda) for k in ("q_on", "q_tg", "wset", "reward", "done")]
    t, p, a = ops.envelope_td(*args, x["gamma"], ops.DOT_UNFUSED, ops.ROWS_REFERENCE)
    t, p, a = t.cpu().numpy(), p.cpu().numpy(), a.cpu().numpy()
    # (1) the reference's own output, bit for bit
    assert cases.digest(t) == str(golden[f"env_{name}_target_sha"])
    assert cases.digest(p) == str(golden[f"env_{name}_pref_sha"])
    assert cases.digest(a) == str(golden[f"env_{name}_act_sha"])
    # (2) every arithmetic mode and both row orders against the oracle
    for mode in (ops.DOT_UNFUSED, ops.DOT_FMA, ops.DOT_PAIRFMA):
        for order in (ops.ROWS_REFERENCE, ops.ROWS_BMAJOR):
            t, p, a = ops.envelope_td(*args, x["gamma"], mode, order)
            to, po, ao = orc.envelope_td(x["q_on"], x["q_tg"], x["wset"], x["reward"], x["done"], x["gamma"], mode, order)
            assert np.array_equal(t.cpu().numpy(), to), (name, mode, order)
            assert np.array_equal(p.cpu().numpy(), po) and np.array_equal(a.cpu().numpy(), ao), (name, mode, order)


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (3, 2, 1, 3), (5, 33, 3, 3), (2, 300, 4, 3), (4, 70, 9, 8), (2, 600, 18, 3), (7, 64, 64, 2)])
def test_envelope_td_edge_shapes(cuda, shape):
    """Ragged / extreme shapes: W not a multiple of 32, W > 256 (several weight chunks), Q tile larger than one shared
    memory stage (W*A*D > 10240 floats), D = 1 and D = 8, a single transition."""
    from morl_baselines_b200 import ops

    B, W, A, D = shape
    rng = np.random.default_rng(B * 1000 + W)
    q_on = rng.standard_normal((B, W, A, D)).astype(np.float32)
    q_tg = rng.standard_normal((B, W, A, D)).astype(np.float32)
    wset = cases.gaussian_weights(rng, W, D)
    reward = rng.standard_normal((B, D)).astype(np.float32)
    done = (rng.random(B) < 0.3).astype(np.float32)
    for order in (ops.ROWS_REFERENCE, ops.ROWS_BMAJOR):
        t, p, a = ops.envelope_td(_t(q_on, cuda), _t(q_tg, cuda), _t(wset, cuda), _t(reward, cuda), _t(done, cuda), 0.97, ops.DOT_UNFUSED, order)
        to, po, ao = orc.envelope_td(q_on, q_tg, wset, reward, done, 0.97, orc.DOT_UNFUSED, order)
        assert np.array_equal(t.cpu().numpy(), to) and np.array_equal(p.cpu().numpy(), po) and np.array_equal(a.cpu().numpy(), ao)


def test_envelope_td_degenerate_values(cuda):
    """All-equal Q (every candidate ties -> index (0,0)), -inf everywhere, and done = 1 rows (target == reward)."""
    from morl_baselines_b200 import ops

    B, W, A, D = 8, 16, 4, 3
    rng = np.random.default_rng(3)
    wset = _t(cases.gaussian_weights(rng, W, D), cuda)
    reward = _t(rng.standard_normal((B, D)).astype(np.float32), cuda)
    q_tg = _t(rng.standard_normal((B, W, A, D)).astype(np.float32), cuda)
    ones = th.ones(B, device=cuda)
    t, p, a = ops.envelope_td(th.zeros(B, W, A, D, device=cuda), q_tg, wset, reward, ones, 0.99)
    assert int(p.abs().sum()) == 0 and int(a.abs().sum()) == 0
    assert th.equal(t.view(W, B, D), reward.unsqueeze(0).expand(W, B, D))  # (1 - done) * gamma == 0
    t, p, a = ops.envelope_td(th.full((B, W, A, D), -float("inf"), device=cuda), q_tg, wset, reward, th.zeros(B, device=cuda), 0.99)
    assert int(p.abs().sum()) == 0 and int(a.abs().sum()) == 0


@pytest.mark.parametrize("shape", [(64, 64, 8, 3), (33, 32, 4, 3), (16, 16, 8, 2), (8, 40, 5, 4)])
def test_envelope_td_near_ties(cuda, shape):
    """Candidates a few ulps apart: the FMA-chain filter of the fast path cannot separate them, so rows must fall back to the
    exact re-scan; FMA and unfused arithmetic genuinely pick different indices here, and every mode must match its oracle."""
    from morl_baselines_b200 import ops

    B, W, A, D = shape
    rng = np.random.default_rng(B + 7 * W)
    base = rng.standard_normal((B, 1, 1, D)).astype(np.float32)
    q_on = (base * (1.0 + rng.integers(0, 6, size=(B, W, A, D)) * np.float32(2.0**-23))).astype(np.float32)
    q_on[::3] = rng.standard_normal((len(q_on[::3]), W, A, D)).astype(np.float32)  # mix in well separated rows
    q_tg = rng.standard_normal((B, W, A, D)).astype(np.float32)
    wset = cases.gaussian_weights(rng, W, D)
    reward = rng.standard_normal((B, D)).astype(np.float32)
    done = np.zeros(B, np.float32)
    n_diff = 0
    ref = {}
    for mode in (ops.DOT_UNFUSED, ops.DOT_FMA, ops.DOT_PAIRFMA):
        t, p, a = ops.envelope_td(_t(q_on, cuda), _t(q_tg, cuda), _t(wset, cuda), _t(reward, cuda), _t(done, cuda), 0.99, mode, ops.ROWS_REFERENCE)
        to, po, ao = orc.envelope_td(q_on, q_tg, wset, reward, done, 0.99, mode, orc.ROWS_REFERENCE)
        assert np.array_equal(p.cpu().numpy(), po) and np.array_equal(a.cpu().numpy(), ao), mode
        assert np.array_equal(t.cpu().numpy(), to), mode
        ref[mode] = (po, ao)
    n_diff = int((ref[ops.DOT_UNFUSED][0] != ref[ops.DOT_FMA][0]).sum() + (ref[ops.DOT_UNFUSED][1] != ref[ops.DOT_FMA][1]).sum())
    assert n_diff > 0  # the construction really separates the arithmetics


def test_envelope_td_full_size_properties(cuda):
    """North-star shape (B=1024, |W|=64, |A|=8, d=3): size-independent properties.
      * optimality: the chosen (j*, a*) attains the maximum scalarised value and no earlier candidate equals it;
      * permutation covariance: permuting the weight set permutes the output rows (REFERENCE order blocks);
      * a weight set made of one repeated vector makes every block identical."""
    from morl_baselines_b200 import ops

    x = cases.envelope_inputs("north_star")
    B, W, A, D = x["B"], x["W"], x["A"], x["D"]
    q_on, q_tg, wset, reward, done = (_t(x[k], cuda) for k in ("q_on", "q_tg", "wset", "reward", "done"))
    t, p, a = ops.envelope_td(q_on, q_tg, wset, reward, done, x["gamma"])
    sc = (wset[:, None, None, None, 0] * q_on[None, ..., 0] + wset[:, None, None, None, 1] * q_on[None, ..., 1]) + wset[:, None, None, None, 2] * q_on[None, ..., 2]
    sc = sc.reshape(W, B, W * A)  # [i, b, (j,a)] computed by torch with the same unfused order
    flat = (p.long() * A + a.long()).view(W, B)
    best = sc.max(dim=2).values
    assert th.equal(sc.gather(2, flat.unsqueeze(2)).squeeze(2), best)
    first = (sc == best.unsqueeze(2)).float().argmax(dim=2)
    assert th.equal(first, flat)
    perm = th.randperm(W, device=cuda)
    t2, p2, a2 = ops.envelope_td(q_on, q_tg, wset[perm].contiguous(), reward, done, x["gamma"])
    assert th.equal(t2.view(W, B, D), t.view(W, B, D)[perm])
    t3, _, _ = ops.envelope_td(q_on, q_tg, wset[:1].expand(W, D).contiguous(), reward, done, x["gamma"])
    assert th.equal(t3.view(W, B, D), t3.view(W, B, D)[:1].expand(W, B, D))


def _env_path(path, *a, **k):
    """Run morl_envelope_td_f32 with the kernel family forced by MORL_ENVELOPE_PATH (read by the library on every call)."""
    import os

    from morl_baselines_b200 import ops

    os.environ["MORL_ENVELOPE_PATH"] = path
    try:
        return ops.envelope_td(*a, **k)
    finally:
        os.environ.pop("MORL_ENVELOPE_PATH", None)


@pytest.mark.parametrize("shape", [(1024, 64, 8, 3), (256, 32, 6, 3), (96, 16, 4, 2), (33, 50, 8, 3), (7, 64, 8, 1), (300, 2, 8, 3), (600, 62, 8, 3),
                                   (64, 128, 8, 3), (16, 256, 8, 3), (9, 96, 4, 4)])
@pytest.mark.parametrize("kind", ["plain", "ties", "neartie", "signed", "special"])
def test_envelope_td_kernel_families_agree_bitwise(cuda, shape, kind):
    """The kernel families of morl_envelope_td_f32 -- generic (v1), CUDA-core fast paths (v3: FMA-chain filter + exact re-check; wp: its
    weight-pair re-blocking, the default at |W| > 32; |W| 96, 128 and 256 run it with several blocks of 64 weights) -- return
    bit-identical targets and indices, in every
    arithmetic mode and row order, on continuous data, exact ties, candidates a few ulps apart, mixed-sign weights / large values,
    and NaN / +-inf / all-zero / huge / tiny blocks.  v1 is pinned to the oracle and the reference's golden vectors above."""
    from morl_baselines_b200 import ops

    B, W, A, D = shape
    g = th.Generator(device=cuda).manual_seed(sum(shape) + len(kind))
    if kind == "ties":
        q_on = th.randint(-2, 3, (B, W, A, D), device=cuda, generator=g).float()
        wset = th.randint(1, 4, (W, D), device=cuda, generator=g).float() / 8.0
    elif kind == "neartie":
        q_on = th.randn(B, 1, A, D, device=cuda, generator=g).repeat(1, W, 1, 1) * (1.0 + 1e-7 * th.randn(B, W, A, D, device=cuda, generator=g))
        wset = th.rand(W, D, device=cuda, generator=g)
    elif kind == "signed":
        q_on = th.randn(B, W, A, D, device=cuda, generator=g) * 100.0
        wset = th.randn(W, D, device=cuda, generator=g)
    elif kind == "special":
        q_on = th.randn(B, W, A, D, device=cuda, generator=g)
        fills = [lambda t: t.fill_(float("nan")), lambda t: t.view(-1)[:1].fill_(float("inf")), lambda t: t.fill_(-float("inf")),
                 lambda t: t.fill_(0.0), lambda t: t.mul_(1e38), lambda t: t.mul_(1e-38), lambda t: t.view(-1)[-1:].fill_(float("nan"))]
        for b, f in enumerate(fills[:B]):
            f(q_on[b])
        wset = th.rand(W, D, device=cuda, generator=g)
    else:
        q_on = th.randn(B, W, A, D, device=cuda, generator=g) * 3.0
        wset = th.rand(W, D, device=cuda, generator=g)
        wset = wset / wset.sum(1, keepdim=True)
    q_tg = th.randn(B, W, A, D, device=cuda, generator=g)
    rew = th.randn(B, D, device=cuda, generator=g)
    done = (th.rand(B, device=cuda, generator=g) < 0.1).float()
    combos = [(ops.DOT_UNFUSED, ops.ROWS_BMAJOR)]
    if kind in ("plain", "ties"):
        combos += [(ops.DOT_UNFUSED, ops.ROWS_REFERENCE), (ops.DOT_FMA, ops.ROWS_BMAJOR), (ops.DOT_PAIRFMA, ops.ROWS_REFERENCE)]
    for mode, order in combos:
        ref = _env_path("v1", q_on, q_tg, wset, rew, done, 0.99, mode, order)
        for path in (("v3", "wp") if W > 32 else ("v3",)):
            got = _env_path(path, q_on, q_tg, wset, rew, done, 0.99, mode, order)
            assert th.equal(ref[0].view(th.int32), got[0].view(th.int32)), (path, mode, order)  # bit pattern (NaN-safe)
            assert th.equal(ref[1], got[1]) and th.equal(ref[2], got[2]), (path, mode, order)


# ------------------------------------------------------------------------------------------------ per-row targets
@pytest.mark.parametrize("name", [c[0] for c in cases.ENVELOPE_CASES])
def test_greedy_td_golden_and_oracle(cuda, golden, name):
    from morl_baselines_b200 import ops

    x = cases.envelope_inputs(name)
    B, W, A, D = x["B"], x["W"], x["A"], x["D"]
    qs = np.ascontiguousarray(x["q_on"].transpose(1, 0, 2, 3)).reshape(W * B, A, D)
    qe = np.ascontiguousarray(x["q_tg"].transpose(1, 0, 2, 3)).reshape(W * B, A, D)
    t, act = ops.greedy_td(_t(qs, cuda), _t(qe, cuda), _t(x["wset"], cuda), _t(x["reward"], cuda), _t(x["done"], cuda), x["gamma"])
    assert cases.digest(t.cpu().numpy()) == str(golden[f"ddqn_{name}_target_sha"])
    for mode in (0, 1, 2):
        t, act = ops.greedy_td(_t(qs, cuda), _t(qe, cuda), _t(x["wset"], cuda), _t(x["reward"], cuda), _t(x["done"], cuda), x["gamma"], mode)
        to, ao = orc.greedy_td(qs, qe, x["wset"], x["reward"], x["done"], x["gamma"], mode)
        assert np.array_equal(t.cpu().numpy(), to) and np.array_equal(act.cpu().numpy(), ao)
    # no Bellman (reward=None) and per-row weights
    wfull = np.repeat(x["wset"], B, axis=0)
    t, act = ops.greedy_td(_t(qs, cuda), _t(qe, cuda), _t(wfull, cuda))
    to, ao = orc.greedy_td(qs, qe, wfull, None, None, 0.0)
    assert np.array_equal(t.cpu().numpy(), to) and np.array_equal(act.cpu().numpy(), ao)


@pytest.mark.parametrize("name", [c[0] for c in cases.GPI_CASES])
def test_gpi_kernels_golden_and_oracle(cuda, golden, name):
    from morl_baselines_b200 import ops

    x = cases.gpi_inputs(name)
    q, w = _t(x["q"], cuda), _t(x["w"], cuda)
    o, p, a = ops.gpi_envelope(q, w)
    assert np.array_equal(o.cpu().numpy(), golden[f"gpi_{name}_maxq"])
    assert np.array_equal(p.cpu().numpy(), golden[f"gpi_{name}_policy"]) and np.array_equal(a.cpu().numpy(), golden[f"gpi_{name}_act"])
    o1, a1 = ops.critic_min_td(q[:, :, 0].contiguous(), w)
    assert np.array_equal(o1.cpu().numpy(), golden[f"gpi_{name}_criticmin"]) and np.array_equal(a1.cpu().numpy(), golden[f"gpi_{name}_criticmin_act"])
    n16 = len(golden[f"gpi_{name}_action16"])
    _, p16, a16 = ops.gpi_envelope(q[:1, :n16].contiguous(), w[:n16].contiguous())
    assert np.array_equal(a16.cpu().numpy(), golden[f"gpi_{name}_action16"]) and np.array_equal(p16.cpu().numpy(), golden[f"gpi_{name}_policy16"])
    # single observation, single shared weight (the shape GPIPD.gpi_action is called with every env step)
    _, p1, a1_ = ops.gpi_envelope(q[:1, :1].contiguous(), w[:1].contiguous())
    assert int(p1[0]) == int(golden[f"gpi_{name}_policy16"][0]) and int(a1_[0]) == int(golden[f"gpi_{name}_action16"][0])
    # Bellman variants + all modes against the oracle
    rew, dn = _t(x["reward"], cuda), _t(x["done"], cuda)
    for mode in (0, 1, 2):
        o, p, a = ops.gpi_envelope(q, w, rew, dn, x["gamma"], mode)
        oo, po, ao = orc.gpi_envelope(x["q"], x["w"], x["reward"], x["done"], x["gamma"], mode)
        assert np.array_equal(o.cpu().numpy(), oo) and np.array_equal(p.cpu().numpy(), po) and np.array_equal(a.cpu().numpy(), ao)
        qc = x["q"][:, :, 0].copy()
        o, a = ops.critic_min_td(_t(qc, cuda), w, rew, dn, x["gamma"], mode)
        oo, ao = orc.critic_min_td(qc, x["w"], x["reward"], x["done"], x["gamma"], mode)
        assert np.array_equal(o.cpu().numpy(), oo) and np.array_equal(a.cpu().numpy(), ao)


def test_critic_min_td_tiled_rows(cuda):
    """GPIPD.update doubles the batch (gpi_pd.py:425-432): rewards/dones tiled x2, weights per row."""
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(11)
    n_nets, B, A, D = 2, 128, 6, 3
    q = rng.standard_normal((n_nets, 2 * B, A, D)).astype(np.float32)
    w = cases.gaussian_weights(rng, 2 * B, D)
    rew = rng.standard_normal((B, D)).astype(np.float32)
    dn = (rng.random(B) < 0.2).astype(np.float32)
    o, a = ops.critic_min_td(_t(q, cuda), _t(w, cuda), _t(rew, cuda), _t(dn, cuda), 0.99, 0, ops.MAP_BLOCK, ops.MAP_TILE)
    oo, ao = orc.critic_min_td(q, w, rew, dn, 0.99, 0, orc.MAP_BLOCK, orc.MAP_TILE)
    assert np.array_equal(o.cpu().numpy(), oo) and np.array_equal(a.cpu().numpy(), ao)
    full = np.concatenate([rew, rew]), np.concatenate([dn, dn])
    o2, _ = orc.critic_min_td(q, w, full[0], full[1], 0.99, 0)
    assert np.array_equal(oo, o2)


@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("D", [2, 3])
def test_actor_critic_td(cuda, variant, D):
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(variant * 10 + D)
    n_nets, N = 2, 257
    q = rng.standard_normal((n_nets, N, D)).astype(np.float32)
    w = cases.gaussian_weights(rng, N if variant != 1 else 1, D)
    rew = rng.standard_normal((N, D)).astype(np.float32)
    dn = (rng.random(N) < 0.2).astype(np.float32)
    logp = rng.standard_normal(N).astype(np.float32) if variant != 2 else None
    got = ops.actor_critic_td(_t(q, cuda), _t(w, cuda), _t(rew, cuda), _t(dn, cuda), None if logp is None else _t(logp, cuda), 0.2, 0.99, variant)
    exp = orc.actor_critic_td(q, w, rew, dn, logp, 0.2, 0.99, variant)
    assert np.array_equal(got.cpu().numpy(), exp)
    # cross-check the oracle itself against a literal torch restatement of the reference lines
    tq, tw, tr, td_ = map(th.from_numpy, (q, w, rew, dn))
    if variant == 0:  # capql.py:329-331
        ref = tr + (1 - td_.reshape(-1, 1)) * 0.99 * (th.min(tq, dim=0)[0] - 0.2 * th.from_numpy(logp).reshape(-1, 1))
        assert np.array_equal(exp, ref.numpy())


# ------------------------------------------------------------------------------------------------ TD loss
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("lam", [0.0, 0.35, 1.0])
@pytest.mark.parametrize("shape", [(64, 8, 8, 3), (37, 5, 7, 3), (256, 32, 6, 2)])
def test_td_mse_priority(cuda, order, lam, shape):
    from morl_baselines_b200 import ops

    B, W, A, D = shape
    rng = np.random.default_rng(B + W)
    qv = rng.standard_normal((B * W, A, D)).astype(np.float32)
    tq = rng.standard_normal((B * W, D)).astype(np.float32)
    wset = cases.gaussian_weights(rng, W, D)
    act = rng.integers(0, A, size=B).astype(np.int32)
    loss, grad, prio = ops.td_mse_priority(_t(qv, cuda), _t(act, cuda), _t(tq, cuda), _t(wset, cuda), lam, B, W, order)
    lo, go, _, po = orc.td_mse(qv, act, tq, wset, lam, B, W, order)
    # loss: float block partials + double final sum vs the oracle's all-double sum: 1e-6 relative
    assert abs(float(loss) - lo) <= 1e-6 * max(1.0, abs(lo))
    assert np.array_equal(prio.cpu().numpy(), po)  # |w . td| in the unfused order: bit-exact
    # gradient: c1*d + c2*aux*w evaluated in float (kernel) vs double-then-rounded (oracle); the two terms may cancel, so the
    # bound is 2 ulp of the larger term: atol = 3e-7 * max|g|
    np.testing.assert_allclose(grad.cpu().numpy(), go, rtol=3e-7, atol=3e-7 * float(np.abs(go).max()))
    # and against torch autograd on the reference's literal loss (envelope.py:301-313) -- 1e-5 relative (north_star tolerance)
    q_t = th.from_numpy(qv).requires_grad_(True)
    i_of = np.arange(B * W) // B if order == 0 else np.arange(B * W) % W
    b_of = np.arange(B * W) % B if order == 0 else np.arange(B * W) // W
    a_rows = th.from_numpy(act[b_of].astype(np.int64))
    q_taken = q_t.gather(1, a_rows.reshape(-1, 1, 1).expand(B * W, 1, D)).reshape(-1, D)
    w_rows = th.from_numpy(wset[i_of])
    ref = th.nn.functional.mse_loss(q_taken, th.from_numpy(tq))
    if lam > 0:
        aux = th.nn.functional.mse_loss(th.einsum("br,br->b", q_taken, w_rows), th.einsum("br,br->b", th.from_numpy(tq), w_rows))
        ref = (1 - lam) * ref + lam * aux
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    np.testing.assert_allclose(grad.cpu().numpy(), q_t.grad.numpy(), rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize("gpi", [False, True])
def test_td_huber_priority(cuda, gpi):
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(5)
    n_nets, B, A, D = 2, 96, 6, 3
    N = 2 * B
    qv = (rng.standard_normal((n_nets, N, A, D)) * 0.02).astype(np.float32)  # straddles min_priority = 0.01
    tq = (rng.standard_normal((N, D)) * 0.02).astype(np.float32)
    tg = (rng.standard_normal((N, D)) * 0.02).astype(np.float32) if gpi else None
    w = cases.gaussian_weights(rng, N, D)
    act = rng.integers(0, A, size=B).astype(np.int32)
    loss, grad, prio = ops.td_huber_priority(_t(qv, cuda), _t(act, cuda), _t(tq, cuda), None if tg is None else _t(tg, cuda), _t(w, cuda), 0.01, B)
    lo, go, po = orc.td_huber(qv, act, tq, tg, w, 0.01, B)
    assert abs(float(loss) - lo) <= 1e-6 * abs(lo)
    assert np.array_equal(prio.cpu().numpy(), po)
    np.testing.assert_allclose(grad.cpu().numpy(), go, rtol=3e-7, atol=1e-12)


# ------------------------------------------------------------------------------------------------ Pareto
@pytest.mark.parametrize("name", cases.PARETO_CASES)
@pytest.mark.parametrize("rd", [True, False])
def test_pareto_mask_golden(cuda, golden, name, rd):
    from morl_baselines_b200 import ops

    pts = cases.pareto_points(name)
    ref = np.unpackbits(golden[f"pareto_{name}_{int(rd)}"])[: len(pts)].astype(bool)
    got = ops.pareto_mask(_t(pts, cuda), rd).cpu().numpy()
    assert np.array_equal(got, ref)
    assert cases.digest(pts[got]) == str(golden[f"pareto_{name}_{int(rd)}_filtered_sha"])


def test_pareto_mask_edge_cases(cuda):
    from morl_baselines_b200 import ops

    nan = float("nan")
    m = ops.pareto_mask(th.tensor([[nan, 1.0], [0.0, 0.0], [1.0, 1.0]], device=cuda, dtype=th.float64), True)
    assert m.tolist() == [False, False, True]
    assert ops.pareto_mask(th.zeros(0, 3, device=cuda), True).numel() == 0
    assert ops.pareto_mask(th.tensor([[1.0, 2.0]], device=cuda), True).tolist() == [True]
    # float32 inputs are compared in float32, not promoted
    a = np.float32(1.0)
    b = np.nextafter(a, np.float32(2.0))
    m = ops.pareto_mask(th.tensor([[a, a], [b, a]], device=cuda, dtype=th.float32), True)
    assert m.tolist() == [False, True]


def test_pareto_mask_large_properties(cuda):
    """N = 20000, d = 4 (beyond anything the reference finishes quickly): idempotence, permutation invariance of the kept
    SET, and agreement with the oracle on a 3000-point subset."""
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(0)
    pts = rng.standard_normal((20000, 4)).astype(np.float32)
    pts[::7] = pts[3]  # heavy duplication of one point
    x = _t(pts, cuda)
    keep = ops.pareto_mask(x, True)
    front = x[keep]
    assert bool(ops.pareto_mask(front, True).all())  # idempotent
    perm = th.randperm(len(pts), device=cuda)
    keep_p = ops.pareto_mask(x[perm].contiguous(), True)
    assert {tuple(r) for r in front.cpu().numpy()} == {tuple(r) for r in x[perm][keep_p].cpu().numpy()}
    sub = pts[:3000]
    assert np.array_equal(ops.pareto_mask(_t(sub, cuda), True).cpu().numpy(), orc.pareto_mask(sub, True))
    assert np.array_equal(ops.pareto_mask(_t(sub, cuda), False).cpu().numpy(), orc.pareto_mask(sub, False))


# ------------------------------------------------------------------------------------------------ replay / polyak
@pytest.mark.parametrize("obs_dim,u8", [(32, True), (11, False), (17, True)])
def test_replay_gather(cuda, obs_dim, u8):
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(obs_dim)
    cap, B, d = 5000, 1024, 3
    obs = rng.standard_normal((cap, obs_dim)).astype(np.float32)
    nobs = rng.standard_normal((cap, obs_dim)).astype(np.float32)
    act = rng.integers(0, 8, size=(cap, 1)).astype(np.uint8) if u8 else rng.standard_normal((cap, 3)).astype(np.float32)
    rew = rng.standard_normal((cap, d)).astype(np.float32)
    done = (rng.random((cap, 1)) < 0.1).astype(np.float32)
    idx = rng.integers(0, cap, size=B)
    o, a, r, no, dn = ops.replay_gather(_t(obs, cuda), _t(nobs, cuda), _t(act, cuda), _t(rew, cuda), _t(done, cuda), _t(idx, cuda))
    assert np.array_equal(o.cpu().numpy(), obs[idx]) and np.array_equal(no.cpu().numpy(), nobs[idx])
    assert np.array_equal(a.cpu().numpy(), act[idx].astype(np.int32) if u8 else act[idx])
    assert np.array_equal(r.cpu().numpy(), rew[idx]) and np.array_equal(dn.cpu().numpy(), done[idx])


@pytest.mark.parametrize("tau", [0.005, 1.0, 0.3])
def test_polyak_golden(cuda, golden, tau):
    from morl_baselines_b200 import ops

    p = _t(golden[f"polyak_{tau}_param"], cuda)
    t = _t(golden[f"polyak_{tau}_target0"], cuda)
    sizes = (24, 256 * 35, 1)
    ps, ts, off = [], [], 0
    for n in sizes:
        ps.append(p[off : off + n].clone())
        ts.append(t[off : off + n].clone())
        off += n
    ops.PolyakPlan(ps, ts).run(tau)
    assert np.array_equal(th.cat(ts).cpu().numpy(), golden[f"polyak_{tau}_target1"])


@pytest.mark.parametrize("max_norm", [None, 1.0, 1e6])
def test_fused_clip_adam_matches_torch(cuda, max_norm):
    """Three steps of clip_grad_norm_ + Adam on the CPU (the reference's optimiser path) vs FusedClipAdam.step_fused.
    Tolerance 2e-6 relative to the parameter scale: same formula, fp32, different operation fusion."""
    from morl_baselines_b200.common.fused_adam import FusedClipAdam

    th.manual_seed(0)
    shapes = [(256, 35), (256,), (256, 256), (24, 256), (24,)]
    ref = [th.nn.Parameter(th.randn(*s)) for s in shapes]
    mine = [th.nn.Parameter(p.detach().clone().to(cuda)) for p in ref]
    o_ref = th.optim.Adam(ref, lr=3e-4)
    o_mine = FusedClipAdam(mine, lr=3e-4)
    for step in range(3):
        for p, q in zip(ref, mine):
            g = th.randn_like(p) * (10.0 if step == 1 else 0.1)
            p.grad = g.clone()
            if q.grad is None:
                q.grad = g.to(cuda)
            else:
                q.grad.copy_(g)
        if max_norm is not None:
            th.nn.utils.clip_grad_norm_(ref, max_norm)
        o_ref.step()
        o_mine.step_fused(max_norm)
    for p, q in zip(ref, mine):
        np.testing.assert_allclose(q.detach().cpu().numpy(), p.detach().numpy(), rtol=2e-6, atol=2e-6)
    sd = o_mine.state_dict()
    assert set(sd["state"][0].keys()) == {"step", "exp_avg", "exp_avg_sq"} and float(sd["state"][0]["step"]) == 3.0


def test_fused_clip_adam_eager_steps_do_not_grow(cuda):
    """ADVICE r1 (high): with ``zero_grad(set_to_none=True)`` callers every eager step presents NEW gradient storage; the optimiser
    must refresh ONE pointer table in place -- no per-step cache entry, no retained gradients, flat device memory over 100 steps."""
    from morl_baselines_b200.common.fused_adam import FusedClipAdam

    th.manual_seed(0)
    ps = [th.nn.Parameter(th.randn(256, 256, device=cuda)), th.nn.Parameter(th.randn(256, device=cuda))]
    opt = FusedClipAdam(ps, lr=1e-3)
    import gc

    held = []
    mem = []
    gc.collect()  # (garbage of earlier tests must not be freed in the middle of the measurement)
    th.cuda.synchronize()
    for step in range(120):
        for p in ps:
            p.grad = th.randn_like(p)  # fresh storage every step
        if step < 4:
            held.extend(p.grad for p in ps)  # (keeps early grads alive so later ones really land at new addresses)
        opt.step_fused(1.0)
        opt.zero_grad(set_to_none=True)
        if step >= 20:
            th.cuda.synchronize()
            mem.append(th.cuda.memory_allocated())
    assert len(opt._cache) == 0
    assert mem[-1] <= mem[0], (mem[0], mem[-1])  # the leak was ~1 MB per step for the Envelope net: it would show as growth here
    assert float(opt.state[ps[0]]["step"]) == 120.0


def test_pareto_archive_matches_reference(cuda, golden):
    """``ParetoArchive.add`` (reference common/pareto.py:149-175) on top of the device prune: the Appendix A.5 sequence and a 120-add
    sequence with duplicates / dominated / dominating arrivals -- same kept evaluations, in the same order, with the same individuals,
    and the same archive size after EVERY add (goldens from the unmodified reference, tests/golden/make_golden.py)."""
    from morl_baselines_b200.common.pareto import ParetoArchive
    from tests.golden import cases

    arch = ParetoArchive()
    for i, e in enumerate([[1, 2], [2, 1], [1, 2], [3, 3], [0, 5]]):
        arch.add(i, np.array(e, dtype=np.float64))
    assert np.array_equal(np.array(arch.evaluations), golden["archive_a5_evals"])
    assert np.array_equal(np.array(arch.individuals), golden["archive_a5_inds"])
    arch = ParetoArchive()
    sizes = []
    for i, e in enumerate(cases.archive_sequence()):
        arch.add(i, e)
        sizes.append(len(arch.evaluations))
    assert np.array_equal(np.array(sizes, np.int32), golden["archive_seq_sizes"])
    assert np.array_equal(np.array(arch.evaluations), golden["archive_seq_evals"])
    assert np.array_equal(np.array(arch.individuals), golden["archive_seq_inds"])


@pytest.mark.parametrize("n,d", [(1, 1), (7, 1), (1, 2), (40, 2), (600, 2), (1, 3), (28, 3), (500, 3), (2048, 3)])
def test_device_hypervolume_matches_host_exact(cuda, n, d):
    """Exact device hypervolume (d <= 3) against the host exact sweep (common/performance_indicators.hypervolume, the routine the HV-parity
    protocol uses): same set -- with dominated points, duplicates, points below the reference point and a NaN row -- to 1e-12 relative
    (float64, different summation order); with a keep mask it equals the hypervolume of the kept subset."""
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.performance_indicators import hypervolume as hv_host

    rng = np.random.default_rng(n * 10 + d)
    pts = rng.random((n, d)) * 10.0 - 1.0  # some coordinates below the reference point 0
    if n > 4:
        pts[1] = pts[0]                     # duplicate
        pts[2] = pts[0] - 0.5               # dominated
        pts[3, 0] = np.nan
    ref = np.zeros(d)
    host_pts = pts[~np.isnan(pts).any(axis=1)]
    expect = hv_host(ref, list(host_pts))
    t = th.from_numpy(pts).to(cuda)
    got = float(ops.hypervolume(t, th.from_numpy(ref)))
    assert abs(got - expect) <= 1e-12 * max(1.0, abs(expect)), (got, expect)
    if n > 4:
        keep = ops.pareto_mask(t, True, raw=True)
        got_k = float(ops.hypervolume(t, th.from_numpy(ref), keep=keep))
        assert abs(got_k - expect) <= 1e-12 * max(1.0, abs(expect))  # pruning dominated points does not change the volume
    with pytest.raises(Exception):
        ops.hypervolume(th.zeros(3, 4, dtype=th.float64, device=cuda), th.zeros(4))


# ------------------------------------------------------------------------------------------------ device-resident PER
@pytest.mark.parametrize("max_size,n0", [(1000, 700), (4096, 4096), (65536, 50000)])
def test_device_sumtree_matches_reference(cuda, golden, max_size, n0):
    """DeviceSumTree against the goldens of the UNMODIFIED reference SumTree (tests/golden/make_golden.py gen_sumtree): same numpy RNG
    stream -> the same sampled indices in every round, and after four duplicate-laden batch_set rounds the same root and the same level
    arrays bit for bit (digest)."""
    from morl_baselines_b200.common.prioritized_buffer import DeviceSumTree

    tree = DeviceSumTree(max_size, cuda)
    rng = np.random.default_rng(max_size)
    tree.batch_set(np.arange(n0), rng.random(n0) + 1e-5)
    for rnd in range(4):
        np.random.seed(100 + rnd)
        idx = tree.sample(256)
        assert np.array_equal(idx, golden[f"sumtree_{max_size}_samples"][rnd])
        upd_idx = np.concatenate([idx, idx[:64]])
        tree.batch_set(upd_idx, rng.random(len(upd_idx)) * 3.0)
    nodes = tree.nodes
    assert nodes[0][0] == float(golden[f"sumtree_{max_size}_root"])
    assert cases.digest(np.concatenate(nodes)) == str(golden[f"sumtree_{max_size}_levels_sha"])


@pytest.mark.parametrize("size", [5, 100, 4096, 100000])
def test_device_sumtree_is_bit_identical_to_host_tree(cuda, size):
    """Random batches (duplicates, up to 1500 indices, beyond the 2048-per-launch limit once), single sets and walks: every level array
    and every walked index equals the host C tree's, which tests/test_host_logic.py pins to numpy's semantics."""
    from morl_baselines_b200.common.prioritized_buffer import DeviceSumTree, SumTree

    rng = np.random.default_rng(size)
    a, b = DeviceSumTree(size, cuda), SumTree(size)
    for it in range(12):
        n = int(rng.integers(1, 1500)) if it != 5 else 5000
        idx = rng.integers(0, size, n)
        pr = rng.random(n) * 10
        a.batch_set(idx, pr)
        b.batch_set(idx.copy(), pr)
        for la, lb in zip(a.nodes, b.nodes):
            assert np.array_equal(la, lb)
        q = rng.uniform(0, b.nodes[0][0], 777)
        assert np.array_equal(a.walk(q), b.walk(q))
    a.set(3 % size, 0.25)
    b.set(3 % size, 0.25)
    minp = th.full((1,), 0.75, device=cuda, dtype=th.float64)
    a.set(1 % size, None, minp)  # priority = the device-resident min_priority
    b.set(1 % size, 0.75)
    assert all(np.array_equal(x, y) for x, y in zip(a.nodes, b.nodes))
    import pickle

    c = pickle.loads(pickle.dumps(a))
    assert all(np.array_equal(x, y) for x, y in zip(a.nodes, c.nodes))
    with pytest.raises(Exception):
        a.batch_set(np.array([1 << 30]), np.array([1.0]))  # out-of-range leaf: flagged on the device, raised on the host


def test_device_per_priority_update(cuda):
    """(|w . td| + min_p) ** alpha in float32 (envelope.py:333), the min_priority ratchet (prioritized_buffer.py:194) and the tree
    write-back as two stream-ordered launches, against numpy: powers within 1 ulp of numpy's float32 power (the kernel rounds the float64
    power once; numpy's own SIMD / libm back ends differ from each other at that level), ratchet and tree exact given those powers."""
    from morl_baselines_b200.common.prioritized_buffer import PrioritizedReplayBuffer

    rb = PrioritizedReplayBuffer((4,), 1, rew_dim=2, max_size=512, device=cuda, tree_on_device=True)
    host = PrioritizedReplayBuffer((4,), 1, rew_dim=2, max_size=512)
    rng = np.random.default_rng(0)
    for k in range(300):
        tr = (rng.standard_normal(4).astype(np.float32), 0, rng.standard_normal(2).astype(np.float32), rng.standard_normal(4).astype(np.float32), False)
        rb.add(*tr)
        host.add(*tr)
    assert all(np.array_equal(x, y) for x, y in zip(rb.tree.nodes, host.tree.nodes))
    for rnd in range(3):
        idx = rng.integers(0, 300, 64)
        raw = (np.abs(rng.standard_normal(64)) * 10.0 ** rng.integers(-6, 2, 64)).astype(np.float32)
        p64 = th.zeros(64, dtype=th.float64, device=cuda)
        p32 = th.zeros(64, dtype=th.float32, device=cuda)
        rb.update_priorities_dev(th.from_numpy(idx).to(cuda), th.from_numpy(raw).to(cuda), 0.6, p64, p32)
        ref = (raw + np.float32(host.min_priority)) ** np.float32(0.6)
        got = p32.cpu().numpy()
        assert np.all(np.abs(got.view(np.int32) - ref.view(np.int32)) <= 1), "more than 1 ulp from numpy's float32 power"
        assert np.array_equal(got, ((raw + np.float32(host.min_priority)).astype(np.float64) ** np.float64(np.float32(0.6))).astype(np.float32))
        host.update_priorities(idx, got)  # same powers -> ratchet and tree must now agree exactly
        assert np.float32(rb.min_priority) == np.float32(host.min_priority)
        assert all(np.array_equal(x, y) for x, y in zip(rb.tree.nodes, host.tree.nodes))
    import pickle

    rb2 = pickle.loads(pickle.dumps(rb))
    assert not rb2.tree_on_device and np.array_equal(np.concatenate(rb2.tree.nodes), np.concatenate(host.tree.nodes))
    rb2.to(cuda)
    assert rb2.tree_on_device and np.array_equal(np.concatenate(rb2.tree.nodes), np.concatenate(host.tree.nodes))
    assert np.float32(rb2.min_priority) == np.float32(host.min_priority)
