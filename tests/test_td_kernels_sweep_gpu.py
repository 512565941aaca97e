"""Argument-space sweep of the per-row TD-target kernels (gpi_td.cu) and the TD-loss kernels (td_loss.cu).

Every case is compared twice:
  * with the CPU oracle (oracle/morl_oracle.c, the contract arithmetic): targets, indices, priorities and gathered Q bit for bit
    (compared on bit patterns, so NaNs compare too); loss scalars within 1e-6 relative;
  * with a float64 restatement in numpy, written here and independent of the oracle, so that an error shared by the kernel and the
    oracle also fails.

Float64 bounds (u = 2^-24, the unit roundoff of float32; every input below is a float32 value, so float64 holds it exactly).

  Scalarised score.  s = w . q over D terms in any of the three dot modes is D roundings (D products or FMAs and D - 1 sums), so
  |fl(s) - s| <= gamma_D * sum_r |w_r q_r| with gamma_D = D u / (1 - D u) < 1.0000005 D u  (Higham, Accuracy and Stability, 3.1).
  If the kernel picks c* from the float32 scores while c_best maximises the float64 ones, then
      s(c*) >= fl(s(c*)) - e >= fl(s(c_best)) - e >= s(c_best) - 2e,   e = gamma_D * max_c sum_r |w_r q_{c,r}|,
  so the INDEX CHECK asserts s(c*) >= max_c s(c) - 4 D u max_c sum|w||q|: twice the derived 2e.  A critic-min score min_n s_n
  moves by at most the same e, so the bound covers the critic-min candidates and the choice of the net (s_{n*} <= min_n s_n + 2e).

  Bellman line.  out = fl(r + fl(fl(nd * gamma) * q)) with nd = 1 - done exact for done in {0, 1}: three roundings, so
      |out - (r + nd gamma q)| <= u |r| + 3u |nd gamma q| + O(u^2) <= 2u (|r| + 2 |nd gamma q|),
  which is the VALUE CHECK (about 2 ulp of the larger of the two summands).  With an entropy term q is replaced by
  fl(q - fl(alpha logp)), which adds u |q| + 2u |alpha logp|; the bound used is 2u (|r| + 3 |nd gamma| (|q| + |alpha logp|)).
  MOSAC's scalar target also carries the score errors of w . r and min_n w . q_n: + 2 D u (sum|w||r| + |nd gamma| max_n sum|w||q_n|).

  Loss scalars.  The kernels square float32 residuals and sum them in a tree of float32 additions (D - 1 per row, 5 shuffle levels
  per warp, 3 across the warps of a block), then add the block partials in double.  A sum of non-negative terms through L levels has
  relative error <= L u, so the MSE term is within (D + 7 + 3) u <= 18 u = 1.07e-6 in the worst case, where every one of the ~10^6
  roundings errs in the same direction; with round-to-nearest on random data the errors have both signs and the observed error is
  far below that.  The test holds the loss to 1e-6 relative, the tolerance that the oracle comparison and torch's float reduction
  also use.  Huber terms are treated the same way; the branch of huber() is decided on the float32 residual, as the reference's
  float32 tensors decide it.

  Gradient.  td_mse: g = c1 d + c2 aux w_r, with c1 = 2 (1 - lambda) / (N D) and c2 = 2 lambda / N each two roundings, d one, the
  products one each and the sum one: |g - G| <= 5u (|T1| + |T2|) + |c2 w_r| |aux - AUX|, and aux = fl(w.q) - fl(w.t) is off by at most
  gamma_D (sum|w||q| + sum|w||t|) + u |aux|.  The bound used is 6u (|T1| + |T2|) + 2 |c2 w_r| D u (sum|w||q| + sum|w||t|).
  td_huber: g = d * fl(fl(1 / (N D)) / n_nets): three roundings, bound 4u |G|.

  Priorities.  |w . (q - t)| unfused: D + 1 roundings with the residual, bound 2 (D + 1) u sum|w||q - t|; the Huber priority scalarises
  max_n |d_n|, with the same bound on sum|w| max_n|d_n|.
"""

import numpy as np
import pytest
import torch as th

from oracle import oracle as orc

pytestmark = pytest.mark.gpu

U = 2.0**-24
MODES = (orc.DOT_UNFUSED, orc.DOT_FMA, orc.DOT_PAIRFMA)
TILE, BLOCK = orc.MAP_TILE, orc.MAP_BLOCK
GAMMA = 0.97


# ------------------------------------------------------------------------------------------------ plumbing
def _t(x, dev):
    return th.from_numpy(np.ascontiguousarray(x)).to(dev)


def _np(x):
    return None if x is None else x.cpu().numpy()


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.int32)


def _assert_bits(got, exp, msg):
    """Bit-pattern equality, except that any two NaNs match: the GPU returns its canonical NaN where x86 keeps or sets the sign and
    payload, and NaN payloads are not part of the contract.  A NaN against a number, or +0 against -0, still fails."""
    assert got.shape == exp.shape, msg
    g, e = got.reshape(-1), exp.reshape(-1)
    bad = np.flatnonzero((_bits(g) != _bits(e)) & ~(np.isnan(g) & np.isnan(e)))
    assert bad.size == 0, f"{msg}: {bad.size} elements differ, first at {bad[:5]}: {got.reshape(-1)[bad[:5]]} vs {exp.reshape(-1)[bad[:5]]}"


def _map_rows(rows, n, m):
    """Row index of X[k] under the maps of include/morl_b200.h, restated here: TILE k % rows, BLOCK k / (n / rows)."""
    k = np.arange(n)
    if rows == n:
        return k
    if rows == 1:
        return np.zeros(n, np.int64)
    return k % rows if m == TILE else k // (n // rows)


def _weights(rng, n, d, quantised=False):
    if quantised:
        return (rng.integers(1, 4, size=(n, d)) / 8.0).astype(np.float32)
    w = np.abs(rng.standard_normal((n, d)))
    return (w / w.sum(1, keepdims=True)).astype(np.float32)


def _values(rng, shape, kind):
    """plain: continuous; ties: small integers (every score exact, many exact ties); neartie: per row one base vector times
    (1 + k 2^-23), k in 0..5, so that the candidates of a row are a few ulps apart and the dot modes round them differently."""
    if kind == "ties":
        return rng.integers(-2, 3, size=shape).astype(np.float32)
    if kind == "neartie":
        base_shape = list(shape)
        base_shape[-2] = 1  # one base per row, shared by the candidates (and the nets)
        base_shape[0] = 1 if len(shape) == 4 else base_shape[0]
        base = rng.standard_normal(base_shape).astype(np.float32)
        q = (base * (1.0 + rng.integers(0, 6, size=shape) * np.float32(2.0**-23))).astype(np.float32)
        return q
    return (rng.standard_normal(shape) * 3.0).astype(np.float32)


def _bellman_bound(r, nd_g, q):
    return 2 * U * (np.abs(r) + 2 * np.abs(nd_g * q))


# ------------------------------------------------------------------------------------------------ kernel calls (numpy in, numpy out)
def _k_greedy(dev, qs, qe, w, rew, done, mode, w_map, r_map):
    from morl_baselines_b200 import ops

    o, a = ops.greedy_td(_t(qs, dev), _t(qe, dev), _t(w, dev), None if rew is None else _t(rew, dev), None if done is None else _t(done, dev),
                         GAMMA, mode, w_map, r_map)
    return _np(o), _np(a)


def _k_critic_min(dev, q, w, rew, done, mode, w_map, r_map):
    from morl_baselines_b200 import ops

    o, a = ops.critic_min_td(_t(q, dev), _t(w, dev), None if rew is None else _t(rew, dev), None if done is None else _t(done, dev),
                             GAMMA, mode, w_map, r_map)
    return _np(o), _np(a)


def _k_gpi(dev, q, w, rew, done, mode, w_map, r_map):
    from morl_baselines_b200 import ops

    o, p, a = ops.gpi_envelope(_t(q, dev), _t(w, dev), None if rew is None else _t(rew, dev), None if done is None else _t(done, dev),
                               GAMMA if rew is not None else 0.0, mode, w_map, r_map)
    return _np(o), _np(p), _np(a)


# ------------------------------------------------------------------------------------------------ float64 target checks
def _scores64(q, w_full):
    """q [n, N, C, D] float32, w_full [N, D] -> float64 scores [n, N, C] and magnitudes sum|w||q| [n, N, C]."""
    q64, w64 = q.astype(np.float64), w_full.astype(np.float64)[None, :, None, :]
    with np.errstate(invalid="ignore", over="ignore"):
        return (q64 * w64).sum(-1), (np.abs(q64) * np.abs(w64)).sum(-1)


def _check_target64(q_sel, q_eval, w_full, idx, out, rew_full, done_full, msg):
    """q_sel, q_eval [n, N, C, D] (q_eval is q_sel for the critic-min kernels); idx [N] chosen candidate; out [N, D].
    Checks the index against the float64 maximum of the critic-min scores and the target against the float64 Bellman line of the
    chosen Q vector of some net whose score is within the bound of the critic-min (the kernels do not report the net)."""
    n, N, C, D = q_sel.shape
    s, mag = _scores64(q_sel, w_full)
    with np.errstate(invalid="ignore"):
        smin = np.where(np.isnan(s).any(0), -np.inf, s.min(0))  # [N, C]; a NaN score never wins
    finite = np.isfinite(smin)
    e_row = np.where(finite, mag.max(0), 0.0).max(1)  # largest sum|w||q| among the finite candidates of the row
    bound = 4 * D * U * e_row
    best = smin.max(1)
    rows = np.arange(N)
    got = smin[rows, idx]
    fin = np.isfinite(best)
    bad = np.flatnonzero(fin & ~(got >= best - bound))
    assert bad.size == 0, f"{msg}: index off the float64 maximum in rows {bad[:5]} ({got[bad[:5]]} vs {best[bad[:5]]})"
    assert np.all(got[best == np.inf] == np.inf), f"{msg}: a +inf candidate exists but did not win"
    assert np.all(idx[best == -np.inf] == 0), f"{msg}: rows without a finite or +inf score must fall back to candidate 0"
    # value: some net within the bound of the critic-min gives the output
    qv = q_eval[:, rows, idx].astype(np.float64)  # [n, N, D]
    s_at = s[:, rows, idx]  # [n, N]
    with np.errstate(invalid="ignore"):
        net_ok = (s_at <= (smin[rows, idx] + bound)[None]) | ~np.isfinite(smin[rows, idx])[None]
    if rew_full is None:
        match = np.stack([np.all(_bits(q_eval[k, rows, idx]) == _bits(out), axis=1) for k in range(n)])
    else:
        r64 = rew_full.astype(np.float64)
        nd_g = ((1.0 - done_full.astype(np.float64)) * GAMMA)[None, :, None]
        with np.errstate(invalid="ignore", over="ignore"):
            ref = r64[None] + nd_g * qv
            err = np.abs(out.astype(np.float64)[None] - ref)
            ok = (err <= _bellman_bound(r64[None], nd_g, qv)) | (out[None] == ref) | (np.isnan(out)[None] & np.isnan(ref))
        match = ok.all(2)
    good = (match & net_ok).any(0)
    bad = np.flatnonzero(~good)
    assert bad.size == 0, f"{msg}: target off the float64 Bellman line of the chosen Q vector in rows {bad[:5]}"


def _greedy_case(dev, rng, N, A, D, kind, modes=MODES, w_rows=None, w_map=BLOCK, r_rows=None, r_map=TILE, reward=True):
    w_rows = N if w_rows is None else w_rows
    r_rows = N if r_rows is None else r_rows
    qs, qe = _values(rng, (N, A, D), kind), rng.standard_normal((N, A, D)).astype(np.float32)
    w = _weights(rng, w_rows, D, kind == "ties")
    rew = rng.standard_normal((r_rows, D)).astype(np.float32) if reward else None
    done = (rng.random(r_rows) < 0.25).astype(np.float32) if reward else None
    wf = w[_map_rows(w_rows, N, w_map)]
    rf = None if rew is None else rew[_map_rows(r_rows, N, r_map)]
    df = None if done is None else done[_map_rows(r_rows, N, r_map)]
    acts = {}
    for mode in modes:
        msg = f"greedy N={N} A={A} D={D} {kind} mode={mode} w={w_rows}/{w_map} r={r_rows}/{r_map}"
        o, a = _k_greedy(dev, qs, qe, w, rew, done, mode, w_map, r_map)
        # the oracle on fully materialised rows: the maps of the kernel are checked against the header's definition
        oo, ao = orc.greedy_td(qs, qe, wf, rf, df, GAMMA, mode)
        assert np.array_equal(a, ao), msg
        _assert_bits(o, oo, msg)
        _check_target64(qs[None], qe[None], wf, a, o, rf, df, msg)
        acts[mode] = ao
    return acts


def _critic_min_case(dev, rng, n_nets, N, A, D, kind, modes=MODES, w_rows=None, w_map=BLOCK, r_rows=None, r_map=TILE, reward=True):
    w_rows = N if w_rows is None else w_rows
    r_rows = N if r_rows is None else r_rows
    q = _values(rng, (n_nets, N, A, D), kind)
    w = _weights(rng, w_rows, D, kind == "ties")
    rew = rng.standard_normal((r_rows, D)).astype(np.float32) if reward else None
    done = (rng.random(r_rows) < 0.25).astype(np.float32) if reward else None
    wf = w[_map_rows(w_rows, N, w_map)]
    rf = None if rew is None else rew[_map_rows(r_rows, N, r_map)]
    df = None if done is None else done[_map_rows(r_rows, N, r_map)]
    acts = {}
    for mode in modes:
        msg = f"critic_min n={n_nets} N={N} A={A} D={D} {kind} mode={mode} w={w_rows}/{w_map} r={r_rows}/{r_map}"
        o, a = _k_critic_min(dev, q, w, rew, done, mode, w_map, r_map)
        oo, ao = orc.critic_min_td(q, wf, rf, df, GAMMA, mode)
        assert np.array_equal(a, ao), msg
        _assert_bits(o, oo, msg)
        _check_target64(q, q, wf, a, o, rf, df, msg)
        acts[mode] = ao
    return acts


def _gpi_case(dev, rng, n_nets, B, P, A, D, kind, modes=MODES, w_rows=None, w_map=BLOCK, r_rows=None, r_map=TILE, reward=True, q=None):
    w_rows = B if w_rows is None else w_rows
    r_rows = B if r_rows is None else r_rows
    if q is None:
        q = _values(rng, (n_nets, B, P * A, D), kind).reshape(n_nets, B, P, A, D)
    w = _weights(rng, w_rows, D, kind == "ties")
    rew = rng.standard_normal((r_rows, D)).astype(np.float32) if reward else None
    done = (rng.random(r_rows) < 0.25).astype(np.float32) if reward else None
    wf = w[_map_rows(w_rows, B, w_map)]
    rf = None if rew is None else rew[_map_rows(r_rows, B, r_map)]
    df = None if done is None else done[_map_rows(r_rows, B, r_map)]
    idx = {}
    for mode in modes:
        msg = f"gpi n={n_nets} B={B} P={P} A={A} D={D} {kind} mode={mode} w={w_rows}/{w_map} r={r_rows}/{r_map}"
        o, p, a = _k_gpi(dev, q, w, rew, done, mode, w_map, r_map)
        oo, po, ao = orc.gpi_envelope(q, wf, rf, df, GAMMA if reward else 0.0, mode)
        assert np.array_equal(p, po) and np.array_equal(a, ao), msg
        _assert_bits(o, oo, msg)
        qf = q.reshape(n_nets, B, P * A, D)
        _check_target64(qf, qf, wf, p * A + a, o, rf, df, msg)
        idx[mode] = po * A + ao
    return idx


# ------------------------------------------------------------------------------------------------ targets: D x dot mode
@pytest.mark.parametrize("D", range(1, 9))
@pytest.mark.parametrize("kernel", ["greedy", "critic_min", "gpi"])
def test_target_every_d_and_dot_mode(cuda, kernel, D):
    """D = 1..8 (one template instance each) in all three dot modes, on continuous, exactly tied and near-tied data.  The near-tie rows
    must make the modes disagree on some indices (D >= 2: unfused vs FMA; D >= 3: pair-FMA vs both), so that a kernel that ignored
    dot_mode, or summed the pair-FMA odd tail in another place, fails the bitwise oracle comparison.  At D = 1 the three modes are the
    same single product, and at D = 2 pair-FMA is the FMA chain; the test asserts that too."""
    rng = np.random.default_rng(100 * D + len(kernel))
    for kind in ("plain", "ties", "neartie"):
        if kernel == "greedy":
            got = _greedy_case(cuda, rng, 1024, 7, D, kind)
        elif kernel == "critic_min":
            got = _critic_min_case(cuda, rng, 2, 1024, 7, D, kind)
        else:
            got = _gpi_case(cuda, rng, 2, 512, 3, 11, D, kind)
        if kind != "neartie":
            continue
        diff = lambda m1, m2: int((got[m1] != got[m2]).sum())  # noqa: E731
        if D == 1:
            assert diff(0, 1) == 0 and diff(0, 2) == 0
        else:
            assert diff(orc.DOT_UNFUSED, orc.DOT_FMA) > 0, "near-tie data does not separate unfused from FMA"
        if D == 2:
            assert diff(orc.DOT_FMA, orc.DOT_PAIRFMA) == 0
        if D >= 3:
            assert diff(orc.DOT_PAIRFMA, orc.DOT_FMA) > 0 and diff(orc.DOT_PAIRFMA, orc.DOT_UNFUSED) > 0, "pair-FMA not separated"


# ------------------------------------------------------------------------------------------------ targets: row maps
W_COMBOS = [(1, 1, BLOCK), (1, 1, TILE), (2, 1, BLOCK), (2, 1, TILE), (3, 1, BLOCK), (3, 1, TILE), (0, 1, BLOCK), (0, 1, TILE)]  # N / k rows


@pytest.mark.parametrize("w_div,_unused,w_map", W_COMBOS, ids=[f"w{'N' if d == 1 else ('1' if d == 0 else f'N/{d}')}-{'block' if m else 'tile'}"
                                                            for d, _, m in W_COMBOS])
@pytest.mark.parametrize("kernel", ["greedy", "critic_min", "gpi"])
def test_target_row_maps(cuda, kernel, w_div, _unused, w_map):
    """w_rows in {N, 1, N/2, N/3} x {BLOCK, TILE} against r_rows in {N, N/2} x {BLOCK, TILE}, at D = 2 and D = 5.  The oracle is called
    with rows materialised by the header's definition of the maps, so a kernel that swapped TILE and BLOCK fails."""
    N = 384
    w_rows = 1 if w_div == 0 else N // w_div
    rng = np.random.default_rng(7 * w_div + w_map + 31 * len(kernel))
    for D in (2, 5):
        for r_rows in (N, N // 2):
            for r_map in (BLOCK, TILE):
                for kind in ("plain", "ties"):
                    kw = dict(modes=(orc.DOT_UNFUSED,), w_rows=w_rows, w_map=w_map, r_rows=r_rows, r_map=r_map)
                    if kernel == "greedy":
                        _greedy_case(cuda, rng, N, 7, D, kind, **kw)
                    elif kernel == "critic_min":
                        _critic_min_case(cuda, rng, 3, N, 7, D, kind, **kw)
                    else:
                        _gpi_case(cuda, rng, 2, N, 3, 5, D, kind, **kw)


@pytest.mark.parametrize("case", ["gpi_pd_doubled_critic_min", "gpi_pd_doubled_gpi_envelope", "envelope_ddqn_greedy", "gpi_action", "max_action"])
def test_target_call_sites(cuda, case):
    """The row-map combinations the algorithms pass:
      * GPI-PD's doubled batch (gpi_pd.py:354 and :451): 2 B0 rows with a weight per row, reward and done un-tiled (B0 rows, TILE);
      * the Envelope's DDQN target (envelope.py:471): N = B W rows in b-major order, w TILE over the W sampled weights, reward BLOCK
        over the B transitions;
      * gpi_action / max_action: one row, one shared weight, one net, no Bellman line."""
    rng = np.random.default_rng(len(case))
    for kind in ("plain", "ties"):
        for D in (2, 3):
            if case == "gpi_pd_doubled_critic_min":
                _critic_min_case(cuda, rng, 2, 256, 6, D, kind, w_rows=256, r_rows=128, r_map=TILE)
            elif case == "gpi_pd_doubled_gpi_envelope":
                _gpi_case(cuda, rng, 2, 256, 5, 6, D, kind, w_rows=256, r_rows=128, r_map=TILE)
            elif case == "envelope_ddqn_greedy":
                B, W = 64, 8
                _greedy_case(cuda, rng, B * W, 8, D, kind, w_rows=W, w_map=TILE, r_rows=B, r_map=BLOCK)
            elif case == "gpi_action":
                _gpi_case(cuda, rng, 1, 1, 9, 6, D, kind, w_rows=1, reward=False)
            else:
                _gpi_case(cuda, rng, 1, 1, 1, 7, D, kind, w_rows=1, reward=False)


# ------------------------------------------------------------------------------------------------ targets: n_nets, A, candidates
@pytest.mark.parametrize("n_nets", [1, 2, 3, 5])
@pytest.mark.parametrize("A", [1, 2, 7, 33])
def test_critic_min_nets_and_actions(cuda, n_nets, A):
    rng = np.random.default_rng(10 * n_nets + A)
    for kind in ("plain", "ties"):
        _critic_min_case(cuda, rng, n_nets, 300, A, 3, kind)
    if n_nets == 1:
        _greedy_case(cuda, rng, 300, A, 3, "plain")
        _greedy_case(cuda, rng, 300, A, 4, "ties")


GPI_PA = [(1, 1), (31, 1), (4, 8), (3, 11), (2, 32), (36, 32)]  # P * A = 1, 31, 32, 33, 64, 1152


@pytest.mark.parametrize("P,A", GPI_PA, ids=[f"PA{p * a}" for p, a in GPI_PA])
def test_gpi_envelope_candidates_and_warps(cuda, P, A):
    """One warp walks the P*A candidates of a row with a stride of 32 lanes; 4 rows per CTA, so B = 1, 3, 4, 5, 129 leaves 3, 1, 0, 3
    and 3 warps of the last CTA idle."""
    rng = np.random.default_rng(P * 100 + A)
    for B in (1, 3, 4, 5, 129):
        for n_nets, kind in ((1, "plain"), (3, "ties"), (2, "neartie")):
            _gpi_case(cuda, rng, n_nets, B, P, A, 3, kind)


# ------------------------------------------------------------------------------------------------ targets: ties
@pytest.mark.parametrize("n_nets", [1, 2, 3, 5])
@pytest.mark.parametrize("kernel", ["greedy", "critic_min", "gpi"])
def test_target_exact_ties(cuda, kernel, n_nets):
    """Quantised Q and weights: exact ties across actions, across nets (equal scores from different Q vectors, so the first argmin
    decides which vector is gathered) and across policies.  First occurrence wins everywhere."""
    rng = np.random.default_rng(n_nets + 11 * len(kernel))
    for D in (1, 2, 3, 6):
        if kernel == "greedy":
            _greedy_case(cuda, rng, 512, 6, D, "ties")
        elif kernel == "critic_min":
            _critic_min_case(cuda, rng, n_nets, 512, 6, D, "ties")
        else:
            _gpi_case(cuda, rng, n_nets, 256, 4, 6, D, "ties")
    # the data really contain ties between nets with different vectors
    q = _values(rng, (2, 512, 6, 2), "ties")
    w = np.full((512, 2), 0.25, np.float32)
    s = (q * w[None, :, None]).sum(-1)
    assert ((s[0] == s[1]) & (q[0] != q[1]).any(-1)).sum() > 100


def test_gpi_envelope_tie_across_lanes(cuda):
    """Two equal best candidates on different lanes (c1 % 32 != c2 % 32): the warp merge's (value desc, index asc) rule must return the
    smaller index whichever lane holds it, and for two on the same lane (c, c + 32) the lane's own strict '>' keeps the first."""
    rng = np.random.default_rng(5)
    n_nets, B, P, A, D = 2, 129, 8, 12, 3  # P * A = 96: three candidates per lane
    q = (rng.standard_normal((n_nets, B, P * A, D)) * 0.1).astype(np.float32)
    top = np.float32(4.0)
    pairs = []
    for b in range(B):
        c1, c2 = sorted(rng.choice(P * A, size=2, replace=False))
        if b % 4 == 0:
            c1, c2 = 1, 16  # lane 0 meets 16 before 1 in the xor tree
        elif b % 4 == 1:
            c1 = c2 % 32  # same lane
        q[:, b, c1] = top
        q[:, b, c2] = top
        pairs.append((c1, c2))
    idx = _gpi_case(cuda, rng, n_nets, B, P, A, D, "plain", q=q.reshape(n_nets, B, P, A, D))
    exp = np.array([min(c) for c in pairs])
    for mode, got in idx.items():
        assert np.array_equal(got, exp), mode


# ------------------------------------------------------------------------------------------------ targets: special values
def _special_rows(rng, n_nets, N, C, D):
    """Rows of scores with +inf, -inf and NaN candidates (whole Q vectors, every net, positive weights: the score is that value in every
    dot mode and in float64).  Returns q [n, N, C, D] and the expected index under the kernels' rule (first argmax from -inf with a strict
    '>': a NaN never wins; all -inf / NaN -> candidate 0), where the rest of the row is well separated."""
    q = rng.standard_normal((n_nets, N, C, D)).astype(np.float32)
    kinds = ["nan0", "nanmid", "allnan", "allneginf", "neginf0_nan", "posinf", "posinf_twice", "nan_then_posinf", "plain"]
    for k in range(N):
        kind = kinds[k % len(kinds)]
        c = rng.integers(1, C) if C > 1 else 0
        if kind == "nan0":
            q[:, k, 0] = np.nan
        elif kind == "nanmid":
            q[:, k, c] = np.nan
        elif kind == "allnan":
            q[:, k] = np.nan
        elif kind == "allneginf":
            q[:, k] = -np.inf
        elif kind == "neginf0_nan":
            q[:, k] = -np.inf
            q[:, k, c] = np.nan
        elif kind == "posinf":
            q[:, k, c] = np.inf
        elif kind == "posinf_twice":
            q[:, k, c] = np.inf
            q[:, k, C - 1] = np.inf
        elif kind == "nan_then_posinf":
            q[:, k, 0] = np.nan
            q[:, k, c] = np.inf
    return q


@pytest.mark.parametrize("kernel", ["greedy", "critic_min", "gpi"])
def test_target_special_values(cuda, kernel):
    """+inf / -inf / NaN scores.  The rule pinned here, against the oracle and the float64 check: first argmax with a strict '>' from
    -inf, so a NaN score never wins (th.argmax would pick it: a deviation that only matters once training has diverged), and a row
    whose every score is -inf or NaN takes candidate 0 (for gpi_envelope with the critic-min net of candidate 0)."""
    rng = np.random.default_rng(len(kernel))
    N = 360
    for D in (1, 3, 5):
        msg = f"{kernel} special D={D}"
        n_nets, C = (1, 7) if kernel == "greedy" else ((2, 7) if kernel == "critic_min" else (2, 40))
        q = _special_rows(rng, n_nets, N, C, D)
        w = _weights(rng, N, D)
        rew = rng.standard_normal((N, D)).astype(np.float32)
        done = (rng.random(N) < 0.3).astype(np.float32)
        for mode in MODES:
            if kernel == "greedy":
                qe = rng.standard_normal((N, C, D)).astype(np.float32)
                o, idx = _k_greedy(cuda, q[0], qe, w, rew, done, mode, BLOCK, TILE)
                oo, io = orc.greedy_td(q[0], qe, w, rew, done, GAMMA, mode)
                _check_target64(q, qe[None], w, idx, o, rew, done, msg)
            elif kernel == "critic_min":
                o, idx = _k_critic_min(cuda, q, w, rew, done, mode, BLOCK, TILE)
                oo, io = orc.critic_min_td(q, w, rew, done, GAMMA, mode)
                _check_target64(q, q, w, idx, o, rew, done, msg)
            else:
                q5 = q.reshape(n_nets, N, 8, 5, D)
                o, p, a = _k_gpi(cuda, q5, w, rew, done, mode, BLOCK, TILE)
                oo, po, ao = orc.gpi_envelope(q5, w, rew, done, GAMMA, mode)
                idx, io = p * 5 + a, po * 5 + ao
                _check_target64(q, q, w, idx, o, rew, done, msg)
            assert np.array_equal(idx, io), msg
            _assert_bits(o, oo, msg)
            assert np.array_equal(idx, _rule_argmax(q, w)), msg


def _rule_argmax(q, w):
    """Expected index for the rows of _special_rows (NaN / inf set on every net at once, finite candidates well separated):
    NaN never wins, a row with only -inf / NaN scores takes candidate 0."""
    with np.errstate(invalid="ignore"):
        s = (q.astype(np.float64) * w.astype(np.float64)[None, :, None, :]).sum(-1).min(0)
    s = np.where(np.isnan(s), -np.inf, s)
    return np.where(s.max(1) == -np.inf, 0, s.argmax(1)).astype(np.int32)


def test_critic_min_nan_in_a_later_net(cuda):
    """A NaN score at net n > 0 never replaces the running minimum (strict '<'); a NaN at net 0 stays and makes the candidate lose."""
    rng = np.random.default_rng(9)
    n_nets, N, A, D = 3, 256, 5, 3
    q = rng.standard_normal((n_nets, N, A, D)).astype(np.float32)
    q[1, ::2, 2] = np.nan  # later net: ignored
    q[0, 1::2, 3] = np.nan  # net 0: the candidate never wins
    w = _weights(rng, N, D)
    o, a = _k_critic_min(cuda, q, w, None, None, 0, BLOCK, TILE)
    oo, ao = orc.critic_min_td(q, w, None, None, 0.0, 0)
    assert np.array_equal(a, ao)
    _assert_bits(o, oo, "critic_min NaN nets")
    assert not np.any(a[1::2] == 3)
    s = (q.astype(np.float64) * w[None, :, None]).sum(-1)
    s_ignore = np.where(np.isnan(s) & (np.arange(n_nets)[:, None, None] > 0), np.inf, s).min(0)
    s_ignore = np.where(np.isnan(s_ignore), -np.inf, s_ignore)
    assert np.array_equal(a, s_ignore.argmax(1))


# ------------------------------------------------------------------------------------------------ targets: NULL outputs
def test_null_outputs_through_the_c_abi(cuda):
    """gpi_envelope with only act_out or only policy_out gives the same indices; greedy_td / critic_min_td with act_out = NULL give the
    same target (called through _lib.load() as ops.py does)."""
    from morl_baselines_b200 import _lib

    lib = _lib.load()
    st = th.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(4)
    n_nets, B, P, A, D = 2, 77, 5, 7, 3
    q = _t(_values(rng, (n_nets, B, P * A, D), "ties"), cuda)
    w = _t(_weights(rng, B, D, True), cuda)
    out, pol, act = (th.empty(B, D, device=cuda), th.full((B,), -7, dtype=th.int32, device=cuda), th.full((B,), -7, dtype=th.int32, device=cuda))
    _lib.check(lib.morl_gpi_envelope_f32(q.data_ptr(), n_nets, w.data_ptr(), B, BLOCK, None, None, B, TILE, 0.0, B, P, A, D, 0, out.data_ptr(),
                                         pol.data_ptr(), act.data_ptr(), st), "gpi")
    pol_only, act_only = th.full_like(pol, -7), th.full_like(act, -7)
    _lib.check(lib.morl_gpi_envelope_f32(q.data_ptr(), n_nets, w.data_ptr(), B, BLOCK, None, None, B, TILE, 0.0, B, P, A, D, 0, None,
                                         pol_only.data_ptr(), None, st), "gpi policy only")
    _lib.check(lib.morl_gpi_envelope_f32(q.data_ptr(), n_nets, w.data_ptr(), B, BLOCK, None, None, B, TILE, 0.0, B, P, A, D, 0, None, None,
                                         act_only.data_ptr(), st), "gpi act only")
    assert th.equal(pol_only, pol) and th.equal(act_only, act)
    N = 300
    qs, qe = _t(_values(rng, (N, A, D), "ties"), cuda), _t(rng.standard_normal((N, A, D)).astype(np.float32), cuda)
    qn = _t(_values(rng, (n_nets, N, A, D), "ties"), cuda)
    wn = _t(_weights(rng, N, D, True), cuda)
    rew, done = _t(rng.standard_normal((N, D)).astype(np.float32), cuda), _t((rng.random(N) < 0.3).astype(np.float32), cuda)
    for name, args in (("morl_greedy_td_f32", (qs.data_ptr(), qe.data_ptr())), ("morl_critic_min_td_f32", (qn.data_ptr(), n_nets))):
        outs = []
        for with_act in (True, False):
            o, a = th.empty(N, D, device=cuda), th.empty(N, dtype=th.int32, device=cuda)
            _lib.check(getattr(lib, name)(*args, wn.data_ptr(), N, BLOCK, rew.data_ptr(), done.data_ptr(), N, TILE, GAMMA, N, A, D, 1, o.data_ptr(),
                                          a.data_ptr() if with_act else None, st), name)
            outs.append(o)
        assert th.equal(outs[0].view(th.int32), outs[1].view(th.int32)), name


# ------------------------------------------------------------------------------------------------ actor-critic targets
@pytest.mark.parametrize("n_nets", [1, 2, 3])
@pytest.mark.parametrize("D", range(1, 9))
@pytest.mark.parametrize("variant", [orc.AC_ELEMENTWISE_MIN, orc.AC_SCALAR_MIN, orc.AC_ARGMIN_GATHER])
def test_actor_critic_td_sweep(cuda, variant, D, n_nets):
    """Every variant x D = 1..8 x n_nets 1..3, w_rows in {1, N/4 (both maps), N}, logp given or None; bitwise against the oracle, within
    the derived bound against float64."""
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(100 * variant + 10 * D + n_nets)
    N = 260
    for w_rows, w_map in ((1, BLOCK), (1, TILE), (N // 4, BLOCK), (N // 4, TILE), (N, BLOCK), (N, TILE)):
        for with_logp in (True, False):
            msg = f"variant={variant} D={D} n={n_nets} w={w_rows}/{w_map} logp={with_logp}"
            q = rng.standard_normal((n_nets, N, D)).astype(np.float32)
            q[:, ::7] = rng.integers(-2, 3, size=(n_nets, len(q[0, ::7]), D))  # exact ties between critics
            w = _weights(rng, w_rows, D, quantised=True)
            w[::2] = _weights(rng, len(w[::2]), D)
            rew = rng.standard_normal((N, D)).astype(np.float32)
            done = (rng.random(N) < 0.25).astype(np.float32)
            logp = rng.standard_normal(N).astype(np.float32) if with_logp else None
            alpha = 0.2
            got = _np(ops.actor_critic_td(_t(q, cuda), _t(w, cuda), _t(rew, cuda), _t(done, cuda), None if logp is None else _t(logp, cuda), alpha,
                                          GAMMA, variant, w_map))
            wf = w[_map_rows(w_rows, N, w_map)]
            exp = orc.actor_critic_td(q, wf, rew, done, logp, alpha, GAMMA, variant)
            _assert_bits(got, exp, msg)
            # float64
            q64, w64, r64 = q.astype(np.float64), wf.astype(np.float64), rew.astype(np.float64)
            ent = np.zeros(N) if logp is None else np.float32(alpha) * logp.astype(np.float64)
            nd_g = (1.0 - done.astype(np.float64)) * GAMMA
            if variant == orc.AC_ELEMENTWISE_MIN:
                m = q64.min(0)
                ref = r64 + nd_g[:, None] * (m - ent[:, None])
                bound = 2 * U * (np.abs(r64) + 3 * np.abs(nd_g[:, None]) * (np.abs(m) + np.abs(ent[:, None])))
                assert np.all(np.abs(got - ref) <= bound), msg
            elif variant == orc.AC_SCALAR_MIN:
                s = (q64 * w64[None]).sum(-1)
                mag = (np.abs(q64) * w64[None]).sum(-1).max(0)
                rs = (r64 * w64).sum(-1)
                m = s.min(0)
                ref = rs + nd_g * (m - ent)
                bound = 2 * U * (np.abs(rs) + 3 * np.abs(nd_g) * (np.abs(m) + np.abs(ent))) + 2 * D * U * ((np.abs(r64) * w64).sum(-1) + np.abs(nd_g) * mag)
                assert np.all(np.abs(got - ref) <= bound), msg
            else:
                s = (q64 * w64[None]).sum(-1)
                mag = (np.abs(q64) * w64[None]).sum(-1).max(0)
                ok_net = s <= s.min(0) + 4 * D * U * mag  # [n, N]
                soft = q64 - ent[None, :, None]
                ref = r64[None] + nd_g[None, :, None] * soft
                bound = 2 * U * (np.abs(r64)[None] + 3 * np.abs(nd_g)[None, :, None] * (np.abs(q64) + np.abs(ent)[None, :, None]))
                match = (np.abs(got[None] - ref) <= bound).all(-1) & ok_net
                assert match.any(0).all(), msg


# ------------------------------------------------------------------------------------------------ td_mse_priority
def _mse_inputs(rng, B, W, A, D):
    qv = rng.standard_normal((B * W, A, D)).astype(np.float32)
    tq = rng.standard_normal((B * W, D)).astype(np.float32)
    wset = _weights(rng, W, D)
    act = rng.integers(0, A, size=B).astype(np.int32)
    return qv, act, tq, wset


def _mse_call(dev, qv, act, tq, wset, lam, B, W, order, **kw):
    from morl_baselines_b200 import ops

    loss, grad, prio = ops.td_mse_priority(_t(qv, dev), _t(act, dev), _t(tq, dev), _t(wset, dev), lam, B, W, order, **kw)
    return float(_np(loss)[0]), _np(grad), _np(prio)


def _check_mse64(loss, grad, prio, qv, act, tq, wset, lam, B, W, order, msg):
    N, A, D = qv.shape
    k = np.arange(N)
    i_of, b_of = (k // B, k % B) if order == orc.ROWS_REFERENCE else (k % W, k // W)
    a = act[b_of]
    q = qv[k, a].astype(np.float64)
    t, w = tq.astype(np.float64), wset[i_of].astype(np.float64)
    lam = float(np.float32(lam))
    d = q - t
    aux = (w * q).sum(1) - (w * t).sum(1)
    ref = (1 - lam) * np.mean(d * d) + lam * np.mean(aux * aux)
    assert abs(loss - ref) <= 1e-6 * abs(ref), f"{msg}: loss {loss} vs float64 {ref}"
    if grad is not None:
        c1, c2 = (1 - lam) * 2 / (N * D), lam * 2 / N
        T1, T2 = c1 * d, c2 * aux[:, None] * w
        G = np.zeros_like(qv, dtype=np.float64)
        G[k, a] = T1 + T2
        gb = np.zeros_like(G)
        gb[k, a] = 6 * U * (np.abs(T1) + np.abs(T2)) + 2 * np.abs(c2 * w) * D * U * ((np.abs(w * q)).sum(1) + (np.abs(w * t)).sum(1))[:, None]
        bad = np.flatnonzero(~(np.abs(grad - G) <= gb))
        assert bad.size == 0, f"{msg}: gradient off float64 at {bad[:5]}"
    if prio is not None:
        first = i_of == 0
        P = np.zeros(B)
        Pb = np.zeros(B)
        P[b_of[first]] = np.abs((w[first] * d[first]).sum(1))
        Pb[b_of[first]] = 2 * (D + 1) * U * (np.abs(w[first] * d[first])).sum(1)
        assert np.all(np.abs(prio - P) <= Pb), f"{msg}: priorities off float64"


@pytest.mark.parametrize("D", range(1, 9))
@pytest.mark.parametrize("order", [orc.ROWS_REFERENCE, orc.ROWS_BMAJOR])
def test_td_mse_sweep(cuda, order, D):
    """Both row orders x lambda in {0, 0.35, 1} x D = 1..8 x A in {4, 7} (A D = 0 mod 4 takes the float4 gradient writer at every D; A = 7
    takes the scalar writer unless D = 4, 8)."""
    rng = np.random.default_rng(10 * D + order)
    for A in (4, 7):
        for lam in (0.0, 0.35, 1.0):
            B, W = 67, 12
            qv, act, tq, wset = _mse_inputs(rng, B, W, A, D)
            msg = f"td_mse order={order} D={D} A={A} lam={lam}"
            loss, grad, prio = _mse_call(cuda, qv, act, tq, wset, lam, B, W, order)
            lo, go, _, po = orc.td_mse(qv, act, tq, wset, lam, B, W, order)
            assert abs(loss - lo) <= 1e-6 * abs(lo), msg
            _assert_bits(prio, po, msg)
            _check_mse64(loss, grad, prio, qv, act, tq, wset, lam, B, W, order, msg)
            assert np.count_nonzero(grad) == np.count_nonzero(go), msg  # zero off the taken action


@pytest.mark.parametrize("B", [1024, 1025])
def test_td_mse_north_star_partials(cuda, B):
    """N = 1024 x 64 = 65,536 rows is exactly 256 block partials, one per finalize thread; N = 1025 x 64 gives 257, so the finalize loop
    runs a second iteration for thread 0."""
    rng = np.random.default_rng(B)
    W, A, D = 64, 8, 3
    qv, act, tq, wset = _mse_inputs(rng, B, W, A, D)
    for lam in (0.0, 0.35):
        loss, grad, prio = _mse_call(cuda, qv, act, tq, wset, lam, B, W, orc.ROWS_BMAJOR)
        lo, _, _, po = orc.td_mse(qv, act, tq, wset, lam, B, W, orc.ROWS_BMAJOR, want_grad=False)
        assert abs(loss - lo) <= 1e-6 * abs(lo), (B, lam, loss, lo)
        _assert_bits(prio, po, f"north star B={B}")
        _check_mse64(loss, grad, prio, qv, act, tq, wset, lam, B, W, orc.ROWS_BMAJOR, f"north star B={B} lam={lam}")


@pytest.mark.parametrize("A,D", [(4, 3), (8, 1), (2, 8), (7, 4), (1, 4)])
def test_td_mse_grad_scalar_path_matches_float4_path(cuda, A, D):
    """A D = 0 mod 4 and a 16-byte aligned row take the float4 gradient writer.  The same call with grad_out one float past an aligned
    buffer forces the scalar writer; both must write the same bits (and the float4 call must match float64)."""
    rng = np.random.default_rng(A * 10 + D)
    B, W = 53, 6
    qv, act, tq, wset = _mse_inputs(rng, B, W, A, D)
    N = B * W
    for lam in (0.0, 0.35):
        _, g_al, _ = _mse_call(cuda, qv, act, tq, wset, lam, B, W, orc.ROWS_BMAJOR)
        buf = th.full((N * A * D + 4,), 7.0, device=cuda)
        view = buf[1 : 1 + N * A * D].view(N, A, D)
        assert view.data_ptr() % 16 == 4
        _, g_un, _ = _mse_call(cuda, qv, act, tq, wset, lam, B, W, orc.ROWS_BMAJOR, grad_out=view)
        _assert_bits(g_un, g_al, f"A={A} D={D} lam={lam}")
        assert float(buf[0]) == 7.0 and float(buf[-3]) == 7.0  # nothing written outside the view
        loss, _, prio = _mse_call(cuda, qv, act, tq, wset, lam, B, W, orc.ROWS_BMAJOR)
        _check_mse64(loss, g_al, prio, qv, act, tq, wset, lam, B, W, orc.ROWS_BMAJOR, f"A={A} D={D} lam={lam}")


def test_td_mse_options(cuda):
    """q_taken_out equals the oracle's gathered Q; want_grad=False / want_prio=False leave the loss unchanged; a device lambda overrides the
    host lambda (host 0, device 0.35 == host 0.35, loss, gradient and priorities bit for bit)."""
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(21)
    B, W, A, D = 96, 10, 6, 5
    qv, act, tq, wset = _mse_inputs(rng, B, W, A, D)
    args = (_t(qv, cuda), _t(act, cuda), _t(tq, cuda), _t(wset, cuda))
    for order in (orc.ROWS_REFERENCE, orc.ROWS_BMAJOR):
        qt = th.empty(B * W, D, device=cuda)
        loss, grad, prio = ops.td_mse_priority(*args, 0.35, B, W, order, q_taken_out=qt)
        _, _, qto, _ = orc.td_mse(qv, act, tq, wset, 0.35, B, W, order)
        _assert_bits(_np(qt), qto, f"q_taken order={order}")
        for kw in (dict(want_grad=False), dict(want_prio=False), dict(want_grad=False, want_prio=False)):
            l2, g2, p2 = ops.td_mse_priority(*args, 0.35, B, W, order, **kw)
            _assert_bits(_np(l2), _np(loss), f"loss with {kw}")
            assert (g2 is None) == (not kw.get("want_grad", True)) and (p2 is None) == (not kw.get("want_prio", True))
        lam_dev = th.tensor([0.35], device=cuda)
        l3, g3, p3 = ops.td_mse_priority(*args, 0.0, B, W, order, lambda_dev=lam_dev)
        _assert_bits(_np(l3), _np(loss), "loss with lambda_dev")
        _assert_bits(_np(g3), _np(grad), "gradient with lambda_dev")
        _assert_bits(_np(p3), _np(prio), "priorities with lambda_dev")
        l0, g0, _ = ops.td_mse_priority(*args, 0.0, B, W, order)
        assert not th.equal(g0, g3)  # lambda really changes the gradient


# ------------------------------------------------------------------------------------------------ td_huber_priority
def _huber_call(dev, q, act, tq, tg, w, mp, p_rows, w_map):
    from morl_baselines_b200 import ops

    loss, grad, prio = ops.td_huber_priority(_t(q, dev), _t(act, dev), _t(tq, dev), None if tg is None else _t(tg, dev), _t(w, dev), mp, p_rows, w_map)
    return float(_np(loss)[0]), _np(grad), _np(prio)


def _check_huber64(loss, grad, prio, q, act, tq, tg, wf, mp, p_rows, msg):
    n, N, A, D = q.shape
    k = np.arange(N)
    a = act[k % len(act)]
    qa = q[:, k, a]  # [n, N, D] float32
    d32 = qa - tq[None]  # float32 residual, as the reference's tensors
    x = np.abs(d32).astype(np.float64)
    mp64 = float(np.float32(mp))
    lin = ~(x < mp64)
    ref = np.where(lin, mp64 * x, 0.5 * x * x).sum() / (N * D) / n
    assert abs(loss - ref) <= 1e-6 * abs(ref), f"{msg}: loss {loss} vs float64 {ref}"
    G = np.zeros(q.shape)
    G[:, k, a] = np.where(lin, mp64 * np.sign(d32), d32.astype(np.float64)) / (N * D) / n
    assert np.all(np.abs(grad - G) <= 4 * U * np.abs(G)), f"{msg}: gradient off float64"
    if p_rows:
        e = np.abs((qa - (tg if tg is not None else tq)[None]).astype(np.float32)).astype(np.float64).max(0)[:p_rows]
        w64 = wf[:p_rows].astype(np.float64)
        P = np.abs((w64 * e).sum(1))
        assert np.all(np.abs(prio - P) <= 2 * (D + 1) * U * (np.abs(w64) * e).sum(1)), f"{msg}: priorities off float64"


@pytest.mark.parametrize("n_nets", [1, 2, 3])
@pytest.mark.parametrize("D", [1, 3, 6, 8])
def test_td_huber_sweep(cuda, D, n_nets):
    """a_rows in {N, N/2}, p_rows in {0, N/2, N}, w_rows in {1, N/2 BLOCK, N/2 TILE, N}, target_gpi given or None."""
    rng = np.random.default_rng(10 * D + n_nets)
    N, A, mp = 192, 5, 0.01
    for a_rows in (N, N // 2):
        for gpi in (False, True):
            q = (rng.standard_normal((n_nets, N, A, D)) * 0.02).astype(np.float32)  # straddles min_priority
            tq = (rng.standard_normal((N, D)) * 0.02).astype(np.float32)
            tg = (rng.standard_normal((N, D)) * 0.02).astype(np.float32) if gpi else None
            act = rng.integers(0, A, size=a_rows).astype(np.int32)
            for w_rows, w_map in ((1, BLOCK), (N // 2, BLOCK), (N // 2, TILE), (N, BLOCK)):
                w = _weights(rng, w_rows, D)
                wf = w[_map_rows(w_rows, N, w_map)]
                for p_rows in (0, N // 2, N):
                    msg = f"huber D={D} n={n_nets} a_rows={a_rows} gpi={gpi} w={w_rows}/{w_map} p_rows={p_rows}"
                    loss, grad, prio = _huber_call(cuda, q, act, tq, tg, w, mp, p_rows, w_map)
                    lo, go, po = orc.td_huber(q, act, tq, tg, wf, mp, p_rows)
                    assert abs(loss - lo) <= 1e-6 * abs(lo), msg
                    if p_rows:
                        _assert_bits(prio, po, msg)
                    else:
                        assert prio is None
                    np.testing.assert_allclose(grad, go, rtol=3e-7, atol=0, err_msg=msg)
                    _check_huber64(loss, grad, prio, q, act, tq, tg, wf, mp, p_rows, msg)


def test_td_huber_residuals_at_min_priority_and_zero(cuda):
    """Residuals of exactly +-min_priority (binary fractions, so q - t == +-mp exactly) take the linear branch: mp |d| = mp^2, not
    0.5 d^2; 40 % of the elements sit there, so the other branch would move the loss by far more than 1e-6.  Residuals of exactly 0 and
    -0.0 contribute nothing and have a zero gradient."""
    rng = np.random.default_rng(17)
    n_nets, N, A, D = 2, 200, 4, 3
    mp = 2.0**-7
    tq = (rng.integers(-64, 64, size=(N, D)) * 2.0**-10).astype(np.float32)
    act = rng.integers(0, A, size=N).astype(np.int32)
    q = (rng.integers(-64, 64, size=(n_nets, N, A, D)) * 2.0**-10).astype(np.float32)
    k = np.arange(N)
    sel = rng.random((n_nets, N, D))
    qa = q[:, k, act]
    qa = np.where(sel < 0.2, tq[None] + np.float32(mp), qa)
    qa = np.where((sel >= 0.2) & (sel < 0.4), tq[None] - np.float32(mp), qa)
    qa = np.where((sel >= 0.4) & (sel < 0.5), tq[None], qa)  # d == +0
    zero_neg = (sel >= 0.5) & (sel < 0.6)
    qa = np.where(zero_neg, np.float32(-0.0), qa)
    q[:, k, act] = qa
    # -0.0 residuals need q = -0.0 and t = +0.0; make the targets of those elements +0 (for every net)
    tq = np.where(zero_neg.any(0), np.float32(0.0), tq).astype(np.float32)
    d = q[:, k, act] - tq[None]
    assert np.sum(np.abs(d) == np.float32(mp)) >= 0.35 * d.size
    assert np.any((d == 0) & np.signbit(d)) and np.any((d == 0) & ~np.signbit(d))
    w = _weights(rng, N, D)
    loss, grad, prio = _huber_call(cuda, q, act, tq, None, w, mp, N, BLOCK)
    lo, go, po = orc.td_huber(q, act, tq, None, w, mp, N)
    assert abs(loss - lo) <= 1e-6 * abs(lo)
    _assert_bits(prio, po, "huber exact residuals")
    g_taken = grad[:, k, act]
    assert np.all(g_taken[d == 0] == 0)
    assert np.array_equal(g_taken, go[:, k, act])
    _check_huber64(loss, grad, prio, q, act, tq, None, w, mp, N, "huber exact residuals")
    x = np.abs(d).astype(np.float64)
    quad_everywhere = np.where(x <= mp, 0.5 * x * x, mp * x).sum() / (N * D) / n_nets
    assert abs(quad_everywhere - loss) > 1e-3 * abs(loss)  # the branch at |d| == mp is visible in the loss
