"""IPRO without a device: Box and the sorted box queue against the reference's Box and sortedcontainers' SortedKeyList, the scalarising
functions against the reference's, the batched hypervolume kernel's supported range, the vectorised float64 hypervolume of the GPU tests
against the recursive host sweep, and the golden file's internal consistency."""

import os

import numpy as np
import pytest
import torch as th

from morl_baselines_b200.common.performance_indicators import hypervolume as host_hypervolume
from morl_baselines_b200.hv_ops import hypervolume_batch_supported
from morl_baselines_b200.multi_policy.ipro.box import Box, BoxQueue
from morl_baselines_b200.multi_policy.ipro.outer_loop import aasf, linear_scalarization
from oracle import ref_harness as rh
from tests.hv_f64 import hv_max
from tests.ipro_standin import CASES

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ipro.npz")
needs_reference = pytest.mark.skipif(not rh.reference_available(), reason="reference not mounted")


def _reference(mod):
    from tests.golden.make_golden_ipro import install_pymoo_standins

    install_pymoo_standins()
    return rh.import_reference(f"morl_baselines.multi_policy.ipro.{mod}")


def _random_box(rng, d):
    a, b = rng.integers(-8, 8, (2, d)) / 4
    if rng.random() < 0.2:
        b[rng.integers(d)] = a[0]  # a degenerate side now and then
    return a, b


@needs_reference
@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_box_matches_reference(d):
    RefBox = _reference("box").Box
    rng = np.random.default_rng(d)
    for _ in range(200):
        p1, p2 = _random_box(rng, d)
        q1, q2 = _random_box(rng, d)
        mine, ref = Box(p1, p2), RefBox(p1, p2)
        other_mine, other_ref = Box(q1, q2), RefBox(q1, q2)
        for attr in ("dimensions", "bounds", "nadir", "ideal", "midpoint", "volume", "max_dist"):
            np.testing.assert_array_equal(getattr(mine, attr), getattr(ref, attr))
        assert mine.is_intersecting(other_mine) == ref.is_intersecting(other_ref)
        assert mine.is_intersecting_with_boundary(other_mine) == ref.is_intersecting_with_boundary(other_ref)
        for dim in range(-d, d):
            assert mine.projection_is_intersecting(other_mine, dim) == ref.projection_is_intersecting(other_ref, dim)
        got, want = mine.get_intersecting_box(other_mine), ref.get_intersecting_box(other_ref)
        assert (got is None) == (want is None)
        if got is not None:
            np.testing.assert_array_equal(got.bounds, want.bounds)
        for pt in (q1, q2, (p1 + p2) / 2, p1):
            assert mine.contains(pt) == ref.contains(pt)
            assert mine.contains_inner(pt) == ref.contains_inner(pt)
        assert mine.vertices() == ref.vertices()
        assert repr(mine) == repr(ref)


def test_box_queue_matches_sorted_key_list():
    sc = pytest.importorskip("sortedcontainers")
    rng = np.random.default_rng(0)
    mine, ref = BoxQueue(), sc.SortedKeyList([], key=lambda b: b.volume)
    for step in range(600):
        if len(ref) and rng.random() < 0.4:
            idx = int(rng.integers(-len(ref), len(ref))) if rng.random() < 0.5 else -1
            assert mine.pop(idx) is ref.pop(idx)
        else:
            # few distinct volumes, so equal keys are common
            box = Box(np.zeros(2), np.array([rng.integers(1, 4), rng.integers(1, 3)], dtype=float))
            mine.add(box), ref.add(box)
        assert len(mine) == len(ref) and bool(mine) == bool(ref)
        assert list(mine) == list(ref)
        if len(ref):
            assert mine[-1] is ref[-1]
    import copy

    dup = copy.deepcopy(mine)
    assert [b.volume for b in dup] == [b.volume for b in mine] and all(a is not b for a, b in zip(dup, mine))


@pytest.mark.parametrize("n,d,ok", [
    (0, 1, True), (2048, 1, True), (2049, 1, False),
    (2048, 2, True), (2049, 2, False),
    (0, 3, True), (2048, 3, True), (2049, 3, False),
    (0, 4, True), (512, 4, True), (513, 4, False),
    (1, 0, False), (1, 5, False), (-1, 2, False),
])
def test_hypervolume_batch_supported_range(n, d, ok):
    assert hypervolume_batch_supported(n, d) is ok


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_vectorised_host_hypervolume_matches_sweep(d):
    rng = np.random.default_rng(10 + d)
    for n in (0, 1, 7, 30):
        p, r = rng.integers(-16, 64, (n, d)) / 8, np.zeros(d)
        assert hv_max(p, r) == host_hypervolume(r, p)
        p, r = rng.random((n, d)), np.full(d, 0.2)
        assert hv_max(p, r) == pytest.approx(host_hypervolume(r, p), rel=1e-13, abs=0)


@needs_reference
def test_scalarisations_match_reference():
    ref = _reference("outer_loop")
    g = th.Generator().manual_seed(0)
    for d in (2, 3, 4):
        batch = th.randn(64, d, generator=g)
        w = th.rand(d, generator=g)
        assert th.equal(linear_scalarization(batch, w), ref.linear_scalarization(batch, w))
        nadir, ideal = -th.rand(d, generator=g) - 1, th.rand(d, generator=g) + 1
        referent = nadir + 0.3 * (ideal - nadir)
        for aug, scale in ((0.1, 100), (0.0, 1.0)):
            assert th.equal(aasf(batch, referent, nadir, ideal, aug=aug, scale=scale),
                            ref.aasf(batch, referent, nadir, ideal, aug=aug, scale=scale))


def _non_dominated(p):
    return not any(np.all(p[j] >= p[i]) and np.any(p[j] > p[i]) for i in range(len(p)) for j in range(len(p)) if i != j)


def test_golden_file_is_consistent():
    g = np.load(GOLDEN)
    replays, empty_queue_ended = 0, False
    for name, c in CASES.items():
        its, n_replay, calls, total_hv = g[f"{name}/final/counters"]
        assert its >= 2 and total_hv > 0
        replays += n_replay
        for k in range(int(its)):
            p = f"{name}/it{k}"
            hv, dom, disc, cov, err = g[f"{p}/scalars"]
            np.testing.assert_array_equal(g[f"{p}/callback"], [k + 1, hv, dom, disc, cov, err])
            assert cov == (dom + disc) / total_hv and 0 <= cov <= 1
        pf, ps = g[f"{name}/final/pf"], g[f"{name}/final/pareto_set"]
        assert _non_dominated(pf)
        sign = -1 if c["ctor"]["direction"] == "minimize" else 1
        assert all(np.any(np.all(np.isclose(sign * v, pf), axis=1)) for v in ps)
        if c["cls"] == "IPRO2D" and its < c["ctor"]["max_iterations"]:
            empty_queue_ended = len(g[f"{name}/final/boxes"]) == 0
    assert replays > 0 and empty_queue_ended
