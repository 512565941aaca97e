"""PGMORL's host pieces (multi_policy/pgmorl/pgmorl.py) against golden vectors from the unmodified reference
(tests/golden/make_golden_pgmorl.py): weight grids and performance buffers exactly, predictions within 1e-9 relative."""

import os

import numpy as np
import pytest

from morl_baselines_b200.multi_policy.pgmorl import pgmorl as pg

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pgmorl.npz"))


@pytest.mark.parametrize("delta,dim", [(0.2, 2), (0.1, 2), (0.05, 2), (0.2, 3), (0.1, 3)])
def test_generate_weights_matches_reference(delta, dim):
    w = pg.generate_weights(delta, dim)
    ref = G[f"weights/{delta}_{dim}"]
    assert w.dtype == ref.dtype and np.array_equal(w, ref)


@pytest.mark.parametrize("d,cls,bins", [(2, pg.PerformanceBuffer2d, 10), (3, pg.PerformanceBuffer3d, 5)])
def test_performance_buffer_matches_reference(d, cls, bins):
    buf = cls(num_bins=bins, max_size=2, origin=np.full(d, -10.0))
    for k, p in enumerate(G[f"buffer{d}/points"]):
        buf.add(k, p)
    assert np.array_equal(np.array(buf.evaluations), G[f"buffer{d}/evaluations"])
    assert np.array_equal(np.array(buf.individuals, np.int64), G[f"buffer{d}/individuals"])
    assert np.array_equal(np.array([len(b) for b in buf.bins]), G[f"buffer{d}/bin_sizes"])


def test_performance_buffer_stores_copies():
    buf = pg.PerformanceBuffer2d(num_bins=4, max_size=2, origin=np.zeros(2))
    cand = [1.0]
    buf.add(cand, np.array([1.0, 1.0]))
    cand[0] = 2.0
    assert buf.individuals == [[1.0]]


@pytest.mark.parametrize("d", [2, 3])
def test_predictor_matches_reference(d):
    pred = pg.PerformancePredictor()
    w, before, after = G[f"predictor{d}/w"], G[f"predictor{d}/before"], G[f"predictor{d}/after"]
    for k in range(len(w)):
        pred.add(w[k], before[k], after[k])
    qw, qe = G[f"predictor{d}/query_w"], G[f"predictor{d}/query_eval"]
    for k in range(len(qw)):
        delta, nxt = pred.predict_next_evaluation(qw[k], qe[k])
        np.testing.assert_allclose(delta, G[f"predictor{d}/deltas"][k], rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(nxt, G[f"predictor{d}/next"][k], rtol=1e-9)


def test_predictor_needs_four_neighbours():
    pred = pg.PerformancePredictor()
    pred.add(np.array([0.5, 0.5], np.float32), np.array([1.0, 1.0]), np.array([2.0, 2.0]))
    with pytest.raises(ValueError):
        pred.predict_next_evaluation(np.array([0.5, 0.5], np.float32), np.array([1.0, 1.0]))
