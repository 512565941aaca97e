"""Golden vectors for PGMORL's host pieces, produced by the unmodified reference (needs the
reference's source tree, so it is run by hand, not by the tests):
    python tests/golden/make_golden_pgmorl.py   ->  tests/golden/pgmorl.npz

multi_policy/pgmorl/pgmorl.py on synthetic evaluations: ``generate_weights`` in 2-D and 3-D, the contents of ``PerformanceBuffer2d`` /
``PerformanceBuffer3d`` after a sequence of adds (candidates are their insertion numbers), and ``PerformancePredictor.
predict_next_evaluation`` for a set of (weight, evaluation) queries after a sequence of samples."""

from __future__ import annotations

import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402

WEIGHT_GRID = ((0.2, 2), (0.1, 2), (0.05, 2), (0.2, 3), (0.1, 3))


def buffer_sequence(d, n, seed):
    g = np.random.default_rng(seed)
    return g.uniform(-20.0, 100.0, (n, d))


def predictor_samples(d, n, seed):
    g = np.random.default_rng(seed)
    before = g.uniform(10.0, 50.0, (n, d))
    w = g.dirichlet(np.ones(d), n).astype(np.float32)
    after = before + g.normal(3.0, 2.0, (n, d)) + 5.0 * w
    return w, before, after


def queries(d, seed):
    g = np.random.default_rng(seed)
    return g.dirichlet(np.ones(d), 6).astype(np.float32), g.uniform(15.0, 45.0, (6, d))


def main():
    assert rh.reference_available()
    rh.install_stubs()
    gym = sys.modules["gymnasium"]
    if getattr(gym, "__graft_stub__", False) and not hasattr(gym, "vector"):
        gym.vector = types.SimpleNamespace(SyncVectorEnv=object)
    pg = rh.import_reference("morl_baselines.multi_policy.pgmorl.pgmorl")
    out = {}
    for delta, dim in WEIGHT_GRID:
        out[f"weights/{delta}_{dim}"] = pg.generate_weights(delta, dim)
    for d, cls, bins in ((2, pg.PerformanceBuffer2d, 10), (3, pg.PerformanceBuffer3d, 5)):
        origin = np.full(d, -10.0)
        pts = buffer_sequence(d, 60, 5 + d)
        buf = cls(num_bins=bins, max_size=2, origin=origin)
        for k, p in enumerate(pts):
            buf.add(k, p)
        out[f"buffer{d}/points"] = pts
        out[f"buffer{d}/evaluations"] = np.array(buf.evaluations)
        out[f"buffer{d}/individuals"] = np.array(buf.individuals, np.int64)
        out[f"buffer{d}/bin_sizes"] = np.array([len(b) for b in buf.bins], np.int64)
    for d in (2, 3):
        w, before, after = predictor_samples(d, 16, 20 + d)
        pred = pg.PerformancePredictor()
        for k in range(len(w)):
            pred.add(w[k], before[k], after[k])
        qw, qe = queries(d, 30 + d)
        deltas, nxt = zip(*[pred.predict_next_evaluation(qw[k], qe[k]) for k in range(len(qw))])
        out[f"predictor{d}/w"], out[f"predictor{d}/before"], out[f"predictor{d}/after"] = w, before, after
        out[f"predictor{d}/query_w"], out[f"predictor{d}/query_eval"] = qw, qe
        out[f"predictor{d}/deltas"], out[f"predictor{d}/next"] = np.array(deltas), np.array(nxt)
    path = os.path.join(HERE, "pgmorl.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
