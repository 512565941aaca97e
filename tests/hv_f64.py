"""Exact maximisation hypervolume for 1 <= d <= 4 in vectorised numpy, float64: the host check of the batched kernel at sizes where the
recursive sweep of common/performance_indicators is too slow (its cost is O(n^(d-1)) interpreter calls).  Slabs over the fourth and third
objectives, the 2-D staircase of each (w, z) slab by a running maximum: O(n^3) array work for d = 4."""

import numpy as np


def hv_max(points, ref) -> float:
    ref = np.asarray(ref, dtype=np.float64)
    d = len(ref)
    q = np.asarray(points, dtype=np.float64).reshape(-1, d) - ref
    q = q[np.all(q > 0, axis=1)]
    if len(q) == 0:
        return 0.0
    q = np.hstack((q, np.ones((len(q), 4 - d))))
    q = q[np.argsort(-q[:, 0], kind="stable")]
    x, y, z, w = q.T
    dx = x - np.append(x[1:], 0.0)
    zs = np.append(np.sort(z)[::-1], 0.0)
    ws = np.append(np.sort(w)[::-1], 0.0)
    total = 0.0
    for j in range(len(q)):
        wh = ws[j] - ws[j + 1]
        if wh <= 0:
            continue
        inw = w >= ws[j]
        mask = (z[None, :] >= zs[:-1, None]) & inw[None, :]  # [z-slab k, point i]
        m = np.maximum.accumulate(np.where(mask, y[None, :], 0.0), axis=1)
        area = (m * dx[None, :]).sum(axis=1)
        total += float((area * (zs[:-1] - zs[1:])).sum()) * wh
    return total
