"""Binding of the batched exact hypervolume kernel (csrc/pareto.cu, ``morl_hypervolume_batch_f64``).

It follows the argument contract of :mod:`ops` (``ops._Args``) and launches through ``ops._launch``, so ``ops.launch_count`` counts it.
"""

from __future__ import annotations

from typing import Optional

import torch as th

from . import _lib
from .ops import _Args, _launch

MAX_N = {1: 2048, 2: 2048, 3: 2048, 4: 512}  # base points per set (include/morl_b200.h)


def hypervolume_batch_supported(n: int, d: int) -> bool:
    """Whether the kernel covers a base set of ``n`` points in ``d`` objectives: 1 <= d <= 4, 0 <= n <= 2048 (d <= 3) or 512 (d = 4).
    Needs no device."""
    return bool(_lib.load().morl_hypervolume_batch_supported(int(n), int(d)))


def hypervolume_batch(base, cand, ref, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Exact hypervolumes (maximisation) above ``ref`` [d] in one launch, float64 CUDA tensors throughout:

    - ``cand`` [n_cand, d] with n_cand >= 1: ``out[k]`` = volume of ``base`` [n_base, d] plus ``cand[k]``, returned as [n_cand];
    - ``cand`` None (or with no rows): ``out[0]`` = volume of ``base`` alone, returned as [1].

    A point that does not exceed ``ref`` in every objective (or holds a NaN) spans nothing.  No host synchronisation."""
    a = _Args("hypervolume_batch")
    base = a.inp(base, "base", (None, None), th.float64)
    n_base, d = base.shape
    cand = a.inp(cand, "cand", (None, d), th.float64, opt=True)
    n_cand = 0 if cand is None else cand.shape[0]
    ref = a.inp(ref, "ref", (d,), th.float64)
    if not hypervolume_batch_supported(n_base, d):
        a.fail("base", f"has shape {tuple(base.shape)}: the kernel supports 1 <= d <= 4 and at most {MAX_N.get(d, 0)} points for d={d}")
    out = a.out(out, "out", (max(n_cand, 1),), th.float64)
    _launch("morl_hypervolume_batch_f64", base, n_base, cand if n_cand else None, n_cand, d, ref, out)
    return out
