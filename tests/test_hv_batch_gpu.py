"""The batched exact hypervolume kernel (morl_hypervolume_batch_f64) against the host in float64, its determinism, its agreement with the
single-set kernel, and the binding's refusals.

Dyadic inputs (multiples of 1/8, |x| <= 64) make every partial sum exact, so the kernel must equal the host bit for bit there.  On
random inputs the bound is relative 1e-12; the worst case measured on an H100 80GB HBM3 (700 W power limit) is 6.5e-16 (d = 2)."""

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import _lib, hv_ops, ops
from morl_baselines_b200.common.performance_indicators import hypervolume as host_sweep
from oracle.hv_oracle import hypervolume_min
from tests.hv_f64 import hv_max

pytestmark = pytest.mark.gpu
REL = 1e-12


def _t(a, dev):
    return th.as_tensor(np.asarray(a, dtype=np.float64), device=dev)


def _dyadic(rng, n, d):
    return rng.integers(-64, 512, (n, d)) / 8


def _host(base, cand, ref):
    sets = [base] if cand is None else [np.vstack((base, c[None])) for c in cand]
    small = len(base) <= 40 or (len(ref) <= 2 and len(base) <= 200)
    # the recursive sweeps at small sizes (both forms), the vectorised one beyond
    return np.array([host_sweep(ref, s) if small else hv_max(s, ref) for s in sets])


@pytest.mark.parametrize("d", [1, 2, 3, 4])
@pytest.mark.parametrize("n_base,n_cand", [(0, 0), (0, 1), (1, 0), (5, 1), (37, 50), (120, 300), ("cap", 0), ("cap", 2)])
def test_batch_matches_host_bit_for_bit_on_dyadic_points(cuda, d, n_base, n_cand):
    rng = np.random.default_rng(7 * d + (0 if n_base == "cap" else n_base) + n_cand)
    if n_base == "cap":
        n_base = hv_ops.MAX_N[d]
    if d == 4 and n_cand > 50 and n_base > 100:
        n_cand = 50
    base, cand, ref = _dyadic(rng, n_base, d), _dyadic(rng, n_cand, d), np.zeros(d)
    got = hv_ops.hypervolume_batch(_t(base, cuda), _t(cand, cuda) if n_cand else None, _t(ref, cuda)).cpu().numpy()
    check = slice(None) if n_cand <= 50 else slice(None, None, 25)  # every 25th of several hundred on the host
    want = _host(base, cand[check] if n_cand else None, ref)
    np.testing.assert_array_equal(got[check], want)
    if n_base <= 40:  # and the minimisation form the reference's pymoo call computes
        assert got[0] == (hypervolume_min(-np.vstack((base, cand[:1])), -ref) if n_cand else hypervolume_min(-base, -ref))


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_batch_matches_host_on_random_points(cuda, d):
    rng = np.random.default_rng(100 + d)
    worst = 0.0
    for n_base, n_cand in ((30, 50), (200, 8)):
        base, cand, ref = rng.random((n_base, d)), rng.random((n_cand, d)), np.full(d, 0.05)
        got = hv_ops.hypervolume_batch(_t(base, cuda), _t(cand, cuda), _t(ref, cuda)).cpu().numpy()
        want = _host(base, cand, ref)
        worst = max(worst, float(np.max(np.abs(got - want) / np.abs(want))))
    print(f"d={d}: worst relative error {worst:.3g} (bound {REL:g})")
    assert worst <= REL


def test_batch_edge_cases(cuda):
    ref = np.array([1.0, 2.0, 3.0])
    base = np.array([[2.0, 3.0, 4.0], [2.0, 3.0, 4.0], [1.0, 5.0, 5.0], [3.0, 2.0, 7.0], [np.nan, 9.0, 9.0], [4.0, 4.0, 4.0]])
    cand = np.array([
        [0.0, 9.0, 9.0],        # outside ref in one objective
        [1.0, 2.0, 3.0],        # on ref
        [1.5, 2.5, 3.5],        # dominated by the base
        [9.0, np.nan, 9.0],     # NaN
        [4.0, 4.0, 4.0],        # duplicate of a base point
        [5.0, 5.0, 5.0],        # adds volume
    ])
    got = hv_ops.hypervolume_batch(_t(base, cuda), _t(cand, cuda), _t(ref, cuda)).cpu().numpy()
    clean = base[~np.isnan(base).any(axis=1)]
    alone = host_sweep(ref, clean)
    np.testing.assert_array_equal(got[:5], [alone] * 5)
    assert got[5] == host_sweep(ref, np.vstack((clean, cand[5:])))
    assert got[5] > alone


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_batch_is_deterministic(cuda, d):
    rng = np.random.default_rng(d)
    n = hv_ops.MAX_N[d] // 4
    base, cand, ref = _t(rng.random((n, d)), cuda), _t(rng.random((64, d)), cuda), _t(np.zeros(d), cuda)
    a = hv_ops.hypervolume_batch(base, cand, ref).cpu().numpy()
    b = hv_ops.hypervolume_batch(base, cand, ref).cpu().numpy()
    assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("n", [0, 1, 33, 1000, 2048])
def test_base_alone_equals_single_set_kernel(cuda, d, n):
    rng = np.random.default_rng(n + d)
    pts, ref = _t(rng.random((n, d)), cuda), _t(np.full(d, 0.1), cuda)
    one = ops.hypervolume(pts, ref).cpu().numpy()
    batch = hv_ops.hypervolume_batch(pts, None, ref).cpu().numpy()
    assert one.tobytes() == batch.tobytes()


def test_single_set_kernel_still_refuses_d4(cuda):
    with pytest.raises(_lib.MorlB200Error):
        ops.hypervolume(th.zeros(3, 4, dtype=th.float64, device=cuda), th.zeros(4))


def test_binding_refuses_bad_arguments_before_launch(cuda):
    base, cand, ref = th.rand(8, 3, device=cuda, dtype=th.float64), th.rand(4, 3, device=cuda, dtype=th.float64), th.zeros(3, device=cuda,
                                                                                                                         dtype=th.float64)
    out = th.full((4,), -1.0, device=cuda, dtype=th.float64)
    bad = [
        dict(base=base.float()),                                     # dtype
        dict(cand=cand.float()),
        dict(ref=ref.float()),
        dict(base=base.cpu()),                                       # device
        dict(ref=ref.cpu()),
        dict(base=base[:, :2]),                                      # shape (cand and ref have 3 columns)
        dict(cand=th.rand(4, 2, device=cuda, dtype=th.float64)),
        dict(ref=th.zeros(2, device=cuda, dtype=th.float64)),
        dict(out=th.empty(3, device=cuda, dtype=th.float64)),
        dict(out=th.empty(8, device=cuda, dtype=th.float64)[::2]),   # non-contiguous output
        dict(base=th.rand(8, 5, device=cuda, dtype=th.float64), cand=None, ref=th.zeros(5, device=cuda, dtype=th.float64)),  # d = 5
        dict(base=th.rand(513, 4, device=cuda, dtype=th.float64), cand=None, ref=th.zeros(4, device=cuda, dtype=th.float64)),  # n > cap
        dict(base=th.rand(2049, 2, device=cuda, dtype=th.float64), cand=None, ref=th.zeros(2, device=cuda, dtype=th.float64)),
        dict(base=th.rand(3, device=cuda, dtype=th.float64)),          # not 2-D
    ]
    for kw in bad:
        args = {**dict(base=base, cand=cand, ref=ref, out=out), **kw}
        before = ops.launch_count
        with pytest.raises(_lib.MorlB200Error):
            hv_ops.hypervolume_batch(args["base"], args["cand"], args["ref"], out=args["out"])
        assert ops.launch_count == before
    assert th.all(out == -1.0)
    # a non-contiguous input is copied, not refused, and gives the same result
    wide = th.rand(8, 6, device=cuda, dtype=th.float64)
    a = hv_ops.hypervolume_batch(wide[:, ::2], cand, ref)
    b = hv_ops.hypervolume_batch(wide[:, ::2].contiguous(), cand, ref)
    assert th.equal(a, b)


def test_library_refuses_out_of_range(cuda):
    lib = _lib.load()
    out = th.empty(1, device=cuda, dtype=th.float64)
    ref = th.zeros(5, device=cuda, dtype=th.float64)
    pts = th.zeros(600, 5, device=cuda, dtype=th.float64)
    s = th.cuda.current_stream().cuda_stream
    assert lib.morl_hypervolume_batch_f64(pts.data_ptr(), 4, None, 0, 5, ref.data_ptr(), out.data_ptr(), s) == -4
    assert lib.morl_hypervolume_batch_f64(pts.data_ptr(), 513, None, 0, 4, ref.data_ptr(), out.data_ptr(), s) == -4
    assert lib.morl_hypervolume_batch_f64(pts.data_ptr(), 4, None, 0, 0, ref.data_ptr(), out.data_ptr(), s) == -4
    assert lib.morl_hypervolume_batch_f64(pts.data_ptr(), 4, None, 2, 3, ref.data_ptr(), out.data_ptr(), s) == -1
    assert lib.morl_hypervolume_batch_f64(pts.data_ptr(), -1, None, 0, 3, ref.data_ptr(), out.data_ptr(), s) == -2
