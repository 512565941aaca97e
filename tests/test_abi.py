"""CPU-only checks of the drop-in boundary: libmorl_b200.so loads, exports exactly the symbols include/morl_b200.h
declares, the ctypes signatures read from the header are the declared ones, and argument errors are reported without touching a device."""

import ctypes as C
import os

import pytest

from morl_baselines_b200 import _lib


def _header_decls():
    with open(_lib.HEADER) as f:
        return _lib.signatures(f.read())


def test_library_builds_and_loads():
    from morl_baselines_b200.csrc import build

    path = build.build()
    assert os.path.exists(path)
    lib = _lib.load()
    assert lib.morl_version() == 200


def test_header_and_library_export_the_same_symbols():
    decls = _header_decls()
    assert len(decls) >= 15
    lib = _lib.load()
    for name, (res, args) in decls.items():
        fn = getattr(lib, name, None)
        assert fn is not None, f"{name} declared in include/morl_b200.h but not exported by libmorl_b200.so"
        assert fn.restype is res and fn.argtypes == args, name


def test_signatures_follow_the_declared_types():
    """Every declaration parses, a few spelled out in full: pointers are c_void_p, value types their own ctypes type."""
    vp, i, f, d, ll, i64, u, sz = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_longlong, C.c_int64, C.c_uint, C.c_size_t
    decls = _header_decls()
    assert decls["morl_last_error"] == (C.c_char_p, [])
    assert decls["morl_version"] == (i, [])
    assert decls["morl_polyak_f32"] == (i, [vp, vp, vp, i, i64, d, vp])
    assert decls["morl_adam_workspace_bytes"] == (sz, [i, i64])
    assert decls["morl_sumtree_set_f64"] == (i, [vp, i, ll, d, i, vp, vp, vp])
    assert decls["morl_philox_advance"] == (i, [vp, u, vp])
    assert decls["morl_gemm_planes_f32"] == (i, [i, vp, ll, vp, vp, ll, vp, i, i, i, i, vp, i, vp, i, vp, i, ll, vp, i, i, vp, vp, vp])
    assert decls["morl_gemm_planes_ln_f32"] == (i, [i, vp, ll, vp, vp, ll, vp, i, i, i, vp, i, vp, vp, f, f, vp, vp, u, vp, i, vp, i, ll, vp, i,
                                                   vp, vp])


@pytest.mark.parametrize("decl", ["MORL_API int morl_x(int n, bool flag);", "MORL_API int morl_x(const int n);",
                                  "MORL_API void morl_x(int n);", "MORL_API int morl_x(int);"])
def test_signatures_refuse_unknown_types(decl):
    with pytest.raises(_lib.MorlB200Error):
        _lib.signatures(decl)


def test_exported_symbols_are_only_the_abi():
    import subprocess

    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    assert exported == set(_header_decls()), exported ^ set(_header_decls())


def test_argument_errors_need_no_device():
    lib = _lib.load()
    rc = lib.morl_envelope_td_f32(None, None, None, None, None, 0.99, 4, 4, 4, 3, 0, 0, None, None, None, None)
    assert rc == -1  # MORL_ERR_NULL
    assert b"NULL" in lib.morl_last_error()
    rc = lib.morl_pareto_mask_f32(16, 10, 9, 1, 16, None)  # D = 9 > MORL_MAX_D
    assert rc == -4
    with pytest.raises(_lib.MorlB200Error):
        _lib.check(rc, "morl_pareto_mask_f32")


def test_ops_refuse_cpu_tensors():
    import torch as th

    from morl_baselines_b200 import ops

    with pytest.raises(_lib.MorlB200Error):
        ops.pareto_mask(th.zeros(4, 2))
    with pytest.raises(_lib.MorlB200Error):
        ops.envelope_td(th.zeros(2, 2, 2, 3), th.zeros(2, 2, 2, 3), th.zeros(2, 3), th.zeros(2, 3), th.zeros(2), 0.99)


def test_fusion_coverage_predicates_need_no_device():
    """The `*_supported` predicates that decide between a fused kernel and the launches it replaces are pure host functions: their answers
    at the BASELINE shapes and just outside them (both sides are CUDA paths; an unsupported shape is refused by the fused entry point)."""
    lib = _lib.load()
    F16, BF16 = _lib.FMT_F16X2, _lib.FMT_BF16X3
    # fused output layers + envelope + Bellman: north-star, configs[1] (minecart: |W| 32, |A| 6, d 3), and what falls outside
    assert lib.morl_qhead_envelope_supported(F16, 1024, 64, 8, 3, 256) == 1
    assert lib.morl_qhead_envelope_supported(F16, 256, 32, 6, 3, 256) == 1
    assert lib.morl_qhead_envelope_supported(BF16, 1024, 64, 8, 3, 256) == 0   # f16x2 planes only
    assert lib.morl_qhead_envelope_supported(F16, 1024, 48, 8, 3, 256) == 0    # |W| must divide 128
    assert lib.morl_qhead_envelope_supported(F16, 1024, 64, 11, 3, 256) == 0   # |A| d > 32 (and |W||A| not a multiple of 16)
    assert lib.morl_qhead_envelope_supported(F16, 1024, 64, 8, 5, 256) == 0    # d in 2..4
    assert lib.morl_qhead_envelope_supported(F16, 1024, 64, 8, 3, 320) == 0    # K <= 256
    assert lib.morl_qhead_gemm_supported(F16, 65536, 24, 256) == 1 and lib.morl_qhead_gemm_supported(F16, 65536, 40, 256) == 0
    assert lib.morl_qhead_gemm_supported(F16, 1000, 24, 256) == 0              # M % 128
    # chained hidden layers: 256-wide layers, at least two 128-row tiles
    assert lib.morl_gemm_chain_supported(F16, 65536, 256) == 1 and lib.morl_gemm_chain_supported(BF16, 8192, 256) == 1
    assert lib.morl_gemm_chain_supported(F16, 65536, 128) == 0 and lib.morl_gemm_chain_supported(F16, 128, 256) == 0
    # refused with an error code and a message, not a crash
    rc = lib.morl_qhead_envelope_td_f32(F16, 16, 16, 0, None, None, 16, 16, 0, None, None, None, None, 256, 16, 16, 16, 0.99, 1024, 48, 8, 3, 0, 0, 0, 16, None, None, None,
                                        None, None)
    assert rc == -4 and b"unsupported configuration" in lib.morl_last_error()


def test_reduction_workspaces_cover_the_chunk_partials():
    """The column-sum reductions write one row of partials per row chunk: up to 296 chunks for the one-pass pairs_grad_reduce (|W| <= 64,
    at most 8 transitions per chunk), up to 74 for the two-pass form (|W| > 64, or a batch too large for 296 chunks of 8).  The library's
    byte counts cover them, so no caller needs to know the chunk arithmetic."""
    lib = _lib.load()
    for B, W, H, chunks in ((1024, 64, 256, 296), (6, 5, 64, 296), (3, 70, 64, 74), (256, 128, 256, 74), (4096, 8, 64, 74)):
        assert lib.morl_pairs_grad_reduce_workspace_bytes(B, W, H) >= chunks * W * H * 4, (B, W, H)
