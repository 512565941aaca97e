"""ctypes loader for libmorl_b200.so (the C-ABI of include/morl_b200.h).

There is NO CPU fallback: if the shared library is missing, or a compute entry point is called without a CUDA device,
the call raises.  The library is built in-tree by ``python -m morl_baselines_b200.csrc.build`` (nvcc, sm_90a) and
travels with the repo snapshot to the GPU box.
"""

from __future__ import annotations

import ctypes as C
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "csrc", "libmorl_b200.so")
HEADER = os.path.join(os.path.dirname(HERE), "include", "morl_b200.h")

# constants of include/morl_b200.h
DOT_UNFUSED, DOT_FMA, DOT_PAIRFMA = 0, 1, 2
MAP_TILE, MAP_BLOCK = 0, 1
ROWS_REFERENCE, ROWS_BMAJOR = 0, 1
AC_ELEMENTWISE_MIN, AC_SCALAR_MIN, AC_ARGMIN_GATHER = 0, 1, 2
MAX_D = 8
PCN_MAX_BATCH = 4096
FMT_BF16X3, FMT_F16X2 = 0, 1

_vp, _i = C.c_void_p, C.c_int

# value types of include/morl_b200.h and their ctypes equivalents (every pointer is passed as c_void_p)
_SCALARS = {"int": _i, "float": C.c_float, "double": C.c_double, "long long": C.c_longlong, "int64_t": C.c_int64, "unsigned int": C.c_uint,
            "size_t": C.c_size_t}
_DECL = re.compile(r"MORL_API\s+([\w\s\*]+?)\s*\b(morl_\w+)\s*\(([^;]*?)\)\s*;", flags=re.S)


def _ctype(decl: str, where: str, ret: bool = False):
    words = decl.replace("*", " * ").split()
    if "*" in words:
        return C.c_char_p if ret and words == ["const", "char", "*"] else _vp
    t = " ".join(words if ret else words[:-1])  # a parameter ends with its name
    if t not in _SCALARS:
        raise MorlB200Error(f"{where}: no ctypes mapping for the C type '{t}' (include/morl_b200.h)")
    return _SCALARS[t]


def signatures(header: str) -> dict:
    """name -> (restype, argtypes) of every MORL_API declaration in the text of include/morl_b200.h."""
    src = re.sub(r"/\*.*?\*/|//[^\n]*", "", header, flags=re.S)
    sigs = {}
    for m in _DECL.finditer(src):
        ret, name, params = m.group(1), m.group(2), m.group(3).strip()
        params = [] if params in ("", "void") else [p for p in params.split(",") if p.strip()]
        sigs[name] = (_ctype(ret, name, ret=True), [_ctype(p, f"{name}({p.strip()})") for p in params])
    return sigs


SPLIT_MAX_JOBS = 16


class SplitJob(C.Structure):
    """MorlSplitJob of include/morl_b200.h"""

    _fields_ = [("src", _vp), ("dst_planes", _vp), ("plane_stride", C.c_longlong), ("scale", _vp), ("rows", _i), ("cols", _i), ("ld_src", _i),
                ("transpose", _i), ("rows_pad", _i), ("ldp", _i), ("auto_scale", _i), ("target_exp", _i)]


_lib = None


class MorlB200Error(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises if it has not been built -- there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MorlB200Error(
            f"{LIB_PATH} not found: build it with `python -m morl_baselines_b200.csrc.build` (nvcc, sm_90a). "
            "morl_baselines_b200 has no CPU / eager fallback for its CUDA operators."
        )
    with open(HEADER) as f:
        sigs = signatures(f.read())
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)  # AttributeError here == ABI drift between header and library
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().morl_last_error().decode("utf-8", "replace")
        raise MorlB200Error(f"{what} failed (code {rc}): {msg}")
