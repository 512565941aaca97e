"""Build libmorl_b200.so in-tree with nvcc for sm_90a (no torch, no JIT cache: the .so travels with the snapshot).

    python -m morl_baselines_b200.csrc.build [--force] [--verbose]

Each .cu is compiled to an object (parallel, cached on mtime) and linked into ONE shared library exporting the
C-ABI of include/morl_b200.h.  Flags: -gencode arch=compute_90a,code=sm_90a -lineinfo -O3; -fmad=false is NOT needed
because every parity-critical operation uses explicit _rn intrinsics.
"""

from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libmorl_b200.so")
SOURCES = ["api.cu", "envelope_td.cu", "gpi_td.cu", "td_loss.cu", "pareto.cu", "replay.cu", "optim.cu", "gemm_planes.cu", "pair_layer1.cu", "host_replay.cu", "sumtree.cu", "qhead_envelope.cu", "dyna.cu", "discrete_sac.cu", "linear_support.cu", "ppo.cu", "pcn.cu", "eupg.cu"]
HEADERS = ["common.cuh", "gemm_tc.cuh", "envelope_wp.cuh", os.path.join(ROOT, "include", "morl_b200.h")]

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-O3",
    "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler",
    "-fPIC,-fvisibility=hidden",
    "-Xptxas",
    "-v",
]


def _nvcc() -> str:
    nv = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nv):
        raise RuntimeError("nvcc not found: cannot build libmorl_b200.so (no CPU fallback exists)")
    return nv


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src: str, verbose: bool) -> str:
    obj = os.path.join(BUILD, src.replace(".cu", ".o"))
    deps = [os.path.join(HERE, src)] + [h if os.path.isabs(h) else os.path.join(HERE, h) for h in HEADERS]
    if _stale(obj, deps):
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(HERE, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(BUILD, src.replace(".cu", ".ptxas.log"))
        with open(log, "w") as f:
            f.write(r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    if force:
        for f in os.listdir(BUILD):
            os.remove(os.path.join(BUILD, f))
        if os.path.exists(LIB):
            os.remove(LIB)
    with cf.ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), SOURCES))
    if _stale(LIB, objs):
        cmd = [_nvcc(), "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
