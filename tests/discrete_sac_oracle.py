"""TEST INFRASTRUCTURE ONLY -- ctypes binding of tests/discrete_sac_oracle.c, the plain-C restatement the discrete-action MOSAC kernels
(morl_discrete_sac_target_f32, morl_discrete_sac_actor_loss_f32) equal bit for bit.  The C file is compiled on first use into a private
temporary directory, so nothing is written into the tree."""

from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "discrete_sac_oracle.c")
MAP_TILE, MAP_BLOCK = 0, 1

_lib = None


def lib():
    global _lib
    if _lib is None:
        out = tempfile.mkdtemp(prefix="discrete_sac_oracle_")
        atexit.register(shutil.rmtree, out, True)
        so = os.path.join(out, "libdiscrete_sac_oracle.so")
        cc = os.environ.get("CC") or shutil.which("gcc") or "cc"
        r = subprocess.run([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall", "-Wextra", "-std=c11", "-o", so, SRC, "-lm"],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"discrete_sac_oracle.c failed to compile:\n{r.stdout}\n{r.stderr}")
        _lib = C.CDLL(so)
        _lib.oracle_ds_exp.restype, _lib.oracle_ds_exp.argtypes = C.c_float, [C.c_float]
        _lib.oracle_ds_log.restype, _lib.oracle_ds_log.argtypes = C.c_float, [C.c_float]
    return _lib


def _f32(x):
    return np.ascontiguousarray(x, dtype=np.float32)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def ds_exp(x):
    """The library's portable fp32 e^x, element-wise."""
    f = lib().oracle_ds_exp
    return np.array([f(float(v)) for v in np.asarray(x, np.float32).reshape(-1)], np.float32).reshape(np.shape(x))


def ds_log(x):
    """The library's portable fp32 log x, element-wise."""
    f = lib().oracle_ds_log
    return np.array([f(float(v)) for v in np.asarray(x, np.float32).reshape(-1)], np.float32).reshape(np.shape(x))


def discrete_sac_target(q_nets, logits, w, reward, done, alpha, gamma, w_map=MAP_BLOCK):
    q_nets, logits, w = _f32(q_nets), _f32(logits), _f32(w)
    n_nets, N, A, D = q_nets.shape
    w = w.reshape(-1, D)
    reward, done = _f32(reward).reshape(N, D), _f32(done).reshape(N)
    out = np.empty(N, np.float32)
    lib().oracle_discrete_sac_target(_p(q_nets), n_nets, _p(logits), _p(w), w.shape[0], w_map, _p(reward), _p(done), C.c_float(alpha),
                                     C.c_float(gamma), N, A, D, _p(out))
    return out


def discrete_sac_actor_loss(logits, q_nets, w, alpha, log_alpha=None, target_entropy=0.0, w_map=MAP_BLOCK):
    """Returns (actor_loss, dlogits [N, A], alpha_loss, dlog_alpha); the last two are None without ``log_alpha``."""
    q_nets, logits, w = _f32(q_nets), _f32(logits), _f32(w)
    n_nets, N, A, D = q_nets.shape
    w = w.reshape(-1, D)
    la = None if log_alpha is None else np.array([log_alpha], np.float32).reshape(1)
    loss, aloss, dla = np.empty(1, np.float32), np.empty(1, np.float32), np.empty(1, np.float32)
    grad = np.empty((N, A), np.float32)
    lib().oracle_discrete_sac_actor_loss(_p(logits), _p(q_nets), n_nets, _p(w), w.shape[0], w_map, C.c_float(alpha), _p(la),
                                         C.c_float(target_entropy), N, A, D, _p(loss), _p(grad), _p(aloss), _p(dla))
    if la is None:
        return loss[0], grad, None, None
    return loss[0], grad, aloss[0], dla[0]
