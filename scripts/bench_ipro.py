"""IPRO's hypervolume work on the device against the host.

    python scripts/bench_ipro.py [--rounds 5] [--out bench_ipro.json]

  hvis : ``compute_hvis``'s 50 volumes "pf U completed U {l}" for 50 lower points l, at d 3 and 4 with |pf U completed| in {32, 128, 512}:
         one launch of the batched kernel (and one copy back), against 50 calls of the host sweep (common/performance_indicators), and at
         d 3 against 50 launches of the single-set kernel (``ops.hypervolume``, one read-back each).  All three must give equal volumes
         (the points are multiples of 1/8, so every sum is exact).  A host variant whose 50 calls would take over ``--host-budget``
         seconds is timed on fewer calls and scaled to 50 (reported as such).
  step : one outer-loop bookkeeping step of IPRO (``update_found`` + ``update_excluded_volume`` + ``estimate_error`` + ``hv``) on the same
         fronts, with the volumes on the device against the host sweep.
Medians over alternating rounds.  Prints one JSON line with the card's name, power limit and SM clock, read in the same call."""

from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time
from functools import partial

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from morl_baselines_b200 import ops  # noqa: E402
from morl_baselines_b200.common.performance_indicators import hypervolume as host_hypervolume  # noqa: E402
from morl_baselines_b200.multi_policy.ipro import outer_loop  # noqa: E402
from morl_baselines_b200.multi_policy.ipro.ipro import IPRO  # noqa: E402


def front(rng, n, d):
    """n mutually (mostly) non-dominated points near a sphere of radius 40, multiples of 1/8."""
    w = np.abs(rng.standard_normal((n, d))) + 0.05
    return np.round(8 * 40 * w / np.linalg.norm(w, axis=1, keepdims=True)) / 8


def state(n, d, seed=0):
    """A bare IPRO state with a front of n points (no learner)."""
    rng = np.random.default_rng(seed)
    a = IPRO.__new__(IPRO)
    a.dim, a.sign = d, 1
    a.nadir, a.ideal = np.full(d, -1.0), np.full(d, 41.0)
    a.ref_point = a.nadir.copy()
    a.pf = front(rng, n, d)
    a.completed = np.empty((0, d))
    a.robust_points = np.empty((0, d))
    a.lower_points = np.round(8 * rng.uniform(0, 30, (200, d))) / 8
    a.upper_points = np.array([a.ideal])
    return a, rng


def timed(fn):
    th.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    th.cuda.synchronize()
    return time.perf_counter() - t0, r


def hvis_case(d, n, rounds, host_budget):
    a, rng = state(n, d)
    lowers = a.lower_points[:50]
    ideal = a.ideal
    base = np.vstack((a.pf, a.completed))

    def kernel():
        return a._improvement_volumes(lowers, device=True)

    def host(k=50):
        return np.array([host_hypervolume(-ideal, -np.vstack((base, l[None]))) for l in lowers[:k]])

    def single():
        out = []
        for l in lowers:
            pts = th.as_tensor(-np.vstack((base, l[None])), device="cuda")
            out.append(float(ops.hypervolume(pts, th.as_tensor(-ideal, device="cuda"))[0]))
        return np.array(out)

    kernel(), (single() if d <= 3 else None)  # warm-up
    if d == 4 and n > 128:  # O(n^3) interpreter calls: minutes for a single volume
        k_host = 0
    else:
        t1, _ = timed(partial(host, 1))
        k_host = 50 if 50 * t1 <= host_budget else max(1, int(host_budget / max(t1, 1e-9)))
    t = {"kernel": [], "host": [], "single": []}
    res = {}
    for r in range(rounds):
        dt, res["kernel"] = timed(kernel)
        t["kernel"].append(dt)
        if d <= 3:
            dt, res["single"] = timed(single)
            t["single"].append(dt)
        if k_host and r < (rounds if k_host == 50 else 1):
            dt, res["host"] = timed(partial(host, k_host))
            t["host"].append(dt * 50 / k_host)
    if k_host:
        assert np.array_equal(res["kernel"][:k_host], res["host"]), "kernel and host volumes differ"
    if d <= 3:
        assert np.array_equal(res["kernel"], res["single"]), "batched and single-set kernels differ"
    out = {k: round(float(np.median(v)) * 1e3, 3) for k, v in t.items() if v}
    out["host_calls_timed"] = k_host
    out["host_rounds"] = len(t["host"])
    return out


def step_case(d, n, rounds):
    """update_found + update_excluded_volume + estimate_error + hv, device volumes against host volumes."""
    a0, rng = state(n, d, seed=1)
    vec = np.round(8 * rng.uniform(10, 30, d)) / 8

    def step(a):
        a.update_found(None, vec)
        a.update_excluded_volume()
        a.estimate_error()
        a.hv = a.compute_hypervolume(-a.sign * a.pf, -a.sign * a.ref_point)
        return np.array([a.dominated_hv, a.discarded_hv, a.error, a.hv])

    orig = outer_loop.max_hypervolumes
    host_hv = partial(orig, device=False)
    t = {"device": [], "host": []}
    res = {}
    step(copy.deepcopy(a0))  # warm-up
    for _ in range(rounds):
        dt, res["device"] = timed(partial(step, copy.deepcopy(a0)))
        t["device"].append(dt)
        outer_loop.max_hypervolumes = host_hv
        try:
            dt, res["host"] = timed(partial(step, copy.deepcopy(a0)))
        finally:
            outer_loop.max_hypervolumes = orig
        t["host"].append(dt)
    assert np.array_equal(res["device"], res["host"]), "device and host bookkeeping differ"
    return {k: round(float(np.median(v)) * 1e3, 3) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-budget", type=float, default=20.0, help="seconds one round of the host sweep may take before it is sampled")
    ap.add_argument("--sizes", default="32,128,512")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bench_ipro.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    result = {"gpu": gpu, "unit": "ms, median over rounds", "hvis": {}, "step": {}}
    for d in (3, 4):
        for n in (int(s) for s in args.sizes.split(",")):
            key = f"d{d}_n{n}"
            result["hvis"][key] = hvis_case(d, n, args.rounds, args.host_budget)
            if d == 4 and n > 128:
                result["step"][key] = "not measured: the host sweep takes minutes per volume"
            else:
                result["step"][key] = step_case(d, n, args.rounds if d == 3 or n <= 32 else 2)
            print(key, result["hvis"][key], result["step"][key], file=sys.stderr, flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
