"""LinearSupport timings in one call.

    python scripts/bench_linear_support.py [--reps 5] [--rep-eval 5]

  * the corner-weight kernel (morl_corner_weights_f64) on a (d, n) grid of random value sets up to the documented candidate bound, timed
    with CUDA events (median of --reps launches into a preallocated buffer), next to the host time of the float64 numpy oracle
    (tests/linear_support_oracle.py) where its enumeration is small enough to run;
  * one GPI-LS ``next_weight`` on the TreasureChain stand-in with a trained GPILS: the batched expanded set (one lockstep round,
    |W_c| x rep_eval episodes) against the reference-shaped serial evaluation (|W_c|^2 x rep_eval episodes, one row per network call).
The card's name and power limit are read in the same call and printed with the numbers (one JSON object on stdout)."""

import argparse
import copy
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch as th

GRID = [(2, 100), (3, 100), (4, 100), (4, 200), (6, 50), (6, 100), (8, 30), (8, 50)]
ORACLE_MAX = 300_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else th.cuda.get_device_name(0)


def kernel_grid(reps):
    from morl_baselines_b200 import _lib, ops
    from tests.linear_support_oracle import candidate_count, corners_oracle

    lib = _lib.load()
    rows = []
    rng = np.random.default_rng(0)
    for d, n in GRID:
        V = np.round(rng.uniform(0, 10, size=(n, d)), 4)
        Vd = th.from_numpy(V).cuda()
        k = ops.corner_weights(Vd).shape[0]
        verts = th.empty((max(k, 1), d + 1), dtype=th.float64, device="cuda")
        count = th.zeros(1, dtype=th.int32, device="cuda")
        ms = []
        for _ in range(reps + 1):
            e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(lib.morl_corner_weights_f64(Vd.data_ptr(), n, d, verts.data_ptr(), max(k, 1), count.data_ptr(), ops._stream()), "corners")
            e1.record()
            th.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        row = {"d": d, "n": n, "candidates": candidate_count(n, d), "corners": k, "kernel_ms_median": float(np.median(ms[1:])),
               "kernel_ms_min": float(np.min(ms[1:]))}
        if candidate_count(n, d) <= ORACLE_MAX:
            t0 = time.perf_counter()
            ref = corners_oracle(V)
            row["oracle_host_ms"] = 1e3 * (time.perf_counter() - t0)
            assert ref.shape[0] == k
        rows.append(row)
    return rows


def gpi_ls_next_weight(rep_eval):
    from morl_baselines_b200.common.evaluation import policy_evaluation_mo
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPILS
    from morl_baselines_b200.multi_policy.linear_support.linear_support import LinearSupport
    from tests.golden.standin_env import TreasureChain

    th.manual_seed(0)
    agent = GPILS(TreasureChain(seed=0), net_arch=[256, 256, 256, 256], batch_size=128, buffer_size=4096, learning_starts=50,
                  gradient_updates=1, log=False, seed=0, device="cuda")
    ls = LinearSupport(num_objectives=3, epsilon=None, verbose=False)
    train_w = [np.eye(3)[i] for i in range(3)] + [np.array([0.4, 0.4, 0.2]), np.array([0.2, 0.3, 0.5]), np.array([0.5, 0.1, 0.4])]
    agent.train_iteration(total_timesteps=600, weight=train_w[3].astype(np.float32), weight_support=[w.astype(np.float32) for w in train_w],
                          change_w_every_episode=True)
    env = TreasureChain(seed=1)
    for w in train_w:  # a CCS with several vectors (the agent's own returns)
        ls.add_solution(policy_evaluation_mo(agent, env, w, rep=1)[3], w)
    agent.set_weight_support(ls.get_weight_support())
    agent.use_gpi = True
    W_corner = ls.compute_corner_weights()

    def batched():
        copy.deepcopy(ls).next_weight(algo="gpi-ls", gpi_agent=agent, env=env, rep_eval=rep_eval)

    def serial():  # the reference's loop: the whole expanded set re-evaluated inside the loop over corner weights
        for _wc in W_corner:
            [policy_evaluation_mo(agent, env, wc2, rep=rep_eval)[3] for wc2 in W_corner]

    out = {"corner_weights": len(W_corner), "ccs": len(ls.ccs), "rep_eval": rep_eval}
    for name, fn in [("batched", batched), ("serial_reference_shape", serial)]:
        fn()
        th.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        th.cuda.synchronize()
        out[f"{name}_s"] = time.perf_counter() - t0
    out["speedup"] = out["serial_reference_shape_s"] / out["batched_s"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rep-eval", type=int, default=5)
    a = ap.parse_args()
    res = {"card": card(), "kernel": kernel_grid(a.reps), "gpi_ls_next_weight": gpi_ls_next_weight(a.rep_eval)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
