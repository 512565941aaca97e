"""Discrete-action MOSAC on the update engine, timed in one call (the shapes of the reference's examples/morld_lunar_lander.py:
8-dim observations, 4 actions, 4 objectives, net_arch [256] * 4, batch 128).

    python scripts/bench_mosac_discrete.py [--reps 50]

  * MOSACDiscrete.update() with use_cuda_graph False (eager) and True (one graph replay per update);
  * one MORL/D improvement pass (``_update_others``, update_passes = 1) over 6 and 64 learners, with and without the population graph
    (all learners' updates replayed as one multi-branch CUDA graph).
Times are a host clock around ``reps`` calls that ends in a device synchronise, after warm-up (which also captures the graphs); the median
of --rounds such windows is reported, with min and max.  The card's name and power limit are read in the same call and printed with the
numbers (one JSON object on stdout)."""

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch as th

OBS, A, D, B, ARCH = 8, 4, 4, 128, [256, 256, 256, 256]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else th.cuda.get_device_name(0)


def window_ms(fn, reps, rounds, warm=5):
    for _ in range(warm):
        fn()
    th.cuda.synchronize()
    per = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        th.cuda.synchronize()
        per.append((time.perf_counter() - t0) * 1e3 / reps)
    return {"median_ms": float(np.median(per)), "min_ms": float(np.min(per)), "max_ms": float(np.max(per))}


def fill(buf, n, rng):
    for _ in range(n):
        buf.add(rng.standard_normal(OBS).astype(np.float32), int(rng.integers(A)), rng.standard_normal(D).astype(np.float32),
                rng.standard_normal(OBS).astype(np.float32), bool(rng.random() < 0.05))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert th.cuda.is_available(), "this benchmark needs a CUDA device"
    from morl_baselines_b200.multi_policy.morld.morld import MORLD
    from morl_baselines_b200.single_policy.ser.mosac_discrete_action import MOSACDiscrete
    from morl_baselines_b200.testing import FakeEnv

    dev = th.device("cuda:0")
    out = {"card": card(), "shape": {"obs": OBS, "actions": A, "objectives": D, "batch": B, "net_arch": ARCH}}
    rng = np.random.default_rng(0)
    upd = {}
    for graph in (False, True):
        th.manual_seed(0)
        agent = MOSACDiscrete(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), weights=np.full(D, 1.0 / D, np.float32), batch_size=B, net_arch=ARCH,
                              buffer_size=4096, update_frequency=1, target_net_freq=200, log=False, device=dev, use_cuda_graph=graph)
        fill(agent.buffer, 2048, rng)

        def step(agent=agent):
            agent.global_step += 1
            agent.update()

        upd["graph" if graph else "eager"] = window_ms(step, args.reps, args.rounds)
    out["update"] = upd
    morld = {}
    for pop in (6, 64):
        for pg in (False, True):
            th.manual_seed(0)
            algo = MORLD(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), pop_size=pop, policy_name="MOSACDiscrete", update_passes=1, log=False, device=dev,
                         seed=0, weight_init_method="random",
                         policy_args={"batch_size": B, "net_arch": ARCH, "buffer_size": 1024, "update_frequency": 1, "target_net_freq": 200})
            algo.population_graph = pg
            for p in algo.population:
                fill(p.wrapped.get_buffer(), 512, rng)
                p.wrapped.global_step = 1

            def one_pass(algo=algo):
                algo._update_others(algo.population[0])

            morld[f"pop{pop}_{'population_graph' if pg else 'per_learner'}"] = window_ms(one_pass, max(2, args.reps // 10), args.rounds, warm=3)
    out["morld_update_others_pass"] = morld
    print(json.dumps(out))


if __name__ == "__main__":
    main()
