"""Pareto Q-learning on the device against the reference's loop restated on the host.

    python scripts/bench_pql.py [--rounds 5] [--steps 3000] [--out bench_pql.json]

  train : ``PQL.train`` steps per second on the treasure grid stand-in of tests/pql_standin.py (d = 2, gamma 1, hypervolume scores, the
          reference's epsilon schedule over the run), against the reference's loop on Python sets restated in numpy (``HostPQL``).  pymoo is
          not installed, so the host scores with this repository's exact vectorised host sweep (tests/hv_f64.hv_max).
  step  : one set update plus one hypervolume scoring, in isolation, on a table whose next state holds a planted front of K points per
          action (action 0's front survives, the others are shifted below it): A * K candidates pruned to K, then A volumes of K points.
          Device: one update launch, one score launch and the copy of the scores back, synchronised.  Host: the same work on Python sets.
Medians over alternating rounds.  Prints one JSON line with the card's name, power limit and SM clock, read in the same call."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from morl_baselines_b200 import pql_ops  # noqa: E402
from morl_baselines_b200.common.utils import linearly_decaying_value  # noqa: E402
from morl_baselines_b200.multi_policy.pareto_q_learning.pql import PQL, _non_dominated  # noqa: E402
from tests.hv_f64 import hv_max  # noqa: E402
from tests.pql_standin import TreasureGrid  # noqa: E402

REF = np.array([0.0, -25.0])
EPS = dict(initial_epsilon=1.0, epsilon_decay_steps=2000, final_epsilon=0.1)


class HostPQL:
    """The reference's PQL loop (pql.py:131-285) on Python sets of tuples, host numpy throughout."""

    def __init__(self, env, ref_point, gamma, seed):
        self.env, self.ref_point, self.gamma = env, ref_point, gamma
        self.np_random = np.random.default_rng(seed)
        self.env_shape = env.observation_space.high - env.observation_space.low + 1
        S, A, d = int(np.prod(self.env_shape)), env.action_space.n, env.reward_dim
        self.num_actions = A
        self.counts = np.zeros((S, A))
        self.avg_reward = np.zeros((S, A, d))
        self.non_dominated = [[{tuple(np.zeros(d))} for _ in range(A)] for _ in range(S)]
        self.epsilon, self.global_step = EPS["initial_epsilon"], 0

    def get_q_set(self, s, a):
        q = self.avg_reward[s, a] + self.gamma * np.array(list(self.non_dominated[s][a]))
        return {tuple(v) for v in q}

    def calc_non_dominated(self, s):
        return _non_dominated(set().union(*[self.get_q_set(s, a) for a in range(self.num_actions)]))

    def score_hypervolume(self, s):
        return [hv_max(list(self.get_q_set(s, a)), self.ref_point) for a in range(self.num_actions)]

    def train(self, total):
        while self.global_step < total:
            state, _ = self.env.reset()
            state = int(np.ravel_multi_index(state, self.env_shape))
            done = False
            while not done and self.global_step < total:
                if self.np_random.uniform(0, 1) < self.epsilon:
                    action = self.np_random.integers(self.num_actions)
                else:
                    sc = np.array(self.score_hypervolume(state))
                    action = self.np_random.choice(np.argwhere(sc == np.max(sc)).flatten())
                nxt, r, term, trunc, _ = self.env.step(action)
                done = term or trunc
                self.global_step += 1
                nxt = int(np.ravel_multi_index(nxt, self.env_shape))
                self.counts[state, action] += 1
                self.non_dominated[state][action] = self.calc_non_dominated(nxt)
                self.avg_reward[state, action] += (r - self.avg_reward[state, action]) / self.counts[state, action]
                state = nxt
            self.epsilon = linearly_decaying_value(EPS["initial_epsilon"], EPS["epsilon_decay_steps"], self.global_step, 0, EPS["final_epsilon"])


def train_case(steps, rounds):
    def device():
        agent = PQL(TreasureGrid(d=2, seed=5), REF, gamma=1.0, seed=1, log=False, **EPS)
        th.cuda.synchronize()
        t0 = time.perf_counter()
        agent.train(total_timesteps=steps, eval_env=TreasureGrid(d=2, seed=6))
        th.cuda.synchronize()
        return steps / (time.perf_counter() - t0)

    def host():
        agent = HostPQL(TreasureGrid(d=2, seed=5), REF, 1.0, 1)
        t0 = time.perf_counter()
        agent.train(steps)
        return steps / (time.perf_counter() - t0)

    device()  # warm-up: module load, first launches
    dev, hst = [], []
    for _ in range(rounds):
        dev.append(device())
        hst.append(host())
    return {"device_steps_per_s": float(np.median(dev)), "host_steps_per_s": float(np.median(hst)),
            "speedup": float(np.median(dev) / np.median(hst))}


def planted(A, K, d, seed=0):
    """Table of 2 states: ND[1][a] = a front of K points on a sphere, action a > 0 shifted down by a."""
    rng = np.random.default_rng(seed)
    w = np.abs(rng.standard_normal((K, d))) + 0.05
    front = 10.0 * w / np.linalg.norm(w, axis=1, keepdims=True)
    nd = np.zeros((2, A, K, d))
    for a in range(A):
        nd[1, a] = front - a
    return nd, np.full((2, A), K, dtype=np.int32)


def step_case(A, K, d, rounds, host_budget):
    nd, cnt = planted(A, K, d)
    ref = np.full(d, -1.0)
    t = pql_ops.PqlTable(2, A, K, d, th.device("cuda"))
    t.nd.copy_(th.from_numpy(nd))
    t.nd_count.copy_(th.from_numpy(cnt))
    host_scores = th.empty(A, dtype=th.float64, pin_memory=True)
    r = np.ones(d)

    def device(n=200):
        th.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            pql_ops.pql_update(t, 0, 0, 1, r, 0.95)
            host_scores.copy_(pql_ops.pql_score(t, 1, pql_ops.HYPERVOLUME, 0.95, ref), non_blocking=True)
            th.cuda.current_stream().synchronize()
        return (time.perf_counter() - t0) / n * 1e3

    h = HostPQL.__new__(HostPQL)
    h.gamma, h.num_actions, h.ref_point = 0.95, A, ref
    h.counts, h.avg_reward = np.zeros((2, A)), np.zeros((2, A, d))
    h.non_dominated = [[{tuple(v) for v in nd[s, a, : cnt[s, a]].tolist()} for a in range(A)] for s in range(2)]

    def host():
        t0 = time.perf_counter()
        h.counts[0, 0] += 1
        h.non_dominated[0][0] = h.calc_non_dominated(1)
        h.avg_reward[0, 0] += (r - h.avg_reward[0, 0]) / h.counts[0, 0]
        h.score_hypervolume(1)
        return (time.perf_counter() - t0) * 1e3

    pql_ops.check_status(t)
    device(5)
    first = host()
    if first > 1e3 * host_budget:
        hst = [first]
        note = "host: one step only (over the budget)"
    else:
        hst = []
        note = None
    dev = []
    for _ in range(rounds):
        dev.append(device())
        if note is None:
            hst.append(host())
    pql_ops.check_status(t)
    out = {"device_ms": float(np.median(dev)), "host_ms": float(np.median(hst)), "speedup": float(np.median(hst) / np.median(dev))}
    if note:
        out["note"] = note
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--host-budget", type=float, default=20.0, help="seconds one host step may take before it is timed once only")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bench_pql.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    result = {"gpu": gpu, "host_hypervolume": "exact vectorised host sweep tests/hv_f64.hv_max (pymoo not installed)",
              "unit": "train: steps/s; step: ms per update + score; medians over rounds", "train": train_case(args.steps, args.rounds),
              "step": {}}
    print("train", result["train"], file=sys.stderr, flush=True)
    for A in (4, 8):
        for d in (2, 3, 4):
            for K in (16, 64, 256):
                key = f"A{A}_d{d}_K{K}"
                result["step"][key] = step_case(A, K, d, args.rounds, args.host_budget)
                print(key, result["step"][key], file=sys.stderr, flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
