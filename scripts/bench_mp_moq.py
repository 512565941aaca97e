"""Multi-policy MO Q-learning: ``train`` steps/s on the treasure grid stand-in (d = 3, slip 0.2), device against the reference's per-step
loop restated on the host (dict tables, python scalarisation, a numpy SumTree), for five configurations at P = 1, 8 and 16 policies;
plus ``eval_batch`` over 100 rows at P = 16 against 100 serial ``eval`` calls, and ``ops.launch_count`` per step.

    python scripts/bench_mp_moq.py [--steps 2000] [--rounds 5]

P policies are built by P - 1 untimed iterations of random weights; the timed iteration is the P-th.  Medians over alternating rounds.
Prints one JSON line with the card's name and power limit, read in the same call."""

from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch as th

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from morl_baselines_b200 import ops  # noqa: E402
from morl_baselines_b200.multi_policy.multi_policy_moqlearning.mp_mo_q_learning import MPMOQLearning  # noqa: E402
from tests.pql_standin import TreasureGrid  # noqa: E402

CONFIGS = {
    "plain": dict(),
    "gpi": dict(use_gpi_policy=True),
    "dyna5": dict(dyna=True, dyna_updates=5),
    "gpi_dyna5": dict(use_gpi_policy=True, dyna=True, dyna_updates=5),
    "gpi_dyna5_pd": dict(use_gpi_policy=True, dyna=True, dyna_updates=5, gpi_pd=True),
}


class HostSumTree:
    """The reference's numpy SumTree (prioritized_buffer.py:12-64), restated."""

    def __init__(self, max_size=int(1e5)):
        self.nodes = [np.zeros(1 << l) for l in range(int(np.ceil(np.log2(max_size))) + 1)]

    def sample(self):
        q = np.random.uniform(0, self.nodes[0][0], size=1)
        i = np.zeros(1, dtype=int)
        for nodes in self.nodes[1:]:
            i *= 2
            left = nodes[i]
            g = np.greater(q, left)
            i += g
            q -= left * g
        return int(i[0])

    def set(self, i, p):
        diff = p - self.nodes[-1][i]
        for nodes in self.nodes[::-1]:
            np.add.at(nodes, i, diff)
            i //= 2


class HostAgent:
    """The reference's MOQLearning step (mo_q_learning.py:123-208), TabularModel and MPMOQLearning GPI, on host dicts."""

    def __init__(self, env, P, kw, seed=0):
        self.env, self.kw = env, kw
        self.rng = np.random.default_rng(seed)
        self.tables = [dict() for _ in range(P)]
        self.W = self.rng.dirichlet(np.ones(3), P)
        self.model, self.pairs, self.sa_ind, self.tree = {}, [], {}, HostSumTree() if kw.get("gpi_pd") else None

    def sq(self, p, s, w):
        t = self.tables[p]
        return np.zeros(4) if s not in t else np.array([np.dot(v, w) for v in t[s]])

    def greedy(self, p, s):
        w = self.W[p]
        if self.kw.get("use_gpi_policy"):
            q = np.stack([self.sq(i, s, w) for i in range(len(self.tables))])
            return int(np.unravel_index(np.argmax(q), q.shape)[1])
        if s not in self.tables[p]:
            return int(self.env.action_space.sample())
        return int(np.argmax(self.sq(p, s, w)))

    def maxs(self, s, w):
        return np.max([self.sq(i, s, w) for i in range(len(self.tables))])

    def td(self, p, s, a, r, s2, term):
        t = self.tables[p]
        for x in (s, s2):
            if x not in t:
                t[x] = np.zeros((4, 3))
        mq = t[s2][self.greedy(p, s2)]
        t[s][a] += 0.1 * (r + (1 - term) * 0.9 * mq - t[s][a])
        if self.tree is not None:
            w = self.W[p]
            pr = np.dot(r, w) + (1 - term) * 0.9 * self.maxs(s2, w) - np.dot(t[s][a], w)
            return max(np.abs(pr), 1e-4) ** 0.6
        return None

    def train(self, p, steps):
        s = tuple(self.env.reset()[0])
        for _ in range(steps):
            a = int(self.env.action_space.sample()) if self.rng.random() < 0.1 else self.greedy(p, s)
            o, r, term, trunc, _ = self.env.step(a)
            s2 = tuple(o)
            prio = self.td(p, s, a, r, s2, term)
            if self.kw.get("dyna"):
                sa, srt = (s, a), (s2, tuple(r), term)
                if sa not in self.model:
                    self.pairs.append(sa)
                    self.model[sa] = {}
                    self.sa_ind[sa] = len(self.pairs) - 1
                self.model[sa][srt] = self.model[sa].get(srt, 0) + 1
                if prio is not None:
                    self.tree.set(self.sa_ind[sa], prio)
                for _ in range(self.kw["dyna_updates"]):
                    ind = self.tree.sample() if self.tree is not None else random.randint(0, len(self.pairs) - 1)
                    ks = list(self.model[self.pairs[ind]].keys())
                    c = np.array(list(self.model[self.pairs[ind]].values()))
                    ns, rr, tt = random.choices(ks, weights=c / c.sum(), k=1)[0]
                    pr = self.td(p, self.pairs[ind][0], self.pairs[ind][1], np.array(rr), ns, tt)
                    if pr is not None:
                        self.tree.set(ind, pr)
            s = tuple(self.env.reset()[0]) if term or trunc else s2


def device_agent(P, kw, steps):
    env = TreasureGrid(d=3, slip=0.2, seed=0)
    agent = MPMOQLearning(env, seed=0, log=False, **kw)
    agent.linear_support.verbose = False
    if P > 1:
        agent.train(total_timesteps=(P - 1) * 50, eval_env=TreasureGrid(d=3, seed=1), ref_point=np.zeros(3), timesteps_per_iteration=50,
                    num_eval_episodes_for_front=1)
    return agent


def time_device(P, kw, steps):
    agent = device_agent(P, kw, steps)
    from morl_baselines_b200.multi_policy.multi_policy_moqlearning.mp_mo_q_learning import DeviceMOQLearning

    learner = DeviceMOQLearning(agent.env, weights=np.ones(3) / 3, parent=agent, log=False, parent_rng=agent.np_random,
                                **{k: v for k, v in kw.items()})
    agent.policies.append(learner)
    learner.train(start_time=0.0, total_timesteps=50, reset_num_timesteps=False)  # warm-up
    th.cuda.synchronize()
    n0 = ops.launch_count
    t0 = time.perf_counter()
    learner.train(start_time=0.0, total_timesteps=steps, reset_num_timesteps=False)
    th.cuda.synchronize()
    dt = time.perf_counter() - t0
    return steps / dt, (ops.launch_count - n0) / steps


def time_host(P, kw, steps):
    h = HostAgent(TreasureGrid(d=3, slip=0.2, seed=0), P, kw)
    for p in range(P - 1):
        h.train(p, 50)
    t0 = time.perf_counter()
    h.train(P - 1, steps)
    return steps / (time.perf_counter() - t0)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"unavailable ({e})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert th.cuda.is_available(), "bench_mp_moq needs a CUDA device"
    res = {"card": card(), "steps": args.steps, "rounds": args.rounds, "train": {}}
    for name, kw in CONFIGS.items():
        for P in (1, 8, 16):
            dev, host, launches = [], [], []
            for _ in range(args.rounds):
                sps, lps = time_device(P, kw, args.steps)
                dev.append(sps)
                launches.append(lps)
                host.append(time_host(P, kw, args.steps))
            res["train"][f"{name}/P{P}"] = {"device_steps_per_s": float(np.median(dev)), "host_steps_per_s": float(np.median(host)),
                                            "launches_per_step": float(np.median(launches))}
            print(name, P, res["train"][f"{name}/P{P}"], file=sys.stderr, flush=True)
    agent = device_agent(16, CONFIGS["gpi"], args.steps)
    rng = np.random.default_rng(0)
    obs = np.stack([rng.integers(0, 6, 100), rng.integers(0, 7, 100)], axis=1).astype(np.int32)
    w = rng.dirichlet(np.ones(3), 100)
    batch, serial = [], []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        agent.eval_batch(obs, w)
        batch.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        for o, wi in zip(obs, w):
            agent.eval(o, wi)
        serial.append(time.perf_counter() - t0)
    res["eval_100_rows_P16_ms"] = {"eval_batch": 1e3 * float(np.median(batch)), "serial_eval": 1e3 * float(np.median(serial))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
