"""PCN on the device at three shapes: minecart (obs 7, 6 actions, d 3, H 64, B 256, U 50, 50 episodes of 100-1000 steps), fruit-tree
(obs 2, 2 actions, d 6, H 64, B 32, U 100, 500 episodes of 6 steps) and a continuous shape (obs 11, act 3, d 3, H 64, B 256, U 50,
50 episodes of 100-1000 steps), on the variable-length stand-in environment of the tests.

    python scripts/bench_pcn.py [--rounds 5] [--out bench_pcn.json]

Per shape, medians over alternating rounds of:
  block  : one U-update block as a CUDA-graph replay (what train() runs), host draws and upload included, against the same class with
           use_cuda_graph=False and against the reference's update loop restated on the device (per-sample Python batch assembly, four
           host-to-device copies, torch eager forward / loss / backward, torch Adam, ``.cpu()`` of loss and prediction per update);
  act    : ``_act``'s single-row forward through pinned memory against a torch-eager forward of the same model plus ``.cpu()``;
  iter   : one train() iteration (U updates, the command choice, 10 rollouts) with its time split between the three.
Prints one JSON line with the card's name, power limit and SM clock."""

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

from morl_baselines_b200.multi_policy.pcn.pcn import PCN, Transition  # noqa: E402
from tests.pcn_standin import VarLengthEnv, random_episode  # noqa: E402

SHAPES = {
    "minecart": dict(env=dict(obs_dim=7, n_actions=6, reward_dim=3, min_len=100, max_len=1000), B=256, U=50, episodes=50),
    "fruit_tree": dict(env=dict(obs_dim=2, n_actions=2, reward_dim=6, min_len=6, max_len=6), B=32, U=100, episodes=500),
    "continuous": dict(env=dict(obs_dim=11, reward_dim=3, continuous_action_dim=3, min_len=100, max_len=1000), B=256, U=50, episodes=50),
}


def sync_time(fn):
    th.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    th.cuda.synchronize()
    return time.perf_counter() - t0


def make_agent(c, graph, seed=0):
    env = VarLengthEnv(**c["env"], seed=seed)
    agent = PCN(env, np.ones(c["env"]["reward_dim"] + 1, np.float32) * 0.1, batch_size=c["B"], log=False, seed=seed, device="cuda",
                use_cuda_graph=graph)
    episodes = []
    for k in range(c["episodes"]):
        o, a, r = random_episode(env, np.random.default_rng(k))
        ts = [Transition(oi, ai, ri.copy(), None, False) for oi, ai, ri in zip(o, a, r)]
        agent._add_episode(ts, max_size=c["episodes"], step=k + 1)
        episodes.append(ts)
    return agent, env, episodes


def reference_block(agent, episodes_by_slot, U, opt):
    """The reference's update loop (pcn.py:202-236) on the device, U times."""
    m, dev = agent.model, agent.device
    heap = agent.experience_replay
    for _ in range(U):
        batch = []
        s_i = agent.np_random.choice(np.arange(len(heap)), size=agent.batch_size, replace=True)
        for i in s_i:
            ep = episodes_by_slot[heap[i][2]]
            t = agent.np_random.integers(0, len(ep))
            batch.append((ep[t].observation, ep[t].action, np.float32(ep[t].reward), np.float32(len(ep) - t)))
        obs, actions, ret, hor = zip(*batch)
        pred = m(th.tensor(np.array(obs)).to(dev), th.tensor(np.array(ret)).to(dev), th.tensor(np.array(hor)).unsqueeze(1).to(dev))
        opt.zero_grad()
        if agent.continuous_action:
            loss = th.nn.functional.mse_loss(th.tensor(np.array(actions)).float().to(dev), pred)
        else:
            onehot = th.nn.functional.one_hot(th.tensor(np.array(actions)).long().to(dev), pred.shape[1])
            loss = th.sum(-onehot * pred, -1).mean()
        loss.backward()
        opt.step()
        loss.detach().cpu().numpy()
        pred.detach().cpu().numpy()


def bench_shape(name, c, rounds):
    graph, env, episodes = make_agent(c, True)
    eager, _, _ = make_agent(c, False)
    ref_agent, _, _ = make_agent(c, False)
    by_slot = dict(enumerate(episodes))  # slots are assigned in insertion order; evicted slots are never drawn
    ref_opt = th.optim.Adam(ref_agent.model.parameters(), lr=ref_agent.learning_rate)
    U = c["U"]
    graph._run_block(U), eager._run_block(U), reference_block(ref_agent, by_slot, 2, ref_opt)  # capture, warm up
    t = {"graph": [], "eager": [], "ref": [], "act_kernel": [], "act_torch": []}
    obs, ret, hor = env.reset()[0], np.ones(c["env"]["reward_dim"], np.float32), np.float32(50)
    m = graph.model
    for _ in range(rounds):
        t["graph"].append(sync_time(lambda: graph._run_block(U)))
        t["eager"].append(sync_time(lambda: eager._run_block(U)))
        t["ref"].append(sync_time(lambda: reference_block(ref_agent, by_slot, U, ref_opt)))
        n = 200
        t0 = time.perf_counter()
        for _ in range(n):
            graph._predict_row(obs, ret, hor)
        t["act_kernel"].append((time.perf_counter() - t0) / n)
        t0 = time.perf_counter()
        with th.no_grad():
            for _ in range(n):
                m(th.tensor(np.array([obs])).float().to("cuda"), th.tensor(np.array([ret])).float().to("cuda"),
                  th.tensor(np.array([hor])).unsqueeze(1).float().to("cuda")).cpu().numpy()
        t["act_torch"].append((time.perf_counter() - t0) / n)
    res = {k + "_ms": round(float(np.median(v)) * 1e3, 4) for k, v in t.items()}
    # one train() iteration split into its phases
    split = {"updates": [], "ranking": [], "rollouts": []}
    max_return = np.full(c["env"]["reward_dim"], 100.0, np.float32)
    for _ in range(rounds):
        split["updates"].append(sync_time(lambda: graph._run_block(U).stats.cpu()))
        t0 = time.perf_counter()
        r, h = graph._choose_commands(20)
        split["ranking"].append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        for _ in range(10):
            ts = graph._run_episode(env, r, h, max_return)
            graph._add_episode(ts, max_size=c["episodes"], step=10**6)
        split["rollouts"].append(time.perf_counter() - t0)
    res.update({f"iter_{k}_ms": round(float(np.median(v)) * 1e3, 3) for k, v in split.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bench_pcn.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    out = {"card": card}
    for name, c in SHAPES.items():
        out[name] = bench_shape(name, c, args.rounds)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
