"""EUPG on the device at two shapes, on the stand-in environment of the tests:
  fishwood : one Discrete observation column, 2 actions, d 2, net_arch [50], 200-step episodes;
  wider    : obs 8, 4 actions, d 3, net_arch [256, 256], 1,000-step episodes.

    python scripts/bench_eupg.py [--rounds 5] [--out bench_eupg.json]

Per shape, medians over alternating rounds of:
  update : one ``update()`` on a full episode on the kernel path, against the same class on its eager path and against the reference's
           update restated on the device (six host-to-device copies, ``.cpu()`` of the episodic return, the Python returns loop, torch eager
           forward / loss / backward and torch Adam);
  act    : one action (the single-row probabilities kernel through pinned memory, sampling on the host), against the reference's
           ``th.Tensor(obs).to(device)``, torch forward, Categorical sample and ``.item()``;
  train  : a ``train()`` of 20,000 steps on the kernel path and on the eager path.
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

from morl_baselines_b200.single_policy.esr.eupg import EUPG  # noqa: E402
from tests.eupg_standin import EupgEnv, fixed_episode, weighted_sum_scalarization  # noqa: E402

SHAPES = {
    "fishwood": dict(env=dict(n_actions=2, reward_dim=2, discrete_obs=2, min_len=200, max_len=200), arch=[50], T=200),
    "wider": dict(env=dict(obs_dim=8, n_actions=4, reward_dim=3, min_len=1000, max_len=1000), arch=[256, 256], T=1000),
}
TRAIN_STEPS = 20000


def sync_time(fn):
    th.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    th.cuda.synchronize()
    return time.perf_counter() - t0


def make_agent(c, fused, seed=0):
    env = EupgEnv(**c["env"], seed=seed)
    d = c["env"]["reward_dim"]
    th.manual_seed(seed)
    agent = EUPG(env, weighted_sum_scalarization(np.ones(d) / d), weights=np.ones(d) / d, net_arch=c["arch"], log=False, device="cuda")
    agent.fused = agent.fused and fused
    for tr in fixed_episode(env, np.random.default_rng(seed), c["T"]):
        agent.buffer.add(*tr)
    return agent


def reference_update(agent, opt):
    """eupg.py:226-251 on the device."""
    dev = agent.device
    obs, acc, actions, rewards, next_obs, dones = agent.buffer.get_all_data(to_tensor=True, device=dev)
    episodic_return = th.sum(rewards, dim=0)
    agent.scalarization(episodic_return.cpu().numpy(), agent.weights)
    flip = rewards.flip(dims=[0])
    c = th.zeros(agent.reward_dim).to(dev)
    for i in range(len(rewards)):
        c = agent.gamma * c + flip[i]
        flip[i] = c
    v = agent.scalarization(flip.flip(dims=[0]))
    loss = -th.mean(agent.net.distribution(obs, acc).log_prob(actions.squeeze()) * v)
    opt.zero_grad()
    loss.backward()
    opt.step()


def reference_act(agent, obs, acc_dev):
    return agent.net.distribution(th.Tensor(obs).to(agent.device), acc_dev).sample().detach().item()


def bench_shape(c, rounds):
    fused, eager, ref = make_agent(c, True), make_agent(c, False), make_agent(c, False)
    ref_opt = th.optim.Adam(ref.net.parameters(), lr=ref.learning_rate)
    fused.update(), eager.update(), reference_update(ref, ref_opt)  # warm up
    S, d = fused.observation_shape[0], fused.reward_dim
    obs = np.ones(S, np.float32)
    acc = np.zeros(d, np.float32)
    acc_dev = th.zeros(d, device="cuda")
    t = {k: [] for k in ("update_kernel", "update_eager", "update_ref", "act_kernel", "act_ref", "train_kernel", "train_eager")}
    for _ in range(rounds):
        t["update_kernel"].append(sync_time(fused.update))
        t["update_eager"].append(sync_time(eager.update))
        t["update_ref"].append(sync_time(lambda: reference_update(ref, ref_opt)))
        n = 500
        t["act_kernel"].append(sync_time(lambda: [fused._choose_action(obs, acc) for _ in range(n)]) / n)
        with th.no_grad():
            t["act_ref"].append(sync_time(lambda: [reference_act(ref, obs, acc_dev) for _ in range(n)]) / n)
    for _ in range(rounds):
        for key, agent in (("train_kernel", make_agent(c, True)), ("train_eager", make_agent(c, False))):
            agent.buffer.cleanup()
            t[key].append(sync_time(lambda: agent.train(total_timesteps=TRAIN_STEPS)))
    return {k + ("_us" if k.startswith("act") else "_ms"): round(float(np.median(v)) * (1e6 if k.startswith("act") else 1e3), 3)
            for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bench_eupg.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    out = {"card": card, "train_steps": TRAIN_STEPS}
    for name, c in SHAPES.items():
        out[name] = bench_shape(c, args.rounds)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
