"""NLMOPPO on the device at three shapes, on the stand-in environment of the tests (4 epochs each):
  test    : 8 envs x 16 steps, 4 minibatches, obs 2, 4 actions, d 2 (the reference test's shape);
  default : 8 envs x 128 steps (the reference's default num_steps: a batch of 1,024), 4 minibatches, obs 2, 4 actions, d 2;
  large   : 64 envs x 128 steps, 8 minibatches, obs 7, 6 actions, d 3.

    python scripts/bench_nl_mo_ppo.py [--rounds 5] [--out bench_nl_mo_ppo.json]

Per shape, medians over alternating rounds of:
  update : one ``update()`` replayed as a CUDA graph, against the same kernels launched eagerly, against the reference's update restated
           on the device (torch eager forward / loss / backward, ``clip_grad_norm_``, torch Adam, one ``.item()`` per minibatch);
  step   : one rollout step (forward kernel, sampling, one copy each way, commit kernel), against the reference's step restated (torch
           forward, ``.cpu()``, three host-to-device copies, the accrued-reward expression);
  act    : one deterministic ``policy_evaluate`` step (the forward kernel's argmax through pinned memory) against the reference's
           ``as_tensor`` copies, torch forward, argmax and ``.item()``.
Prints one JSON line with the card's name, power limit and SM clock, read in the same call."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th
from torch import nn, optim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from morl_baselines_b200.single_policy.ser.nl_mo_ppo import NLMOPPO  # noqa: E402
from tests.nl_ppo_standin import RingEnv, RingVecEnv  # noqa: E402

SHAPES = {
    "test": dict(envs=8, steps=16, mb=4, env=dict(obs_dim=2, n_actions=4, d=2)),
    "default": dict(envs=8, steps=128, mb=4, env=dict(obs_dim=2, n_actions=4, d=2)),
    "large": dict(envs=64, steps=128, mb=8, env=dict(obs_dim=7, n_actions=6, d=3)),
}


def sync_time(fn):
    th.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    th.cuda.synchronize()
    return time.perf_counter() - t0


def u_func(v):
    return -th.logsumexp(-4.0 * v, 0) / 4.0


def make(c, graph=True, seed=0):
    th.manual_seed(seed)
    ag = NLMOPPO(0, RingVecEnv(c["envs"], **c["env"]), num_steps=c["steps"], num_minibatches=c["mb"], device="cuda", seed=seed,
                 use_cuda_graph=graph)
    ag.u_func = u_func
    ag._set_pref(np.ones(c["env"]["d"]) / c["env"]["d"])
    obs, _ = ag.envs.reset(seed=seed)
    ag._next_obs.copy_(th.as_tensor(obs))
    ag._collect_rollouts(0)
    ag._compute_advantages_and_returns()
    return ag


def reference_update(ag, opt):
    """nl_mo_ppo.py:325-398 on the device."""
    B0 = ag.init_obs.shape[0]
    v0 = ag.agent.get_value(ag.init_obs, acc_reward=th.zeros((B0, ag.num_objectives), device=ag.device), pref=ag.pref).mean(0)
    v0 = v0.detach().requires_grad_(True)
    (w,) = th.autograd.grad(ag.u_func(v0), v0)
    B, mb = ag.batch_size, ag.minibatch_size
    b_obs, b_acc, b_act, b_logp, b_adv, b_ret, b_val = ag._batch()
    b_pref = ag.pref.expand(B, -1)
    b_inds = np.arange(B)
    clipfracs = []
    for _ in range(ag.update_epochs):
        ag.rng.shuffle(b_inds)
        for start in range(0, B, mb):
            i = b_inds[start:start + mb]
            _, newlogprob, entropy, newvalue = ag.agent.get_action_and_value(b_obs[i], acc_reward=b_acc[i], action=b_act.long()[i], pref=b_pref[i])
            logratio = newlogprob - b_logp[i]
            ratio = logratio.exp()
            with th.no_grad():
                clipfracs.append(((ratio - 1.0).abs() > ag.clip_coef).float().mean().item())
            a = b_adv[i]
            a = (a - a.mean(dim=0, keepdim=True)) / (a.std(dim=0, keepdim=True) + 1e-8)
            pg = (th.max(-a * ratio.unsqueeze(-1), -a * th.clamp(ratio, 1 - ag.clip_coef, 1 + ag.clip_coef).unsqueeze(-1)).mean(0) * w).sum()
            vc = b_val[i] + th.clamp(newvalue - b_val[i], -ag.clip_coef, ag.clip_coef)
            v_loss = 0.5 * th.max((newvalue - b_ret[i]) ** 2, (vc - b_ret[i]) ** 2).mean()
            loss = pg - ag.ent_coef * entropy.mean() + ag.vf_coef * v_loss
            opt.zero_grad()
            loss.backward()
            nn.utils.clip_grad_norm_(ag.agent.parameters(), ag.max_grad_norm)
            opt.step()


def reference_step(ag, state):
    """One step of nl_mo_ppo.py:249-275 on the device."""
    next_obs, next_acc, next_done, timestep = state
    ag.obs[0] = next_obs
    ag.acc_rewards[0] = next_acc
    ag.dones[0] = next_done
    with th.no_grad():
        action, logprob, _, value = ag.agent.get_action_and_value(next_obs, acc_reward=next_acc, pref=ag.pref)
        ag.values[0] = value
    ag.actions[0] = action
    ag.logprobs[0] = logprob
    o, r, te, tr, _ = ag.envs.step(action.detach().cpu().numpy())
    ag.rewards[0] = th.as_tensor(r, device=ag.device, dtype=th.float32)
    next_obs = th.as_tensor(o, device=ag.device, dtype=th.float32)
    next_done = th.as_tensor(np.logical_or(te, tr), device=ag.device, dtype=th.float32)
    next_acc = (next_acc + (ag.gamma ** timestep) * ag.rewards[0]) * (1.0 - next_done.unsqueeze(-1))
    timestep = (timestep + 1) * (1 - next_done.int().unsqueeze(-1))
    return next_obs, next_acc, next_done, timestep


def bench_shape(c, rounds):
    graph, eager, ref = make(c, True), make(c, False), make(c, True)
    ref_opt = optim.Adam(ref.agent.parameters(), lr=ref.learning_rate, eps=1e-5)
    graph.update(), eager.update(), reference_update(ref, ref_opt)  # warm up, capture
    E, d = c["envs"], c["env"]["d"]
    state = (ref._next_obs.clone(), ref._next_acc.clone(), ref._next_done.clone(), th.zeros((E, 1), dtype=th.int32, device="cuda"))
    obs1, _ = RingEnv(**c["env"]).reset(seed=0)
    acc1 = np.zeros(d, np.float32)
    t = {k: [] for k in ("update_graph_ms", "update_eager_ms", "update_ref_ms", "step_kernel_us", "step_ref_us", "act_kernel_us", "act_ref_us")}
    n = 200
    for _ in range(rounds):
        t["update_graph_ms"].append(sync_time(graph.update) * 1e3)
        t["update_eager_ms"].append(sync_time(eager.update) * 1e3)
        t["update_ref_ms"].append(sync_time(lambda: reference_update(ref, ref_opt)) * 1e3)
        T, graph.num_steps = graph.num_steps, 1  # one step per call
        t["step_kernel_us"].append(sync_time(lambda: [graph._collect_rollouts(0) for _ in range(n)]) / n * 1e6)
        graph.num_steps = T
        box = [state]
        t["step_ref_us"].append(sync_time(lambda: [box.append(reference_step(ref, box.pop())) for _ in range(n)]) / n * 1e6)
        t["act_kernel_us"].append(sync_time(lambda: [graph._act(obs1, acc1, True) for _ in range(n)]) / n * 1e6)
        with th.no_grad():
            t["act_ref_us"].append(sync_time(lambda: [ref.agent.get_greedy_action(th.as_tensor(obs1, device="cuda", dtype=th.float32),
                                                                                  acc_reward=th.as_tensor(acc1, device="cuda", dtype=th.float32),
                                                                                  pref=ref.pref).item() for _ in range(n)]) / n * 1e6)
    return {k: round(float(np.median(v)), 3) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bench_nl_mo_ppo.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    out = {"card": card}
    for name, c in SHAPES.items():
        out[name] = bench_shape(c, args.rounds)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
