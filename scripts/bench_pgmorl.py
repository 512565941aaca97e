"""PGMORL's population update phase on the device, at the halfcheetah shape of the reference's examples/pgmorl_halfcheetah.py:
pop 6, 4 envs x 2048 steps, 32 minibatches x 10 epochs, obs 17, act 6, d 2, [64, 64].

    python scripts/bench_pgmorl.py [--rounds 5] [--out bench_pgmorl.json]

Compared in one process, alternating round by round on the same seeded batches:
  graph  : every agent's update as ONE PopulationGraph replay (what PGMORL runs)
  eager  : the same MOPPO classes with use_cuda_graph=False, agent after agent
  ref    : a restatement of the reference's update loop (mo_ppo.py:433-558): the per-step Python GAE loop, torch autograd for the loss,
           clip_grad_norm_ + torch Adam (eps 1e-5) and the per-minibatch ``.item()`` of the clip fraction
and the GAE kernel alone against the Python loop.  Before timing, one update of each path starts from the same parameters and batch:
graph and eager must be bit-identical, and the restatement close (float32 rounding only).  Prints one JSON line with the card's name,
power limit and SM clock."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from morl_baselines_b200 import ops  # noqa: E402
from morl_baselines_b200.common.graphed import PopulationGraph  # noqa: E402
from morl_baselines_b200.single_policy.ser.mo_ppo import MOPPO, MOPPONet, PPOReplayBuffer  # noqa: E402

POP, E, T, MB, EPOCHS, OBS, ACT, D, ARCH = 6, 4, 2048, 32, 10, 17, 6, 2, [64, 64]
GAMMA, LAM = 0.995, 0.95


class _Envs:
    num_envs = E


def make_population(dev, use_cuda_graph):
    th.manual_seed(0)
    agents = []
    for i in range(POP):
        net = MOPPONet((OBS,), (ACT,), D, ARCH).to(dev)
        w = np.array([i / (POP - 1), 1 - i / (POP - 1)], np.float32)
        a = MOPPO(i, net, w, _Envs(), steps_per_iteration=T, num_minibatches=MB, update_epochs=EPOCHS, gamma=GAMMA, device=dev,
                  rng=np.random.default_rng(100 + i), use_cuda_graph=use_cuda_graph)
        g = np.random.default_rng(i)
        b = a.batch
        b.obs.copy_(th.from_numpy(g.standard_normal((T, E, OBS)).astype(np.float32)))
        b.actions.copy_(th.from_numpy(g.standard_normal((T, E, ACT)).astype(np.float32) * 0.5))
        with th.no_grad():
            _, lp, _, v = net.get_action_and_value(b.obs.reshape(-1, OBS), b.actions.reshape(-1, ACT))
        b.logprobs.copy_((lp + th.from_numpy(g.standard_normal(T * E).astype(np.float32) * 0.05).to(dev)).reshape(T, E))
        b.values.copy_(v.reshape(T, E, D))
        b.rewards.copy_(th.from_numpy(g.standard_normal((T, E, D)).astype(np.float32)))
        b.dones.copy_(th.from_numpy((g.random((T, E)) < 0.002).astype(np.float32)))
        a._next = (th.from_numpy(g.standard_normal((E, D)).astype(np.float32)).to(dev), th.zeros(E, device=dev))
        ops.vector_gae(b.rewards, b.values, b.dones, a._next[0], a._next[1], a._w32, GAMMA, LAM, True, returns_out=a.returns, adv_out=a.advantages)
        agents.append(a)
    return agents


def python_gae(b, next_value, next_done, w):
    """The reference's loop (mo_ppo.py:439-476)."""
    adv = th.zeros_like(b.rewards)
    last = 0
    ext = lambda x: x.unsqueeze(1).repeat(1, D)  # noqa: E731
    for t in reversed(range(T)):
        nnt, nv = (1.0 - next_done, next_value) if t == T - 1 else (1.0 - b.dones[t + 1], b.values[t + 1])
        nnt = ext(nnt)
        delta = b.rewards[t] + GAMMA * nv * nnt - b.values[t]
        adv[t] = last = delta + GAMMA * LAM * nnt * last
    return adv + b.values, adv @ w


class RefUpdate:
    """The reference's update of one agent (mo_ppo.py:492-558), with its own torch Adam over the agent's network."""

    def __init__(self, a):
        self.a = a
        self.opt = th.optim.Adam(a.networks.parameters(), lr=a.learning_rate, eps=1e-5)
        self.rng = np.random.default_rng(100 + a.id)

    def __call__(self):
        a, net = self.a, self.a.networks
        returns, advantages = python_gae(a.batch, a._next[0], a._next[1], a.weights)
        b_obs, b_act = a.batch.obs.reshape(-1, OBS), a.batch.actions.reshape(-1, ACT)
        b_lp, b_adv, b_ret, b_val = a.batch.logprobs.reshape(-1), advantages.reshape(-1), returns.reshape(-1, D), a.batch.values.reshape(-1, D)
        b_inds = np.arange(a.batch_size)
        clipfracs = []
        for _ in range(EPOCHS):
            self.rng.shuffle(b_inds)
            for start in range(0, a.batch_size, a.minibatch_size):
                mb = b_inds[start:start + a.minibatch_size]
                _, newlp, ent, newv = net.get_action_and_value(b_obs[mb], b_act[mb])
                logratio = newlp - b_lp[mb]
                ratio = logratio.exp()
                with th.no_grad():
                    clipfracs += [((ratio - 1.0).abs() > a.clip_coef).float().mean().item()]
                adv = b_adv[mb]
                adv = (adv - adv.mean()) / (adv.std() + 1e-8)
                pg = th.max(-adv * ratio, -adv * th.clamp(ratio, 1 - a.clip_coef, 1 + a.clip_coef)).mean()
                newv = newv.view(-1, D)
                vc = b_val[mb] + th.clamp(newv - b_val[mb], -a.clip_coef, a.clip_coef)
                v_loss = 0.5 * th.max((newv - b_ret[mb]) ** 2, (vc - b_ret[mb]) ** 2).mean()
                loss = pg - a.ent_coef * ent.mean() + v_loss * a.vf_coef
                self.opt.zero_grad()
                loss.backward()
                th.nn.utils.clip_grad_norm_(net.parameters(), a.max_grad_norm)
                self.opt.step()


def timed(fn, n=1):
    th.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    th.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = th.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()

    graph_pop, eager_pop, ref_pop = make_population(dev, True), make_population(dev, False), make_population(dev, False)
    pg = PopulationGraph([a._variant("all").step for a in graph_pop], lambda: [t for a in graph_pop for t in a._mutated_tensors()])

    def run_graph():
        for a in graph_pop:
            a.prepare_update()
        pg()

    def run_eager():
        for a in eager_pop:
            a.update()

    refs = [RefUpdate(a) for a in ref_pop]

    def run_ref():
        for r in refs:
            r()

    # agreement at the timed size, from identical parameters and batches
    run_graph()
    run_eager()
    run_ref()
    th.cuda.synchronize()
    bit_identical = all(th.equal(p, q) for a, b in zip(graph_pop, eager_pop) for p, q in zip(a.networks.parameters(), b.networks.parameters()))
    ref_dev = max(float((p - q).abs().max() / q.abs().max().clamp_min(1e-12)) for a, b in zip(graph_pop, ref_pop)
                  for p, q in zip(a.networks.parameters(), b.networks.parameters()))
    a0 = graph_pop[0]
    r_py, adv_py = python_gae(a0.batch, a0._next[0], a0._next[1], a0._w32)
    r_k, adv_k = ops.vector_gae(a0.batch.rewards, a0.batch.values, a0.batch.dones, a0._next[0], a0._next[1], a0._w32, GAMMA, LAM, True)
    gae_returns_equal = bool(th.equal(r_py, r_k))
    gae_adv_maxdiff = float((adv_py - adv_k).abs().max())

    res = {"graph": [], "eager": [], "ref": [], "gae_kernel": [], "gae_python": []}
    for _ in range(args.rounds):
        res["graph"].append(timed(run_graph))
        res["eager"].append(timed(run_eager))
        res["ref"].append(timed(run_ref))
        res["gae_kernel"].append(timed(lambda: ops.vector_gae(a0.batch.rewards, a0.batch.values, a0.batch.dones, a0._next[0], a0._next[1], a0._w32,
                                                              GAMMA, LAM, True), n=50))
        res["gae_python"].append(timed(lambda: python_gae(a0.batch, a0._next[0], a0._next[1], a0._w32), n=3))
    med = {k: float(np.median(v)) for k, v in res.items()}
    out = {"card": card, "shape": dict(pop=POP, envs=E, steps=T, minibatches=MB, epochs=EPOCHS, obs=OBS, act=ACT, d=D, arch=ARCH),
           "median_ms": med, "rounds_ms": res, "graph_eager_bit_identical": bit_identical, "graph_vs_ref_max_rel_dev": ref_dev,
           "gae_returns_bit_exact": gae_returns_equal, "gae_adv_max_abs_diff": gae_adv_maxdiff,
           "speedup_graph_vs_eager": med["eager"] / med["graph"], "speedup_graph_vs_ref": med["ref"] / med["graph"],
           "speedup_gae": med["gae_python"] / med["gae_kernel"]}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
