"""GPI-PD's Dyna path with continuous actions at the sizes of the reference's examples/gpi_pd_hopper.py: hopper dimensions (observations 11,
actions 3, d = 3), ensemble 5 x [200] * 4, rollouts of 50,000 rows (5 chunks of 10,000) for 5 steps, model buffer 200,000.

    python scripts/bench_gpipd_continuous_dyna.py [--rounds R]        # on the GPU: prints one JSON object
    python scripts/bench_gpipd_continuous_dyna.py --impl reference    # the reference's rollout, one chunk, on the CPU (needs the reference)

GPU figures:
  * ``rollout_ms``: ``_rollout_dynamics`` with the fused commit (morl_dyna_commit_f32) against the same step composed from existing code
    (``ModelEnv.step_device`` -> boolean masks -> ``ReplayBuffer.add_batch``), alternating in one process, at two uncertainty thresholds: 2.0
    (the example's) and 1e9 (every row kept, the worst case for the append);
  * ``update_ms``: one ``update()`` (20 gradient steps, batch 128, 10 % real rows) with model samples, as graph replays and eagerly;
  * ``fit_epoch_ms``: one ``ProbabilisticEnsemble.fit`` epoch on 100,000 transitions (bootstrapped minibatches of 256, graph replays).
The ensemble and the agent are untrained (seeded), so the figures measure the engine, not a learned model.  The card name, power limit and
SM clocks are read in the same run."""

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

OBS, ACT, D = 11, 3, 3


def make_env():
    from morl_baselines_b200.testing import FakeEnv, _Spec

    env = FakeEnv(obs_dim=OBS, continuous_action_dim=ACT, reward_dim=D)
    env.spec = _Spec("mo-hopper-v4")
    return env


def fill_real(rb, n, rng):
    """n hopper-like real transitions (heights around 1.2, small angles) so that imagined rows survive several steps."""
    obs = (rng.standard_normal((n, OBS)) * 0.3).astype(np.float32)
    obs[:, 0] += 1.2
    rb.obs[:n], rb.next_obs[:n] = obs, obs + 0.01 * rng.standard_normal((n, OBS)).astype(np.float32)
    rb.actions[:n] = rng.uniform(-1, 1, (n, ACT)).astype(np.float32)
    rb.rewards[:n] = rng.standard_normal((n, D)).astype(np.float32)
    rb.dones[:n] = 0.0
    rb.size, rb.ptr = n, n % rb.max_size
    if hasattr(rb, "mark_all_dirty"):
        rb.mark_all_dirty()
    if hasattr(rb, "tree"):
        rb.tree.batch_set(np.arange(n), rng.random(n) + 0.1)


def shape_model(model, rb):
    """Input statistics of the real data (an unfitted ensemble normalises by zero), small state deltas and a narrow aleatoric part, so that
    imagined rows survive several steps and the uncertainties spread around the example's threshold."""
    model._fit_input_stats(np.hstack((rb.obs[:rb.size], rb.actions[:rb.size])))
    with th.no_grad():
        model.layers[-1].W.mul_(0.1)
        model.max_logvar.fill_(-8.0)


def make_agent(dev, threshold):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import GPIPDContinuousAction

    th.manual_seed(0)
    agent = GPIPDContinuousAction(make_env(), gradient_updates=20, min_priority=0.1, batch_size=128, buffer_size=int(4e5), dynamics_rollout_starts=0,
                                  dynamics_rollout_len=5, dynamics_rollout_freq=250, dynamics_rollout_batch_size=50000, dynamics_train_freq=250,
                                  dynamics_buffer_size=200000, dynamics_real_ratio=0.1, dynamics_min_uncertainty=threshold, dyna=True, per=True, log=False,
                                  seed=0, device=dev)
    fill_real(agent.replay_buffer, 100000, np.random.default_rng(0))
    agent.replay_buffer.flush()
    shape_model(agent.dynamics, agent.replay_buffer)
    agent.set_weight_support([np.array([1.0, 0.0, 0.0], np.float32), np.array([0.0, 1.0, 0.0], np.float32), np.array([0.3, 0.3, 0.4], np.float32)])
    return agent


@th.no_grad()
def composed_rollout(agent, weight):
    """The same rollout composed from existing code: ModelEnv.step_device, boolean masks, ReplayBuffer.add_batch (the discrete path's step)."""
    from morl_baselines_b200.common.model_based.utils import ModelEnv

    num_times = int(np.ceil(agent.dynamics_rollout_batch_size / 10000))
    batch_size = min(agent.dynamics_rollout_batch_size, 10000)
    model_env = ModelEnv(agent.dynamics, agent.env.unwrapped.spec.id, rew_dim=agent.reward_dim)
    db = agent.dynamics_buffer
    for _ in range(num_times):
        obs = th.from_numpy(agent.replay_buffer.sample_obs(batch_size)).to(agent.device)
        for _h in range(agent.dynamics_rollout_len):
            actions = agent.policy(obs, weight.reshape(1, -1).repeat(obs.shape[0], 1), noise=agent.policy_noise, noise_clip=agent.noise_clip)
            next_obs, r, dones, info = model_env.step_device(obs, actions)
            keep = info["uncertainty"] < agent.dynamics_min_uncertainty
            if int(keep.sum()):
                db.add_batch(obs[keep], actions[keep], r[keep], next_obs[keep], dones[keep].float())
            nonterm = ~dones.squeeze(-1)
            if int(nonterm.sum()) == 0:
                break
            obs = next_obs[nonterm]


def timed(fn, n=1):
    th.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    th.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def gpu_main(args):
    dev = th.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    res = {"bench": "gpipd_continuous_dyna", "card": card, "shape": {"obs": OBS, "act": ACT, "d": D, "ensemble": "5 x [200]*4", "rollout_rows": 50000,
                                                                         "rollout_len": 5, "model_buffer": 200000}}
    w = th.tensor([0.3, 0.3, 0.4], device=dev)
    res["rollout_ms"] = {}
    for thr in (2.0, 1e9):
        agent = make_agent(dev, thr)
        fused, composed, rows = [], [], []
        agent._rollout_dynamics(w)  # warm-up of both arms
        composed_rollout(agent, w)
        for _ in range(args.rounds):
            s0 = agent.dynamics_buffer.ptr
            fused.append(timed(lambda: agent._rollout_dynamics(w)))
            rows.append((agent.dynamics_buffer.ptr - s0) % agent.dynamics_buffer.max_size)
            composed.append(timed(lambda: composed_rollout(agent, w)))
        res["rollout_ms"][f"threshold_{thr:g}"] = {"fused": sorted(fused), "composed": sorted(composed), "rows_kept_per_rollout": rows,
                                                   "median_speedup": float(np.median(composed) / np.median(fused))}
    # one update() with model samples, graph replays and eager
    agent = make_agent(dev, 1e9)
    agent._rollout_dynamics(w)
    agent.global_step = 1
    res["update_ms"] = {}
    for mode in (True, False):
        agent.use_cuda_graph = mode
        agent.update(w)  # warm-up (capture)
        res["update_ms"]["graph" if mode else "eager"] = sorted(timed(lambda: agent.update(w)) for _ in range(args.rounds))
    # one fit epoch on 100,000 transitions
    ens = agent.dynamics
    rb = agent.replay_buffer
    m_obs, m_act, m_rew, m_nobs, _ = rb.get_all_data()
    X, Y = np.hstack((m_obs, m_act)), np.hstack((m_rew, m_nobs - m_obs))
    t_fit = []
    for _ in range(args.rounds + 1):
        th.cuda.synchronize()
        t0 = time.perf_counter()
        ens.fit(X, Y, max_epochs=1)
        th.cuda.synchronize()
        t_fit.append((time.perf_counter() - t0) * 1e3)
    res["fit_epoch_ms"] = {"transitions": int(X.shape[0]), "holdout": 5000, "batch": 256, "ms_incl_upload_and_holdout": sorted(t_fit[1:])}
    print(json.dumps(res))


def reference_main(args):
    """One chunk (10,000 rows x 5 steps) of the reference's _rollout_dynamics on the CPU, same shapes."""
    from oracle import ref_harness as rh

    if not rh.reference_available():
        raise SystemExit("the reference is not available here")
    gm = rh.import_reference("morl_baselines.multi_policy.gpi_pd.gpi_pd_continuous_action")
    th.manual_seed(0)
    agent = gm.GPIPDContinuousAction(make_env(), batch_size=128, buffer_size=int(4e5), dynamics_rollout_starts=0, dynamics_rollout_len=5,
                                     dynamics_rollout_batch_size=10000, dynamics_buffer_size=200000, dynamics_min_uncertainty=1e9, dyna=True, per=True,
                                     log=False, seed=0, device="cpu")
    fill_real(agent.replay_buffer, 100000, np.random.default_rng(0))
    shape_model(agent.dynamics, agent.replay_buffer)
    w = th.tensor([0.3, 0.3, 0.4])
    times = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        agent._rollout_dynamics(w)
        times.append((time.perf_counter() - t0) * 1e3)
    print(json.dumps({"bench": "gpipd_continuous_dyna", "impl": "reference", "device": "cpu", "threads": th.get_num_threads(),
                      "rollout_chunk_10000x5_ms": sorted(times), "model_buffer_size": int(agent.dynamics_buffer.size)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--impl", choices=("engine", "reference"), default="engine")
    args = ap.parse_args()
    (reference_main if args.impl == "reference" else gpu_main)(args)


if __name__ == "__main__":
    main()
