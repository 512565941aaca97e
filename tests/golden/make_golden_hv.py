"""Hypervolume-parity reference run (SURVEY.md section 8(d), "HV parity protocol"): the UNMODIFIED reference Envelope is trained on
CPU on the stand-in MDP (tests/golden/standin_env.py) for a fixed number of environment steps / gradient updates per seed; the
discounted returns of its greedy policy for a fixed list of evaluation weights, the non-dominated front and its hypervolume are
frozen into tests/golden/hv_parity.json.  tests/test_hv_parity_gpu.py trains the CUDA engine with the same hyper-parameters, seeds,
environment and evaluation weights and requires the mean hypervolume to agree within 1 %.

    python tests/golden/make_golden_hv.py         (build container only: needs /root/reference)
"""

from __future__ import annotations

import json
import os
import sys
import time

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402
from morl_baselines_b200.common.performance_indicators import hypervolume as hypervolume_exact  # noqa: E402  (the ONE exact-HV routine both engines' fronts go through)
from tests.golden.standin_env import HV_REF_POINT, TreasureChain, robust_eval_weights  # noqa: E402

HP = dict(learning_rate=1e-3, initial_epsilon=1.0, final_epsilon=0.05, epsilon_decay_steps=3000, tau=1.0, target_net_update_freq=200,
          buffer_size=4096, net_arch=[256, 256, 256, 256], batch_size=32, learning_starts=200, gradient_updates=1, gamma=0.98,
          max_grad_norm=1.0, envelope=True, num_sample_w=4, per=True, per_alpha=0.6, initial_homotopy_lambda=0.0,
          final_homotopy_lambda=1.0, homotopy_decay_steps=None)
TOTAL_STEPS = 6000
SEEDS = [0, 1, 2]


def evaluate(agent, gamma, weights):
    pm = rh.import_reference("morl_baselines.common.pareto")
    env = TreasureChain(seed=123)
    returns = []
    for w in weights:
        obs, _ = env.reset()
        done, g, disc = False, 1.0, np.zeros(3)
        while not done:
            obs, r, term, trunc, _ = env.step(agent.eval(obs, w))
            disc += g * r
            g *= gamma
            done = term or trunc
        returns.append(disc)
    front = pm.filter_pareto_dominated(returns)
    return returns, front, hypervolume_exact(HV_REF_POINT, front)


def main():
    assert rh.reference_available()
    em = rh.import_reference("morl_baselines.multi_policy.envelope.envelope")
    # Envelope.train builds its (unused when log=False) evaluation-weight list with pymoo's Riesz-energy generator, which is not
    # installed; hand it the deterministic simplex grid instead (module attribute patched at run time, reference source untouched)
    em.equally_spaced_weights = lambda dim, n, seed=42: [w for w, _, _ in robust_eval_weights(HP["gamma"])]
    th.set_num_threads(min(8, os.cpu_count() or 1))
    ew = robust_eval_weights(HP["gamma"])
    weights = [w for w, _, _ in ew]
    out = {"hyper_parameters": HP, "total_timesteps": TOTAL_STEPS, "ref_point": HV_REF_POINT.tolist(),
           "eval_weights": [list(map(float, w)) for w in weights], "eval_weight_margins": [g for _, g, _ in ew],
           "env": "TreasureChain (tests/golden/standin_env.py)", "seeds": {}}
    env0 = TreasureChain()
    true_front = env0.pareto_front(HP["gamma"])
    out["true_front_hv"] = hypervolume_exact(HV_REF_POINT, true_front)
    for seed in SEEDS:
        t0 = time.time()
        th.manual_seed(seed)
        np.random.seed(seed)
        env = TreasureChain(seed=seed)
        agent = em.Envelope(env, log=False, seed=seed, device="cpu", **HP)
        agent.train(total_timesteps=TOTAL_STEPS)
        returns, front, hv = evaluate(agent, HP["gamma"], weights)
        out["seeds"][str(seed)] = {"hv": hv, "front": [list(map(float, p)) for p in front], "n_front": len(front),
                                   "returns": [list(map(float, p)) for p in returns]}
        print(f"seed {seed}: hv {hv:.4f} (true front {out['true_front_hv']:.4f}), |front| {len(front)}, {time.time() - t0:.0f} s", flush=True)
    out["hv_mean"] = float(np.mean([v["hv"] for v in out["seeds"].values()]))
    with open(os.path.join(HERE, "hv_parity.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("hv mean", out["hv_mean"])


if __name__ == "__main__":
    main()
