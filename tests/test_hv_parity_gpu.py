"""Hypervolume parity after equal updates (SURVEY.md section 8(d) "HV parity protocol"; BASELINE.json: "hypervolume within 1 % of
reference after equal updates").

The unmodified reference Envelope was trained on CPU in the build container (tests/golden/make_golden_hv.py -> hv_parity.json) on
the stand-in vector-reward MDP of tests/golden/standin_env.py (mo-gymnasium is not installed, so BOTH engines use the stand-in, as
the protocol prescribes).  Here the CUDA engine is trained with the same hyper-parameters, seeds, environment, number of
environment steps (= gradient updates) and evaluation-weight list; both fronts go through the same exact hypervolume routine.
Bar: |mean_seeds HV_b200 - mean_seeds HV_ref| / mean HV_ref <= 1 %  (3 seeds).
"""

import json
import os

import numpy as np
import pytest
import torch as th

from tests.golden.standin_env import HV_REF_POINT, TreasureChain

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _evaluate(agent, gamma, weights):
    from morl_baselines_b200.common.pareto import filter_pareto_dominated
    from morl_baselines_b200.common.performance_indicators import hypervolume

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
    front = filter_pareto_dominated(returns)
    return front, hypervolume(HV_REF_POINT, list(front))


def test_envelope_hypervolume_within_one_percent_of_reference(cuda):
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "hv_parity.json")))
    hp = gold["hyper_parameters"]
    hvs = []
    for seed_s, ref in sorted(gold["seeds"].items()):
        seed = int(seed_s)
        th.manual_seed(seed)
        np.random.seed(seed)
        env = TreasureChain(seed=seed)
        agent = Envelope(env, log=False, seed=seed, device=cuda, **hp)
        agent.train(total_timesteps=gold["total_timesteps"])
        assert agent.global_step == gold["total_timesteps"]
        front, hv = _evaluate(agent, hp["gamma"], [np.asarray(w, dtype=np.float32) for w in gold["eval_weights"]])
        hvs.append(hv)
        print(f"seed {seed}: hv b200 {hv:.4f} vs reference {ref['hv']:.4f} (true front {gold['true_front_hv']:.4f}), |front| {len(front)} vs {ref['n_front']}")
    mean_b200, mean_ref = float(np.mean(hvs)), float(gold["hv_mean"])
    rel = abs(mean_b200 - mean_ref) / mean_ref
    print(f"mean hv b200 {mean_b200:.4f}, reference {mean_ref:.4f}, relative difference {rel * 100:.3f} %")
    assert rel <= 0.01
    # sanity: neither engine can exceed the hypervolume of the true Pareto front of the deterministic MDP (returns are accumulated
    # from float32 rewards, the true front in float64: allow rounding)
    assert max(hvs) <= gold["true_front_hv"] * (1 + 1e-6)


def test_envelope_hypervolume_config2_unsaturated(cuda):
    """Same protocol at BASELINE configs[1] hyper-parameters (|W| = 32, batch 256, 4 x 256, per=True) on a budget where the REFERENCE has
    not reached the true front (tests/golden/make_golden_hv_config2.py: 400 environment steps, 300 updates, uniformly random behaviour
    policy so that both engines learn from identical replay contents) -- unlike the saturated fixture above, a moderate regression of
    the update path moves this hypervolume."""
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    path = os.path.join(ROOT, "tests", "golden", "hv_parity_config2.json")
    gold = json.load(open(path))
    hp, total = gold["hyper_parameters"], gold["total_timesteps"]
    assert gold["hv_mean"] < 0.98 * gold["true_front_hv"], "fixture must be unsaturated"
    hvs, refs = [], []
    for seed_s, rec in sorted(gold["seeds"].items()):
        seed, ref = int(seed_s), rec[str(total)]
        th.manual_seed(seed)
        np.random.seed(seed)
        env = TreasureChain(seed=seed)
        agent = Envelope(env, log=False, seed=seed, device=cuda, **hp)
        agent.train(total_timesteps=total)
        front, hv = _evaluate(agent, hp["gamma"], [np.asarray(w, dtype=np.float32) for w in gold["eval_weights"]])
        hvs.append(hv)
        refs.append(ref["hv"])
        print(f"seed {seed}: hv b200 {hv:.4f} vs reference {ref['hv']:.4f} ({100 * ref['hv'] / gold['true_front_hv']:.1f} % of the true front), "
              f"|front| {len(front)} vs {ref['n_front']}")
    rel = abs(float(np.mean(hvs)) - float(np.mean(refs))) / float(np.mean(refs))
    print(f"mean hv b200 {np.mean(hvs):.4f}, reference {np.mean(refs):.4f}, relative difference {rel * 100:.3f} %")
    assert rel <= 0.01


def test_batched_evaluation_round_equals_serial(cuda):
    """SURVEY 8(f)4: the lockstep evaluation round (one batched network call per environment step for all weights x episodes) returns
    exactly what the reference's serial loop of ``policy_eval`` calls returns (deterministic stand-in environment), and the device
    hypervolume of the resulting front equals the host routine's."""
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.evaluation import policy_evaluation_mo_batched
    from morl_baselines_b200.common.performance_indicators import hypervolume
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    th.manual_seed(1)
    np.random.seed(1)
    env = TreasureChain(seed=1)
    agent = Envelope(env, log=False, seed=1, device=cuda, net_arch=[64, 64], batch_size=32, num_sample_w=4, learning_starts=50, buffer_size=1024)
    agent.train(total_timesteps=300)
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "hv_parity.json")))
    weights = [np.asarray(w, dtype=np.float32) for w in gold["eval_weights"]]
    serial = [agent.policy_eval(TreasureChain(seed=123), weights=w, num_episodes=3) for w in weights]
    batched = policy_evaluation_mo_batched(agent, TreasureChain(seed=123), weights, rep=3)
    for s_, b_ in zip(serial, batched):
        for x, y in zip(s_, b_):
            assert np.array_equal(np.asarray(x), np.asarray(y))
    front = np.array([b[3] for b in batched], dtype=np.float64)
    pts = th.from_numpy(front).to(cuda)
    keep = ops.pareto_mask(pts, True, raw=True)
    hv_dev = float(ops.hypervolume(pts, th.from_numpy(HV_REF_POINT), keep=keep))
    from morl_baselines_b200.common.pareto import filter_pareto_dominated

    hv_host = hypervolume(HV_REF_POINT, list(filter_pareto_dominated(front)))
    assert abs(hv_dev - hv_host) <= 1e-12 * max(1.0, hv_host)
