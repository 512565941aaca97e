"""Golden vectors for NLMOPPO, produced by the unmodified reference on CPU (needs the reference's source tree, so it is run by hand, not
by the tests):
    python tests/golden/make_golden_nl_mo_ppo.py   ->  tests/golden/nl_mo_ppo.npz

The cases are ``UPDATE_CASES`` and ``TRAIN_CASES`` of tests/nl_ppo_standin.py, on its ring environment.

  update_<case> : a seeded learner (``th.manual_seed(seed)`` before construction) whose rollout storage is filled with a synthetic batch
                  from ``np.random.default_rng(100 + seed)``: obs, accrued rewards, actions, rewards, values, dones, the carried next
                  obs / accrued reward / done, and old log-probabilities equal to the current ones plus noise (zero noise on every fifth
                  row, so those ratios are exactly 1).  Recorded: the initial parameters, the inputs, the bootstrap value, the
                  per-objective advantages and returns of ``_compute_advantages_and_returns``, the loss weights, the parameters after the
                  first minibatch step and after ``update()``, the number of shuffles drawn and the returned statistics.
  train_<case>  : a seeded ``train(eval_env, u, pref, deterministic=True)`` with ``Categorical.sample`` returning the rows of
                  ``action_table``: every storage tensor of the last iteration, the final parameters and the evaluation result.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402
from tests.nl_ppo_standin import TRAIN_CASES, UPDATE_CASES, UTILITIES, FixedSampling, RingEnv, RingVecEnv, action_table  # noqa: E402

STORAGE = ("obs", "acc_rewards", "actions", "logprobs", "rewards", "dones", "values", "advantages", "returns")


def params(net) -> dict:
    return {k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}


def put(out: dict, prefix: str, d: dict):
    for k, v in d.items():
        out[f"{prefix}/{k}"] = np.asarray(v)


class CountingRng:
    """The learner's generator, counting the shuffles drawn from it."""

    def __init__(self, rng):
        self.rng, self.shuffles = rng, 0

    def shuffle(self, x):
        self.shuffles += 1
        self.rng.shuffle(x)


def synthetic_batch(c):
    T, E, (S, A, d) = c["T"], c["E"], (c["env"]["obs_dim"], c["env"]["n_actions"], c["env"]["d"])
    rng = np.random.default_rng(100 + c["seed"])
    f = lambda *s: rng.standard_normal(s).astype(np.float32)  # noqa: E731
    b = dict(obs=f(T, E, S), acc_rewards=f(T, E, d), actions=rng.integers(0, A, (T, E)), rewards=f(T, E, d), values=f(T, E, d),
             dones=(rng.random((T, E)) < 0.15).astype(np.float32), next_obs=f(E, S), next_acc=f(E, d),
             next_done=(rng.random(E) < 0.3).astype(np.float32))
    noise = 0.3 * f(T * E)
    noise[::5] = 0.0
    return b, noise


def update_cases(out: dict):
    nl = rh.import_reference("morl_baselines.single_policy.ser.nl_mo_ppo")
    for name, c in UPDATE_CASES.items():
        th.manual_seed(c["seed"])
        agent = nl.NLMOPPO(0, RingVecEnv(c["E"], **c["env"]), num_steps=c["T"], device="cpu", seed=c["seed"], **c["ctor"])
        pre = f"update_{name}"
        put(out, f"{pre}/init", params(agent.agent))
        b, noise = synthetic_batch(c)
        for k in ("obs", "acc_rewards", "rewards", "values", "dones"):
            getattr(agent, k).copy_(th.from_numpy(b[k]))
        agent.actions.copy_(th.from_numpy(b["actions"]))
        agent.pref = None if c["pref"] is None else th.tensor(c["pref"], dtype=th.float32)
        agent.u_func = UTILITIES[c["u"]]
        T, E, S, d = c["T"], c["E"], c["env"]["obs_dim"], c["env"]["d"]
        with th.no_grad():
            _, lp, _, _ = agent.agent.get_action_and_value(agent.obs.reshape(-1, S), agent.acc_rewards.reshape(-1, d), action=agent.actions.reshape(-1),
                                                           pref=agent.pref)
        agent.logprobs.copy_((lp + th.from_numpy(noise)).reshape(T, E))
        b["logprobs"] = agent.logprobs.numpy().copy()
        nobs, nacc, ndone = (th.from_numpy(b[k]) for k in ("next_obs", "next_acc", "next_done"))
        with th.no_grad():
            b["next_value"] = agent.agent.get_value(nobs, nacc, agent.pref).numpy()
        agent.advantages, agent.returns = agent._compute_advantages_and_returns(nobs, nacc, ndone)
        b["advantages"], b["returns"] = agent.advantages.numpy().copy(), agent.returns.numpy().copy()
        put(out, f"{pre}/in", b)
        out[f"{pre}/loss_weights"] = agent._compute_loss_weights().numpy()
        first = {}
        step = agent.optimizer.step

        def first_step(*a, step=step, first=first, agent=agent, **k):
            r = step(*a, **k)
            if not first:
                first.update(params(agent.agent))
            return r

        agent.optimizer.step = first_step
        agent.rng = CountingRng(agent.rng)
        stats = agent.update()
        put(out, f"{pre}/first", first)
        put(out, f"{pre}/after", params(agent.agent))
        out[f"{pre}/shuffles"] = np.array(agent.rng.shuffles)
        out[f"{pre}/stats"] = np.array([float(s.detach()) if isinstance(s, th.Tensor) else float(s) for s in stats], np.float64)  # v, pg, entropy, old_approx_kl, approx_kl, clipfrac


def train_cases(out: dict):
    nl = rh.import_reference("morl_baselines.single_policy.ser.nl_mo_ppo")
    for name, c in TRAIN_CASES.items():
        th.manual_seed(c["seed"])
        agent = nl.NLMOPPO(0, RingVecEnv(c["E"], **c["env"]), num_steps=c["T"], device="cpu", seed=c["seed"], **c["ctor"])
        pre = f"train_{name}"
        put(out, f"{pre}/init", params(agent.agent))
        table = action_table(c["seed"], agent.num_iterations * c["T"], c["E"], c["env"]["n_actions"])
        with FixedSampling(table) as fs:
            res = agent.train(RingEnv(**c["env"]), UTILITIES[c["u"]], c["pref"], deterministic=True)
        assert fs.k == len(table)
        put(out, f"{pre}/final", params(agent.agent))
        put(out, f"{pre}/last", {k: getattr(agent, k).detach().numpy().copy() for k in STORAGE})
        out[f"{pre}/eval"] = np.asarray(res, np.float64)


def main():
    th.set_num_threads(1)
    out: dict = {}
    update_cases(out)
    train_cases(out)
    path = os.path.join(HERE, "nl_mo_ppo.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
