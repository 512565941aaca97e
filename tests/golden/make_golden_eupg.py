"""Golden vectors for EUPG and its accrued-reward buffer, produced by the unmodified reference on CPU (needs the reference's source tree,
so it is run by hand, not by the tests):
    python tests/golden/make_golden_eupg.py   ->  tests/golden/eupg.npz

  update_<case> : the initial state dict, then for each of the case's fixed episodes (``eupg_standin.fixed_episode`` from a numpy seed,
                  added to the buffer and followed by ``update()`` and ``cleanup()``) the loss and the parameters after the update.
                  "box" (Box observations truncated to int32, S 3, d 2, 3 actions, [50]) has an episode of T = 1; "wrap" (Discrete
                  observations, d 3, 4 actions, [17, 5], max_size 16) has episodes longer than the ring; "a1" has one action, where every
                  gradient is zero.
  train_<case>  : a seeded ``train()`` (``th.manual_seed``) with ``eupg_standin.RecordingScalarization``: every sampled action, the final
                  parameters and every call the scalarisation received, in order.
  buffer        : an int32-observation buffer's arrays after adds that wrap, a ``sample(use_cer=True)`` under ``np.random.seed`` and
                  ``cleanup``.
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
from tests.eupg_standin import EupgEnv, RecordingScalarization, fixed_episode, pack_calls, weighted_sum_scalarization  # noqa: E402

UPDATE_CASES = {
    "box": dict(env=dict(obs_dim=3, n_actions=3, reward_dim=2), ctor=dict(net_arch=[50], gamma=0.99, learning_rate=1e-3),
                weights=[0.7, 0.3], lengths=[23, 1, 40, 9], seed=3),
    "wrap": dict(env=dict(n_actions=4, reward_dim=3, discrete_obs=6), ctor=dict(net_arch=[17, 5], gamma=0.9, learning_rate=3e-3,
                                                                                  buffer_size=16),
                 weights=[0.5, 0.2, 0.3], lengths=[12, 37, 16, 20], seed=4),
    "a1": dict(env=dict(obs_dim=2, n_actions=1, reward_dim=2), ctor=dict(net_arch=[8], gamma=0.95, learning_rate=1e-2),
               weights=[1.0, 1.0], lengths=[6, 11], seed=5),
}

TRAIN_CASES = {
    "box": dict(env=dict(obs_dim=3, n_actions=3, reward_dim=2, seed=41), ctor=dict(net_arch=[50], gamma=0.99, learning_rate=1e-2),
                weights=[0.6, 0.4], steps=400, seed=7),
    "disc": dict(env=dict(n_actions=2, reward_dim=2, discrete_obs=5, seed=42), ctor=dict(net_arch=[50], gamma=0.99, learning_rate=1e-2),
                 weights=[1.0, 1.0], steps=300, seed=8),
}


def params(net) -> dict:
    return {k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}


def put(out: dict, prefix: str, d: dict):
    for k, v in d.items():
        out[f"{prefix}/{k}"] = np.asarray(v)


def reference_loss(agent) -> np.ndarray:
    """The loss the reference's next ``update()`` computes (eupg.py:228-247), evaluated with its own code before the update runs."""
    obs, acc, actions, rewards, _, _ = agent.buffer.get_all_data(to_tensor=True, device="cpu")
    with th.no_grad():
        v = agent.scalarization(agent._forward_cumulative_rewards(rewards))
        lp = agent.net.distribution(obs, acc).log_prob(actions.squeeze())
        return (-th.mean(lp * v)).numpy().astype(np.float32)


def update_cases(out: dict):
    eupg = rh.import_reference("morl_baselines.single_policy.esr.eupg")
    for name, c in UPDATE_CASES.items():
        env = EupgEnv(**c["env"], seed=c["seed"])
        th.manual_seed(c["seed"])
        agent = eupg.EUPG(env, weighted_sum_scalarization(c["weights"]), weights=np.array(c["weights"]), log=False, device="cpu", **c["ctor"])
        put(out, f"update_{name}/init", params(agent.net))
        losses = []
        for k, T in enumerate(c["lengths"]):
            for tr in fixed_episode(env, np.random.default_rng(1000 * c["seed"] + k), T):
                agent.buffer.add(*tr)
            losses.append(reference_loss(agent))
            agent.update()
            agent.buffer.cleanup()
            put(out, f"update_{name}/after{k}", params(agent.net))
        out[f"update_{name}/loss"] = np.array(losses, np.float32)


def train_cases(out: dict):
    eupg = rh.import_reference("morl_baselines.single_policy.esr.eupg")
    for name, c in TRAIN_CASES.items():
        env = EupgEnv(**c["env"])
        scal = RecordingScalarization(env.reward_dim)
        th.manual_seed(c["seed"])
        agent = eupg.EUPG(env, scal, weights=np.array(c["weights"]), log=False, device="cpu", **c["ctor"])
        put(out, f"train_{name}/init", params(agent.net))
        actions = []
        step = env.step

        def recording(a, step=step, actions=actions):
            actions.append(a)
            return step(a)

        env.step = recording
        agent.train(total_timesteps=c["steps"])
        put(out, f"train_{name}/final", params(agent.net))
        out[f"train_{name}/actions"] = np.array(actions, np.int64)
        kinds, rets, ws, fwd, lens = pack_calls(scal.calls)
        out[f"train_{name}/call_kinds"] = kinds
        out[f"train_{name}/call_returns"] = rets
        out[f"train_{name}/call_weights"] = ws
        out[f"train_{name}/call_forward"] = fwd
        out[f"train_{name}/call_forward_len"] = lens
        out[f"train_{name}/num_episodes"] = np.array(agent.num_episodes)


def buffer_case(out: dict):
    mod = rh.import_reference("morl_baselines.common.accrued_reward_buffer")
    buf = mod.AccruedRewardReplayBuffer((3,), (1,), rew_dim=2, max_size=5, obs_dtype=np.int32, action_dtype=np.int32)
    rng = np.random.default_rng(12)
    for i in range(8):
        obs = rng.uniform(-4, 4, 3)
        buf.add(obs, rng.standard_normal(2).astype(np.float32), i % 3, rng.standard_normal(2), obs + 0.5, i == 7)
    for k in ("obs", "next_obs", "actions", "rewards", "accrued_rewards", "dones"):
        out[f"buffer/{k}"] = getattr(buf, k).copy()
    out["buffer/ptr_size"] = np.array([buf.ptr, buf.size])
    np.random.seed(5)
    for k, v in zip(("obs", "accrued_rewards", "actions", "rewards", "next_obs", "dones"), buf.sample(4, use_cer=True)):
        out[f"buffer/sample_{k}"] = v
    buf.cleanup()
    out["buffer/after_cleanup"] = np.array([buf.ptr, buf.size, len(buf)])


def main():
    th.set_num_threads(1)
    out: dict = {}
    update_cases(out)
    train_cases(out)
    buffer_case(out)
    path = os.path.join(HERE, "eupg.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
