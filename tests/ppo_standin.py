"""A synchronous vector env over ``testing.FakeEnv`` with continuous actions: the stand-in for mo-gymnasium's MOSyncVectorEnv that the
MO-PPO and PGMORL tests drive (same reset / step / num_envs surface, episodes restarted on termination or truncation)."""

from __future__ import annotations

import numpy as np

from morl_baselines_b200.testing import FakeEnv


class FakeVecEnv:
    def __init__(self, envs):
        self.envs = list(envs)
        self.num_envs = len(self.envs)
        self.observation_space = self.envs[0].observation_space
        self.action_space = self.envs[0].action_space
        self.reward_space = self.envs[0].reward_space
        self.unwrapped = self

    def reset(self, seed=None, options=None):
        obs = [e.reset(seed=None if seed is None else seed + i)[0] for i, e in enumerate(self.envs)]
        return np.stack(obs), {}

    def step(self, actions):
        obs, rew, term, trunc = [], [], [], []
        for e, a in zip(self.envs, actions):
            o, r, te, tr, _ = e.step(a)
            if te or tr:
                o, _ = e.reset()
            obs.append(o)
            rew.append(r)
            term.append(te)
            trunc.append(tr)
        return np.stack(obs), np.stack(rew).astype(np.float64), np.array(term), np.array(trunc), {}

    def close(self):
        pass


def fake_env(obs_dim=11, act_dim=3, reward_dim=2, seed=0, horizon=20):
    return FakeEnv(obs_dim=obs_dim, reward_dim=reward_dim, continuous_action_dim=act_dim, seed=seed, horizon=horizon)


def fake_vec_env(num_envs=2, **kw):
    return FakeVecEnv([fake_env(seed=i, **kw) for i in range(num_envs)])
