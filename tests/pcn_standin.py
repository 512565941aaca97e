"""Stand-in environment for the PCN / LCN tests: episodes end at varying lengths (a length drawn at every reset), so the episode store
holds variable-length episodes and the minibatch draws depend on them.  Shared by tests/golden/make_golden_pcn.py (which runs the
reference on it) and the tests (which run this package on it)."""

from __future__ import annotations

import numpy as np

from oracle.ref_harness import Box, Discrete, _Spec


class VarLengthEnv:
    """A smooth random MDP: state <- tanh(0.8 state + drive(action)), reward = R state + 1 (float32), length uniform in [min_len, max_len]."""

    def __init__(self, obs_dim: int = 4, n_actions: int = 3, reward_dim: int = 2, continuous_action_dim=None, min_len: int = 2,
                 max_len: int = 12, seed: int = 0):
        self.observation_space = Box(-1.0, 1.0, shape=(obs_dim,))
        if continuous_action_dim is None:
            self.action_space = Discrete(n_actions)
        else:
            self.action_space = Box(-1.0, 1.0, shape=(continuous_action_dim,))
        self.action_space.seed(seed + 1)
        self.reward_space = Box(-np.inf, np.inf, shape=(reward_dim,))
        self.reward_dim = reward_dim
        self.unwrapped = self
        self.spec = _Spec("var-length-v0")
        self.metadata = {"render_modes": []}
        self._continuous = continuous_action_dim is not None
        self._rng = np.random.default_rng(seed)
        self._min, self._max = min_len, max_len
        gen = np.random.default_rng(4321)
        n_feat = continuous_action_dim if self._continuous else n_actions
        self._A = (gen.standard_normal((n_feat, obs_dim)) * 0.8).astype(np.float32)
        self._R = gen.standard_normal((reward_dim, obs_dim)).astype(np.float32)
        self._obs_dim = obs_dim

    def reset(self, seed=None, options=None):
        if seed is not None:
            self._rng = np.random.default_rng(seed)
        self._t = 0
        self._len = int(self._rng.integers(self._min, self._max + 1))
        self._state = (self._rng.standard_normal(self._obs_dim) * 0.5).astype(np.float32)
        return self._state.copy(), {}

    def step(self, action):
        drive = np.asarray(action, dtype=np.float32) @ self._A if self._continuous else self._A[int(action)]
        self._state = np.tanh(0.8 * self._state + drive).astype(np.float32)
        reward = (self._R @ self._state + 1.0).astype(np.float32)
        self._t += 1
        return self._state.copy(), reward, self._t >= self._len, False, {}

    def close(self):
        pass


def random_episode(env, rng: np.random.Generator):
    """One episode of uniformly random actions drawn from ``rng``: (obs [L, S], actions, rewards [L, d]) as float32 / int arrays."""
    obs, _ = env.reset()
    o, a, r = [], [], []
    done = False
    while not done:
        act = rng.uniform(-1, 1, env.action_space.shape).astype(np.float32) if env._continuous else int(rng.integers(env.action_space.n))
        n_obs, rew, term, trunc, _ = env.step(act)
        o.append(obs)
        a.append(act)
        r.append(np.float32(rew).copy())
        obs, done = n_obs, term or trunc
    return o, a, r
