"""Synthetic inputs and an environment shell shared by bench.py, __graft_entry__.smoke(), the tests and the golden-vector generators.

Nothing here is on the update path: ``FakeEnv`` only carries the spaces ``MOAgent.extract_env_info`` reads (reference
``morl_baselines/common/morl_algorithm.py:248-273``) plus a deterministic random-walk MDP so ``train()`` loops can be driven without
mo-gymnasium (not installed in this image), and ``synthetic_store`` is the synthetic replay content of BASELINE.md section 3 / SURVEY.md 8(d).
"""

from __future__ import annotations

import numpy as np


# ----------------------------------------------------------------------------------------------
# gymnasium.spaces stand-ins (only .n / .shape / .low / .high / .sample are read by the reference)
# ----------------------------------------------------------------------------------------------
class _Space:
    def __init__(self):
        self._rng = np.random.default_rng(0)

    def seed(self, seed=None):
        self._rng = np.random.default_rng(seed)


class Discrete(_Space):
    def __init__(self, n):
        super().__init__()
        self.n = int(n)
        self.shape = ()

    def sample(self):
        return int(self._rng.integers(self.n))


class MultiBinary(_Space):
    def __init__(self, n):
        super().__init__()
        self.n = int(n)
        self.shape = (self.n,)

    def sample(self):
        return self._rng.integers(0, 2, size=self.n)


class MultiDiscrete(_Space):
    def __init__(self, nvec):
        super().__init__()
        self.nvec = np.asarray(nvec, dtype=np.int64)
        self.shape = self.nvec.shape

    def sample(self):
        return self._rng.integers(0, self.nvec)


class Box(_Space):
    def __init__(self, low=-1.0, high=1.0, shape=None, dtype=np.float32):
        super().__init__()
        if shape is None:
            shape = np.shape(low)
        self.shape = tuple(shape)
        self.low = np.broadcast_to(np.asarray(low, dtype=dtype), self.shape).copy()
        self.high = np.broadcast_to(np.asarray(high, dtype=dtype), self.shape).copy()
        self.dtype = dtype

    def is_bounded(self, manner="both"):
        below, above = bool(np.all(np.isfinite(self.low))), bool(np.all(np.isfinite(self.high)))
        return {"both": below and above, "below": below, "above": above}[manner]

    def sample(self):
        if not (np.all(np.isfinite(self.low)) and np.all(np.isfinite(self.high))):
            return self._rng.standard_normal(self.shape).astype(self.dtype)  # unbounded box: gymnasium samples a normal as well
        return self._rng.uniform(self.low, self.high).astype(self.dtype)


class _Spec:
    def __init__(self, id):
        self.id = id


class FakeEnv:
    """Vector-reward environment shell: spaces + a deterministic random-walk MDP.

    The dynamics are not part of any parity claim; they exist so ``train()`` loops of both engines
    can be driven by the same host-side rollout (SURVEY.md section 8(d) "stand-in MOMDP").
    """

    def __init__(self, obs_dim=32, n_actions=8, reward_dim=3, continuous_action_dim=None, seed=0, horizon=50):
        self.observation_space = Box(-np.inf, np.inf, shape=(obs_dim,))
        if continuous_action_dim is None:
            self.action_space = Discrete(n_actions)
        else:
            self.action_space = Box(-1.0, 1.0, shape=(continuous_action_dim,))
        self.reward_space = Box(-np.inf, np.inf, shape=(reward_dim,))
        self.reward_dim = reward_dim
        self.unwrapped = self
        self.spec = _Spec("fake-momdp-v0")
        self.metadata = {"render_modes": []}
        self._rng = np.random.default_rng(seed)
        self._obs_dim = obs_dim
        self._horizon = horizon
        self._t = 0
        self._state = np.zeros(obs_dim, dtype=np.float32)
        n_act_feat = n_actions if continuous_action_dim is None else continuous_action_dim
        gen = np.random.default_rng(1234)
        self._A = (gen.standard_normal((n_act_feat, obs_dim)) * 0.3).astype(np.float32)
        self._R = (gen.standard_normal((reward_dim, obs_dim)) / np.sqrt(obs_dim)).astype(np.float32)
        self._continuous = continuous_action_dim is not None

    def reset(self, seed=None, options=None):
        if seed is not None:
            self._rng = np.random.default_rng(seed)
        self._t = 0
        self._state = self._rng.standard_normal(self._obs_dim).astype(np.float32)
        return self._state.copy(), {}

    def step(self, action):
        if self._continuous:
            drive = np.asarray(action, dtype=np.float32) @ self._A
        else:
            drive = self._A[int(action)]
        self._state = (0.9 * self._state + drive).astype(np.float32)
        reward = (self._R @ self._state).astype(np.float32)
        self._t += 1
        terminated = False
        truncated = self._t >= self._horizon
        return self._state.copy(), reward, terminated, truncated, {}


def synthetic_store(n, obs_dim=32, n_actions=8, rew_dim=3, seed=0):
    """The synthetic replay contents of BASELINE.md section 3 / SURVEY.md 8(d) (numpy PCG64: bit-reproducible everywhere)."""
    rng = np.random.default_rng(seed)
    return dict(
        obs=rng.standard_normal((n, obs_dim)).astype(np.float32),
        next_obs=rng.standard_normal((n, obs_dim)).astype(np.float32),
        actions=rng.integers(0, n_actions, size=(n, 1)).astype(np.uint8),
        rewards=rng.standard_normal((n, rew_dim)).astype(np.float32),
        dones=(rng.random((n, 1)) < 0.02).astype(np.float32),
    )
