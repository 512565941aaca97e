"""Stand-ins for the EUPG tests: a Box-observation environment whose observations are not integers (the learner stores them in an int32
buffer, so they are truncated), a Discrete-observation one (observations are python ints), a stateful scalarisation that records every
call, and fixed episodes.  Shared by tests/golden/make_golden_eupg.py (which runs the reference on them) and the tests."""

from __future__ import annotations

import numpy as np
import torch as th

from oracle.ref_harness import Box, Discrete, _Spec


class EupgEnv:
    """A smooth random MDP with ``n_actions`` actions and episodes of uniform length in [min_len, max_len].  With ``discrete_obs`` the
    observation is a python int in [0, n_states); otherwise a float32 vector of ``obs_dim`` values in (-3, 3)."""

    def __init__(self, obs_dim: int = 3, n_actions: int = 3, reward_dim: int = 2, discrete_obs: int = 0, min_len: int = 5, max_len: int = 40,
                 seed: int = 0):
        self.discrete_obs = discrete_obs
        self.observation_space = Discrete(discrete_obs) if discrete_obs else Box(-3.0, 3.0, shape=(obs_dim,))
        self.action_space = Discrete(n_actions)
        self.reward_space = Box(-np.inf, np.inf, shape=(reward_dim,))
        self.reward_dim = reward_dim
        self.unwrapped = self
        self.spec = _Spec("eupg-standin-v0")
        self.metadata = {"render_modes": []}
        self._rng = np.random.default_rng(seed)
        self._min, self._max = min_len, max_len
        gen = np.random.default_rng(97)
        self._dim = 2 if discrete_obs else obs_dim
        self._A = (gen.standard_normal((n_actions, self._dim)) * 0.9).astype(np.float32)
        self._R = gen.standard_normal((reward_dim, self._dim)).astype(np.float32)

    def _obs(self):
        if self.discrete_obs:
            return int(np.floor((self._state[0] + 1.0) * 0.5 * self.discrete_obs)) % self.discrete_obs
        return (3.0 * self._state).astype(np.float32)

    def reset(self, seed=None, options=None):
        if seed is not None:
            self._rng = np.random.default_rng(seed)
        self._t = 0
        self._len = int(self._rng.integers(self._min, self._max + 1))
        self._state = (self._rng.standard_normal(self._dim) * 0.5).astype(np.float32)
        return self._obs(), {}

    def step(self, action):
        self._state = np.tanh(0.8 * self._state + self._A[int(action)]).astype(np.float32)
        reward = (self._R @ self._state + 0.5).astype(np.float32)
        self._t += 1
        return self._obs(), reward, self._t >= self._len, False, {}

    def close(self):
        pass


class RecordingScalarization:
    """Stateful Tchebicheff-like utility that records its calls.  With (return, weights) it is called on an episodic return (numpy):
    the utopian point z tracks max(r + tau) and it returns -max_i w_i |r_i - z_i|.  With one argument it is called on the discounted
    forward returns [T, d] (a tensor) and returns -max_i |c_ti - z_i| per row, a [T] tensor on the same device."""

    def __init__(self, reward_dim: int, tau: float = 0.1):
        self.utopia = np.full(reward_dim, -np.inf)
        self.tau = tau
        self.calls = []  # ("ret", r, w) or ("fwd", c)

    def __call__(self, reward, weights=None):
        if isinstance(reward, th.Tensor):
            self.calls.append(("fwd", reward.detach().cpu().numpy().copy()))
            z = th.as_tensor(self.utopia, dtype=reward.dtype, device=reward.device)
            return -th.max(th.abs(reward - z), dim=1).values
        r = np.asarray(reward, dtype=np.float64)
        self.calls.append(("ret", np.asarray(reward).copy(), np.asarray(weights, dtype=np.float64).copy()))
        np.maximum(self.utopia, r + self.tau, out=self.utopia)
        return -float(np.max(np.abs(r - self.utopia) * np.asarray(weights, dtype=np.float64)))


def pack_calls(calls):
    """(kinds int8 [n], returns [n_ret, d], weights [n_ret, d], forward returns concatenated [sum T, d], their lengths [n_fwd])."""
    kinds = np.array([0 if c[0] == "ret" else 1 for c in calls], np.int8)
    rets = np.array([c[1] for c in calls if c[0] == "ret"], np.float64)
    ws = np.array([c[2] for c in calls if c[0] == "ret"], np.float64)
    fwd = [c[1] for c in calls if c[0] == "fwd"]
    return kinds, rets, ws, np.concatenate(fwd).astype(np.float32), np.array([len(f) for f in fwd], np.int64)


def weighted_sum_scalarization(weights):
    """Stateless linear utility for the update cases: ``w . r`` on numpy returns, ``c @ w`` (float32, same device) on forward returns."""
    w64 = np.asarray(weights, dtype=np.float64)

    def scalarize(reward, w=None):
        if isinstance(reward, th.Tensor):
            return reward @ th.as_tensor(w64, dtype=reward.dtype, device=reward.device)
        return float(np.dot(reward, w64))

    return scalarize


def fixed_episode(env: EupgEnv, rng: np.random.Generator, length: int):
    """One episode of ``length`` steps with actions from ``rng``: the (obs, accrued reward, action, reward, next_obs, terminated) tuples in
    the order the learner adds them; the accrued reward follows the reference's in-place float32 rule."""
    obs, _ = env.reset()
    acc = th.zeros(env.reward_dim, dtype=th.float32)
    out = []
    for t in range(length):
        a = int(rng.integers(env.action_space.n))
        n_obs, r, _, _, _ = env.step(a)
        o = [obs] if type(obs) is int else obs
        out.append((o, acc.numpy().copy(), a, r, n_obs, t == length - 1))
        acc += th.from_numpy(r)
        obs = n_obs
    return out
