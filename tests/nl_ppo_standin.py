"""A small discrete-action multi-objective environment for NLMOPPO's tests: a point on a ring of ``n_pos`` cells with a heading, an
observation of ``obs_dim`` features, ``n_actions`` moves and ``d`` reward components, episodes of at most ``horizon`` steps.  Seeded by
``reset(seed=...)`` only, so a run replays exactly."""

from __future__ import annotations

from types import SimpleNamespace

import numpy as np


def _box(n):
    return SimpleNamespace(shape=(n,), dtype=np.float32)


class RingEnv:
    """Single environment: reset(seed) -> (obs [S], info); step(a) -> (obs, reward [d], terminated, truncated, info)."""

    def __init__(self, obs_dim=2, n_actions=4, d=2, horizon=12, n_pos=7):
        self.obs_dim, self.n_actions, self.d, self.horizon, self.n_pos = obs_dim, n_actions, d, horizon, n_pos
        self.observation_space, self.reward_space = _box(obs_dim), _box(d)
        self.action_space = SimpleNamespace(n=n_actions, shape=())
        self._rng = np.random.default_rng(0)
        self._table = None

    def _obs(self):
        k = np.arange(self.obs_dim)
        return np.cos(2 * np.pi * (self.pos + 1) * (k + 1) / self.n_pos + 0.3 * self.t).astype(np.float32)

    def reset(self, seed=None):
        if seed is not None:
            self._rng = np.random.default_rng(seed)
            tr = np.random.default_rng(1234)
            self._table = tr.standard_normal((self.n_pos, self.n_actions, self.d)).astype(np.float64)
        self.pos, self.t = int(self._rng.integers(self.n_pos)), 0
        return self._obs(), {}

    def step(self, a):
        a = int(a)
        r = self._table[self.pos, a] * 0.5
        self.pos = (self.pos + a - self.n_actions // 2) % self.n_pos
        self.t += 1
        terminated = bool(self.pos == 0 and a == 0)
        truncated = self.t >= self.horizon
        return self._obs(), r, terminated, truncated, {}


class RingVecEnv:
    """``num_envs`` RingEnvs stepped in lockstep with autoreset in the same step (the returned observation of a finished env is its
    reset observation), exposing the attributes NLMOPPO reads."""

    def __init__(self, num_envs=8, **kw):
        self.envs = [RingEnv(**kw) for _ in range(num_envs)]
        self.num_envs = num_envs
        e = self.envs[0]
        self.single_observation_space, self.single_action_space, self.reward_space = e.observation_space, e.action_space, e.reward_space

    def reset(self, seed=None):
        obs = [env.reset(seed=None if seed is None else seed + i)[0] for i, env in enumerate(self.envs)]
        return np.stack(obs), {}

    def step(self, actions):
        out = [env.step(a) for env, a in zip(self.envs, np.asarray(actions).reshape(-1))]
        obs, rew, term, trunc = [], [], [], []
        for env, (o, r, te, tr, _) in zip(self.envs, out):
            if te or tr:
                o = env.reset()[0]
            obs.append(o), rew.append(r), term.append(te), trunc.append(tr)
        return np.stack(obs), np.stack(rew), np.array(term), np.array(trunc), {}


# ---- the golden cases of tests/golden/nl_mo_ppo.npz (shared by the generator and the tests) --------------------------------------------
def u_linear(v):
    """Linear utility with weights 1..d, normalised."""
    import torch as th

    w = th.arange(1, v.shape[-1] + 1, dtype=v.dtype, device=v.device)
    return (v * w / w.sum()).sum()


def u_cheb(v):
    """Smooth Chebyshev-like utility: a soft minimum of v - (-1)."""
    import torch as th

    return -th.logsumexp(-8.0 * (v + 1.0), 0) / 8.0


UTILITIES = {"linear": u_linear, "cheb": u_cheb}

# ctor: NLMOPPO keyword arguments; env: RingVecEnv arguments; pref: None or a list; u: a key of UTILITIES
UPDATE_CASES = {
    "d2_lin": dict(E=4, T=16, env=dict(obs_dim=2, n_actions=4, d=2), pref=None, u="linear", seed=3,
                   ctor=dict(num_minibatches=4, update_epochs=2, norm_adv=True, clip_vloss=True, ent_coef=0.01, target_kl=None)),
    "d3_pref_cheb": dict(E=4, T=16, env=dict(obs_dim=3, n_actions=5, d=3), pref=[0.2, 0.5, 0.3], u="cheb", seed=4,
                         ctor=dict(num_minibatches=3, update_epochs=2, norm_adv=False, clip_vloss=False, ent_coef=0.0, target_kl=None)),
    "d2_pref_kl": dict(E=4, T=16, env=dict(obs_dim=2, n_actions=4, d=2), pref=[0.6, 0.4], u="cheb", seed=5,
                       ctor=dict(num_minibatches=4, update_epochs=4, norm_adv=True, clip_vloss=True, ent_coef=0.01, target_kl=1e-3)),
    "a40_fallback": dict(E=2, T=16, env=dict(obs_dim=2, n_actions=40, d=2), pref=None, u="linear", seed=6,
                         ctor=dict(num_minibatches=2, update_epochs=2, norm_adv=True, clip_vloss=True, ent_coef=0.01, target_kl=None)),
}

TRAIN_CASES = {
    "lin": dict(E=4, T=16, env=dict(obs_dim=2, n_actions=4, d=2), pref=None, u="linear", seed=7,
                ctor=dict(num_minibatches=4, update_epochs=2, anneal_lr=False, total_timesteps=3 * 64)),
    "anneal": dict(E=4, T=16, env=dict(obs_dim=3, n_actions=4, d=3), pref=[0.3, 0.3, 0.4], u="cheb", seed=8,
                   ctor=dict(num_minibatches=4, update_epochs=2, anneal_lr=True, total_timesteps=3 * 64)),
}


def action_table(seed: int, n_calls: int, E: int, A: int) -> np.ndarray:
    """The actions ``Categorical.sample`` returns in a replayable train() run: call k gets row k."""
    return np.random.default_rng(1000 + seed).integers(0, A, (n_calls, E))


class FixedSampling:
    """Context manager patching ``torch.distributions.Categorical.sample`` to return the rows of ``table`` in order (on the device of the
    distribution's logits), so a train() run replays whatever the sampled distributions are."""

    def __init__(self, table: np.ndarray):
        self.table, self.k = table, 0

    def __enter__(self):
        import torch as th
        from torch.distributions import Categorical

        self._orig = Categorical.sample
        fs = self

        def sample(dist, sample_shape=()):
            row = fs.table[fs.k]
            fs.k += 1
            return th.as_tensor(row[: dist.logits.shape[0]] if dist.logits.dim() > 1 else row[0], dtype=th.long, device=dist.logits.device)

        Categorical.sample = sample
        return self

    def __exit__(self, *exc):
        from torch.distributions import Categorical

        Categorical.sample = self._orig


class single_thread:
    """Context manager running torch's CPU ops on one thread: the QR of ``orthogonal_`` rounds differently with more threads, and the
    golden file was made with one."""

    def __enter__(self):
        import torch as th

        self.n = th.get_num_threads()
        th.set_num_threads(1)

    def __exit__(self, *exc):
        import torch as th

        th.set_num_threads(self.n)
