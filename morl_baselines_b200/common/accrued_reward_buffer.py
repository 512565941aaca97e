"""Replay buffer with the accrued reward of every step, for ESR learners -- drop-in for reference
morl_baselines/common/accrued_reward_buffer.py.

Plain numpy with the reference's semantics: a ring of ``max_size`` rows, typed arrays that cast what is assigned into them (a float
observation stored in an ``int32`` buffer is truncated toward zero), ``sample`` drawing from the global ``np.random`` state.  It holds no
device memory, so it pickles as the reference's does (``get_save_dict(save_replay_buffer=True)`` stores it).  ``EUPG`` stages its rows
``[0, size)`` to the device itself, in one copy per episode.
"""

from __future__ import annotations

import numpy as np
import torch as th


class AccruedRewardReplayBuffer:
    """Ring of transitions that also keeps, for each step, the reward accrued before it."""

    def __init__(self, obs_shape, action_shape, rew_dim=1, max_size=100000, obs_dtype=np.float32, action_dtype=np.float32):
        """Ring of ``max_size`` transitions: obs / next_obs ``obs_dtype``, actions ``action_dtype``, rewards, accrued rewards and dones
        float32."""
        self.max_size = max_size
        self.ptr, self.size = 0, 0
        self.obs = np.zeros((max_size,) + obs_shape, dtype=obs_dtype)
        self.next_obs = np.zeros((max_size,) + obs_shape, dtype=obs_dtype)
        self.actions = np.zeros((max_size,) + action_shape, dtype=action_dtype)
        self.rewards = np.zeros((max_size, rew_dim), dtype=np.float32)
        self.accrued_rewards = np.zeros((max_size, rew_dim), dtype=np.float32)
        self.dones = np.zeros((max_size, 1), dtype=np.float32)

    def add(self, obs, accrued_reward, action, reward, next_obs, done):
        """Store one transition at ``ptr`` and advance the ring."""
        self.obs[self.ptr] = np.array(obs).copy()
        self.next_obs[self.ptr] = np.array(next_obs).copy()
        self.actions[self.ptr] = np.array(action).copy()
        self.rewards[self.ptr] = np.array(reward).copy()
        self.accrued_rewards[self.ptr] = np.array(accrued_reward).copy()
        self.dones[self.ptr] = np.array(done).copy()
        self.ptr = (self.ptr + 1) % self.max_size
        self.size = min(self.size + 1, self.max_size)

    def _rows(self, inds, to_tensor, device):
        out = (self.obs[inds], self.accrued_rewards[inds], self.actions[inds], self.rewards[inds], self.next_obs[inds], self.dones[inds])
        if to_tensor:
            return tuple(th.tensor(x).to(device) for x in out)
        return out

    def sample(self, batch_size, replace=True, use_cer=False, to_tensor=False, device=None):
        """``batch_size`` rows drawn with the global ``np.random.choice``; with ``use_cer`` the first is the newest row (``ptr - 1``).
        Returns (obs, accrued_rewards, actions, rewards, next_obs, dones)."""
        inds = np.random.choice(self.size, batch_size, replace=replace)
        if use_cer:
            inds[0] = self.ptr - 1  # combined experience replay: the newest row is always in the batch
        return self._rows(inds, to_tensor, device)

    def cleanup(self):
        """Empty the buffer (the arrays keep their contents)."""
        self.size, self.ptr = 0, 0

    def get_all_data(self, to_tensor=False, device=None):
        """Rows ``[0, size)`` in storage order: (obs, accrued_rewards, actions, rewards, next_obs, dones)."""
        return self._rows(np.arange(self.size), to_tensor, device)

    def __len__(self):
        """Number of rows currently held."""
        return self.size
