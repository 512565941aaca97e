"""ModelEnv and the termination rules of GPI-PD's Dyna path, on the device (mirrors reference common/model_based/utils.py:13-188; the
plotting helper ``visualize_eval`` is not part of the update path and is not mirrored).

``ModelEnv.step`` keeps observations, predictions, termination flags and uncertainties in HBM: the imagined transitions are consumed
by a masked bulk insert into the dynamics replay buffer (``ReplayBuffer.add_batch``) -- the reference copies every tensor to the host
and appends row by row in a python loop (gpi_pd.py:394-397, up to 25,000 iterations per rollout)."""

from __future__ import annotations

from typing import Tuple

import numpy as np
import torch as th

from ... import ops


def termination_fn_false(obs, act, next_obs, rew):
    return th.zeros((obs.shape[0], 1), dtype=th.bool, device=obs.device)


def termination_fn_dst(obs, act, next_obs, rew):
    raise NotImplementedError("deep-sea-treasure needs mo_gymnasium's CONCAVE_MAP (not installed in this image)")


def termination_fn_mountaincar(obs, act, next_obs, rew):
    done = (next_obs[:, 0] >= 0.45) & (next_obs[:, 1] >= 0.0)
    return done[:, None]


def termination_fn_minecart(obs, act, next_obs, rew):
    old_pos, pos = obs[:, 0:2], next_obs[:, 0:2]
    in_base = th.sqrt((pos * pos).sum(1)) < 0.15
    was_out_base = th.sqrt((old_pos * old_pos).sum(1)) >= 0.15
    return (was_out_base & in_base)[:, None]


def termination_fn_hopper(obs, act, next_obs, rew):
    height, angle = next_obs[:, 0], next_obs[:, 1]
    # (the reference's `np.abs(next_obs[:, 1:] < 100)` takes |.| of the comparison, i.e. the test is next_obs[:, 1:] < 100)
    not_done = th.isfinite(next_obs).all(-1) & (next_obs[:, 1:] < 100).all(-1) & (height > 0.7) & (angle.abs() < 0.2)
    return (~not_done)[:, None]


def termination_fn_lunarlander(obs, act, next_obs, rew):
    has_exited_screen = next_obs[:, 0].abs() >= 1.0
    has_crashed_or_landed = (rew[:, 0] != 0) & (next_obs[:, 6] >= 0.95) & (next_obs[:, 7] >= 0.95)
    return (has_exited_screen | has_crashed_or_landed)[:, None]


def termination_fn_humanoid(obs, act, next_obs, rew):
    min_z, max_z = 1.0, 2.0
    not_done = (min_z < next_obs[:, 0]) & (next_obs[:, 0] < max_z)
    return (~not_done)[:, None]


# env id -> (rule, rule id of the fused device step ``ops.dyna_commit`` or None where it has none): the reference's ModelEnv.__init__ table
# (utils.py:119-138), first match wins.  Minecart and deep-sea-treasure are discrete-action environments and have no device rule.
_RULE_TABLE = (
    (lambda e: "hopper" in e, termination_fn_hopper, ops.TERM_HOPPER),
    (lambda e: "halfcheetah" in e, termination_fn_false, ops.TERM_NONE),
    (lambda e: "humanoid" in e, termination_fn_humanoid, ops.TERM_HUMANOID),
    (lambda e: "lunar-lander" in e, termination_fn_lunarlander, ops.TERM_LUNARLANDER),
    (lambda e: "mo-reacher" in e, termination_fn_false, ops.TERM_NONE),
    (lambda e: "mountaincar" in e, termination_fn_mountaincar, ops.TERM_MOUNTAINCAR),
    (lambda e: "minecart" in e, termination_fn_minecart, None),
    (lambda e: e == "mo-highway-fast-v0" or e == "mo-highway-v0", termination_fn_false, ops.TERM_NONE),
    (lambda e: e == "deep-sea-treasure-v0", termination_fn_dst, None),
)


def _rule_entry(env_id: str):
    for matches, fn, rule_id in _RULE_TABLE:
        if matches(env_id):
            return fn, rule_id
    raise NotImplementedError(f"no termination rule for environment {env_id!r}")


def termination_fn_for(env_id: str):
    """Rule table of the reference's ModelEnv.__init__ (utils.py:119-138)."""
    return _rule_entry(env_id)[0]


def termination_rule_id(env_id: str) -> int:
    """The ``ops.TERM_*`` id of ``env_id``'s termination rule, for the fused rollout step; NotImplementedError when the environment has no
    rule, or only one that the device step does not implement (minecart, deep-sea-treasure)."""
    rule_id = _rule_entry(env_id)[1]
    if rule_id is None:
        raise NotImplementedError(f"the termination rule of {env_id!r} has no device form (discrete-action environments only)")
    return rule_id


class ModelEnv:
    """The learned model as an environment (reference utils.py:105-188)."""

    def __init__(self, model, env_id=None, rew_dim=1):
        self.model = model
        self.rew_dim = rew_dim
        self.termination_func = termination_fn_for(env_id)

    @th.no_grad()
    def step_device(self, obs: th.Tensor, act: th.Tensor, deterministic: bool = False):
        """Batched step with device tensors in and out: (next_obs [N, obs], rewards [N, rew_dim], terminals [N, 1] bool, info)."""
        inputs = th.cat((obs, act), dim=-1).float().to(self.model.device)
        obs_f = obs.float().contiguous()
        samples, vars_, unc = self.model.sample_device(inputs, deterministic=deterministic, obs=obs_f, rew_dim=self.rew_dim)
        rewards, next_obs = samples[:, : self.rew_dim], samples[:, self.rew_dim:]
        terminals = self.termination_func(obs_f, act, next_obs, rewards)
        info = {"uncertainty": unc, "var_obs": vars_[:, self.rew_dim:], "var_rewards": vars_[:, : self.rew_dim]}
        return next_obs, rewards, terminals, info

    def step(self, obs: th.Tensor, act: th.Tensor, deterministic: bool = False) -> Tuple[np.ndarray, np.ndarray, np.ndarray, dict]:
        """Reference signature (utils.py:140-188): numpy results; a single (1-D) observation is accepted and squeezed again."""
        assert len(obs.shape) == len(act.shape)
        single = len(obs.shape) == 1
        if single:
            obs, act = obs.unsqueeze(0), act.unsqueeze(0)
        next_obs, rewards, terminals, info = self.step_device(obs.to(self.model.device), act.to(self.model.device), deterministic)
        next_obs, rewards, terminals = next_obs.cpu().numpy(), rewards.cpu().numpy(), terminals.cpu().numpy()
        info = {k: v.cpu().numpy() for k, v in info.items()}
        if single:
            next_obs, rewards, terminals = next_obs[0], rewards[0], terminals[0]
            info = {k: v[0] for k, v in info.items()}
        return next_obs, rewards, terminals, info
