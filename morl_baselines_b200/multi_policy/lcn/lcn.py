"""Lorenz Conditioned Networks on the CUDA update engine -- drop-in for reference morl_baselines/multi_policy/lcn/lcn.py (``lorenz_vector``
and ``LCN`` with the same constructor and ``train`` arguments).

LCN is PCN (multi_policy/pcn/pcn.py) with episodes ranked and commands chosen by Lorenz dominance (``distance_ref="nondominated"``) or
lambda-Lorenz dominance (``"lambda_lorenz"``), and a configurable crowding threshold.  The model, the device episode store, the graphed
update block and the rollouts are PCN's; only the host-side ranking differs, computed in numpy exactly as the reference computes it.
"""

from __future__ import annotations

from typing import List, Optional, Type, Union

import numpy as np
import torch as th

from ... import ops
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.pareto import get_non_dominated_inds
from ..pcn.pcn import (  # noqa: F401  (the reference's lcn module re-exports these)
    PCN,
    BasePCNModel,
    ContinuousActionsDefaultModel,
    DiscreteActionsDefaultModel,
    Transition,
    crowding_distance,
    front_distance_scores,
)


def lorenz_vector(points: np.ndarray, proportional: bool = False) -> np.ndarray:
    """Lorenz vector of each point: the cumulative sum of its objectives sorted in increasing order, optionally divided by their sum
    (reference lcn.py:26-45)."""
    lv = np.cumsum(np.sort(points, axis=1), axis=1)
    if proportional:
        lv = lv / np.sum(points, axis=1, keepdims=True)
    return lv


def lcn_scores(returns: np.ndarray, threshold: float, distance_ref: str, lcn_lambda: Optional[float]) -> np.ndarray:
    """LCN's episode scores (reference lcn.py:213-268): distance to the Lorenz (or lambda-Lorenz) front with PCN's penalties.  With
    ``"lambda_lorenz"`` the distances are measured between the SORTED returns."""
    crowded = np.argwhere(crowding_distance(returns) <= threshold).flatten()
    if distance_ref == "lambda_lorenz":
        assert lcn_lambda is not None, "lcn_lambda must be set when using distance_ref='lambda_lorenz'"
        returns = np.sort(returns, axis=1)
        nd = get_non_dominated_inds(lcn_lambda * returns + (1 - lcn_lambda) * lorenz_vector(returns))
    else:
        nd = get_non_dominated_inds(lorenz_vector(returns))
    return front_distance_scores(returns, nd, crowded)


class LCN(PCN):
    """Lorenz Conditioned Networks (Michailidis et al., JAIR 2026) on the CUDA update engine (reference lcn.py:48-480)."""

    checkpoint_every = 100

    def __init__(self, env, scaling_factor: np.ndarray, learning_rate: float = 1e-2, gamma: float = 1.0, batch_size: int = 32,
                 hidden_dim: int = 64, noise: float = 0.1, distance_ref: str = "nondominated", lcn_lambda: Optional[float] = None,
                 project_name: str = "MORL-Baselines", experiment_name: str = "LCN", wandb_entity: Optional[str] = None, log: bool = True,
                 seed: Optional[int] = None, device: Union[th.device, str] = "auto", model_class: Optional[Type[BasePCNModel]] = None,
                 use_cuda_graph: bool = True) -> None:
        MOAgent.__init__(self, env, device=device, seed=seed)
        MOPolicy.__init__(self, device=device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.LCN needs a CUDA device: the update path is CUDA-only")
        ops._lib.load()
        self.distance_ref = distance_ref
        self.lcn_lambda = lcn_lambda
        self.cd_threshold = 0.2
        self._init_common(scaling_factor, learning_rate, gamma, batch_size, hidden_dim, noise, model_class, use_cuda_graph)
        self.log = log
        if log:
            experiment_name += " continuous action" if self.continuous_action else ""
            self.setup_wandb(project_name, experiment_name, wandb_entity)

    def get_config(self) -> dict:
        """Configuration of the LCN agent."""
        return {
            "env_id": self.env.unwrapped.spec.id,
            "reward_dim": self.reward_dim,
            "batch_size": self.batch_size,
            "gamma": self.gamma,
            "learning_rate": self.learning_rate,
            "hidden_dim": self.hidden_dim,
            "scaling_factor": self.scaling_factor,
            "continuous_action": self.continuous_action,
            "noise": self.noise,
            "distance_ref": self.distance_ref,
            "lcn_lambda": self.lcn_lambda,
            "seed": self.seed,
        }

    def _scores(self, returns: np.ndarray, threshold: float) -> np.ndarray:
        return lcn_scores(returns, threshold, self.distance_ref, self.lcn_lambda)

    def _front(self, returns: np.ndarray) -> np.ndarray:
        return get_non_dominated_inds(lorenz_vector(returns))

    def _threshold(self) -> float:
        return self.cd_threshold

    def save(self, filename: str = "LCN_model", save_dir: str = "weights"):
        """Save the whole model module with ``th.save``."""
        super().save(filename, save_dir)

    def _checkpoint(self, n_checkpoints: int, save_dir: str):
        self.save(save_dir=save_dir, filename=f"LCN_model_{n_checkpoints}")

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              num_eval_weights_for_eval: int = 50, num_er_episodes: int = 500, num_step_episodes: int = 10, num_model_updates: int = 100,
              max_return: np.ndarray = None, max_buffer_size: int = 500, num_points_pf: int = 100, save_dir: str = "weights",
              cd_threshold: float = 0.2):
        """Train LCN (reference lcn.py:358-480)."""
        self.cd_threshold = cd_threshold
        self._train(total_timesteps, eval_env, ref_point, known_pareto_front, num_eval_weights_for_eval, num_er_episodes, num_step_episodes,
                    num_model_updates, max_return, max_buffer_size, num_points_pf, save_dir,
                    {"save_dir": save_dir, "distance_ref": self.distance_ref, "lcn_lambda": self.lcn_lambda, "cd_threshold": cd_threshold})
        self.env.close()
