"""IPRO-2D (reference multi_policy/ipro/ipro_2d.py): IPRO for two objectives, where the open region is a set of boxes.

Each iteration takes the largest open box and asks the learner to improve on its nadir; a found point splits the box into two, the
parts it dominates and is dominated by are added to the dominated and discarded volumes.  The boxes wait in a :class:`BoxQueue` ordered
by volume (the reference keeps a ``sortedcontainers.SortedKeyList``).
"""

from __future__ import annotations

from copy import deepcopy
from typing import Literal, Optional, Union

import numpy as np
import torch

from ...common.pareto import filter_pareto_dominated, pareto_dominates, strict_pareto_dominates
from .box import Box, BoxQueue
from .outer_loop import OuterLoop, Subproblem


class IPRO2D(OuterLoop):
    """IPRO-2D with the non-linear MO-PPO learner."""

    def __init__(
        self,
        env,
        direction: Literal["maximize", "minimize"] = "maximize",
        offset: float = 1,
        tolerance: float = 1e-6,
        max_iterations: Optional[int] = None,
        reset_agent: bool = False,
        aug: float = 0.1,
        scale: float = 100,
        iter_total_timesteps: int = 500000,
        learning_rate: float = 2.5e-4,
        num_steps: int = 128,
        anneal_lr: bool = True,
        gamma: float = 0.99,
        gae_lambda: float = 0.95,
        num_minibatches: int = 4,
        update_epochs: int = 4,
        norm_adv: bool = True,
        clip_coef: float = 0.2,
        clip_vloss: bool = True,
        ent_coef: float = 0.01,
        vf_coef: float = 0.5,
        max_grad_norm: float = 0.5,
        target_kl: float = None,
        mc_k: int = 32,
        device: Union[torch.device, str] = "auto",
        log: bool = False,
        experiment_name: Optional[str] = "IPRO-2D",
        project_name: str = "MORL-Baselines",
        wandb_entity: str = None,
        wandb_mode: Literal["online", "offline", "disabled"] = "online",
        seed: int = 1,
        rng: Union[np.random.Generator, None] = None,
    ):
        """Arguments as :class:`IPRO`'s, without ``update_freq``."""
        super().__init__(
            env, method="IPRO-2D", direction=direction, offset=offset, tolerance=tolerance, max_iterations=max_iterations,
            reset_agent=reset_agent, aug=aug, scale=scale, total_timesteps=iter_total_timesteps, learning_rate=learning_rate,
            num_steps=num_steps, anneal_lr=anneal_lr, gamma=gamma, gae_lambda=gae_lambda, num_minibatches=num_minibatches,
            update_epochs=update_epochs, norm_adv=norm_adv, clip_coef=clip_coef, clip_vloss=clip_vloss, ent_coef=ent_coef, vf_coef=vf_coef,
            max_grad_norm=max_grad_norm, target_kl=target_kl, mc_k=mc_k, device=device, log=log, experiment_name=experiment_name,
            project_name=project_name, wandb_entity=wandb_entity, wandb_mode=wandb_mode, seed=seed, rng=rng,
        )
        self.box_queue = BoxQueue()

    def reset(self):
        self.box_queue = BoxQueue()
        super().reset()

    def estimate_error(self):
        """The longest side of an open box (0 when none is left)."""
        self.error = max(box.max_dist for box in self.box_queue) if len(self.box_queue) else 0

    def split_box(self, box, point):
        """The two boxes of ``box`` left open by ``point`` (upper left and lower right); the part ``point`` dominates and the part that
        dominates it are added to the dominated and discarded volumes."""
        upper_left = Box(np.array([point[0], box.ideal[1]]), np.array([box.nadir[0], point[1]]))
        lower_right = Box(np.array([box.ideal[0], point[1]]), np.array([point[0], box.nadir[1]]))
        self.dominated_hv += Box(box.nadir, point).volume
        self.discarded_hv += Box(point, box.ideal).volume
        return [upper_left, lower_right]

    def update_box_queue(self, box, point):
        """Queue the parts of ``box`` that ``point`` leaves open and that are larger than the tolerance and not degenerate."""
        for part in self.split_box(box, point):
            if part.volume > self.tolerance and pareto_dominates(part.ideal, part.nadir):
                self.box_queue.add(part)

    def init_phase(self, extrema=None, deterministic: bool = False, eval_env=None) -> tuple:
        """Without ``extrema``, maximise each objective alone: the two vectors give the bounding box (widened by ``offset``) and the
        first front.  The bounding box is the first open box."""
        subsolutions = []
        if extrema is None:
            found = []
            for weight_vec in np.eye(2):
                vec, sol = self.linear_train(weight_vec=weight_vec, deterministic=deterministic, eval_env=eval_env)
                print(f"Found solution {vec} for weight vector {weight_vec}")
                vec *= self.sign
                found.append(vec)
                subsolutions.append((weight_vec, vec, sol))
            found = np.array(found)
            self.nadir = np.min(found, axis=0) - self.offset
            self.ideal = np.max(found, axis=0) + self.offset
            self.pf = filter_pareto_dominated(np.array(found))
        else:
            self.nadir, self.ideal = extrema

        self.ref_point = np.copy(self.nadir) if self.ref_point is None else np.array(self.ref_point)
        self.bounding_box = Box(self.nadir, self.ideal)
        self.box_queue.add(self.bounding_box)
        self.estimate_error()
        self.total_hv = self.bounding_box.volume
        self.hv = self.compute_hypervolume(-self.sign * self.pf, -self.sign * self.ref_point)
        self.agent.reset_agent(pref_dim=self.dim)  # the utility changes from linear to AASF
        return subsolutions, len(self.pf) == 1

    def is_done(self, step):
        return not self.box_queue or super().is_done(step)

    def get_iterable_for_replay(self):
        """(index, box) of a copy of the open boxes, largest first."""
        return reversed(list(enumerate(deepcopy(self.box_queue))))

    def maybe_add_solution(self, subproblem: Subproblem, point: np.ndarray, item: tuple):
        """Accept ``point`` for the open box ``item`` = (index, box) if it strictly dominates the box's nadir; returns the new subproblem
        or False."""
        idx, box = item
        if not strict_pareto_dominates(point, box.nadir):
            return False
        new_subproblem = Subproblem(referent=box.nadir, nadir=box.nadir, ideal=box.ideal)
        self.update_found(new_subproblem, point, box_idx=idx)
        return new_subproblem

    def maybe_add_completed(self, subproblem: Subproblem, point: np.ndarray, item: tuple):
        """Close the open box ``item`` = (index, box) if its nadir dominates the subproblem's referent; returns the new subproblem or
        False."""
        idx, box = item
        if not pareto_dominates(box.nadir, subproblem.referent):
            return False
        new_subproblem = Subproblem(referent=box.nadir, nadir=box.nadir, ideal=box.ideal)
        self.update_not_found(new_subproblem, point, box_idx=idx)
        return new_subproblem

    def update_found(self, subproblem, vec, box_idx=-1):
        self.update_box_queue(self.box_queue.pop(box_idx), vec)
        self.pf = np.vstack((self.pf, vec))

    def update_not_found(self, subproblem, vec, box_idx=-1):
        self.discarded_hv += self.box_queue.pop(box_idx).volume
        self.completed = np.vstack((self.completed, np.copy(subproblem.referent)))
        if strict_pareto_dominates(vec, self.nadir):
            self.robust_points = np.vstack((self.robust_points, vec))

    def decompose_problem(self, iteration, method="first"):
        box = self.box_queue[-1]
        return Subproblem(referent=box.nadir, nadir=box.nadir, ideal=box.ideal)

    def update_excluded_volume(self):
        """Nothing to do: splitting and closing boxes keeps the volumes."""
