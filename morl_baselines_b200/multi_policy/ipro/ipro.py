"""IPRO (reference multi_policy/ipro/ipro.py): iterated Pareto referent optimisation for any number of objectives.

The open region is described by its lower points (candidate referents) and upper points.  Each iteration asks the learner to improve on
the lower point with the largest hypervolume improvement; those improvements are recomputed every ``update_freq`` iterations for up to 50
sampled lower points in ONE launch of the batched hypervolume kernel (:func:`outer_loop.max_hypervolumes`).  The lower / upper point
updates and the error estimate are host numpy on the device Pareto filter, with the reference's expressions.
"""

from __future__ import annotations

from typing import Literal, Optional, Union

import numpy as np
import torch

from ...common.pareto import batched_pareto_dominates, batched_strict_pareto_dominates, filter_pareto_dominated, pareto_dominates, strict_pareto_dominates
from .box import Box
from .outer_loop import OuterLoop, Subproblem, max_hypervolumes


class IPRO(OuterLoop):
    """IPRO with the non-linear MO-PPO learner."""

    def __init__(
        self,
        env,
        direction: Literal["maximize", "minimize"] = "maximize",
        offset: float = 1,
        tolerance: float = 1e-6,
        max_iterations: Optional[int] = None,
        update_freq: int = 1,
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
        experiment_name: Optional[str] = "IPRO",
        project_name: str = "MORL-Baselines",
        wandb_entity: str = None,
        wandb_mode: Literal["online", "offline", "disabled"] = "online",
        seed: int = 1,
        rng: Union[np.random.Generator, None] = None,
    ):
        """``iter_total_timesteps`` is the learner's ``total_timesteps`` for each problem; the PPO arguments go to the learner.  With
        ``rng`` given, IPRO and the learner draw from it; otherwise each seeds its own generator with ``seed``."""
        super().__init__(
            env, method="IPRO", direction=direction, offset=offset, tolerance=tolerance, max_iterations=max_iterations, reset_agent=reset_agent,
            aug=aug, scale=scale, total_timesteps=iter_total_timesteps, learning_rate=learning_rate, num_steps=num_steps, anneal_lr=anneal_lr,
            gamma=gamma, gae_lambda=gae_lambda, num_minibatches=num_minibatches, update_epochs=update_epochs, norm_adv=norm_adv,
            clip_coef=clip_coef, clip_vloss=clip_vloss, ent_coef=ent_coef, vf_coef=vf_coef, max_grad_norm=max_grad_norm, target_kl=target_kl,
            mc_k=mc_k, device=device, log=log, experiment_name=experiment_name, project_name=project_name, wandb_entity=wandb_entity,
            wandb_mode=wandb_mode, seed=seed, rng=rng,
        )
        self.update_freq = update_freq
        self.lower_points = []
        self.upper_points = []
        self.rng = np.random.default_rng(seed) if rng is None else rng

    def reset(self):
        self.lower_points = []
        self.upper_points = []
        super().reset()

    def init_phase(self, extrema=None, deterministic: bool = False, eval_env=None) -> tuple:
        """Bound the front: without ``extrema``, maximise and minimise each objective alone (the ideal is exact, the nadir pessimistic)
        and widen both by ``offset``.  Then set up the lower and upper points and the first hypervolume improvements.  Returns the
        linear subsolutions and whether the front is a single point."""
        subsolutions = []
        if extrema is None:
            nadir, ideal, pf = np.zeros(self.dim), np.zeros(self.dim), []
            for i, weight_vec in enumerate(np.eye(self.dim)):
                ideal_vec, ideal_sol = self.linear_train(weight_vec=weight_vec, deterministic=deterministic, eval_env=eval_env)
                print(f"Found solution {ideal_vec} for weight vector {weight_vec}")
                nadir_vec, _ = self.linear_train(weight_vec=-1 * weight_vec, deterministic=deterministic, eval_env=eval_env)
                ideal_vec *= self.sign
                nadir_vec *= self.sign
                ideal[i], nadir[i] = ideal_vec[i], nadir_vec[i]
                pf.append(ideal_vec)
                subsolutions.append((weight_vec, ideal_vec, ideal_sol))
            self.pf = filter_pareto_dominated(np.array(pf))
            # the offset makes every Pareto-optimal point strictly dominate the nadir
            self.nadir = np.copy(nadir - self.offset)
            self.ideal = np.copy(ideal + self.offset)
            if len(self.pf) == 1:
                return subsolutions, True
        else:
            self.nadir, self.ideal = extrema

        self.ref_point = np.copy(self.nadir) if self.ref_point is None else np.array(self.ref_point)
        self.hv = self.compute_hypervolume(-self.sign * self.pf, -self.sign * self.ref_point)
        self.bounding_box = Box(self.nadir, self.ideal)
        self.total_hv = self.bounding_box.volume
        self.lower_points = np.array([self.nadir])
        for point in self.pf:
            self.update_lower_points(np.array(point))
        self.upper_points = np.array([self.ideal])
        self.error = max(self.ideal - self.nadir)
        self.compute_hvis()
        return subsolutions, False

    def compute_hvis(self, num=50):
        """Order the lower points by decreasing hypervolume improvement, estimated on up to ``num`` of them drawn without replacement
        (the others count as 0).  The improvement of lower point l is ranked by the volume between pf U completed U {l} and the ideal,
        which differs from it by a constant.  One kernel launch for all drawn points."""
        hvis = np.zeros(len(self.lower_points))
        drawn = self.rng.choice(len(self.lower_points), min(num, len(self.lower_points)), replace=False)
        if len(drawn):
            hvis[drawn] = self._improvement_volumes(self.lower_points[drawn])
        self.lower_points = self.lower_points[np.argsort(hvis)[::-1]]

    def _improvement_volumes(self, lowers: np.ndarray, device: bool = True) -> np.ndarray:
        """compute_hypervolume(pf U completed U {l}, ideal) for each row l of ``lowers``, over the points the ideal weakly dominates: the
        maximisation volume of the negated points above -ideal.  A lower point the ideal does not dominate leaves pf U completed alone."""
        ideal = np.asarray(self.ideal)
        base = np.vstack((self.pf, self.completed))
        base = base[batched_pareto_dominates(ideal, base)]
        keep = batched_pareto_dominates(ideal, lowers)
        vols = np.zeros(len(lowers))
        if keep.any():
            vols[keep] = max_hypervolumes(-base, -lowers[keep], -ideal, device=device)
        if not keep.all():
            vols[~keep] = max_hypervolumes(-base, None, -ideal, device=device)[0]
        return vols

    def max_hypervolume_improvement(self):
        """Recompute the improvements; the lower point with the largest one."""
        self.compute_hvis()
        return self.lower_points[0]

    def estimate_error(self):
        """Largest distance (in the worst objective) from an upper point to its closest point of the front."""
        if len(self.upper_points) == 0:
            self.error = 0
            return
        pf = np.array(list(self.pf))
        self.error = np.max(np.min(np.max(self.upper_points[:, None, :] - pf[None, :, :], axis=2), axis=1))

    def update_upper_points(self, vec):
        """Replace each upper point that strictly dominates ``vec`` by its d projections onto ``vec`` that still dominate the nadir."""
        beats = batched_strict_pareto_dominates(self.upper_points, vec)
        shifted = np.stack([self.upper_points[beats == 1]] * self.dim)
        shifted[range(self.dim), :, range(self.dim)] = np.expand_dims(vec, -1)
        shifted = shifted.reshape(-1, self.dim)
        shifted = shifted[np.all(shifted > self.nadir, axis=-1)]
        self.upper_points = filter_pareto_dominated(np.vstack((self.upper_points[beats == 0], shifted)))

    def update_lower_points(self, vec):
        """Replace each lower point that ``vec`` strictly dominates by its d projections onto ``vec`` that the ideal still dominates."""
        beaten = batched_strict_pareto_dominates(vec, self.lower_points)
        shifted = np.stack([self.lower_points[beaten == 1]] * self.dim)
        shifted[range(self.dim), :, range(self.dim)] = np.expand_dims(vec, -1)
        shifted = shifted.reshape(-1, self.dim)
        shifted = shifted[np.all(self.ideal > shifted, axis=-1)]
        self.lower_points = -filter_pareto_dominated(-np.vstack((self.lower_points[beaten == 0], shifted)))

    def select_referent(self, method="random"):
        if method == "random":
            return self.lower_points[self.rng.integers(0, len(self.lower_points))]
        if method == "first":
            return self.lower_points[0]
        raise ValueError(f"Unknown method {method}")

    def get_iterable_for_replay(self):
        return np.copy(self.lower_points)

    def maybe_add_solution(self, subproblem: Subproblem, point: np.ndarray, lower: np.ndarray):
        """Accept ``point`` as the answer for referent ``lower`` if it strictly dominates it; returns the new subproblem or False."""
        if not strict_pareto_dominates(point, lower):
            return False
        new_subproblem = Subproblem(referent=lower, nadir=self.nadir, ideal=self.ideal)
        self.update_found(new_subproblem, point)
        return new_subproblem

    def maybe_add_completed(self, subproblem: Subproblem, point: np.ndarray, lower: np.ndarray):
        """Close referent ``lower`` if it dominates the subproblem's referent; returns the new subproblem or False."""
        if not pareto_dominates(lower, subproblem.referent):
            return False
        new_subproblem = Subproblem(referent=lower, nadir=self.nadir, ideal=self.ideal)
        self.update_not_found(new_subproblem, point)
        return new_subproblem

    def update_found(self, subproblem, vec):
        self.pf = np.vstack((self.pf, vec))
        self.update_lower_points(vec)
        self.update_upper_points(vec)

    def update_not_found(self, subproblem, vec):
        self.completed = np.vstack((self.completed, subproblem.referent))
        self.lower_points = self.lower_points[np.any(self.lower_points != subproblem.referent, axis=1)]
        self.update_upper_points(subproblem.referent)
        if strict_pareto_dominates(vec, self.nadir):
            self.robust_points = np.vstack((self.robust_points, vec))

    def decompose_problem(self, iteration, method="first"):
        if iteration % self.update_freq == 0:
            self.compute_hvis()
        return Subproblem(referent=self.select_referent(method=method), nadir=self.nadir, ideal=self.ideal)

    def update_excluded_volume(self):
        """The volume the front dominates above the nadir, and the volume above pf U completed below the ideal."""
        self.dominated_hv = self.compute_hypervolume(-self.pf, -self.nadir)
        self.discarded_hv = self.compute_hypervolume(np.vstack((self.pf, self.completed)), self.ideal)

