"""IPRO's outer loop (reference multi_policy/ipro/outer_loop.py): it splits the search for a Pareto front into single-objective problems,
hands each to the non-linear MO-PPO learner (:class:`NLMOPPO`) with an achievement-scalarising utility, and keeps the bookkeeping of what
has been found, excluded and is still open.

The exact hypervolumes of the bookkeeping run on the device: :func:`max_hypervolumes` is one launch of the batched kernel
(``hv_ops.hypervolume_batch``) for any number of "base set plus one candidate" volumes, with one device-to-host copy.  Sets the kernel does
not cover (more than 2048 points for d <= 3 or 512 for d = 4, or d >= 5) are computed by the host sweep of
``common.performance_indicators``.
"""

from __future__ import annotations

import random
import time
from dataclasses import dataclass
from functools import partial
from typing import Any, Callable, Iterable, Literal, Optional

import numpy as np
import torch

from ... import hv_ops
from ...common.morl_algorithm import MOAgent
from ...common.pareto import (
    batched_pareto_dominates,
    batched_strict_pareto_dominates,
    filter_pareto_dominated,
    strict_pareto_dominates,
)
from ...common.performance_indicators import hypervolume as host_hypervolume
from ...single_policy.ser.nl_mo_ppo import NLMOPPO


def max_hypervolumes(base: np.ndarray, cand: Optional[np.ndarray], ref: np.ndarray, device: bool = True) -> np.ndarray:
    """Exact maximisation hypervolumes above ``ref`` [d]: of ``base`` [n, d] plus each row of ``cand`` [m, d] (float64 [m]), or of
    ``base`` alone when ``cand`` is None (float64 [1]).  One kernel launch inside its range; the host sweep outside it, or when
    ``device`` is False."""
    base = np.ascontiguousarray(base, dtype=np.float64).reshape(-1, len(ref))
    ref = np.asarray(ref, dtype=np.float64)
    if device and hv_ops.hypervolume_batch_supported(len(base), len(ref)):
        dev = torch.device("cuda", torch.cuda.current_device())
        as_dev = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)  # noqa: E731
        out = hv_ops.hypervolume_batch(as_dev(base), None if cand is None else as_dev(cand).reshape(-1, len(ref)), as_dev(ref))
        return out.cpu().numpy()
    if cand is None:
        return np.array([host_hypervolume(ref, base)])
    return np.array([host_hypervolume(ref, np.vstack((base, c))) for c in np.asarray(cand, dtype=np.float64).reshape(-1, len(ref))])


@dataclass
class Subproblem:
    """A referent with the nadir and ideal of the region it was drawn from."""

    referent: np.ndarray
    nadir: np.ndarray
    ideal: np.ndarray


Subsolution = tuple  # (Subproblem, vector, solution)
IPROCallback = Callable[[int, float, float, float, float, float], Any]


def linear_scalarization(batch: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
    """Weighted sum over the last axis."""
    return torch.sum(batch * weights, dim=-1)


def aasf(batch, referent, nadir, ideal, aug=0.0, scale=100):
    """Augmented achievement scalarising function: the smallest scaled improvement over ``referent``, relative to the extent
    ``ideal - nadir``, plus ``aug`` times their mean."""
    frac = scale * (batch - referent) / (ideal - nadir)
    return torch.min(frac, dim=-1)[0] + aug * torch.mean(frac, dim=-1)


class OuterLoop(MOAgent):
    """State and control flow shared by IPRO and IPRO-2D; not meant to be used directly."""

    def __init__(
        self,
        env,
        method: str = "IPRO",
        direction: Literal["maximize", "minimize"] = "maximize",
        offset: float = 1,
        tolerance: float = 1e-1,
        max_iterations: Optional[int] = None,
        aug: float = 0.1,
        scale: float = 100,
        reset_agent: bool = False,
        log: bool = False,
        experiment_name: Optional[str] = None,
        project_name: Optional[str] = None,
        wandb_entity: Optional[str] = None,
        wandb_mode: Literal["online", "offline", "disabled"] = "online",
        seed: Optional[int] = None,
        **kwargs,
    ):
        """``kwargs`` (which must hold ``device``) are the learner's: ``NLMOPPO(0, env, seed=seed, **kwargs)``."""
        MOAgent.__init__(self, env, device=kwargs["device"], seed=seed)
        self.env = env
        self.dim = self.env.reward_space.shape[0]
        self.agent = NLMOPPO(0, env, seed=seed, **kwargs)

        self.method = method
        self.direction = direction
        self.ref_point = None
        self.offset = offset
        self.tolerance = tolerance
        self.max_iterations = np.inf if max_iterations is None else max_iterations
        self.aug = aug
        self.scale = scale
        self.reset_agent = reset_agent
        self.sign = 1 if direction == "maximize" else -1

        self.track = log
        self.run_id = None
        self.exp_name = experiment_name
        self.wandb_project_name = project_name
        self.wandb_entity = wandb_entity
        self.wandb_mode = wandb_mode
        self.seed = seed
        OuterLoop.reset(self)

    def reset(self):
        """Forget the bounding box, the fronts and the measures."""
        self.bounding_box = None
        self.ideal = None
        self.nadir = None
        self.pf = np.empty((0, self.dim))
        self.robust_points = np.empty((0, self.dim))
        self.completed = np.empty((0, self.dim))
        self.hv = 0
        self.total_hv = 0
        self.dominated_hv = 0
        self.discarded_hv = 0
        self.coverage = 0
        self.error = np.inf
        self.replay_triggered = 0

    def get_config(self) -> dict:
        return {
            "method": self.method,
            "env_id": self.env.spec.id,
            "dimensions": self.dim,
            "tolerance": self.tolerance,
            "max_iterations": self.max_iterations,
            "seed": self.seed,
        }

    def setup(self) -> float:
        """Start the wandb run when logging; returns the start time."""
        if self.track:
            import wandb

            self.setup_wandb(project_name=self.wandb_project_name, experiment_name=self.exp_name, entity=self.wandb_entity,
                             mode=self.wandb_mode)
            wandb.define_metric("iteration")
            for name in ("hypervolume", "dominated_hv", "discarded_hv", "coverage", "error"):
                wandb.define_metric(f"outer/{name}", step_metric="iteration")
            self.run_id = wandb.run.id
        return time.time()

    def get_pareto_set(self, subsolutions: list) -> list:
        """(vector, solution) of every subsolution whose vector is (close to) a point of the front, in the caller's sign."""
        return [(self.sign * vec, sol) for _, vec, sol in subsolutions if np.any(np.all(np.isclose(vec, self.pf), axis=1))]

    def get_pareto_front(self) -> np.ndarray:
        return self.pf * self.sign

    def finish(self, start_time: float, iteration: int):
        """Merge the robust points into the front and take the final volumes."""
        self.pf = filter_pareto_dominated(np.vstack((self.pf, self.robust_points)))
        self.dominated_hv = self.compute_hypervolume(-self.sign * self.pf, -self.sign * self.nadir)
        self.hv = self.compute_hypervolume(-self.sign * self.pf, -self.sign * self.ref_point)
        self.log_iteration(iteration + 1)
        print(f"Iterations {iteration + 1} | Time {time.time() - start_time:.2f} | HV {self.hv:.2f} | PF size {len(self.pf)} |")
        self.close_wandb()

    def close_wandb(self):
        if self.track:
            import wandb

            wandb.log({"pareto_front": wandb.Table(data=self.pf, columns=[f"obj_{i}" for i in range(self.dim)])})
            wandb.run.summary["PF_size"] = len(self.pf)
            wandb.finish()

    def log_iteration(self, iteration: int, subproblem: Optional[Subproblem] = None, pareto_point: Optional[np.ndarray] = None):
        """Log the measures of this iteration (and its referent, ideal and found point) to wandb, retrying on a wandb error."""
        if not self.track:
            return
        import wandb

        while True:
            try:
                wandb.log({"outer/hypervolume": self.hv, "outer/dominated_hv": self.dominated_hv, "outer/discarded_hv": self.discarded_hv,
                           "outer/coverage": self.coverage, "outer/error": self.error, "iteration": iteration})
                break
            except wandb.Error as e:
                print(f"wandb got error {e}")
                time.sleep(random.randint(10, 100))
        summary = wandb.run.summary
        if subproblem is not None:
            summary[f"referent_{iteration}"] = self.sign * subproblem.referent
            summary[f"ideal_{iteration}"] = self.sign * subproblem.ideal
            summary[f"pareto_point_{iteration}"] = self.sign * pareto_point
        summary["hypervolume"] = self.hv
        summary["PF_size"] = len(self.pf)
        summary["replay_triggered"] = self.replay_triggered

    def compute_hypervolume(self, points: np.ndarray, ref: np.ndarray) -> float:
        """Hypervolume of ``points`` in the minimisation form (the region between each point and ``ref``), over the points ``ref`` weakly
        dominates (reference outer_loop.py:250-256; pymoo's exact HV there).  Computed as the maximisation volume of the negated points."""
        points = points[batched_pareto_dominates(ref, points)]
        if points.size == 0:
            return 0
        return float(max_hypervolumes(-points, None, -np.asarray(ref))[0])

    # ---- the steps each method defines ---------------------------------------------------------------------------------------------
    def init_phase(self, extrema=None, deterministic: bool = False, eval_env=None) -> tuple:
        raise NotImplementedError

    def is_done(self, step: int) -> bool:
        return 1 - self.coverage <= self.tolerance or step >= self.max_iterations

    def decompose_problem(self, iteration: int, method: str = "first") -> Subproblem:
        raise NotImplementedError

    def update_found(self, subproblem: Subproblem, vec: np.ndarray):
        raise NotImplementedError

    def update_not_found(self, subproblem: Subproblem, vec: np.ndarray):
        raise NotImplementedError

    def update_excluded_volume(self):
        raise NotImplementedError

    def estimate_error(self):
        raise NotImplementedError

    def get_iterable_for_replay(self) -> Iterable[Any]:
        raise NotImplementedError

    def maybe_add_solution(self, subproblem: Subproblem, vec: np.ndarray, item: Any):
        raise NotImplementedError

    def maybe_add_completed(self, subproblem: Subproblem, vec: np.ndarray, item: Any):
        raise NotImplementedError

    # ---- replay after a non-optimal oracle answer ----------------------------------------------------------------------------------
    def replay(self, vec: np.ndarray, sol: Any, iter_pairs: list) -> list:
        """Rebuild the state from the extrema after ``vec`` turned out to strictly dominate an earlier answer: the earlier subproblems are
        replayed in order until ``vec`` takes the place of the first answer it beats (or fits the first referent it beats), and each
        remaining answer is then offered to the open items of the rebuilt state.  Returns the new subsolutions."""
        nadir, ideal, replays = self.nadir, self.ideal, self.replay_triggered
        self.reset()
        self.replay_triggered = replays + 1
        self.init_phase(extrema=(nadir, ideal), eval_env=None)

        new_subsolutions = []
        consumed = 0
        for old_subproblem, old_vec, old_sol in iter_pairs:
            consumed += 1
            was_found = strict_pareto_dominates(old_vec, old_subproblem.referent)
            if strict_pareto_dominates(vec, old_vec if was_found else old_subproblem.referent):
                self.update_found(old_subproblem, vec)
                new_subsolutions.append((old_subproblem, vec, sol))
                break
            if was_found:
                self.update_found(old_subproblem, old_vec)
                new_subsolutions.append((old_subproblem, old_vec, old_sol))
            else:
                self.update_not_found(old_subproblem, old_vec)
                new_subsolutions.append((old_subproblem, old_vec, old_vec))

        for old_subproblem, old_vec, old_sol in iter_pairs[consumed:]:
            items = self.get_iterable_for_replay()
            add = self.maybe_add_solution if strict_pareto_dominates(old_vec, old_subproblem.referent) else self.maybe_add_completed
            for item in items:
                res = add(old_subproblem, old_vec, item)
                if res:
                    new_subsolutions.append((res, old_vec, old_sol))
                    break
        return new_subsolutions

    def eval(self, obs, disc_vec_return, pref=None):
        return self.agent.eval(obs, disc_vec_return, pref=pref)

    # ---- the learner's problems ----------------------------------------------------------------------------------------------------
    def linear_train(self, weight_vec: np.ndarray, deterministic: bool, eval_env) -> tuple:
        """Train the learner on the weighted sum with ``weight_vec``; returns its vector (learner's sign) and its Agent."""
        if self.reset_agent:
            self.agent.reset_agent(pref_dim=self.dim)
        weights = torch.tensor(weight_vec, device=self.device, dtype=torch.float32)
        vec = self.agent.train(eval_env, partial(linear_scalarization, weights=weights), pref=weights, deterministic=deterministic)
        return vec, self.agent.agent

    def oracle_train(self, referent: np.ndarray, deterministic: bool, eval_env) -> tuple:
        """Train the learner on the AASF of ``referent``; returns its vector, multiplied in place into the maximisation sign, and its
        Agent."""
        if self.reset_agent:
            self.agent.reset_agent(pref_dim=self.dim)
        as_dev = lambda v: self.sign * torch.tensor(v, device=self.device, dtype=torch.float32)  # noqa: E731
        referent, nadir, ideal = as_dev(referent), as_dev(self.nadir), as_dev(self.ideal)
        u_func = partial(aasf, referent=referent, nadir=nadir, ideal=ideal, aug=self.aug, scale=self.scale)
        vec = self.agent.train(eval_env, u_func, pref=referent, deterministic=deterministic)
        vec *= self.sign
        return vec, self.agent.agent

    def train(self, eval_env, ref_point: np.ndarray, deterministic: bool = False, extrema=None,
              callback: Optional[IPROCallback] = None) -> list:
        """Run the outer loop until the covered share of the bounding box reaches ``1 - tolerance`` (or ``max_iterations``); returns the
        Pareto set as (vector, Agent) pairs."""
        self.ref_point = ref_point
        start = self.setup()
        linear_subsolutions, done = self.init_phase(extrema=extrema, deterministic=deterministic, eval_env=eval_env)
        if done:
            print("The problem is solved in the initial phase.")
            return self.get_pareto_set(linear_subsolutions)

        iteration = 0
        self.log_iteration(iteration)
        subsolutions = []
        while not self.is_done(iteration):
            begin = time.time()
            print(f"Iter {iteration} - Covered {self.coverage:.5f}% - Error {self.error:.5f}")
            subproblem = self.decompose_problem(iteration)
            vec, sol = self.oracle_train(referent=subproblem.referent, deterministic=deterministic, eval_env=eval_env)

            found = strict_pareto_dominates(vec, subproblem.referent)
            earlier = np.vstack((self.pf, self.completed)) if found else self.completed
            if np.any(batched_strict_pareto_dominates(vec, earlier)):
                subsolutions = self.replay(vec, sol, subsolutions)
            else:
                (self.update_found if found else self.update_not_found)(subproblem, vec)
                subsolutions.append((subproblem, vec, sol))

            self.update_excluded_volume()
            self.estimate_error()
            self.coverage = (self.dominated_hv + self.discarded_hv) / self.total_hv
            self.hv = self.compute_hypervolume(-self.sign * self.pf, -self.sign * self.ref_point)

            iteration += 1
            self.log_iteration(iteration, subproblem=subproblem, pareto_point=vec)
            if callback is not None:
                callback(iteration, self.hv, self.dominated_hv, self.discarded_hv, self.coverage, self.error)
            print(f"Ref {self.sign * subproblem.referent} - Found {self.sign * vec} - Time {time.time() - begin:.2f}s")
            print("---------------------")

        self.finish(start, iteration)
        return self.get_pareto_set(linear_subsolutions + subsolutions)
