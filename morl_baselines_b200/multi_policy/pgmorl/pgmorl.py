"""Prediction-guided MORL (PGMORL, Xu et al., ICML 2020) on the CUDA update engine -- drop-in for reference
morl_baselines/multi_policy/pgmorl/pgmorl.py (``PerformancePredictor``, ``generate_weights``, ``PerformanceBuffer2d``,
``PerformanceBuffer3d`` and ``PGMORL`` with the same constructor, ``get_config`` and ``train``).  As in the reference, the
post-processing phase of the paper is not implemented.

The host logic is the reference's: the hyperbolic performance model is fitted by ``scipy.optimize.least_squares`` and tasks are scored
by the host hypervolume and sparsity.  The population's learning runs on the device:
  * every iteration runs all agents' rollouts one after the other, in the reference's order (they share one vector env, whose
    normalisation statistics carry from agent to agent), then all agents' updates as ONE ``PopulationGraph`` replay.  This equals the
    reference's rollout 0, update 0, rollout 1, ... because an update reads only its own agent's batch and network, a rollout never reads
    another agent's network, updates consume only numpy generators (the host draws the shuffles in agent order) and only rollouts consume
    torch's generator.  With ``target_kl`` set (one host read per epoch) the agents update one after the other.
  * task selection does not replace ``self.agents[i]``: the selected snapshot is written into slot ``i``'s existing tensors with a zeroed
    (fresh) Adam (``MOPPO.become_copy_of``), so the captured population graph stays valid.  The performance buffer and the archive hold
    deep copies, which never alias live parameters.

mo-gymnasium is resolved through the module-level helpers ``mo_make``, ``make_env`` and ``make_vector_env``.
"""

from __future__ import annotations

import time
from copy import deepcopy
from itertools import product
from typing import List, Optional, Tuple, Union

import numpy as np
import torch as th
from scipy.optimize import least_squares

from ...common.evaluation import log_all_multi_policy_metrics
from ...common.graphed import PopulationGraph
from ...common.morl_algorithm import MOAgent
from ...common.pareto import ParetoArchive
from ...common.performance_indicators import hypervolume, sparsity
from ...single_policy.ser.mo_ppo import MOPPO, MOPPONet, make_env


def mo_make(env_id: str, **kwargs):
    """``mo_gymnasium.make``."""
    import mo_gymnasium as mo_gym

    return mo_gym.make(env_id, **kwargs)


def make_vector_env(env_fns):
    """mo-gymnasium's synchronous vector env over the thunks ``env_fns``."""
    import mo_gymnasium as mo_gym

    return mo_gym.wrappers.vector.MOSyncVectorEnv(env_fns)


def _wandb_log(d):
    import wandb

    wandb.log(d)


class PerformancePredictor:
    """Predicts the evaluation a policy reaches after training with a weight, from the (weight, before, after) samples of earlier
    generations: one hyperbolic model per objective, fitted on the policy's neighbourhood (reference pgmorl.py:27-202)."""

    def __init__(self, neighborhood_threshold: float = 0.1, sigma: float = 0.03, A_bound_min: float = 1.0, A_bound_max: float = 500.0,
                 f_scale: float = 20.0):
        self.previous_performance, self.next_performance, self.used_weight = [], [], []
        self.neighborhood_threshold, self.A_bound_min, self.A_bound_max, self.f_scale, self.sigma = (neighborhood_threshold, A_bound_min,
                                                                                                      A_bound_max, f_scale, sigma)

    def add(self, weight: np.ndarray, eval_before_pg: np.ndarray, eval_after_pg: np.ndarray) -> None:
        self.previous_performance.append(eval_before_pg)
        self.next_performance.append(eval_after_pg)
        self.used_weight.append(weight)

    def _fit_and_predict(self, weights, deltas, next_perfs, dim: int, current_eval: np.ndarray, weight_candidate: np.ndarray, sigma: float):
        """Fit delta_dim = A tanh-like(a (w_dim - b)) + c on the neighbours, each weighted by a Gaussian of its distance to
        ``current_eval``, and evaluate it at the candidate weight."""
        x = np.array([w[dim] for w in weights])
        y = np.array([dl[dim] for dl in deltas])
        sw = np.array([np.exp(-((np.linalg.norm(np.abs(p - current_eval) / np.abs(current_eval)) / sigma) ** 2) / 2.0) for p in next_perfs])

        def model(p, xs):
            ex = np.exp(p[1] * (xs - p[2]))
            return p[0] * (ex - 1) / (ex + 1) + p[3]

        def residual(p, xs, ys):
            return (p[0] * (np.exp(p[1] * (xs - p[2])) - 1.0) / (np.exp(p[1] * (xs - p[2])) + 1) + p[3] - ys) * sw

        def jacobian(p, xs, ys):
            A, a, b = p[0], p[1], p[2]
            ex = np.exp(a * (xs - b))
            J = np.zeros([len(p), len(xs)])
            J[0] = ((ex - 1) / (ex + 1)) * sw
            J[1] = (A * (xs - b) * (2.0 * ex) / ((ex + 1) ** 2)) * sw
            J[2] = (A * (-a) * (2.0 * ex) / ((ex + 1) ** 2)) * sw
            J[3] = sw
            return np.transpose(J)

        # the amplitude's upper bound is the spread of the deltas clipped to [1, 500], as in the reference
        upper_A = np.clip(np.max(y) - np.min(y), 1.0, 500.0)
        fit = least_squares(residual, np.ones(4), loss="soft_l1", f_scale=self.f_scale, args=(x, y), jac=jacobian,
                            bounds=([0, 0.1, -5.0, -500.0], [upper_A, 20.0, 5.0, 500.0]))
        return model(fit.x, weight_candidate[dim])

    def predict_next_evaluation(self, weight_candidate: np.ndarray, policy_eval: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """(predicted delta, predicted next evaluation) of training ``policy_eval``'s policy with ``weight_candidate``.  The neighbourhood
        (and sigma) doubles until it holds at least 4 distinct samples."""
        nb_w, nb_delta, nb_next = [], [], []
        sigma, threshold = self.sigma / 2.0, self.neighborhood_threshold / 2.0
        while len(nb_w) < 4:
            sigma *= 2.0
            threshold *= 2.0
            if threshold == np.inf or sigma == np.inf:
                raise ValueError("Cannot find at least 4 neighbors by enlarging the neighborhood.")
            for prev, nxt, w in zip(self.previous_performance, self.next_performance, self.used_weight):
                if np.all(np.abs(prev - policy_eval) < threshold * np.abs(policy_eval)) and tuple(nxt) not in list(map(tuple, nb_next)):
                    nb_w.append(w)
                    nb_delta.append(nxt - prev)
                    nb_next.append(nxt)
        deltas = np.array([self._fit_and_predict(nb_w, nb_delta, nb_next, k, policy_eval, weight_candidate, sigma)
                           for k in range(weight_candidate.size)])
        return deltas, deltas + policy_eval


def generate_weights(delta_weight: float, dimensions: int = 2) -> np.ndarray:
    """Every weight vector on the grid of step ``delta_weight`` (float32) whose components sum to 1 (reference pgmorl.py:205-223)."""
    grid = np.arange(0.0, 1.0 + delta_weight, delta_weight, dtype=np.float32)
    combos = np.array(list(product(grid, repeat=dimensions)), dtype=np.float32)
    return combos[np.isclose(combos.sum(axis=1), 1.0)]


class _PerformanceBuffer:
    """Population store: ``num_bins`` bins of at most ``max_size`` individuals, each bin sorted by ascending norm of the evaluation
    shifted by ``origin`` (the worst is dropped first).  Individuals are stored as deep copies."""

    def __init__(self, max_size: int, origin: np.ndarray):
        self.max_size = max_size
        self.origin = -origin

    def _init_bins(self):
        self.bins = [[] for _ in range(self.num_bins)]
        self.bins_evals = [[] for _ in range(self.num_bins)]

    @property
    def evaluations(self) -> List[np.ndarray]:
        return [e for b in self.bins_evals for e in b]

    @property
    def individuals(self) -> list:
        return [i for b in self.bins for i in b]

    def _centered(self, evaluation):
        return np.clip(evaluation + self.origin, 0.0, float("inf"))

    def _insert(self, bin_id: int, candidate, evaluation, norm_eval):
        pos = len(self.bins_evals[bin_id])
        for k, existing in enumerate(self.bins_evals[bin_id]):
            if norm_eval < np.linalg.norm(self._centered(existing)):
                pos = k
                break
        self.bins[bin_id].insert(pos, deepcopy(candidate))
        self.bins_evals[bin_id].insert(pos, evaluation)
        if len(self.bins[bin_id]) > self.max_size:
            self.bins[bin_id].pop(0)
            self.bins_evals[bin_id].pop(0)


class PerformanceBuffer2d(_PerformanceBuffer):
    """Two objectives: bins are equal sectors of the angle in the positive quadrant (reference pgmorl.py:226-296)."""

    def __init__(self, num_bins: int, max_size: int, origin: np.ndarray):
        super().__init__(max_size, origin)
        self.num_bins = num_bins
        self.dtheta = np.pi / 2.0 / self.num_bins
        self._init_bins()

    def add(self, candidate, evaluation: np.ndarray):
        c = self._centered(evaluation)
        norm_eval = np.linalg.norm(c)
        bin_id = int(np.arccos(np.clip(c[1] / (norm_eval + 1e-3), -1.0, 1.0)) // self.dtheta)
        if 0 <= bin_id < self.num_bins:
            self._insert(bin_id, candidate, evaluation, norm_eval)


class PerformanceBuffer3d(_PerformanceBuffer):
    """Three objectives: one bin per unit direction of a ``num_bins - 1`` simplex grid; an evaluation goes to the direction with the
    largest dot product (reference pgmorl.py:299-368)."""

    def __init__(self, num_bins: int, max_size: int, origin: np.ndarray):
        super().__init__(max_size, origin)
        self.pbuffer_vec = generate_weights(1.0 / (num_bins - 1), 3)
        for i in range(len(self.pbuffer_vec)):
            self.pbuffer_vec[i] = self.pbuffer_vec[i] / np.linalg.norm(self.pbuffer_vec[i])
        self.num_bins = len(self.pbuffer_vec)
        self._init_bins()

    def add(self, candidate, evaluation: np.ndarray):
        c = self._centered(evaluation)
        best, bin_id = -np.inf, -1
        for i in range(self.num_bins):
            dot = np.dot(self.pbuffer_vec[i], c)
            if dot > best:
                best, bin_id = dot, i
        self._insert(bin_id, candidate, evaluation, np.linalg.norm(c))


class PGMORL(MOAgent):
    """Prediction-Guided Multi-Objective Reinforcement Learning (J. Xu, Y. Tian, P. Ma, D. Rus, S. Sueda, W. Matusik, ICML 2020)."""

    def __init__(self, env_id: str, origin: np.ndarray, num_envs: int = 4, pop_size: int = 6, warmup_iterations: int = 80,
                 steps_per_iteration: int = 2048, evolutionary_iterations: int = 20, num_weight_candidates: int = 7,
                 num_performance_buffer: int = 100, performance_buffer_size: int = 2, min_weight: float = 0.0, max_weight: float = 1.0,
                 delta_weight: float = 0.2, sparsity_coef: float = -1.0, env=None, gamma: float = 0.995, project_name: str = "MORL-baselines",
                 experiment_name: str = "PGMORL", wandb_entity: Optional[str] = None, seed: Optional[int] = None, log: bool = True,
                 net_arch: List = [64, 64], num_minibatches: int = 32, update_epochs: int = 10, learning_rate: float = 3e-4,
                 anneal_lr: bool = False, clip_coef: float = 0.2, ent_coef: float = 0.0, vf_coef: float = 0.5, clip_vloss: bool = True,
                 max_grad_norm: float = 0.5, norm_adv: bool = True, target_kl: Optional[float] = None, gae: bool = True, gae_lambda: float = 0.95,
                 device: Union[th.device, str] = "auto", group: Optional[str] = None):
        super().__init__(env, device=device, seed=seed)
        self.tmp_env = mo_make(env_id)
        self.extract_env_info(self.tmp_env)
        self.env_id, self.num_envs = env_id, num_envs
        assert hasattr(self.action_space, "low"), "only continuous action space is supported"
        if hasattr(self.tmp_env, "close"):
            self.tmp_env.close()
        self.gamma = gamma
        self.pop_size, self.warmup_iterations, self.steps_per_iteration = pop_size, warmup_iterations, steps_per_iteration
        self.evolutionary_iterations, self.num_weight_candidates = evolutionary_iterations, num_weight_candidates
        self.min_weight, self.max_weight, self.delta_weight, self.sparsity_coef = min_weight, max_weight, delta_weight, sparsity_coef
        self.num_performance_buffer, self.performance_buffer_size = num_performance_buffer, performance_buffer_size
        self.archive = ParetoArchive()
        if self.reward_dim == 2:
            self.population = PerformanceBuffer2d(num_bins=num_performance_buffer, max_size=performance_buffer_size, origin=origin)
        elif self.reward_dim == 3:
            self.population = PerformanceBuffer3d(num_bins=num_performance_buffer, max_size=performance_buffer_size, origin=origin)
        else:
            raise ValueError("Only 2D and 3D objectives are supported.")
        self.predictor = PerformancePredictor()

        self.net_arch = net_arch
        self.batch_size = int(self.num_envs * self.steps_per_iteration)
        self.num_minibatches = num_minibatches
        self.minibatch_size = int(self.batch_size // self.num_minibatches)
        self.update_epochs, self.learning_rate, self.anneal_lr, self.clip_coef = update_epochs, learning_rate, anneal_lr, clip_coef
        self.vf_coef, self.ent_coef, self.max_grad_norm, self.norm_adv = vf_coef, ent_coef, max_grad_norm, norm_adv
        self.target_kl, self.clip_vloss, self.gae_lambda, self.gae = target_kl, clip_vloss, gae_lambda, gae

        if env is not None:
            raise ValueError("Environments should be vectorized for PPO. You should provide an environment id instead.")
        self.env = make_vector_env([make_env(env_id, (self.seed if self.seed is not None else 0) + i, i, experiment_name, self.gamma)
                                    for i in range(self.num_envs)])

        self.log = log
        if self.log:
            self.setup_wandb(project_name, experiment_name, wandb_entity, group)

        self.networks = [MOPPONet(self.observation_shape, self.action_space.shape, self.reward_dim, self.net_arch).to(self.device)
                         for _ in range(self.pop_size)]
        weights = generate_weights(self.delta_weight, self.reward_dim)
        print(f"Warmup phase - sampled weights: {weights}")
        self.agents = [MOPPO(i, self.networks[i], weights[i], self.env, log=self.log, gamma=self.gamma, device=self.device, seed=self.seed,
                             steps_per_iteration=self.steps_per_iteration, num_minibatches=self.num_minibatches, update_epochs=self.update_epochs,
                             learning_rate=self.learning_rate, anneal_lr=self.anneal_lr, clip_coef=self.clip_coef, ent_coef=self.ent_coef,
                             vf_coef=self.vf_coef, clip_vloss=self.clip_vloss, max_grad_norm=self.max_grad_norm, norm_adv=self.norm_adv,
                             target_kl=self.target_kl, gae=self.gae, gae_lambda=self.gae_lambda, rng=self.np_random)
                       for i in range(self.pop_size)]
        self._population_graph = None

    def get_config(self) -> dict:
        return {"env_id": self.env_id, "num_envs": self.num_envs, "pop_size": self.pop_size, "warmup_iterations": self.warmup_iterations,
                "evolutionary_iterations": self.evolutionary_iterations, "num_weight_candidates": self.num_weight_candidates,
                "num_performance_buffer": self.num_performance_buffer, "performance_buffer_size": self.performance_buffer_size,
                "min_weight": self.min_weight, "max_weight": self.max_weight, "delta_weight": self.delta_weight,
                "sparsity_coef": self.sparsity_coef, "gamma": self.gamma, "seed": self.seed, "net_arch": self.net_arch,
                "batch_size": self.batch_size, "minibatch_size": self.minibatch_size, "update_epochs": self.update_epochs,
                "learning_rate": self.learning_rate, "anneal_lr": self.anneal_lr, "clip_coef": self.clip_coef, "vf_coef": self.vf_coef,
                "ent_coef": self.ent_coef, "max_grad_norm": self.max_grad_norm, "norm_adv": self.norm_adv, "target_kl": self.target_kl,
                "clip_vloss": self.clip_vloss, "gae": self.gae, "gae_lambda": self.gae_lambda}

    # ---- one iteration of the population ----------------------------------------------------------------------------------------
    def _update_all_agents(self):
        """Every agent's update, in agent order; as ONE population-graph replay when the agents update without early stopping."""
        if self.target_kl is not None or not all(a.use_cuda_graph for a in self.agents):
            for a in self.agents:
                a.update()
            return
        steps = [a.prepare_update().step for a in self.agents]  # host: shuffles drawn in agent order
        if self._population_graph is None:
            agents = list(self.agents)
            self._population_graph = PopulationGraph(steps, lambda: [t for a in agents for t in a._mutated_tensors()])
        self._population_graph()
        if self.log:
            for a in self.agents:
                a._log_update()

    def __train_all_agents(self, iteration: int, max_iterations: int):
        for agent in self.agents:
            agent.global_step = self.global_step
            agent.rollout(iteration, max_iterations)
            self.global_step += self.steps_per_iteration * self.num_envs
        self._update_all_agents()
        if self.log:
            _wandb_log({"charts/SPS": int(self.global_step / (time.time() - self.start_time)), "global_step": self.global_step})

    def __eval_all_agents(self, eval_env, evaluations_before_train: List[np.ndarray], ref_point: np.ndarray,
                          known_pareto_front: Optional[List[np.ndarray]] = None, add_to_prediction: bool = True):
        """Evaluate every agent; store the result in the population buffer, the archive and (after training) the predictor."""
        for i, agent in enumerate(self.agents):
            _, _, _, discounted_reward = agent.policy_eval(eval_env, weights=agent.np_weights, log=self.log)
            self.population.add(agent, discounted_reward)
            self.archive.add(agent, discounted_reward)
            if add_to_prediction:
                self.predictor.add(agent.weights.detach().cpu().numpy(), evaluations_before_train[i], discounted_reward)
            evaluations_before_train[i] = discounted_reward
        if self.log:
            print("Current pareto archive:")
            print(self.archive.evaluations)
            log_all_multi_policy_metrics(current_front=self.archive.evaluations, hv_ref_point=ref_point, reward_dim=self.reward_dim,
                                         global_step=self.global_step, n_sample_weights=self.num_eval_weights_for_eval, ref_front=known_pareto_front)

    def __task_weight_selection(self, ref_point: np.ndarray):
        """Greedily choose, for each agent slot, the (population member, weight) pair whose predicted evaluation most improves
        hypervolume + sparsity_coef * sparsity of the front extended by the earlier choices (reference pgmorl.py:652-731)."""
        candidate_weights = generate_weights(self.delta_weight / 2.0, self.reward_dim)
        self.np_random.shuffle(candidate_weights)
        current_front = deepcopy(self.archive.evaluations)
        population, population_eval = self.population.individuals, self.population.evaluations
        selected_tasks = []
        for i in range(len(self.agents)):
            max_improv, best_candidate, best_eval, best_predicted_eval = float("-inf"), None, None, None
            for candidate, last_eval in zip(population, population_eval):
                cand_weights = [w for w in candidate_weights if (tuple(last_eval), tuple(w)) not in selected_tasks]
                predicted = [self.predictor.predict_next_evaluation(w, last_eval)[1] for w in cand_weights]
                hvs = [hypervolume(ref_point, current_front + [p]) for p in predicted]
                sps = [sparsity(current_front + [p]) for p in predicted]
                mixture = [hv + self.sparsity_coef * sp for hv, sp in zip(hvs, sps)]
                if self.log:
                    _wandb_log({"metrics/hypervolume_improvement": np.mean(hvs), "metrics/sparsity_improvement": np.mean(sps),
                                "metrics/mixture_improvement": np.mean(mixture), "global_step": self.global_step})
                k = int(np.argmax(np.array(mixture)))
                if max_improv < np.max(np.array(mixture)):
                    max_improv = np.max(np.array(mixture))
                    best_candidate, best_eval, best_predicted_eval = (candidate, cand_weights[k]), last_eval, predicted[k]
            selected_tasks.append((tuple(best_eval), tuple(best_candidate[1])))
            current_front.append(best_predicted_eval)
            # the reference assigns deepcopy(candidate) to the slot; the copy is written into the slot's own tensors instead
            slot = self.agents[i]
            step = slot.global_step
            slot.become_copy_of(best_candidate[0])
            slot.global_step, slot.id = step, i
            slot.change_weights(deepcopy(best_candidate[1]))
            print(f"Agent #{slot.id} - weights {best_candidate[1]}")
            print(f"current eval: {best_eval} - estimated next: {best_predicted_eval} - deltas {(best_predicted_eval - best_eval)}")

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              num_eval_weights_for_eval: int = 50):
        """Warm-up iterations on the initial weights, then generations of task selection followed by ``evolutionary_iterations``
        iterations (reference pgmorl.py:733-819)."""
        if self.log:
            self.register_additional_config({"total_timesteps": total_timesteps, "ref_point": ref_point.tolist(), "known_front": known_pareto_front,
                                             "num_eval_weights_for_eval": num_eval_weights_for_eval})
        self.num_eval_weights_for_eval = num_eval_weights_for_eval
        max_iterations = total_timesteps // self.steps_per_iteration // self.num_envs // self.pop_size
        iteration = 0
        current_evaluations = [np.zeros(self.reward_dim) for _ in range(len(self.agents))]
        self.__eval_all_agents(eval_env, current_evaluations, ref_point, known_pareto_front, add_to_prediction=False)
        self.start_time = time.time()
        for i in range(1, self.warmup_iterations + 1):
            print(f"Warmup iteration #{iteration}, global step: {self.global_step}")
            if self.log:
                _wandb_log({"charts/warmup_iterations": i, "global_step": self.global_step})
            self.__train_all_agents(iteration=iteration, max_iterations=max_iterations)
            iteration += 1
        self.__eval_all_agents(eval_env, current_evaluations, ref_point, known_pareto_front)

        max_iterations = max(max_iterations, self.warmup_iterations + self.evolutionary_iterations)
        generation = 1
        while iteration < max_iterations:
            self.__task_weight_selection(ref_point=ref_point)
            print(f"Evolutionary generation #{generation}")
            if self.log:
                _wandb_log({"charts/evolutionary_generation": generation, "global_step": self.global_step})
            for _ in range(self.evolutionary_iterations):
                if self.log:
                    print(f"Evolutionary iteration #{iteration - self.warmup_iterations}")
                    _wandb_log({"charts/evolutionary_iterations": iteration - self.warmup_iterations, "global_step": self.global_step})
                self.__train_all_agents(iteration=iteration, max_iterations=max_iterations)
                iteration += 1
            self.__eval_all_agents(eval_env, current_evaluations, ref_point, known_pareto_front)
            generation += 1
        print("Done training!")
        self.env.close()
        if self.log:
            self.close_wandb()
