"""Pareto Q-learning (reference multi_policy/pareto_q_learning/pql.py) on the device set table of csrc/pql.cu.

The stored sets ND[s][a], the average rewards and the visit counts live on the device (:class:`pql_ops.PqlTable`).  Each step is one
launch of the exact set update; a greedy step adds one launch of the action scores and one device-to-host copy of them.  The agent's random
draws stay on the host and are the reference's, in the reference's order, so a seeded run takes the reference's actions.  The stored sets
and averages are bit-identical to the reference's float64 arithmetic.

One documented difference: ``track_policy`` scans the vectors stored for one action in the table's canonical order (descending coordinate
sum, then lexicographically descending), not in Python-set iteration order.  The tracked action and target differ from the reference's only
when two stored vectors of the same action are equally close to the target, or both lie within ``tol`` of it.
"""

from __future__ import annotations

import numbers
from typing import Callable, List, Optional

import numpy as np
import torch as th

from ... import pql_ops
from ..._lib import MorlB200Error
from ...common.evaluation import log_all_multi_policy_metrics
from ...common.morl_algorithm import MOAgent
from ...common.utils import linearly_decaying_value


def _non_dominated(candidates: set) -> set:
    """The points of a set of tuples that no distinct point is >= in every coordinate (the kernels' prune)."""
    if len(candidates) == 0:
        return set()
    pts = np.array(list(candidates), dtype=np.float64)
    ge = np.all(pts[None, :, :] >= pts[:, None, :], axis=-1)
    eq = np.all(pts[None, :, :] == pts[:, None, :], axis=-1)
    keep = ~np.any(ge & ~eq, axis=1)
    return {tuple(p) for p in pts[keep].tolist()}


class _Snapshot:
    """One host copy of the device table."""

    def __init__(self, t: pql_ops.PqlTable):
        self.counts = t.counts.cpu().numpy()
        self.avg_reward = t.avg_reward.cpu().numpy()
        self.nd_count = t.nd_count.cpu().numpy()
        self.nd = t.nd.cpu().numpy()

    def stored(self, s: int, a: int) -> np.ndarray:
        return self.nd[s, a, : self.nd_count[s, a]]


class PQL(MOAgent):
    """Pareto Q-learning.

    Tabular method relying on pareto pruning.
    Paper: K. Van Moffaert and A. Nowé, “Multi-objective reinforcement learning using sets of pareto dominating policies,” The Journal of
    Machine Learning Research, vol. 15, no. 1, pp. 3483–3512, 2014.
    """

    def __init__(
        self,
        env,
        ref_point: np.ndarray,
        gamma: float = 0.8,
        initial_epsilon: float = 1.0,
        epsilon_decay_steps: int = 100000,
        final_epsilon: float = 0.1,
        seed: Optional[int] = None,
        project_name: str = "MORL-Baselines",
        experiment_name: str = "Pareto Q-Learning",
        wandb_entity: Optional[str] = None,
        log: bool = True,
        max_set_size: int = 64,
    ):
        """Initialize the Pareto Q-learning algorithm.

        Args:
            env: The environment.
            ref_point: The reference point for the hypervolume metric.
            gamma: The discount factor.
            initial_epsilon: The initial epsilon value.
            epsilon_decay_steps: The number of steps to decay epsilon.
            final_epsilon: The final epsilon value.
            seed: The random seed.
            project_name: The name of the project used for logging.
            experiment_name: The name of the experiment used for logging.
            wandb_entity: The wandb entity used for logging.
            log: Whether to log or not.
            max_set_size: Capacity K of every stored set ND[s][a].  A step whose set would need more points raises MorlB200Error at the
                next check (a greedy step, an episode end or the end of ``train``), naming the size it needs.
        """
        if not th.cuda.is_available():
            raise MorlB200Error("morl_baselines_b200.PQL needs a CUDA device: the set table is CUDA-only (no CPU fallback)")
        super().__init__(env, device="cuda", seed=seed)
        # Learning parameters
        self.gamma = gamma
        self.epsilon = initial_epsilon
        self.initial_epsilon = initial_epsilon
        self.epsilon_decay_steps = epsilon_decay_steps
        self.final_epsilon = final_epsilon

        # Algorithm setup
        self.ref_point = ref_point

        self._classify_spaces()
        self.num_objectives = self.env.unwrapped.reward_space.shape[0]
        self.max_set_size = int(max_set_size)
        self._table = pql_ops.PqlTable(self.num_states, self.num_actions, self.max_set_size, self.num_objectives, th.device("cuda"))
        self._scores_host = th.empty(self.num_actions, dtype=th.float64, pin_memory=True)
        self._status_host = th.empty(3, dtype=th.int32, pin_memory=True)

        # Logging
        self.project_name = project_name
        self.experiment_name = experiment_name
        self.log = log

        if self.log:
            self.setup_wandb(
                project_name=self.project_name,
                experiment_name=self.experiment_name,
                entity=wandb_entity,
            )

    def _classify_spaces(self):
        """Number of actions, state shape and number of states from the spaces, recognised by their attributes (gymnasium's spaces and
        their stand-ins alike), as the reference's constructor classifies them (pql.py:64-86)."""
        act = self.env.action_space
        if hasattr(act, "nvec"):
            self.num_actions = int(np.prod(act.nvec))
        elif hasattr(act, "n") and tuple(getattr(act, "shape", ())) == ():
            self.num_actions = int(act.n)
        else:
            raise Exception("PQL only supports (multi)discrete action spaces.")

        obs = self.env.observation_space
        if hasattr(obs, "nvec"):
            self.env_shape = obs.nvec
        elif hasattr(obs, "n") and tuple(getattr(obs, "shape", ())) == ():
            self.env_shape = (obs.n,)
        elif (
            hasattr(obs, "low")
            and hasattr(obs, "high")
            and np.all(np.isfinite(obs.low))
            and np.all(np.isfinite(obs.high))
            and issubclass(np.dtype(obs.dtype).type, numbers.Integral)
        ):
            low_bound = np.array(obs.low)
            high_bound = np.array(obs.high)
            self.env_shape = high_bound - low_bound + 1
        else:
            raise Exception("PQL only supports discretizable observation spaces.")

        self.num_states = int(np.prod(self.env_shape))

    # ---- host snapshots of the device table ----------------------------------------------------------------------------------------------
    @property
    def counts(self) -> np.ndarray:
        """Visit counts [S, A] (float64, as the reference keeps them)."""
        return self._table.counts.cpu().numpy()

    @property
    def avg_reward(self) -> np.ndarray:
        """Average immediate rewards [S, A, d]."""
        return self._table.avg_reward.cpu().numpy()

    @property
    def non_dominated(self) -> list:
        """ND[s][a] as the reference keeps it: a list (states) of lists (actions) of sets of float64 tuples."""
        snap = _Snapshot(self._table)
        return [[{tuple(v) for v in snap.stored(s, a).tolist()} for a in range(self.num_actions)] for s in range(self.num_states)]

    def get_config(self) -> dict:
        """Get the configuration dictionary.

        Returns:
            Dict: A dictionary of parameters and values.
        """
        return {
            "env_id": self.env.unwrapped.spec.id,
            "ref_point": list(self.ref_point),
            "gamma": self.gamma,
            "initial_epsilon": self.initial_epsilon,
            "epsilon_decay_steps": self.epsilon_decay_steps,
            "final_epsilon": self.final_epsilon,
            "seed": self.seed,
        }

    def _check_status(self):
        pql_ops.check_status(self._table)

    def _scores(self, state: int, mode: int) -> np.ndarray:
        """Device scores of ``state``, copied back together with the overflow status behind one synchronisation."""
        dev = pql_ops.pql_score(self._table, state, mode, self.gamma, self.ref_point if mode == pql_ops.HYPERVOLUME else None)
        self._scores_host.copy_(dev, non_blocking=True)
        self._status_host.copy_(self._table.status, non_blocking=True)
        th.cuda.current_stream().synchronize()
        pql_ops.check_status(self._table, self._status_host.numpy())
        return self._scores_host.numpy().copy()

    def score_pareto_cardinality(self, state: int):
        """Compute the action scores based upon the Pareto cardinality metric.

        Args:
            state (int): The current state.

        Returns:
            ndarray: A score per action.
        """
        return self._scores(state, pql_ops.CARDINALITY)

    def score_hypervolume(self, state: int):
        """Compute the action scores based upon the hypervolume metric.

        Args:
            state (int): The current state.

        Returns:
            A list with a score per action.
        """
        return self._scores(state, pql_ops.HYPERVOLUME).tolist()

    def get_q_set(self, state: int, action: int):
        """Compute the Q-set for a given state-action pair.

        Args:
            state (int): The current state.
            action (int): The action.

        Returns:
            A set of Q vectors.
        """
        nd_array = self._table.nd[state, action, : int(self._table.nd_count[state, action])].cpu().numpy()
        q_array = self._table.avg_reward[state, action].cpu().numpy() + self.gamma * nd_array
        return {tuple(vec) for vec in q_array.tolist()}

    def select_action(self, state: int, score_func: Callable):
        """Select an action in the current state.

        Args:
            state (int): The current state.
            score_func (callable): A function that returns a score per action.

        Returns:
            int: The selected action.
        """
        if self.np_random.uniform(0, 1) < self.epsilon:
            return self.np_random.integers(self.num_actions)
        else:
            action_scores = score_func(state)
            return self.np_random.choice(np.argwhere(action_scores == np.max(action_scores)).flatten())

    def calc_non_dominated(self, state: int):
        """Get the non-dominated vectors in a given state.

        Args:
            state (int): The current state.

        Returns:
            Set: A set of Pareto non-dominated vectors.
        """
        candidates = set().union(*[self.get_q_set(state, action) for action in range(self.num_actions)])
        return _non_dominated(candidates)

    def _get_state_index(self, state: int | np.ndarray) -> int:
        if np.issubdtype(type(state), np.integer):
            return int(state)
        return int(np.ravel_multi_index(state, self.env_shape))

    def train(
        self,
        total_timesteps: int,
        eval_env,
        ref_point: Optional[np.ndarray] = None,
        known_pareto_front: Optional[List[np.ndarray]] = None,
        num_eval_weights_for_eval: int = 50,
        log_every: Optional[int] = 10000,
        action_eval: Optional[str] = "hypervolume",
    ):
        """Learn the Pareto front.

        Args:
            total_timesteps (int, optional): The number of episodes to train for.
            eval_env (gym.Env): The environment to evaluate the policies on.
            ref_point (ndarray, optional): The reference point for the hypervolume metric during evaluation. If none, use the same ref
                point as training.  Action scores always use the constructor's ``ref_point``.
            known_pareto_front (List[ndarray], optional): The optimal Pareto front, if known.
            num_eval_weights_for_eval (int): Number of weights use when evaluating the Pareto front, e.g., for computing expected utility.
            log_every (int, optional): Log the results every number of timesteps. (Default value = 1000)
            action_eval (str, optional): The action evaluation function name. (Default value = 'hypervolume')

        Returns:
            Set: The final Pareto front.
        """
        if action_eval == "hypervolume":
            score_func = self.score_hypervolume
        elif action_eval == "pareto_cardinality":
            score_func = self.score_pareto_cardinality
        else:
            raise Exception("No other method implemented yet")
        if not pql_ops.pql_supported(self.num_actions, self.max_set_size, self.num_objectives, pql_ops.MODES[action_eval]):
            raise MorlB200Error(f"PQL: {action_eval} scores are not supported for {self.num_actions} actions, max_set_size="
                                f"{self.max_set_size} and {self.num_objectives} objectives (hypervolume scores need at most 4 objectives)")
        if ref_point is None:
            ref_point = self.ref_point
        if self.log:
            self.register_additional_config(
                {
                    "total_timesteps": total_timesteps,
                    "ref_point": ref_point.tolist(),
                    "known_front": known_pareto_front,
                    "num_eval_weights_for_eval": num_eval_weights_for_eval,
                    "log_every": log_every,
                    "action_eval": action_eval,
                }
            )

        while self.global_step < total_timesteps:
            state, _ = self.env.reset()
            state = self._get_state_index(state)
            terminated = False
            truncated = False

            while not (terminated or truncated) and self.global_step < total_timesteps:
                action = self.select_action(state, score_func)
                next_state, reward, terminated, truncated, _ = self.env.step(action)
                self.global_step += 1
                next_state = self._get_state_index(next_state)

                pql_ops.pql_update(self._table, state, action, next_state, np.asarray(reward, dtype=np.float64), self.gamma)
                state = next_state

                if self.log and self.global_step % log_every == 0:
                    import wandb

                    wandb.log({"global_step": self.global_step})
                    pf = self._eval_all_policies(eval_env)
                    log_all_multi_policy_metrics(
                        current_front=pf,
                        hv_ref_point=ref_point,
                        reward_dim=self.reward_dim,
                        global_step=self.global_step,
                        n_sample_weights=num_eval_weights_for_eval,
                        ref_front=known_pareto_front,
                    )

            self.epsilon = linearly_decaying_value(
                self.initial_epsilon,
                self.epsilon_decay_steps,
                self.global_step,
                0,
                self.final_epsilon,
            )
            self._check_status()

        self._check_status()
        return self.get_local_pcs(state=0)

    def _eval_all_policies(self, env) -> List[np.ndarray]:
        """Evaluate all learned policies by tracking them, on one host snapshot of the table."""
        snap = _Snapshot(self._table)
        pf = []
        for vec in self._local_pcs(snap, 0):
            pf.append(self._track(snap, vec, env))

        return pf

    def track_policy(self, vec, env, tol=1e-3):
        """Track a policy from its return vector.

        Args:
            vec (array_like): The return vector to track.
            env (gym.Env): The environment to track the policy in.
            tol (float, optional): The tolerance for the return vector. (Default value = 1e-3)
        """
        return self._track(_Snapshot(self._table), vec, env, tol)

    def _track(self, snap: _Snapshot, vec, env, tol=1e-3):
        target = np.array(vec)
        state, _ = env.reset()
        terminated = False
        truncated = False
        total_rew = np.zeros(self.num_objectives)
        current_gamma = 1.0

        while not (terminated or truncated):
            state = self._get_state_index(state)
            closest_dist = np.inf
            closest_action = 0
            found_action = False
            new_target = target

            for action in range(self.num_actions):
                im_rew = snap.avg_reward[state, action]
                non_dominated_set = snap.stored(state, action)

                for q in non_dominated_set:
                    q = np.array(q)
                    dist = np.sum(np.abs(self.gamma * q + im_rew - target))
                    if dist < closest_dist:
                        closest_dist = dist
                        closest_action = action
                        new_target = q

                        if dist < tol:
                            found_action = True
                            break

                if found_action:
                    break

            state, reward, terminated, truncated, _ = env.step(closest_action)
            total_rew += current_gamma * reward
            current_gamma *= self.gamma
            target = new_target

        return total_rew

    def _local_pcs(self, snap: _Snapshot, state: int) -> set:
        candidates = set()
        for action in range(self.num_actions):
            q_array = snap.avg_reward[state, action] + self.gamma * snap.stored(state, action)
            candidates |= {tuple(vec) for vec in q_array.tolist()}
        return _non_dominated(candidates)

    def get_local_pcs(self, state: int = 0):
        """Collect the local PCS in a given state.

        Args:
            state (int): The state to get a local PCS for. (Default value = 0)

        Returns:
            Set: A set of Pareto optimal vectors.
        """
        return self._local_pcs(_Snapshot(self._table), state)
