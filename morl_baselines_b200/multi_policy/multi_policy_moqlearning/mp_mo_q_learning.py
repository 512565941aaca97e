"""Multi-policy scalarised Q-learning (reference multi_policy/multi_policy_moqlearning/mp_mo_q_learning.py) with its inner learner's Dyna-Q
(reference single_policy/ser/mo_q_learning.py and common/model_based/tabular_model.py) on the device table of csrc/moq.cu.

Every policy's Q-table, the shared Dyna model and its priority sum tree live on the device (:class:`moq_ops.MoqTable`); the keys live in
one host index (:class:`moq_ops.MoqIndex`).  An environment step is at most two launches: the greedy (or GPI) action when the ε coin says
greedy, and the step itself (TD update, GPI-PD priority, model update and every Dyna update).  The random draws stay on the host, from the
reference's generators in the reference's order, and reach the kernels by value, so a seeded run takes the reference's actions and its
tables are bit-identical.

Documented differences from the reference:
- ``q_table`` is a read-only host snapshot ``{state tuple: float64 [A, d]}`` of the visited states, keyed by python scalars and ordered by
  the first time any policy saw the state, not by this policy's insertion order.
- ``model`` is the shared device table, not a host ``TabularModel``.
- Only ``weighted_sum`` scalarisation is supported (``NotImplementedError`` otherwise).
- ``gpi_pd=True`` or ``use_gpi_policy=True`` without a parent raises ``ValueError`` (the reference fails with ``AttributeError`` at the
  first step).
- Without CUDA the classes raise ``MorlB200Error``.
- ``equally_spaced_weights`` is computed only when ``log`` is on; it consumes no global draws either way.
- With ``log`` on, the inner learner logs ε but not the TD error, which stays on the device.
"""

from __future__ import annotations

import time
from copy import deepcopy
from typing import List, Optional

import numpy as np
import torch as th

from ... import moq_ops
from ..._lib import MorlB200Error
from ...common.evaluation import log_all_multi_policy_metrics, policy_evaluation_mo
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.scalarization import weighted_sum
from ...common.utils import linearly_decaying_value
from ...common.weights import equally_spaced_weights, random_weights
from ..linear_support.linear_support import LinearSupport


def _need_cuda(who: str):
    if not th.cuda.is_available():
        raise MorlB200Error(f"morl_baselines_b200.{who} needs a CUDA device: the Q-tables are CUDA-only (no CPU fallback)")


def _check_scalarization(scalarization):
    if scalarization is not weighted_sum:
        raise NotImplementedError("only weighted_sum scalarisation is supported: the device tables scalarise with w . q")


class MoqStore:
    """The state shared by the policies of one agent: the host index, the device table and pinned buffers for the act round trip."""

    def __init__(self, action_dim: int, reward_dim: int, model: bool):
        self.index = moq_ops.MoqIndex()
        self.table = moq_ops.MoqTable(action_dim, reward_dim, th.device("cuda"), model)
        self.n_policies = 0
        self._out = th.empty((moq_ops.ACT_ROWS, 2), dtype=th.int32, pin_memory=True)
        self._value = th.empty(moq_ops.ACT_ROWS, dtype=th.float64, pin_memory=True)
        self._status = th.empty(2, dtype=th.int32, pin_memory=True)

    def add_policy(self) -> int:
        p = self.n_policies
        self.table.reserve(P=p + 1)
        self.table.clear_policy(p)
        self.n_policies += 1
        return p

    def act(self, states, policies, w):
        """(actions, visited, values) of greedy rows, copied back with the status word behind one synchronisation."""
        n = len(states)
        if n > self._out.shape[0]:
            self._out = th.empty((n, 2), dtype=th.int32, pin_memory=True)
            self._value = th.empty(n, dtype=th.float64, pin_memory=True)
        out, value = moq_ops.moq_act(self.table, self.n_policies, states, policies, w)
        self._out[:n].copy_(out, non_blocking=True)
        self._value[:n].copy_(value, non_blocking=True)
        self._status.copy_(self.table.status, non_blocking=True)
        th.cuda.current_stream().synchronize()
        moq_ops.check_status(self.table, self._status.numpy())
        o = self._out[:n].numpy()
        return o[:, 0].copy(), o[:, 1].copy(), self._value[:n].numpy().copy()

    def check_status(self):
        moq_ops.check_status(self.table)


class DeviceMOQLearning(MOPolicy, MOAgent):
    """Scalarised Q-learning for one weight vector (reference MOQLearning), on one policy slot of a :class:`MoqStore`.

    Paper: K. Van Moffaert, M. Drugan, and A. Nowe, Scalarized Multi-Objective Reinforcement Learning: Novel Design Techniques. 2013.
    """

    def __init__(self, env, id: Optional[int] = None, weights: np.ndarray = np.array([0.5, 0.5]), scalarization=weighted_sum,
                 learning_rate: float = 0.1, gamma: float = 0.9, initial_epsilon: float = 0.1, final_epsilon: float = 0.1,
                 epsilon_decay_steps: int = None, learning_starts: int = 0, use_gpi_policy: bool = False, dyna: bool = False,
                 dyna_updates: int = 5, model: Optional[MoqStore] = None, gpi_pd: bool = False, min_priority: float = 0.0001, alpha: float = 0.6,
                 parent=None, project_name: str = "MORL-baselines", experiment_name: str = "MO Q-Learning", wandb_entity: Optional[str] = None,
                 log: bool = True, seed: Optional[int] = None, parent_rng: Optional[np.random.Generator] = None):
        """Same arguments, in the same order, as the reference constructor (mo_q_learning.py:26-52).  ``model``: a shared
        :class:`MoqStore` (the parent passes its own)."""
        _need_cuda("DeviceMOQLearning")
        _check_scalarization(scalarization)
        if parent is None and (gpi_pd or use_gpi_policy):
            raise ValueError("gpi_pd and use_gpi_policy need a parent MPMOQLearning (its policies are the GPI set)")
        MOAgent.__init__(self, env, device="cuda")
        MOPolicy.__init__(self, id, device="cuda")
        self.learning_rate = learning_rate
        self.id, self.seed = id, seed
        self.np_random = parent_rng if parent_rng is not None else np.random.default_rng(seed)
        self.idstr = "" if id is None else f"_{id}"
        self.gamma = gamma
        self.initial_epsilon, self.epsilon, self.final_epsilon = initial_epsilon, initial_epsilon, final_epsilon
        self.epsilon_decay_steps, self.learning_starts = epsilon_decay_steps, learning_starts
        self.use_gpi_policy, self.dyna, self.dyna_updates, self.gpi_pd = use_gpi_policy, dyna, dyna_updates, gpi_pd
        self.min_priority, self.alpha = min_priority, alpha
        self.parent = parent
        self.weights = weights
        self.scalarization = scalarization
        store = parent._store if parent is not None else model
        self._store = store if store is not None else MoqStore(self.action_dim, self.reward_dim, dyna)
        if dyna and not self._store.table.model:
            raise ValueError("dyna=True needs a store created with a model")
        self.slot = self._store.add_policy()
        self.log = log
        if self.log and parent_rng is None:
            self.setup_wandb(project_name, experiment_name, wandb_entity)

    @property
    def model(self) -> Optional[MoqStore]:
        """The shared device model (the store), or None without Dyna."""
        return self._store if self.dyna else None

    @property
    def q_table(self) -> dict:
        """Host snapshot ``{state tuple: float64 [A, d]}`` of the states this policy visited (global first-seen order)."""
        t, idx = self._store.table, self._store.index
        n = len(idx.states)
        vis = t.visited[:n, self.slot].cpu().numpy()
        q = t.q[:n, self.slot].cpu().numpy()
        return {idx.states[s]: q[s].copy() for s in range(n) if vis[s]}

    def _act(self, obs) -> int:
        """ε-greedy action (reference mo_q_learning.py:123-129): one draw of the policy's generator per step."""
        if self.np_random.random() < self.epsilon:
            return int(self.env.action_space.sample())
        return self.eval(obs, self.weights)

    @staticmethod
    def _state_to_tuple(obs) -> tuple:
        return moq_ops.state_key(obs)

    def scalarized_q_values(self, obs, w: np.ndarray) -> np.ndarray:
        """Scalarised Q value of every action for the observation and weights (reference :137-142); a host read of one row."""
        s = self._store.index.find(obs)
        if s < 0 or not bool(self._store.table.visited[s, self.slot]):
            return np.zeros(self.action_dim)
        return np.array([self.scalarization(v, w) for v in self._store.table.q[s, self.slot].cpu().numpy()])

    def eval(self, obs, w: Optional[np.ndarray] = None) -> int:
        """Greedy action under the policy's own weights (reference :160-171: ``w`` only goes to a GPI parent); a state the policy never
        visited gets a random action from the environment's sampler."""
        if self.use_gpi_policy:
            return self.parent.eval(obs, w)
        act, seen, _ = self._store.act([self._store.index.find(obs)], [self.slot], np.asarray(self.weights, dtype=np.float64))
        if not seen[0]:
            return int(self.env.action_space.sample())
        return int(act[0])

    def update(self):
        """One step on ``self.obs / action / reward / next_obs / terminated`` (reference :173-227): one device launch (one per 64 Dyna
        updates) after the host draws of the Dyna updates."""
        st = self._store
        s = st.index.add_state(self.obs)
        s2 = st.index.add_state(self.next_obs)
        st.table.reserve(S=len(st.index.states))
        flags = (moq_ops.GPI if self.use_gpi_policy else 0) | (moq_ops.MODEL if self.dyna else 0) | (moq_ops.PRIORITIZE if self.gpi_pd else 0)
        kw = {}
        if self.dyna:
            m, o = st.index.add_outcome(s, int(self.action), s2, self.reward, self.terminated)
            n_pairs = len(st.index.pairs)
            st.table.reserve(M=n_pairs, K=o + 1)
            pick, u, choice = moq_ops.dyna_draws(self.dyna_updates, n_pairs, self.gpi_pd)
            kw = dict(pair=m, outcome=o, n_pairs=n_pairs, pick=pick, u=u, choice=choice)
        moq_ops.moq_step(st.table, st.n_policies, self.slot, s, int(self.action), s2, bool(self.terminated), np.asarray(self.weights, dtype=np.float64),
                         np.asarray(self.reward, dtype=np.float64), flags, self.gamma, self.learning_rate, self.min_priority, self.alpha, **kw)
        if self.epsilon_decay_steps is not None:
            self.epsilon = linearly_decaying_value(self.initial_epsilon, self.epsilon_decay_steps, self.global_step, self.learning_starts,
                                                   self.final_epsilon)
        if self.log and self.global_step % 1000 == 0:
            import wandb

            wandb.log({f"charts{self.idstr}/epsilon": self.epsilon, "global_step": self.global_step})

    def get_config(self) -> dict:
        return {"env_id": self.env.unwrapped.spec.id, "learning_rate": self.learning_rate, "gamma": self.gamma,
                "initial_epsilon": self.initial_epsilon, "final_epsilon": self.final_epsilon, "epsilon_decay_steps": self.epsilon_decay_steps,
                "use_gpi_policy": self.use_gpi_policy, "dyna": self.dyna, "dyna_updates": self.dyna_updates, "gpi_pd": self.gpi_pd,
                "min_priority": self.min_priority, "alpha": self.alpha, "weight": self.weights, "scalarization": self.scalarization.__name__,
                "seed": self.seed}

    def train(self, start_time, total_timesteps: int = int(5e5), reset_num_timesteps: bool = True, eval_env=None, eval_freq: int = 1000):
        """Interaction loop (reference :249-311): act, step, update, reset at episode ends.  A walk beyond the model's pairs raises
        MorlB200Error at the next greedy step or at the end."""
        self.obs, _ = self.env.reset()
        self.global_step = 0 if reset_num_timesteps else self.global_step
        self.num_episodes = 0 if reset_num_timesteps else self.num_episodes
        for _ in range(1, total_timesteps + 1):
            self.global_step += 1
            self.action = self._act(self.obs)
            self.next_obs, self.reward, self.terminated, self.truncated, info = self.env.step(self.action)
            self.update()
            if eval_env is not None and self.log and self.global_step % eval_freq == 0:
                self.policy_eval(eval_env, scalarization=self.scalarization, weights=self.weights, log=self.log)
            if self.terminated or self.truncated:
                self.obs, _ = self.env.reset()
                self.num_episodes += 1
                if self.log and self.global_step % 1000 == 0:
                    import wandb

                    wandb.log({f"charts{self.idstr}/SPS": int(self.global_step / (time.time() - start_time)), "global_step": self.global_step})
            else:
                self.obs = self.next_obs
        self._store.check_status()


class MPMOQLearning(MOAgent):
    """Multi-policy MOQ-Learning: outer loop of scalarised Q-learning over weight vectors (random, OLS or GPI-LS).

    Paper: K. Van Moffaert, M. Drugan, and A. Nowe, Scalarized Multi-Objective Reinforcement Learning: Novel Design Techniques. 2013.
    """

    def __init__(self, env, scalarization=weighted_sum, learning_rate: float = 0.1, gamma: float = 0.9, initial_epsilon: float = 0.1,
                 final_epsilon: float = 0.1, epsilon_decay_steps: int = None, weight_selection_algo: str = "random", epsilon_ols: Optional[float] = None,
                 use_gpi_policy: bool = False, transfer_q_table: bool = True, dyna: bool = False, dyna_updates: int = 5, gpi_pd: bool = False,
                 project_name: str = "MORL-Baselines", experiment_name: str = "MultiPolicy MO Q-Learning", wandb_entity: Optional[str] = None,
                 seed: Optional[int] = None, log: bool = True):
        """Same arguments, in the same order, as the reference constructor (mp_mo_q_learning.py:28-72)."""
        _need_cuda("MPMOQLearning")
        _check_scalarization(scalarization)
        MOAgent.__init__(self, env, device="cuda", seed=seed)
        self.scalarization = scalarization
        self.learning_rate = learning_rate
        self.gamma = gamma
        self.initial_epsilon = initial_epsilon
        self.final_epsilon = final_epsilon
        self.epsilon_decay_steps = epsilon_decay_steps
        self.use_gpi_policy = use_gpi_policy
        self.dyna = dyna
        self.dyna_updates = dyna_updates
        self.gpi_pd = gpi_pd
        self.transfer_q_table = transfer_q_table
        self.policies = []
        self.weight_selection_algo = weight_selection_algo
        self.epsilon_ols = epsilon_ols
        assert self.weight_selection_algo in ["random", "ols", "gpi-ls"], f"Unknown weight selection algorithm: {self.weight_selection_algo}."
        self.linear_support = LinearSupport(num_objectives=self.reward_dim, epsilon=epsilon_ols)
        self._store = MoqStore(self.action_dim, self.reward_dim, dyna)
        self.project_name = project_name
        self.experiment_name = experiment_name
        self.log = log
        if self.log:
            self.setup_wandb(project_name=self.project_name, experiment_name=self.experiment_name, entity=wandb_entity)

    def get_config(self) -> dict:
        return {"env_id": self.env.unwrapped.spec.id, "learning_rate": self.learning_rate, "gamma": self.gamma,
                "initial_epsilon": self.initial_epsilon, "final_epsilon": self.final_epsilon, "epsilon_decay_steps": self.epsilon_decay_steps,
                "scalarization": self.scalarization.__name__, "use_gpi_policy": self.use_gpi_policy,
                "weight_selection_algo": self.weight_selection_algo, "epsilon_ols": self.epsilon_ols, "transfer_q_table": self.transfer_q_table,
                "dyna": self.dyna, "dyna_updates": self.dyna_updates, "gpi_pd": self.gpi_pd, "seed": self.seed}

    def _gpi_row(self, states, w):
        w = np.asarray(w, dtype=np.float64).reshape(len(states), -1)
        return self._store.act([self._store.index.find(s) for s in states], [-1] * len(states), w)

    def _gpi_action(self, state, w: np.ndarray) -> int:
        """GPI(s, w) = argmax_a max_pi Q^pi(s, a) . w: the first maximum of the stacked [policies, actions] values (one launch)."""
        return int(self._gpi_row([state], w)[0][0])

    def max_scalar_q_value(self, state, w: np.ndarray) -> float:
        """Maximum scalarised Q value over all policies and actions for the state and weights (one launch)."""
        return float(self._gpi_row([state], w)[2][0])

    def eval(self, obs, w: Optional[np.ndarray] = None) -> int:
        """The GPI action with use_gpi_policy; otherwise the action of the CCS policy best for w."""
        if self.use_gpi_policy:
            return self._gpi_action(obs, w)
        best_policy = np.argmax([np.dot(w, v) for v in self.linear_support.ccs])
        return self.policies[best_policy].eval(obs, w)

    @property
    def eval_batch(self):
        """``eval_batch(obs [N, ...], w [N, d]) -> actions [N]``: the GPI action of every row, in one round trip.  Exists only with
        use_gpi_policy: without GPI an unvisited state draws a random action, and lockstep evaluation would reorder those draws."""
        if not self.use_gpi_policy:
            raise AttributeError("eval_batch needs use_gpi_policy=True")
        return self._eval_batch

    def _eval_batch(self, obs, w) -> np.ndarray:
        obs = np.asarray(obs)
        return self._gpi_row([obs[i] for i in range(obs.shape[0])], w)[0].astype(np.int64)

    def delete_policies(self, delete_indx: List[int]):
        """Delete the policies with the given indices (their slots are compacted out of the device table)."""
        for i in sorted(delete_indx, reverse=True):
            self.policies.pop(i)
        keep = [p.slot for p in self.policies]
        if keep != list(range(self._store.n_policies)):
            self._store.table.keep_policies(keep)
            for j, p in enumerate(self.policies):
                p.slot = j
        self._store.n_policies = len(self.policies)

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              timesteps_per_iteration: int = int(2e5), num_eval_weights_for_front: int = 100, num_eval_episodes_for_front: int = 5,
              num_eval_weights_for_eval: int = 50, eval_freq: int = 1000):
        """Learn a set of policies (reference mp_mo_q_learning.py:158-279)."""
        if self.log:
            self.register_additional_config({"total_timesteps": total_timesteps, "ref_point": ref_point.tolist(), "known_front": known_pareto_front,
                                             "timesteps_per_iteration": timesteps_per_iteration,
                                             "num_eval_weights_for_front": num_eval_weights_for_front,
                                             "num_eval_episodes_for_front": num_eval_episodes_for_front,
                                             "num_eval_weights_for_eval": num_eval_weights_for_eval, "eval_freq": eval_freq})
        num_iterations = int(total_timesteps / timesteps_per_iteration)
        if eval_env is None:
            eval_env = deepcopy(self.env)
        eval_weights = equally_spaced_weights(self.reward_dim, n=num_eval_weights_for_front) if self.log else None

        for iter in range(num_iterations):
            if self.weight_selection_algo == "ols" or self.weight_selection_algo == "gpi-ls":
                w = self.linear_support.next_weight(algo=self.weight_selection_algo,
                                                    gpi_agent=self if self.weight_selection_algo == "gpi-ls" else None,
                                                    env=eval_env if self.weight_selection_algo == "gpi-ls" else None,
                                                    rep_eval=num_eval_episodes_for_front)
                if w is None:
                    print("OLS has no more corner weights to try. Using a random weight instead.")
                    w = random_weights(self.reward_dim, rng=self.np_random)
            elif self.weight_selection_algo == "random":
                w = random_weights(self.reward_dim, rng=self.np_random)

            new_agent = DeviceMOQLearning(env=self.env, id=iter, weights=w, scalarization=self.scalarization, learning_rate=self.learning_rate,
                                          gamma=self.gamma, initial_epsilon=self.initial_epsilon, final_epsilon=self.final_epsilon,
                                          epsilon_decay_steps=self.epsilon_decay_steps, use_gpi_policy=self.use_gpi_policy, dyna=self.dyna,
                                          dyna_updates=self.dyna_updates, gpi_pd=self.gpi_pd, parent=self, log=self.log,
                                          parent_rng=self.np_random, seed=self.seed)
            if self.transfer_q_table and len(self.policies) > 0:
                reuse_ind = np.argmax([np.dot(w, v) for v in self.linear_support.ccs])
                self._store.table.copy_policy(self.policies[reuse_ind].slot, new_agent.slot)
            self.policies.append(new_agent)

            start_time = time.time()
            new_agent.global_step = self.global_step
            new_agent.train(start_time=start_time, total_timesteps=timesteps_per_iteration, reset_num_timesteps=False, eval_freq=eval_freq,
                            eval_env=eval_env)
            self.global_step = new_agent.global_step

            value = policy_evaluation_mo(agent=new_agent, env=eval_env, w=w, rep=num_eval_episodes_for_front)[3]
            removed_inds = self.linear_support.add_solution(value, w)
            if self.weight_selection_algo != "random":
                self.delete_policies(removed_inds)

            if self.log:
                if self.use_gpi_policy:
                    front = [policy_evaluation_mo(agent=self, env=eval_env, w=w_eval, rep=num_eval_episodes_for_front)[3] for w_eval in eval_weights]
                else:
                    front = self.linear_support.ccs
                log_all_multi_policy_metrics(current_front=front, hv_ref_point=ref_point, reward_dim=self.reward_dim, global_step=self.global_step,
                                             n_sample_weights=num_eval_weights_for_eval, ref_front=known_pareto_front)

        if self.log:
            self.close_wandb()
