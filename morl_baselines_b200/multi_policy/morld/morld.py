"""MORL/D (decomposition-based MORL) on the CUDA update engine -- drop-in for reference
morl_baselines/multi_policy/morld/morld.py with MOSAC or MOSACDiscrete inner learners (config 5 of BASELINE.json).

What changes under the API (SURVEY.md section 8, rows a13, a18, a19 and 8(e)):
  * the population shards across GPUs: policy p lives on rank ``p % world`` (one process per GPU, torch.distributed / NCCL);
    ``__update_others`` -- the strictly serial ``update_passes x (pop-1)`` learner updates of the reference (morld.py:423-433) --
    runs only over the rank's own policies, with no communication;
  * once per evaluation round every rank prunes its local evaluations + archive with the CUDA dominance kernel and the ranks
    exchange the fronts with ONE all-gather (parallel.allgather_fronts); every rank then holds the identical global front
    used for the metrics (hypervolume etc.);
  * ParetoArchive.add re-filters on the GPU (common/pareto.py).
EUPG, the reference's third inner learner (morld.py:30-34), is an on-policy ESR learner and is outside the accelerated path.
Single-process behaviour (world size 1) is the reference's.
"""

from __future__ import annotations

import math
import os
import time
from typing import Callable, List, Optional, Tuple, Union

import numpy as np
import torch as th
import torch.distributed as dist
from torch import optim

from ...common.graphed import GraphCache, PopulationGraph
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.networks import polyak_update
from ...common.pareto import ParetoArchive
from ...common.scalarization import tchebicheff, weighted_sum
from ...common.utils import nearest_neighbors
from ...common.weights import equally_spaced_weights, random_weights
from ...parallel import allgather_fronts
from ...single_policy.ser.mosac_continuous_action import MOSAC
from ...single_policy.ser.mosac_discrete_action import MOSACDiscrete

POLICIES = {"MOSAC": MOSAC, "MOSACDiscrete": MOSACDiscrete}


class Policy:
    """Individual of the population: id, weight vector, wrapped MOPolicy (reference morld.py:37-51)."""

    def __init__(self, id: int, weights: np.ndarray, wrapped: MOPolicy):
        self.id = id
        self.weights = weights
        self.wrapped = wrapped


def _world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


class MORLD(MOAgent):
    """MORL/D (Felten, Talbi, Danoy, JAIR 2024)."""

    def __init__(
        self,
        env,
        scalarization_method: str = "ws",
        evaluation_mode: str = "ser",
        policy_name: str = "MOSAC",
        policy_args: dict = {},
        gamma: float = 0.995,
        pop_size: int = 6,
        seed: int = 42,
        rng: Optional[np.random.Generator] = None,
        exchange_every: int = int(4e4),
        neighborhood_size: int = 1,
        dist_metric: Callable[[np.ndarray, np.ndarray], float] = lambda a, b: np.sum(np.square(a - b)),
        shared_buffer: bool = False,
        sharing_mechanism: List[str] = [],
        update_passes: int = 10,
        weight_init_method: str = "uniform",
        weight_adaptation_method: Optional[str] = None,
        project_name: str = "MORL-Baselines",
        experiment_name: str = "MORL-D",
        wandb_entity: Optional[str] = None,
        log: bool = True,
        device: Union[th.device, str] = "auto",
    ):
        self.env = env
        super().__init__(self.env, device, seed=seed)
        self.gamma = gamma
        self.seed = seed
        self.np_random = rng if rng is not None else np.random.default_rng(self.seed)
        try:  # reward normalisation wrapper of mo-gymnasium, applied per objective as in the reference (morld.py:119-121)
            from mo_gymnasium.wrappers import MONormalizeReward

            for i in range(env.unwrapped.reward_space.shape[0]):
                env = MONormalizeReward(env, idx=i)
        except Exception:
            pass
        self.evaluation_mode = evaluation_mode
        self.pop_size = pop_size
        self.weight_init_method = weight_init_method
        self.weight_adaptation_method = weight_adaptation_method
        self.delta = 0.1 if weight_adaptation_method == "PSA" else None
        if weight_init_method == "uniform":
            self.weights = np.array(equally_spaced_weights(self.reward_dim, self.pop_size, self.seed))
        elif weight_init_method == "random":
            self.weights = random_weights(self.reward_dim, n=self.pop_size, dist="dirichlet", rng=self.np_random)
        else:
            raise Exception(f"Unsupported weight init method: ${weight_init_method}")
        self.scalarization_method = scalarization_method
        if scalarization_method == "ws":
            self.scalarization = weighted_sum
        elif scalarization_method == "tch":
            self.scalarization = tchebicheff(tau=0.5, reward_dim=self.reward_dim)
        else:
            raise Exception(f"Unsupported scalarization method: ${scalarization_method}")
        self.neighborhood_size = neighborhood_size
        self.transfer = "transfer" in sharing_mechanism
        self.update_passes = update_passes
        self.exchange_every = exchange_every
        self.shared_buffer = shared_buffer
        self.dist_metric = dist_metric
        self.neighborhoods = [nearest_neighbors(n=neighborhood_size, current_weight=w, all_weights=self.weights, dist_metric=dist_metric)
                              for w in self.weights] if neighborhood_size > 0 else [[] for _ in self.weights]
        self.global_step = 0
        self.iteration = 0
        self.project_name = project_name
        self.experiment_name = experiment_name + f"({policy_name})"
        self.log = log
        if shared_buffer:
            self.experiment_name += "-SB"
        if weight_adaptation_method is not None:
            self.experiment_name += ("+" if shared_buffer else "-") + weight_adaptation_method
        if self.transfer:
            self.experiment_name += "+transfer"
        if policy_name not in POLICIES:
            raise NotImplementedError(f"inner policy {policy_name!r} is outside the accelerated path (MOSAC and MOSACDiscrete only; "
                                      "EUPG is an on-policy ESR learner, SURVEY.md section 2 #29)")
        self.policy_factory = POLICIES[policy_name]
        self.policy_name = policy_name
        self.policy_args = policy_args
        self.rank, self.world = _world()
        self.current_policy = 0
        self.population = [
            Policy(id=i, weights=w, wrapped=self.policy_factory(id=i, env=self.env, weights=w,
                                                                scalarization=th.matmul if scalarization_method == "ws" else self.scalarization,
                                                                gamma=gamma, log=self.log, seed=self.seed, parent_rng=self.np_random,
                                                                device=self.device, **policy_args))
            for i, w in enumerate(self.weights)
        ]
        self.archive = ParetoArchive()
        self.global_front = None
        self.population_graph = True  # replay a rank's learners as one multi-branch CUDA graph in _update_others
        self._pop_graphs = GraphCache()
        self._front_prune = None  # dominance test of the front exchange: None = the CUDA kernel (tests on CPU/gloo inject one)
        if self.log:
            self.setup_wandb(project_name=self.project_name, experiment_name=self.experiment_name, entity=wandb_entity)
        if self.shared_buffer:
            self._share_buffers()

    def get_config(self) -> dict:
        return {"env_id": self.env.unwrapped.spec.id, "scalarization_method": self.scalarization_method, "evaluation_mode": self.evaluation_mode,
                "gamma": self.gamma, "pop_size": self.pop_size, "exchange_every": self.exchange_every,
                "neighborhood_size": self.neighborhood_size, "shared_buffer": self.shared_buffer, "update_passes": self.update_passes,
                "transfer": self.transfer, "weight_init_method": self.weight_init_method, "weight_adapt_method": self.weight_adaptation_method,
                "delta_adapt": self.delta, "project_name": self.project_name, "experiment_name": self.experiment_name, "seed": self.seed,
                "log": self.log, "device": self.device, "policy_name": self.policy_name, **self.population[0].wrapped.get_config(),
                **self.policy_args}

    # ------------------------------------------------------------------------------------------ sharding helpers
    def owner(self, policy_id: int) -> int:
        """Rank that owns (updates and evaluates) a policy."""
        return policy_id % self.world

    def local_policies(self) -> List[Policy]:
        return [p for p in self.population if self.owner(p.id) == self.rank]

    def _share_buffers(self, neighborhood: bool = False):
        """Share replay buffers (reference morld.py:245-261)."""
        if neighborhood:
            for p in self.population:
                buf = p.wrapped.get_buffer()
                for n in self.neighborhoods[p.id]:
                    self.population[n].wrapped.set_buffer(buf)
        else:
            buf = self.population[0].wrapped.get_buffer()
            for p in self.population:
                p.wrapped.set_buffer(buf)

    def _select_candidate(self) -> Policy:
        """Turn-by-turn candidate selection (reference morld.py:263-269)."""
        candidate = self.population[self.current_policy]
        if self.current_policy + 1 == self.pop_size:
            self.iteration += 1
        self.current_policy = (self.current_policy + 1) % self.pop_size
        return candidate

    def _eval_policy(self, policy: Policy, eval_env, num_eval_episodes_for_front: int) -> np.ndarray:
        """Average discounted vector return (reference morld.py:271-304)."""
        acc = np.zeros(self.reward_dim)
        for _ in range(num_eval_episodes_for_front):
            if self.evaluation_mode == "ser":
                _, _, _, disc = policy.wrapped.policy_eval(eval_env, weights=policy.weights, scalarization=self.scalarization, log=self.log)
            elif self.evaluation_mode == "esr":
                _, _, _, disc = policy.wrapped.policy_eval_esr(eval_env, weights=policy.weights, scalarization=self.scalarization, log=self.log)
            else:
                raise Exception("Evaluation mode must either be esr or ser.")
            acc += disc
        return acc / num_eval_episodes_for_front

    def _eval_all_policies(self, eval_env, num_eval_episodes_for_front: int, num_eval_weights_for_eval: int, ref_point: np.ndarray,
                           known_front: Optional[List[np.ndarray]] = None):
        """Evaluate the (local) policies, update the archive, exchange fronts (reference morld.py:306-335 + 8(e))."""
        evals = [None] * self.pop_size
        for agent in self.local_policies():
            disc = self._eval_policy(agent, eval_env, num_eval_episodes_for_front)
            evals[agent.id] = disc
            self.archive.add(agent, disc)
        # ONE collective per round: the record of a rank carries its local non-dominated front AND the evaluations of the policies it owns
        # (every rank needs all of them for the weight adaptation); NaN marks the slots of policies other ranks own
        mine = np.full((self.pop_size, self.reward_dim), np.nan, dtype=np.float64)
        for p in self.local_policies():
            mine[p.id] = np.asarray(evals[p.id], dtype=np.float64)
        local = np.array(self.archive.evaluations, dtype=np.float64).reshape(-1, self.reward_dim)
        front, gathered = allgather_fronts(th.from_numpy(local).to(self.device), cap=max(64, 2 * self.pop_size), prune=self._front_prune,
                                           extras=th.from_numpy(mine.reshape(-1)).to(self.device))
        gathered = gathered.numpy().reshape(self.world, self.pop_size, self.reward_dim)
        for pid in range(self.pop_size):
            evals[pid] = gathered[self.owner(pid), pid]
        self.global_front = front.numpy()
        if self.log and self.rank == 0:
            from ...common.evaluation import log_all_multi_policy_metrics

            log_all_multi_policy_metrics(list(self.global_front), ref_point, self.reward_dim, self.global_step,
                                         n_sample_weights=num_eval_weights_for_eval, ref_front=known_front)
        return evals

    def _share(self, last_trained: Policy):
        """Neighbour weight transfer on the first iteration (reference morld.py:337-366)."""
        if self.transfer and self.iteration == 0:
            src = last_trained.wrapped.get_policy_net()
            for n in self.neighborhoods[last_trained.id]:
                if n > last_trained.id:
                    dst_policy = self.population[n]
                    dst = dst_policy.wrapped.get_policy_net()
                    polyak_update(params=src.parameters(), target_params=dst.parameters(), tau=1.0)
                    if hasattr(dst_policy.wrapped, "_graphs"):  # MOSAC(Discrete): capture-safe fused Adam; captured graphs reference the old optimiser
                        from ...common.fused_adam import FusedClipAdam

                        eps = getattr(dst_policy.wrapped, "ADAM_EPS", 1e-8)  # MOSACDiscrete's optimisers all use eps 1e-4, as its reference
                        dst_policy.wrapped.actor_optimizer = FusedClipAdam(dst.parameters(), lr=dst_policy.wrapped.policy_lr, eps=eps)
                        dst_policy.wrapped._graphs.clear()
                    else:
                        dst_policy.wrapped.actor_optimizer = optim.Adam(dst.parameters(), lr=dst_policy.wrapped.policy_lr)

    def _adapt_weights(self, evals: List[np.ndarray]):
        """PSA weight adaptation (reference morld.py:368-417)."""
        if self.weight_adaptation_method != "PSA":
            return
        front = self.global_front if self.global_front is not None else np.array(self.archive.evaluations)

        def closest_non_dominated(ev):
            best, best_d = None, math.inf
            for cand in front:
                d = np.sum(np.square(ev - cand))
                if best_d > d > 0.01:
                    best, best_d = cand, d
            return best

        for i, p in enumerate(self.population):
            ev = evals[i]
            closest = closest_non_dominated(ev)
            new_w = np.array(p.weights, dtype=np.float64)
            if closest is not None:
                for k in range(len(ev)):
                    new_w[k] = p.weights[k] * (1 + self.delta) if ev[k] >= closest[k] else p.weights[k] / (1 + self.delta)
            normalized = new_w / np.linalg.norm(new_w, ord=1)
            p.wrapped.set_weights(normalized)
            p.weights = normalized

    def _update_others(self, current: Policy):
        """``update_passes`` improvement passes over every policy except ``current`` (reference morld.py:423-433), restricted to the policies
        this rank owns -- the population is embarrassingly parallel across GPUs -- and, within a rank, replayed as ONE CUDA graph with
        parallel branches (common/graphed.PopulationGraph) instead of one graph replay per policy.  The host halves (replay-index draws
        from the global numpy RNG) run in the reference's policy order, so RNG consumption is unchanged."""
        pols = [p for p in self.local_policies() if len(p.wrapped.get_buffer()) > 0 and p != current]
        if not pols:
            return
        batched = self.population_graph and len(pols) > 1 and all(getattr(p.wrapped, "graph_update_ready", lambda: False)() for p in pols)
        for _ in range(self.update_passes):
            if not batched:
                for p in pols:
                    p.wrapped.update()
                continue
            variants = [p.wrapped._prepare_graph_update() for p in pols]
            key = tuple((p.id, v.key) for p, v in zip(pols, variants))
            pg = self._pop_graphs.get_or_build(key, lambda: PopulationGraph([v.step for v in variants],
                                                                            lambda pols=pols: [t for p in pols for t in p.wrapped._mutated_tensors()]))
            pg()

    def save(self, save_dir="weights/", filename=None, save_replay_buffer=True):
        """Save population and archive with the reference's keys (morld.py:435-457)."""
        os.makedirs(save_dir, exist_ok=True)
        filename = filename or "morld_save"
        params = {}
        for i, policy in enumerate(self.population):
            params[f"population_policy_{i}"] = policy.wrapped.get_save_dict(save_replay_buffer)
        for i, (policy, ev) in enumerate(zip(self.archive.individuals, self.archive.evaluations)):
            params[f"archive_policy_{i}"] = policy.wrapped.get_save_dict(save_replay_buffer=False)
            params[f"archive_policy_{i}_eval"] = ev
        th.save(params, os.path.join(save_dir, filename + ".tar"))

    def load(self, path, load_replay_buffer=True):
        params = th.load(path, map_location=self.device, weights_only=False)
        for i, policy in enumerate(self.population):
            key = f"population_policy_{i}"
            if key in params:
                policy.wrapped.load(params[key], load_replay_buffer=load_replay_buffer)
                policy.weights = policy.wrapped.weights
        self.archive.individuals, self.archive.evaluations = [], []
        i = 0
        import copy

        while f"archive_policy_{i}" in params and f"archive_policy_{i}_eval" in params and len(self.population) > 0:
            ap = copy.deepcopy(self.population[0])
            ap.wrapped.load(params[f"archive_policy_{i}"], load_replay_buffer=False)
            ap.weights = ap.wrapped.weights
            self.archive.individuals.append(ap)
            self.archive.evaluations.append(params[f"archive_policy_{i}_eval"])
            i += 1

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              num_eval_episodes_for_front: int = 5, num_eval_weights_for_eval: int = 50, reset_num_timesteps: bool = False,
              checkpoints: bool = True, save_freq: int = 10000):
        """Main loop (reference morld.py:494-584).  With several ranks the candidate's owner runs the environment interaction;
        every rank then improves and evaluates its own shard and the fronts are exchanged once per round."""
        if self.log:
            self.register_additional_config({"total_timesteps": total_timesteps, "ref_point": ref_point.tolist(),
                                             "known_front": known_pareto_front, "num_eval_weights_for_eval": num_eval_weights_for_eval,
                                             "num_eval_episodes_for_front": num_eval_episodes_for_front})
        self.global_step = 0 if reset_num_timesteps else self.global_step
        self.num_episodes = 0 if reset_num_timesteps else self.num_episodes
        start_time = time.time()
        self.env.reset()
        self._eval_all_policies(eval_env, num_eval_episodes_for_front, num_eval_weights_for_eval, ref_point, known_pareto_front)
        while self.global_step < total_timesteps:
            policy = self._select_candidate()
            if self.owner(policy.id) == self.rank:
                policy.wrapped.train(self.exchange_every, eval_env=eval_env, start_time=start_time)
            self.global_step += self.exchange_every
            for p in self.population:
                p.wrapped.global_step = self.global_step
            self._update_others(policy)
            evals = self._eval_all_policies(eval_env, num_eval_episodes_for_front, num_eval_weights_for_eval, ref_point, known_pareto_front)
            self._share(policy)
            self._adapt_weights(evals)
            if checkpoints and self.global_step % save_freq == 0 and self.rank == 0:
                self.save(filename=f"{self.experiment_name} step={self.global_step}", save_replay_buffer=False)
        if self.log:
            self.close_wandb()
