"""Pareto Conditioned Networks on the CUDA update engine -- drop-in for reference morl_baselines/multi_policy/pcn/pcn.py
(``crowding_distance``, ``Transition``, ``BasePCNModel``, ``DiscreteActionsDefaultModel``, ``ContinuousActionsDefaultModel`` and ``PCN``
with the same constructor arguments, public methods and state-dict keys).

What runs where:
  * Episodes live in a device transition pool (``EpisodeStore``): each episode's observations, return-to-go and actions are appended
    with one host-to-device copy.  The host keeps only the heap the reference keeps, as ``(score, step, slot)`` entries driven by
    ``heapq`` exactly as the reference drives ``(score, step, transitions)`` (``EpisodeHeap``), so minibatch positions, evictions and
    the ranking are the reference's.
  * Ranking (crowding distance, non-dominated mask, distance to the front, penalties) stays on the host in numpy: the heap order depends
    on these float32 scores bit for bit, and there are a few hundred episodes at most.
  * An update is one kernel pair (``morl_pcn_update_f32``: gather, forward, loss, backward into the ``.grad`` storages) and one fused
    Adam step.  ``train()`` draws the indices of all ``num_model_updates`` updates up front, in the reference's order, uploads them once
    and replays ONE CUDA graph for the block (``use_cuda_graph``); loss and entropy are read back once per iteration.
  * ``_act`` runs the forward kernel on one row through pinned host memory; sampling stays on the host with the reference's generators.

The fused kernels cover the default models inside ``ops.pcn_supported``; a user-supplied ``model_class`` or a shape outside that range
runs the same learner with the model evaluated eagerly by torch on the same device store, without graph capture (an arbitrary model
may not be capturable).

Differences from the reference, each deliberate:
  * ``load()`` also rebuilds the optimiser on the loaded model (the reference keeps optimising the replaced model's parameters);
  * ``update()`` returns detached tensors.
"""

from __future__ import annotations

import heapq
import os
from abc import ABC
from dataclasses import dataclass
from typing import Callable, List, Optional, Type, Union

import numpy as np
import torch as th
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.morl_algorithm import MOAgent, MOPolicy, _is_discrete
from ...common.pareto import get_non_dominated_inds


def crowding_distance(points: np.ndarray) -> np.ndarray:
    """Crowding distance of each point (reference pcn.py:22-38): per objective, the gap between the two neighbours in sorted order of the
    min-max normalised points (1 for the extremes), summed over objectives."""
    norm = (points - points.min(axis=0)) / (np.ptp(points, axis=0) + 1e-8)
    order = np.argsort(norm, axis=0)
    ranked = np.take_along_axis(norm, order, axis=0)
    gaps = np.pad(np.abs(ranked[:-2] - ranked[2:]), ((1,), (0,)), constant_values=1)
    per_dim = np.zeros(norm.shape)
    per_dim[order, np.arange(norm.shape[-1])] = gaps
    return np.sum(per_dim, axis=-1)


def return_to_go(rewards: np.ndarray, gamma: float) -> np.ndarray:
    """Discounted return-to-go of an episode's float32 rewards [L, d], in place, in the reference's order (pcn.py:239-241)."""
    for i in reversed(range(len(rewards) - 1)):
        rewards[i] += gamma * rewards[i + 1]
    return rewards


def front_distance_scores(points: np.ndarray, non_dominated: np.ndarray, crowded: np.ndarray) -> np.ndarray:
    """Negative distance of each point to the closest point of the front ``points[non_dominated]``, 1e-5 less for all but the first copy
    of each front point, doubled where the crowding distance is small (reference pcn.py:250-268)."""
    front = points[non_dominated]
    diff = np.tile(np.expand_dims(points, 1), (1, len(front), 1)) - front
    scores = np.min(np.linalg.norm(diff, axis=-1), axis=-1) * -1
    front_i = np.nonzero(non_dominated)[0]
    _, first = np.unique(front, axis=0, return_index=True)
    duplicate = np.ones(len(scores), dtype=bool)
    duplicate[front_i[first]] = False
    scores[duplicate] -= 1e-5
    scores[crowded] *= 2
    return scores


def pcn_scores(returns: np.ndarray, threshold: float) -> np.ndarray:
    """PCN's episode scores: distance to the Pareto front of the returns with the crowding penalty."""
    crowded = np.argwhere(crowding_distance(returns) <= threshold).flatten()
    return front_distance_scores(returns, get_non_dominated_inds(returns), crowded)


def pcn_front(returns: np.ndarray) -> np.ndarray:
    """Mask of the returns PCN conditions on (pcn.py:279)."""
    return get_non_dominated_inds(returns)


def draw_update_indices(rng: np.random.Generator, lengths: np.ndarray, batch_size: int, n_updates: int):
    """The minibatch draws of ``n_updates`` consecutive reference updates (pcn.py:205-211): per update, ``batch_size`` heap positions from
    ``rng.choice`` and then one timestep per sample from ``rng.integers(0, len(episode))``.  Returns positions and timesteps [U, B]."""
    n = len(lengths)
    pos = np.empty((n_updates, batch_size), dtype=np.int64)
    t = np.empty((n_updates, batch_size), dtype=np.int64)
    for u in range(n_updates):
        pos[u] = rng.choice(np.arange(n), size=batch_size, replace=True)
        # one call with a vector of bounds consumes the generator exactly as the reference's per-sample scalar calls do
        t[u] = rng.integers(0, lengths[pos[u]])
    return pos, t


class EpisodeHeap:
    """The reference's experience-replay heap with the transitions replaced by store slots: a list of ``(score, step, slot)`` that
    ``heapq`` drives exactly as the reference drives ``(score, step, transitions)``, plus each slot's return and length."""

    def __init__(self):
        self.entries: list = []
        self.returns: dict = {}  # slot -> float32 return of the episode's first step
        self.lengths: dict = {}

    def __len__(self):
        return len(self.entries)

    def add(self, slot: int, ret0: np.ndarray, length: int, step: int, max_size: int) -> Optional[int]:
        """Push a new episode with score 1 (pcn.py:242-248); returns the slot that left the heap, if any."""
        self.returns[slot], self.lengths[slot] = ret0, int(length)
        if len(self.entries) == max_size:
            out = heapq.heappushpop(self.entries, (1, step, slot))[2]
            del self.returns[out], self.lengths[out]
            return out
        heapq.heappush(self.entries, (1, step, slot))
        return None

    def episode_returns(self, entries=None) -> np.ndarray:
        return np.array([self.returns[e[2]] for e in (self.entries if entries is None else entries)])

    def episode_lengths(self, entries=None) -> np.ndarray:
        return np.array([self.lengths[e[2]] for e in (self.entries if entries is None else entries)], dtype=np.int64)

    def nlargest(self, n: int, scores: np.ndarray) -> list:
        """The ``n`` best entries by ``scores`` (one per heap position), then every score is written into the heap and it is heapified
        (pcn.py:270-276)."""
        order = np.argsort(scores)
        largest = [self.entries[i] for i in order[-n:]]
        for i in range(len(scores)):
            self.entries[i] = (scores[i], self.entries[i][1], self.entries[i][2])
        heapq.heapify(self.entries)
        return largest


class EpisodeStore:
    """Device transition pool f32 [capacity, S + d + action columns] (obs | return-to-go | action, a discrete action as int32 bits), one
    row per transition, episodes contiguous.  Appending never reallocates unless the live rows need more room; then ``on_realloc`` runs
    (captured graphs read the pool's storage).  Space freed by evicted episodes is reclaimed by compacting in place."""

    def __init__(self, obs_dim: int, reward_dim: int, action_cols: int, discrete: bool, device, on_realloc: Callable[[], None],
                 capacity: int = 4096):
        self.S, self.d, self.ac, self.discrete = obs_dim, reward_dim, action_cols, discrete
        self.ld = obs_dim + reward_dim + action_cols
        self.device, self.on_realloc = device, on_realloc
        self.pool = th.zeros((capacity, self.ld), dtype=th.float32, device=device)
        self.tail = 0
        self.start: dict = {}  # slot -> first row
        self.length: dict = {}
        self._next_slot = 0
        self._pin = th.zeros((0, self.ld), dtype=th.float32)
        self._copied = th.cuda.Event()

    def _staging(self, rows: int) -> np.ndarray:
        self._copied.synchronize()  # the previous episode's copy has read the pinned rows
        if self._pin.shape[0] < rows:
            self._pin = th.zeros((max(rows, 2 * self._pin.shape[0]), self.ld), dtype=th.float32).pin_memory()
        return self._pin.numpy()[:rows]

    def add(self, obs: np.ndarray, actions: np.ndarray, rtg: np.ndarray) -> int:
        L = len(obs)
        if self.tail + L > self.pool.shape[0]:
            self._make_room(L)
        host = self._staging(L)
        S, d = self.S, self.d
        host[:, :S] = obs.reshape(L, S)
        host[:, S:S + d] = rtg
        if self.discrete:
            host.view(np.int32)[:, S + d] = actions.reshape(L)
        else:
            host[:, S + d:] = actions.reshape(L, self.ac)
        self.pool[self.tail:self.tail + L].copy_(self._pin[:L], non_blocking=True)
        self._copied.record()
        slot = self._next_slot
        self._next_slot += 1
        self.start[slot], self.length[slot] = self.tail, L
        self.tail += L
        return slot

    def remove(self, slot: int):
        del self.start[slot], self.length[slot]

    def _make_room(self, rows: int):
        live = sum(self.length.values())
        slots = sorted(self.start, key=self.start.get)
        idx = th.from_numpy(np.concatenate([np.arange(self.start[s], self.start[s] + self.length[s]) for s in slots] or [np.zeros(0, np.int64)]))
        idx = idx.to(self.device)
        if 2 * (live + rows) > self.pool.shape[0]:  # keep at least half the pool free after the move, so compactions stay rare
            pool = th.zeros((max(2 * self.pool.shape[0], 2 * (live + rows)), self.ld), dtype=th.float32, device=self.device)
            pool[:live] = self.pool.index_select(0, idx)
            self.pool = pool
            self.on_realloc()
        else:
            self.pool[:live] = self.pool.index_select(0, idx)
        row = 0
        for s in slots:
            self.start[s] = row
            row += self.length[s]
        self.tail = live


@dataclass
class Transition:
    """Transition dataclass."""

    observation: np.ndarray
    action: Union[float, int]
    reward: np.ndarray
    next_observation: np.ndarray
    terminal: bool


class BasePCNModel(nn.Module, ABC):
    """Base model of PCN (reference pcn.py:51-72): ``forward(state, desired_return, desired_horizon)``."""

    def __init__(self, state_dim: int, action_dim: int, reward_dim: int, scaling_factor: np.ndarray, hidden_dim: int):
        super().__init__()
        self.state_dim = state_dim
        self.action_dim = action_dim
        self.reward_dim = reward_dim
        self.scaling_factor = nn.Parameter(th.tensor(scaling_factor).float(), requires_grad=False)
        self.hidden_dim = hidden_dim

    def forward(self, state, desired_return, desired_horizon):
        """Log-probabilities of the actions, or the action itself for continuous actions."""
        c = th.cat((desired_return, desired_horizon), dim=-1) * self.scaling_factor
        return self.fc(self.s_emb(state.float()) * self.c_emb(c))


class DiscreteActionsDefaultModel(BasePCNModel):
    """PCN model for discrete actions (reference pcn.py:75-89)."""

    def __init__(self, state_dim: int, action_dim: int, reward_dim: int, scaling_factor: np.ndarray, hidden_dim: int):
        super().__init__(state_dim, action_dim, reward_dim, scaling_factor, hidden_dim)
        self.s_emb = nn.Sequential(nn.Linear(self.state_dim, self.hidden_dim), nn.Sigmoid())
        self.c_emb = nn.Sequential(nn.Linear(self.reward_dim + 1, self.hidden_dim), nn.Sigmoid())
        self.fc = nn.Sequential(nn.Linear(self.hidden_dim, self.hidden_dim), nn.ReLU(), nn.Linear(self.hidden_dim, self.action_dim),
                                nn.LogSoftmax(dim=1))


class ContinuousActionsDefaultModel(BasePCNModel):
    """PCN model for continuous actions (reference pcn.py:92-103)."""

    def __init__(self, state_dim: int, action_dim: int, reward_dim: int, scaling_factor: np.ndarray, hidden_dim: int):
        super().__init__(state_dim, action_dim, reward_dim, scaling_factor, hidden_dim)
        self.s_emb = nn.Sequential(nn.Linear(self.state_dim, self.hidden_dim), nn.Sigmoid())
        self.c_emb = nn.Sequential(nn.Linear(self.reward_dim + 1, self.hidden_dim), nn.Sigmoid())
        self.fc = nn.Sequential(nn.Linear(self.hidden_dim, self.hidden_dim), nn.ReLU(), nn.Linear(self.hidden_dim, self.action_dim))


DEFAULT_MODELS = (DiscreteActionsDefaultModel, ContinuousActionsDefaultModel)


def default_model_tensors(model: BasePCNModel) -> List[th.Tensor]:
    """The 8 trainable tensors of a default model in the kernels' order (state-dict order)."""
    return [model.s_emb[0].weight, model.s_emb[0].bias, model.c_emb[0].weight, model.c_emb[0].bias, model.fc[0].weight, model.fc[0].bias,
            model.fc[2].weight, model.fc[2].bias]


class PCN(MOAgent, MOPolicy):
    """Pareto Conditioned Networks (Reymond, Bargiacchi & Nowé, AAMAS 2022) on the CUDA update engine (reference pcn.py:106-503)."""

    experiment_default = "PCN"
    checkpoint_every = 1000  # train() saves and evaluates every total_timesteps / checkpoint_every steps

    def __init__(self, env, scaling_factor: np.ndarray, learning_rate: float = 1e-3, gamma: float = 1.0, batch_size: int = 256,
                 hidden_dim: int = 64, noise: float = 0.1, project_name: str = "MORL-Baselines", experiment_name: str = "PCN",
                 wandb_entity: Optional[str] = None, log: bool = True, seed: Optional[int] = None, device: Union[th.device, str] = "auto",
                 model_class: Optional[Type[BasePCNModel]] = None, use_cuda_graph: bool = True) -> None:
        MOAgent.__init__(self, env, device=device, seed=seed)
        MOPolicy.__init__(self, device=device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error(f"morl_baselines_b200.{type(self).__name__} needs a CUDA device: the update path is CUDA-only")
        ops._lib.load()
        self._init_common(scaling_factor, learning_rate, gamma, batch_size, hidden_dim, noise, model_class, use_cuda_graph)
        self.log = log
        if log:
            experiment_name += " continuous action" if self.continuous_action else ""
            self.setup_wandb(project_name, experiment_name, wandb_entity)

    def _init_common(self, scaling_factor, learning_rate, gamma, batch_size, hidden_dim, noise, model_class, use_cuda_graph):
        self.batch_size = batch_size
        self.gamma = gamma
        self.learning_rate = learning_rate
        self.hidden_dim = hidden_dim
        self.scaling_factor = scaling_factor
        self.desired_return = None
        self.desired_horizon = None
        self.continuous_action = not _is_discrete(self.env.action_space)
        self.noise = noise
        self.use_cuda_graph = use_cuda_graph
        if model_class and not issubclass(model_class, BasePCNModel):
            raise ValueError("model_class must be a subclass of BasePCNModel")
        if model_class is None:
            model_class = ContinuousActionsDefaultModel if self.continuous_action else DiscreteActionsDefaultModel
        self._graphs = GraphCache()
        self._set_model(model_class(self.observation_dim, self.action_dim, self.reward_dim, self.scaling_factor,
                                    hidden_dim=self.hidden_dim).to(self.device))
        self._heap = EpisodeHeap()
        self._store = self._new_store()
        self._act_in = None

    # ---- model, optimiser and the kernel path's state ---------------------------------------------------------------------------------
    def _set_model(self, model: BasePCNModel):
        self.model = model
        self.opt = FusedClipAdam(self.model.parameters(), lr=self.learning_rate)
        self._clear_on_load = self.model.register_load_state_dict_post_hook(lambda module, keys: self._graphs.clear())
        self._graphs.clear()
        self.fused = type(model) in DEFAULT_MODELS and ops.pcn_supported(self.observation_dim, self.reward_dim, self.hidden_dim, self.action_dim,
                                                                          self.batch_size)
        self._forward_fused = type(model) in DEFAULT_MODELS and ops.pcn_supported(self.observation_dim, self.reward_dim, self.hidden_dim,
                                                                                   self.action_dim)
        if self._forward_fused:
            tensors = default_model_tensors(model)
            self._param_table = ops.pcn_pointer_table(tensors)
        if self.fused:
            for t in tensors:  # persistent .grad storages the update kernel overwrites (captured graphs keep their addresses)
                t.grad = th.zeros_like(t)
            self._grad_table = ops.pcn_pointer_table([t.grad for t in tensors])
            self._ws = ops.pcn_workspace(self.observation_dim, self.reward_dim, self.hidden_dim, self.action_dim, self.batch_size, self.device)

    def _new_store(self) -> EpisodeStore:
        return EpisodeStore(self.observation_dim, self.reward_dim, self.action_dim if self.continuous_action else 1, not self.continuous_action,
                            self.device, self._graphs.clear)

    def get_config(self) -> dict:
        """Configuration of the PCN agent."""
        return {
            "env_id": self.env.unwrapped.spec.id,
            "batch_size": self.batch_size,
            "gamma": self.gamma,
            "learning_rate": self.learning_rate,
            "hidden_dim": self.hidden_dim,
            "scaling_factor": self.scaling_factor,
            "continuous_action": self.continuous_action,
            "noise": self.noise,
            "seed": self.seed,
        }

    @property
    def experience_replay(self) -> list:
        """The heap as ``(score, step, slot)`` entries; ``slot`` names the episode's rows in the device store."""
        return self._heap.entries

    # ---- update ----------------------------------------------------------------------------------------------------------------------
    def _updates(self, v: Variant, n: int):
        """Device half of ``n`` updates whose (row, horizon) pairs are row u of ``v.idx``: kernel pair + fused Adam per update."""
        S, d = self.observation_dim, self.reward_dim
        for u in range(n):
            rows, hor = v.idx.dev[u, 0], v.idx.dev[u, 1]
            pred = v.pred if u == n - 1 else None
            if self.fused:
                ops.pcn_update(self._param_table, self._grad_table, self.model.scaling_factor, self._store.pool, S, d, rows, hor, self.batch_size,
                               self.hidden_dim, self.action_dim, self.continuous_action, v.stats[0, u:u + 1],
                               None if self.continuous_action else v.stats[1, u:u + 1], pred, self._ws)
            else:
                self._eager_loss(rows, hor, v.stats[:, u], pred)
            self.opt.step_fused(None)

    def _eager_loss(self, rows: th.Tensor, hor: th.Tensor, stats: th.Tensor, pred_out: Optional[th.Tensor]):
        """The model evaluated by torch on the rows of the device store: loss, entropy and the gradients (reference pcn.py:213-234)."""
        S, d = self.observation_dim, self.reward_dim
        batch = self._store.pool.index_select(0, rows.long())
        prediction = self.model(batch[:, :S], batch[:, S:S + d], hor.float().unsqueeze(1))
        if self.continuous_action:
            loss = F.mse_loss(batch[:, S + d:S + d + self.action_dim], prediction)
        else:
            actions = batch[:, S + d].contiguous().view(th.int32).long()
            loss = th.sum(-F.one_hot(actions, prediction.shape[1]) * prediction, -1).mean()
            stats[1].copy_(th.sum(-th.exp(prediction.detach()) * prediction.detach()))
        stats[0].copy_(loss.detach())
        if pred_out is not None:
            pred_out.copy_(prediction.detach())
        self.opt.zero_grad(set_to_none=True)
        loss.backward()

    def _mutated(self):
        return list(self.model.parameters()) + optimizer_tensors(self.opt)

    def _variant(self, n: int) -> Variant:
        """The block of ``n`` updates: static (row, horizon) inputs [n, 2, B], loss / entropy [2, n], the last update's prediction."""
        def build():
            v = Variant(n, lambda: self._updates(v, n), self._mutated, idx=Staging((n, 2, self.batch_size), th.int32, self.device),
                        stats=th.zeros((2, n), device=self.device), pred=th.zeros((self.batch_size, self.action_dim), device=self.device))
            return v

        return self._graphs.get_or_build(n, build)

    def _prepare_block(self, n: int) -> Variant:
        """Host half: draw the indices of ``n`` updates in the reference's order, resolve heap positions to store rows and upload them."""
        v = self._variant(n)
        slots = np.array([e[2] for e in self._heap.entries], dtype=np.int64)
        lengths = np.array([self._store.length[s] for s in slots], dtype=np.int64)
        starts = np.array([self._store.start[s] for s in slots], dtype=np.int64)
        pos, t = draw_update_indices(self.np_random, lengths, self.batch_size, n)
        host = v.idx.host()
        host[:, 0] = starts[pos] + t
        host[:, 1] = lengths[pos] - t
        v.idx.upload()
        return v

    def _run_block(self, n: int) -> Variant:
        v = self._prepare_block(n)
        if self.use_cuda_graph and self.fused:  # a model torch evaluates (user class, unsupported shape) runs eagerly, uncaptured
            v.graph()
        else:
            v.step()
        return v

    def update(self):
        """One update (reference pcn.py:202-236); returns the loss and the prediction (log-probabilities or actions) of its minibatch."""
        v = self._run_block(1)
        return v.stats[0, 0].clone(), v.pred.clone()

    # ---- episodes and ranking -------------------------------------------------------------------------------------------------------
    def _add_episode(self, transitions: List[Transition], max_size: int, step: int) -> None:
        rewards = return_to_go(np.array([t.reward for t in transitions], dtype=np.float32), self.gamma)
        for t, r in zip(transitions, rewards):
            t.reward = r
        obs = np.array([t.observation for t in transitions], dtype=np.float32)
        acts = np.array([t.action for t in transitions], dtype=np.float32 if self.continuous_action else np.int32)
        slot = self._store.add(obs, acts, rewards)
        out = self._heap.add(slot, rewards[0].copy(), len(transitions), step, max_size)
        if out is not None:
            self._store.remove(out)

    def _scores(self, returns: np.ndarray, threshold: float) -> np.ndarray:
        return pcn_scores(returns, threshold)

    def _front(self, returns: np.ndarray) -> np.ndarray:
        return pcn_front(returns)

    def _threshold(self) -> float:
        return 0.2

    def _nlargest(self, n, threshold=0.2):
        """The ``n`` most promising episodes; rewrites every heap score (reference pcn.py:250-276)."""
        return self._heap.nlargest(n, self._scores(self._heap.episode_returns(), threshold))

    def _choose_commands(self, num_episodes: int):
        episodes = self._nlargest(num_episodes, self._threshold())
        returns, horizons = self._heap.episode_returns(episodes), self._heap.episode_lengths(episodes)
        nd = self._front(returns)
        returns, horizons = returns[nd], horizons[nd]
        r_i = self.np_random.integers(0, len(returns))
        desired_horizon = np.float32(horizons[r_i] - 2)
        s = np.std(returns, axis=0)
        desired_return = returns[r_i].copy()
        r_i = self.np_random.integers(0, len(desired_return))
        desired_return[r_i] += self.np_random.uniform(high=s[r_i])
        return np.float32(desired_return), desired_horizon

    # ---- acting ----------------------------------------------------------------------------------------------------------------------
    def _act_buffers(self):
        if self._act_in is None:
            S, d, A = self.observation_dim, self.reward_dim, self.action_dim
            self._act_in = th.zeros(S + d + 1, dtype=th.float32).pin_memory()
            self._act_out = th.zeros((1, A), dtype=th.float32).pin_memory()
            self._act_views = (self._act_in[:S].view(1, S), self._act_in[S:S + d].view(1, d), self._act_in[S + d:])
        return self._act_in.numpy(), self._act_out.numpy()

    def _predict_row(self, obs, desired_return, desired_horizon) -> np.ndarray:
        """The model on one row: log-probabilities or the action (float32 [A])."""
        if not self._forward_fused:
            with th.no_grad():
                pred = self.model(th.tensor(np.array([obs])).float().to(self.device), th.tensor(np.array([desired_return])).float().to(self.device),
                                  th.tensor(np.array([desired_horizon])).unsqueeze(1).float().to(self.device))
            return pred.cpu().numpy()[0]
        host_in, host_out = self._act_buffers()
        S, d = self.observation_dim, self.reward_dim
        host_in[:S] = np.asarray(obs, dtype=np.float32).reshape(-1)
        host_in[S:S + d] = np.asarray(desired_return, dtype=np.float32).reshape(-1)
        host_in[S + d] = np.float32(desired_horizon)
        o, r, h = self._act_views
        ops.pcn_forward(self._param_table, self.model.scaling_factor, o, r, h, self.hidden_dim, not self.continuous_action, self._act_out)
        th.cuda.current_stream().synchronize()
        return host_out[0].copy()

    def _act(self, obs: np.ndarray, desired_return, desired_horizon, eval_mode=False):
        out = self._predict_row(obs, desired_return, desired_horizon)
        if self.continuous_action:
            return out if eval_mode else out + np.random.normal(0.0, self.noise)
        if eval_mode:
            return np.argmax(out)
        return self.np_random.choice(np.arange(len(out)), p=np.exp(out))

    def _run_episode(self, env, desired_return, desired_horizon, max_return, eval_mode=False):
        transitions = []
        obs, _ = env.reset()
        done = False
        while not done:
            action = self._act(obs, desired_return, desired_horizon, eval_mode)
            n_obs, reward, terminated, truncated, _ = env.step(action)
            done = terminated or truncated
            transitions.append(Transition(observation=obs, action=action, reward=np.float32(reward).copy(), next_observation=n_obs,
                                          terminal=terminated))
            obs = n_obs
            desired_return = np.clip(desired_return - reward, None, max_return, dtype=np.float32)
            desired_horizon = np.float32(max(desired_horizon - 1, 1.0))
        return transitions

    def set_desired_return_and_horizon(self, desired_return: np.ndarray, desired_horizon: int):
        """Set desired return and horizon for evaluation."""
        self.desired_return = desired_return
        self.desired_horizon = desired_horizon

    def eval(self, obs, w=None):
        """Greedy action for the observation under the set desired return and horizon."""
        return self._act(obs, self.desired_return, self.desired_horizon, eval_mode=True)

    def evaluate(self, env, max_return, n=10):
        """Run the policy conditioned on the ``n`` best episodes' returns and horizons (reference pcn.py:365-383)."""
        n = min(n, len(self._heap))
        episodes = self._nlargest(n, self._threshold())
        returns = np.float32(self._heap.episode_returns(episodes))
        horizons = np.float32(self._heap.episode_lengths(episodes))
        e_returns = []
        for i in range(n):
            transitions = self._run_episode(env, returns[i], np.float32(horizons[i]), max_return, eval_mode=True)
            rewards = return_to_go(np.array([t.reward for t in transitions], dtype=np.float32), self.gamma)
            e_returns.append(rewards[0])
        distances = np.linalg.norm(np.array(returns) - np.array(e_returns), axis=-1)
        return e_returns, np.array(returns), distances

    def save(self, filename: str = "PCN_model", save_dir: str = "weights"):
        """Save the whole model module with ``th.save``."""
        os.makedirs(save_dir, exist_ok=True)
        self._clear_on_load.remove()  # the hook closes over this agent: the saved module carries no hook, as the reference's
        try:
            th.save(self.model, f"{save_dir}/{filename}.pt")
        finally:
            self._clear_on_load = self.model.register_load_state_dict_post_hook(lambda module, keys: self._graphs.clear())

    def load(self, path: str):
        """Load a model saved by ``save``; the optimiser restarts on the loaded parameters."""
        if not os.path.isfile(path):
            raise FileNotFoundError(f"Model file {path} does not exist.")
        self._set_model(th.load(path, map_location=self.device, weights_only=False))

    # ---- training --------------------------------------------------------------------------------------------------------------------
    def _fill_random(self, num_er_episodes: int, max_buffer_size: int):
        self._heap = EpisodeHeap()
        self._store = self._new_store()
        self._graphs.clear()
        for _ in range(num_er_episodes):
            transitions = []
            obs, _ = self.env.reset()
            done = False
            while not done:
                action = self.env.action_space.sample()
                n_obs, reward, terminated, truncated, _ = self.env.step(action)
                transitions.append(Transition(obs, action, np.float32(reward).copy(), n_obs, terminated))
                done = terminated or truncated
                obs = n_obs
                self.global_step += 1
            self._add_episode(transitions, max_size=max_buffer_size, step=self.global_step)

    def _train_iteration(self, num_model_updates: int, num_er_episodes: int, num_step_episodes: int, max_buffer_size: int, max_return,
                         ref_point, total_episodes: int):
        """One iteration of the reference's loop: the update block, a new command, ``num_step_episodes`` rollouts."""
        v = self._run_block(num_model_updates)
        stats = v.stats.cpu().numpy()
        loss = list(stats[0])
        entropy = [] if self.continuous_action else list(stats[1])
        desired_return, desired_horizon = self._choose_commands(num_er_episodes)
        if self.log:
            import wandb

            from ...common.performance_indicators import hypervolume

            leaves_r = self._heap.episode_returns(self._heap.entries[len(self._heap) // 2:])
            wandb.log({"train/hypervolume": hypervolume(ref_point, leaves_r), "train/loss": np.mean(loss), "global_step": self.global_step})
            if not self.continuous_action:
                wandb.log({"train/entropy": np.mean(entropy), "global_step": self.global_step})
        returns, horizons = [], []
        for _ in range(num_step_episodes):
            transitions = self._run_episode(self.env, desired_return, desired_horizon, max_return)
            self.global_step += len(transitions)
            self._add_episode(transitions, max_size=max_buffer_size, step=self.global_step)
            returns.append(transitions[0].reward)
            horizons.append(len(transitions))
        if self.log:
            import wandb

            wandb.log({"train/episode": total_episodes + num_step_episodes, "train/horizon_desired": desired_horizon,
                       "train/mean_horizon_distance": np.linalg.norm(np.mean(horizons) - desired_horizon), "global_step": self.global_step})
            for i in range(self.reward_dim):
                wandb.log({f"train/desired_return_{i}": desired_return[i], f"train/mean_return_{i}": np.mean(np.array(returns)[:, i]),
                           f"train/mean_return_distance_{i}": np.linalg.norm(np.mean(np.array(returns)[:, i]) - desired_return[i]),
                           "global_step": self.global_step})
        print(f"step {self.global_step} \t return {np.mean(returns, axis=0)}, ({np.std(returns, axis=0)}) \t loss {np.mean(loss):.3E} \t "
              f"horizons {np.mean(horizons)}")
        return desired_return, desired_horizon

    def _checkpoint(self, n_checkpoints: int, save_dir: str):
        self.save()

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              num_eval_weights_for_eval: int = 50, num_er_episodes: int = 20, num_step_episodes: int = 10, num_model_updates: int = 50,
              max_return: np.ndarray = None, max_buffer_size: int = 100, num_points_pf: int = 100):
        """Train PCN (reference pcn.py:396-503)."""
        self._train(total_timesteps, eval_env, ref_point, known_pareto_front, num_eval_weights_for_eval, num_er_episodes, num_step_episodes,
                    num_model_updates, max_return, max_buffer_size, num_points_pf, "weights", {})

    def _train(self, total_timesteps, eval_env, ref_point, known_pareto_front, num_eval_weights_for_eval, num_er_episodes, num_step_episodes,
               num_model_updates, max_return, max_buffer_size, num_points_pf, save_dir, extra_config):
        max_return = max_return if max_return is not None else np.full(self.reward_dim, 100.0, dtype=np.float32)
        if self.log:
            self.register_additional_config({
                "total_timesteps": total_timesteps, "ref_point": ref_point.tolist(), "known_front": known_pareto_front,
                "num_eval_weights_for_eval": num_eval_weights_for_eval, "num_er_episodes": num_er_episodes,
                "num_step_episodes": num_step_episodes, "num_model_updates": num_model_updates, "max_return": max_return.tolist(),
                "max_buffer_size": max_buffer_size, "num_points_pf": num_points_pf, **extra_config})
        self.global_step = 0
        total_episodes = num_er_episodes
        n_checkpoints = 0
        self._fill_random(num_er_episodes, max_buffer_size)
        while self.global_step < total_timesteps:
            self._train_iteration(num_model_updates, num_er_episodes, num_step_episodes, max_buffer_size, max_return, ref_point, total_episodes)
            total_episodes += num_step_episodes
            if self.global_step >= (n_checkpoints + 1) * total_timesteps / self.checkpoint_every:
                self._checkpoint(n_checkpoints, save_dir)
                n_checkpoints += 1
                e_returns, _, _ = self.evaluate(eval_env, max_return, n=num_points_pf)
                if self.log:
                    from ...common.evaluation import log_all_multi_policy_metrics

                    log_all_multi_policy_metrics(current_front=e_returns, hv_ref_point=ref_point, reward_dim=self.reward_dim,
                                                 global_step=self.global_step, n_sample_weights=num_eval_weights_for_eval,
                                                 ref_front=known_pareto_front)
