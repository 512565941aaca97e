"""GPI-PD / GPI-LS with continuous actions on the CUDA update engine -- drop-in for reference
morl_baselines/multi_policy/gpi_pd/gpi_pd_continuous_action.py (same classes ``Policy / QNetwork / GPIPDContinuousAction /
GPILSContinuousAction``, constructor arguments, method names and checkpoint keys).

Hot-path row a11 of SURVEY.md section 8 (BASELINE.json configs[2]: GPI-PD on mo-hopper-v4):

* the TD3-style vector target -- stack the N target critics, scalarise with the per-row weight, argmin over the critics, gather the
  winning critic's vector, vector Bellman line (gpi_pd_continuous_action.py:396-403) -- is ONE kernel
  (``morl_actor_critic_td_f32``, variant ARGMIN_GATHER);
* the GPI evaluation over the |M| x |M| (critic-conditioning weight, candidate action) pairs (``eval``, :463-478) is one batched
  critic call followed by the fused double-argmax kernel (``morl_gpi_envelope_f32`` with B = 1);
* target-network syncs are one multi-tensor launch per network (``polyak_update``), Adam steps the fused two-launch optimiser;
* the reference's update is ~200 tiny tensor operations (launch bound): the device
  side of one gradient update -- gather from the HBM replay mirror, weight tiling, target, critic step, priorities, target syncs and
  the delayed actor step -- is captured in CUDA graphs over static index / weight / noise buffers (``use_cuda_graph``,
  common/graphed.py); per update the host only walks the PER sum-tree, replays one graph and writes the priorities back.

The Dyna path (``dyna=True``, the reference's default; :216-235, :336-371, :548-562): the probabilistic ensemble is fitted on the real
transitions (``ProbabilisticEnsemble.fit``, device-resident), and every imagined step of ``_rollout_dynamics`` is one actor forward, one
ensemble forward and ONE fused commit (``morl_dyna_commit_f32``: sample, termination rule, uncertainty gate, ring append into the model
buffer's HBM store, compaction of the alive rows) followed by a read-back of two counts -- the reference appends the survivors row by row in
a python loop.  Mixed real / imagined minibatches take the same CUDA-graph path as real ones (two gathers into one batch).  The termination
rule is resolved at construction (``termination_rule_id``): an environment without one raises there, not at the first rollout.
``visualize_eval`` (matplotlib) is not mirrored.
"""

from __future__ import annotations

import os
import random
from itertools import chain
from typing import List, Optional, Union

import numpy as np
import torch as th
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...common.buffer import ReplayBuffer
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.model_based.probabilistic_ensemble import ProbabilisticEnsemble
from ...common.model_based.utils import termination_rule_id
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.networks import layer_init, mlp, polyak_update
from ...common.prioritized_buffer import PrioritizedReplayBuffer
from ...common.utils import unique_tol
from ...common.weights import equally_spaced_weights


class Policy(nn.Module):
    """Deterministic weight-conditioned actor with tanh squashing (reference gpi_pd_continuous_action.py:34-58)."""

    def __init__(self, obs_dim, rew_dim, output_dim, action_space, net_arch=[256, 256]):
        super().__init__()
        self.action_space = action_space
        self.latent_pi = mlp(obs_dim + rew_dim, -1, net_arch)
        self.mean = nn.Linear(net_arch[-1], output_dim)
        self.register_buffer("action_scale", th.tensor((action_space.high - action_space.low) / 2.0, dtype=th.float32))
        self.register_buffer("action_bias", th.tensor((action_space.high + action_space.low) / 2.0, dtype=th.float32))
        self.apply(layer_init)

    def forward(self, obs, w, noise=None, noise_clip=None, eps: Optional[th.Tensor] = None):
        """``eps`` (standard normal, shape of the action) may be injected for parity tests; otherwise ``th.randn_like`` as in the
        reference (:54-56)."""
        h = self.latent_pi(th.concat((obs, w), dim=obs.dim() - 1))
        action = th.tanh(self.mean(h))
        if noise is not None:
            e = th.randn_like(action) if eps is None else eps
            n = (e * noise).clamp(-noise_clip, noise_clip)
            action = (action + n).clamp(-1, 1)
        return action * self.action_scale + self.action_bias


class QNetwork(nn.Module):
    """Vector critic S x A x W -> R^d with Dropout + LayerNorm (reference gpi_pd_continuous_action.py:61-73)."""

    def __init__(self, obs_dim, action_dim, rew_dim, net_arch=[256, 256], layer_norm=True, drop_rate=0.01):
        super().__init__()
        self.net = mlp(obs_dim + action_dim + rew_dim, rew_dim, net_arch, drop_rate=drop_rate, layer_norm=layer_norm)
        self.apply(layer_init)

    def forward(self, obs, action, w):
        return self.net(th.cat((obs, action, w), dim=obs.dim() - 1))


class GPIPDContinuousAction(MOAgent, MOPolicy):
    """GPI-PD with continuous actions (Alegre et al., AAMAS 2023, appendix): TD3 extended to weight-conditioned vector critics."""

    def __init__(self, env, learning_rate: float = 3e-4, gamma: float = 0.99, tau: float = 0.005, buffer_size: int = 400000,
                 net_arch: List = [256, 256], batch_size: int = 128, num_q_nets: int = 2, delay_policy_update: int = 2,
                 learning_starts: int = 100, gradient_updates: int = 20, use_gpi: bool = False, policy_noise: float = 0.2,
                 noise_clip: float = 0.5, per: bool = True, min_priority: float = 0.1, alpha: float = 0.6, dyna: bool = True,
                 dynamics_net_arch: List = [200, 200, 200, 200], dynamics_train_freq: int = 250, dynamics_rollout_len: int = 5,
                 dynamics_rollout_starts: int = 1000, dynamics_rollout_freq: int = 250, dynamics_rollout_batch_size: int = 50000,
                 dynamics_buffer_size: int = 200000, dynamics_min_uncertainty: float = 2.0, dynamics_real_ratio: float = 0.1,
                 project_name: str = "MORL-Baselines", experiment_name: str = "GPI-PD Continuous Action", wandb_entity: Optional[str] = None,
                 log: bool = True, seed: Optional[int] = None, device: Union[th.device, str] = "auto", use_cuda_graph: bool = True):
        """The reference's arguments in the reference's order (gpi_pd_continuous_action.py:86-121) + ``use_cuda_graph``."""
        MOAgent.__init__(self, env, device=device, seed=seed)
        MOPolicy.__init__(self, device=device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.GPIPDContinuousAction needs a CUDA device: the update path is CUDA-only "
                                         "(no CPU fallback)")
        ops._lib.load()
        self.learning_rate, self.tau, self.gamma = learning_rate, tau, gamma
        self.use_gpi, self.policy_noise, self.noise_clip = use_gpi, policy_noise, noise_clip
        self.buffer_size, self.batch_size, self.learning_starts, self.gradient_updates = buffer_size, batch_size, learning_starts, gradient_updates
        self.num_q_nets, self.delay_policy_update = num_q_nets, delay_policy_update
        self.net_arch, self.dynamics_net_arch = net_arch, dynamics_net_arch
        self.per, self.min_priority, self.alpha = per, min_priority, alpha
        if self.per:
            self.replay_buffer = PrioritizedReplayBuffer(self.observation_shape, self.action_dim, rew_dim=self.reward_dim, max_size=buffer_size,
                                                         device=self.device)
        else:
            self.replay_buffer = ReplayBuffer(self.observation_shape, self.action_dim, rew_dim=self.reward_dim, max_size=buffer_size, device=self.device)

        mk = lambda: QNetwork(self.observation_dim, self.action_dim, self.reward_dim, net_arch=net_arch).to(self.device)  # noqa: E731
        self.q_nets = [mk() for _ in range(num_q_nets)]
        self.target_q_nets = [mk() for _ in range(num_q_nets)]
        for q_net, target_q_net in zip(self.q_nets, self.target_q_nets):
            target_q_net.load_state_dict(q_net.state_dict())
            for param in target_q_net.parameters():
                param.requires_grad = False
        self.policy = Policy(self.observation_dim, self.reward_dim, self.action_dim, self.env.action_space, net_arch=net_arch).to(self.device)
        self.target_policy = Policy(self.observation_dim, self.reward_dim, self.action_dim, self.env.action_space, net_arch=net_arch).to(self.device)
        self.target_policy.load_state_dict(self.policy.state_dict())
        for param in self.target_policy.parameters():
            param.requires_grad = False
        # torch.optim.Adam subclasses with the reference's arithmetic and state_dict layout, two launches per step, capture-safe
        self.q_optim = FusedClipAdam(chain(*[net.parameters() for net in self.q_nets]), lr=self.learning_rate)
        self.policy_optim = FusedClipAdam(list(self.policy.parameters()), lr=self.learning_rate)
        self.use_cuda_graph = use_cuda_graph
        self._graphs = GraphCache()

        self.dyna, self.dynamics, self.dynamics_buffer = dyna, None, None
        if self.dyna:
            # resolved here, so that an environment without a termination rule fails at construction (the reference fails at the first rollout)
            self._termination_rule = termination_rule_id(self.env.unwrapped.spec.id)
            self.dynamics = ProbabilisticEnsemble(input_dim=self.observation_dim + self.action_dim, output_dim=self.observation_dim + self.reward_dim,
                                                  arch=self.dynamics_net_arch, device=self.device)
            self.dynamics_buffer = ReplayBuffer(self.observation_shape, self.action_dim, rew_dim=self.reward_dim, max_size=dynamics_buffer_size,
                                                device=self.device)
        self.dynamics_buffer_size = dynamics_buffer_size
        self.dynamics_train_freq, self.dynamics_rollout_len, self.dynamics_rollout_starts = dynamics_train_freq, dynamics_rollout_len, dynamics_rollout_starts
        self.dynamics_rollout_freq, self.dynamics_rollout_batch_size = dynamics_rollout_freq, dynamics_rollout_batch_size
        self.dynamics_min_uncertainty, self.dynamics_real_ratio = dynamics_min_uncertainty, dynamics_real_ratio

        self.weight_support = []
        self.stacked_weight_support = []
        self._n_updates = 0
        self._noise_hook = None  # tests may set a callable(shape) -> standard-normal tensor (device) replacing th.randn_like
        self._last_losses = None
        self.log = log
        if self.log:
            self.setup_wandb(project_name, experiment_name, wandb_entity)

    def get_config(self):
        return {
            "env_id": self.env.unwrapped.spec.id, "learning_rate": self.learning_rate, "num_q_nets": self.num_q_nets,
            "batch_size": self.batch_size, "tau": self.tau, "gamma": self.gamma, "policy_noise": self.policy_noise, "net_arch": self.net_arch,
            "gradient_updates": self.gradient_updates, "delay_policy_update": self.delay_policy_update, "min_priority": self.min_priority,
            "per": self.per, "buffer_size": self.buffer_size, "alpha": self.alpha, "learning_starts": self.learning_starts, "dyna": self.dyna,
            "dynamics_net_arch": self.dynamics_net_arch, "dynamics_rollout_len": self.dynamics_rollout_len,
            "dynamics_min_uncertainty": self.dynamics_min_uncertainty, "dynamics_real_ratio": self.dynamics_real_ratio,
            "dynamics_train_freq": self.dynamics_train_freq, "dynamics_rollout_starts": self.dynamics_rollout_starts,
            "dynamics_rollout_freq": self.dynamics_rollout_freq, "dynamics_rollout_batch_size": self.dynamics_rollout_batch_size,
            "seed": self.seed,
        }

    def save(self, save_dir="weights/", filename=None, save_replay_buffer=True):
        """Checkpoint with the reference's keys (gpi_pd_continuous_action.py:290-309)."""
        os.makedirs(save_dir, exist_ok=True)
        saved_params = {"policy_state_dict": self.policy.state_dict(), "policy_optimizer_state_dict": self.policy_optim.state_dict()}
        for i, (q_net, target_q_net) in enumerate(zip(self.q_nets, self.target_q_nets)):
            saved_params["q_net_" + str(i) + "_state_dict"] = q_net.state_dict()
            saved_params["target_q_net_" + str(i) + "_state_dict"] = target_q_net.state_dict()
        saved_params["q_nets_optimizer_state_dict"] = self.q_optim.state_dict()
        saved_params["M"] = self.weight_support
        if self.dyna:
            saved_params["dynamics_state_dict"] = self.dynamics.state_dict()
        if save_replay_buffer:
            saved_params["replay_buffer"] = self.replay_buffer
        filename = getattr(self, "experiment_name", "GPI-PD Continuous Action") if filename is None else filename
        th.save(saved_params, save_dir + "/" + filename + ".tar")

    def load(self, path, load_replay_buffer=True):
        params = th.load(path, map_location=self.device, weights_only=False)
        self.weight_support = params["M"]
        self.stacked_weight_support = th.stack(self.weight_support) if len(self.weight_support) > 0 else []
        self.policy.load_state_dict(params["policy_state_dict"])
        self.policy_optim.load_state_dict(params["policy_optimizer_state_dict"])
        for i, (q_net, target_q_net) in enumerate(zip(self.q_nets, self.target_q_nets)):
            q_net.load_state_dict(params["q_net_" + str(i) + "_state_dict"])
            target_q_net.load_state_dict(params["target_q_net_" + str(i) + "_state_dict"])
        self.q_optim.load_state_dict(params["q_nets_optimizer_state_dict"])
        if self.dyna:
            self.dynamics.load_state_dict(params["dynamics_state_dict"])
        if load_replay_buffer and "replay_buffer" in params:
            self.replay_buffer = params["replay_buffer"]
            if hasattr(self.replay_buffer, "to"):
                self.replay_buffer.to(self.device)
        self._graphs.clear()  # optimiser state tensors / the buffer / the support may have been replaced

    # ------------------------------------------------------------------------------------------ the update
    def _uses_model_samples(self) -> bool:
        return self.dyna and self.global_step >= self.dynamics_rollout_starts and len(self.dynamics_buffer) > 0

    def _num_real(self) -> int:
        return int(self.batch_size * self.dynamics_real_ratio) if self._uses_model_samples() else self.batch_size

    def _sample_batch_experiences(self):
        """Real minibatch, or -- once the model has been rolled out -- ``dynamics_real_ratio`` real rows followed by imagined ones (reference
        :311-334).  Always a 6-tuple; the indices are those of the real rows."""
        if not self._uses_model_samples():
            return self.replay_buffer.sample(self.batch_size, to_tensor=True, device=self.device)
        num_real = self._num_real()
        parts, idxes = [], th.zeros(0, dtype=th.int64)
        if num_real > 0:
            *real, idxes = self.replay_buffer.sample(num_real, to_tensor=True, device=self.device)
            parts.append(real)
        if self.batch_size > num_real:
            parts.append(self.dynamics_buffer.sample(self.batch_size - num_real, to_tensor=True, device=self.device)[:5])
        return tuple(th.cat(cols, dim=0) for cols in zip(*parts)) + (idxes,)

    @th.no_grad()
    def _rollout_dynamics(self, weight: th.Tensor):
        """Dyna planning (reference :336-371): ``ceil(batch / 10000)`` chunks of up to 10,000 replayed states, each rolled through the model
        for ``dynamics_rollout_len`` steps under the target-noised policy.  A step is one actor forward, one ensemble forward, one fused
        commit into the model buffer's device store and one read-back of {kept, alive}; the host only moves ``ptr`` / ``size``.  Random
        numbers are consumed as in the reference: numpy for the start states and the elite draws, torch for the policy and model noise.  The
        written ring range is copied back into the buffer's numpy arrays once, at the end."""
        num_times = int(np.ceil(self.dynamics_rollout_batch_size / 10000))
        batch_size = min(self.dynamics_rollout_batch_size, 10000)
        dev, db, model, hook = self.device, self.dynamics_buffer, self.dynamics, self._noise_hook
        S, A, D, E = self.observation_dim, self.action_dim, self.reward_dim, model.ensemble_size
        db.flush()
        stores = db._dev
        ws = ops.dyna_commit_workspace(batch_size, dev)
        alive_bufs = (th.empty(batch_size, S, device=dev), th.empty(batch_size, S, device=dev))
        unc = th.empty(batch_size, device=dev)
        counts = th.empty(2, dtype=th.int32, device=dev)
        counts_pin = th.empty(2, dtype=th.int32).pin_memory()
        stream = th.cuda.current_stream()
        start, written, last_n = db.ptr, 0, 0
        for _ in range(num_times):
            obs = th.from_numpy(self.replay_buffer.sample_obs(batch_size)).to(dev)
            n = batch_size
            for plan_step in range(self.dynamics_rollout_len):
                w = weight.reshape(1, -1).repeat(n, 1)
                actions = self.policy(obs, w, noise=self.policy_noise, noise_clip=self.noise_clip, eps=hook((n, A)) if hook is not None else None)
                out = model._raw(th.cat((obs, actions), dim=-1))
                model_inds = np.random.choice(model.elites, size=n)
                idx = th.from_numpy(np.ascontiguousarray(model_inds, dtype=np.int32)).to(dev, non_blocking=True)
                noise = model._randn((E, n, S + D)).contiguous()
                nxt = alive_bufs[plan_step % 2]
                ops.dyna_commit(out, model.max_logvar, model.min_logvar, idx, noise, obs, actions, D, self._termination_rule, self.dynamics_min_uncertainty,
                                stores, db.ptr, nxt[:n], unc[:n], counts, ws)
                counts_pin.copy_(counts, non_blocking=True)
                stream.synchronize()
                kept, alive = (int(c) for c in counts_pin)
                db.ptr = (db.ptr + kept) % db.max_size
                db.size = min(db.size + kept, db.max_size)
                written += kept
                last_n = n
                if alive == 0:
                    break
                obs, n = nxt[:alive], alive
        # the rows written on the device form one ring interval from `start`: mirror it into the numpy arrays (async copies, one sync)
        cnt = min(written, db.max_size)
        first = min(cnt, db.max_size - start)
        for h, d in zip(db._host_tensors(), stores):
            for a, b in ((start, start + first), (0, cnt - first)):
                if b > a:
                    h[a:b].copy_(d[a:b], non_blocking=True)
        stream.synchronize()
        if self.log and last_n > 0:
            import wandb

            u = unc[:last_n].cpu().numpy()
            wandb.log({"dynamics/uncertainty_mean": u.mean(), "dynamics/uncertainty_max": u.max(), "dynamics/uncertainty_min": u.min(),
                       "global_step": self.global_step})

    def _train_dynamics(self):
        """Fit the ensemble on every real transition: X = [s | a], Y = [r | s' - s] (reference :548-555)."""
        m_obs, m_actions, m_rewards, m_next_obs, _ = self.replay_buffer.get_all_data()
        X = np.hstack((m_obs, m_actions))
        Y = np.hstack((m_rewards, m_next_obs - m_obs))
        mean_holdout_loss = self.dynamics.fit(X, Y)
        if self.log:
            import wandb

            wandb.log({"dynamics/mean_holdout_loss": mean_holdout_loss, "global_step": self.global_step})
        return mean_holdout_loss

    def _tile_weights(self, weight, picks, B0):
        """Effective-batch weights: ``weight`` for the first B0 rows, support weights ``picks`` for the doubled half (:381-391)."""
        D = self.reward_dim
        if picks is not None:
            return th.cat([weight.reshape(1, D).expand(B0, D), self.stacked_weight_support.index_select(0, picks)], dim=0).contiguous()
        return weight.reshape(1, D).repeat(B0, 1)

    def _device_update(self, s_obs, s_actions, s_rewards, s_next_obs, s_dones, w, with_policy: bool, eps, n_prio: int, prio_out=None):
        """The device side of one gradient update (reference :393-446) on the effective batch."""
        with th.no_grad():
            next_actions = self.target_policy(s_next_obs, w, noise=self.policy_noise, noise_clip=self.noise_clip, eps=eps)
            q_targets = th.stack([q_target(s_next_obs, next_actions, w) for q_target in self.target_q_nets])  # [n, N, D]
            # argmin_n w . Q_n -> gather -> r + (1 - done) * gamma * Q: one kernel (:396-403)
            target_q = ops.actor_critic_td(q_targets, w, s_rewards, s_dones, None, 0.0, self.gamma, ops.AC_ARGMIN_GATHER)
        q_values = [q_net(s_obs, s_actions, w) for q_net in self.q_nets]
        critic_loss = (1 / self.num_q_nets) * sum([F.mse_loss(q_value, target_q) for q_value in q_values])
        self.q_optim.zero_grad(set_to_none=True)
        critic_loss.backward()
        self.q_optim.step_fused(None)
        prio = None
        if n_prio > 0:
            per = (q_values[0] - target_q)[:n_prio].detach().abs() * 0.05
            prio = th.einsum("br,br->b", per, w[:n_prio])
            if prio_out is not None:
                prio_out.copy_(prio)
        for q_net, target_q_net in zip(self.q_nets, self.target_q_nets):
            polyak_update(q_net.parameters(), target_q_net.parameters(), self.tau)
        if with_policy:
            actions = self.policy(s_obs, w)
            q_values_pi = (1 / self.num_q_nets) * sum(q_net(s_obs, actions, w) for q_net in self.q_nets)
            policy_loss = -th.einsum("br,br->b", q_values_pi, w).mean()
            self.policy_optim.zero_grad(set_to_none=True)
            policy_loss.backward()
            self.policy_optim.step_fused(None)
            polyak_update(self.policy.parameters(), self.target_policy.parameters(), self.tau)
            self._last_policy_loss = policy_loss.detach()
        self._last_critic_loss = critic_loss.detach()
        return prio

    def _mutated_tensors(self):
        ts = [p for m in [self.policy, self.target_policy] + self.q_nets + self.target_q_nets for p in m.parameters()]
        return ts + optimizer_tensors(self.q_optim) + optimizer_tensors(self.policy_optim)

    def update(self, weight: th.Tensor):
        """``gradient_updates`` critic steps (+ delayed actor steps) for the given weight (reference :373-452)."""
        D, B0, rb = self.reward_dim, self.batch_size, self.replay_buffer
        hook = self._noise_hook
        graphable = self.use_cuda_graph and getattr(rb, "_dev", None) is not None and B0 <= len(rb)
        priority = None
        for _ in range(self.gradient_updates):
            P = len(self.weight_support)
            N = 2 * B0 if P > 1 else B0
            with_policy = self._n_updates % self.delay_policy_update == 0
            if not graphable:
                smp = self._sample_batch_experiences()
                s_obs, s_actions, s_rewards, s_next_obs, s_dones = smp[:5]
                idxes = smp[5] if self.per else None
                picks = None
                if P > 1:
                    # half of the effective batch uses `weight`, the other half weights drawn from the support (:381-391);
                    # random.choices on range(P) consumes python's RNG exactly like random.choices(self.weight_support, k=B)
                    picks = th.tensor(random.choices(range(P), k=B0), device=self.device)
                    s_obs, s_actions, s_rewards, s_next_obs, s_dones = (s_obs.repeat(2, 1), s_actions.repeat(2, 1), s_rewards.repeat(2, 1),
                                                                        s_next_obs.repeat(2, 1), s_dones.repeat(2, 1))
                w = self._tile_weights(weight, picks, B0)
                n_prio = len(idxes) if self.per else 0
                prio = self._device_update(s_obs, s_actions, s_rewards, s_next_obs, s_dones, w, with_policy,
                                           hook((N, self.action_dim)) if hook is not None else None, n_prio)
                if n_prio > 0:
                    priority = prio.cpu().numpy().flatten().clip(min=self.min_priority) ** self.alpha
                    rb.update_priorities(np.asarray(idxes.cpu() if th.is_tensor(idxes) else idxes), priority)
            else:
                # graph path: the host walks the PER tree / draws the support picks (same RNG consumption and order as the reference),
                # fills the static buffers, replays one graph, and writes the priorities back
                # with model samples the first num_real rows of the static index buffer are real indices, the rest model-buffer indices
                db = self.dynamics_buffer if self._uses_model_samples() else None
                nr = self._num_real()
                n_prio = nr if self.per else 0
                key = (P > 1, with_policy, hook is not None, id(rb), id(self.stacked_weight_support) if P > 1 else 0, db is not None, id(db))

                def build(doubled=P > 1, with_policy=with_policy, nr=nr, n_prio=n_prio, db=db):
                    inds = Staging(2 * B0, th.int64, self.device)  # replay indices (real, then imagined), support picks
                    w_in, prio = th.zeros(D, device=self.device), Staging(B0, th.float32, self.device)
                    eps = th.zeros(N, self.action_dim, device=self.device) if hook is not None else None

                    def step():
                        if db is None:
                            obs, act, rew, nobs, done = ops.replay_gather(*rb._dev, inds.dev[:B0])
                        else:  # two gathers into one batch: real rows, then imagined rows
                            obs, nobs = th.empty(B0, self.observation_dim, device=self.device), th.empty(B0, self.observation_dim, device=self.device)
                            act, rew = th.empty(B0, self.action_dim, device=self.device), th.empty(B0, D, device=self.device)
                            done = th.empty(B0, 1, device=self.device)
                            for store, lo, hi in ((rb, 0, nr), (db, nr, B0)):
                                if hi > lo:
                                    ops.replay_gather(*store._dev, inds.dev[lo:hi], outs=(obs[lo:hi], act[lo:hi], rew[lo:hi], nobs[lo:hi], done[lo:hi]))
                        if doubled:
                            obs, act, rew, nobs, done = obs.repeat(2, 1), act.repeat(2, 1), rew.repeat(2, 1), nobs.repeat(2, 1), done.repeat(2, 1)
                        w = self._tile_weights(w_in, inds.dev[B0:] if doubled else None, B0)
                        self._device_update(obs, act, rew, nobs, done, w, with_policy, eps, n_prio, prio.dev[:n_prio])

                    return Variant(key, step, self._mutated_tensors, inds=inds, w=w_in, eps=eps, prio=prio)

                v = self._graphs.get_or_build(key, build)
                hostv = v.inds.host()
                # host draws in the reference's order: PER tree (or uniform real draw), model-buffer draw, support picks
                idxes = rb.tree.sample(nr) if self.per else rb._draw(nr)
                hostv[:nr] = idxes
                if db is not None:
                    hostv[nr:B0] = db._draw(B0 - nr)
                if P > 1:
                    hostv[B0:] = random.choices(range(P), k=B0)
                v.inds.upload()
                v.w.copy_(weight.reshape(-1))
                if hook is not None:
                    v.eps.copy_(hook((N, self.action_dim)))
                rb.flush()
                if db is not None:
                    db.flush()
                v.graph()
                if n_prio > 0:
                    priority = v.prio.fetch(n_prio).clip(min=self.min_priority) ** self.alpha
                    rb.update_priorities(np.asarray(idxes), priority)
            self._n_updates += 1

        self._last_losses = (getattr(self, "_last_critic_loss", None), getattr(self, "_last_policy_loss", None))
        if self.log and self.global_step % 100 == 0:
            import wandb

            if self.per and priority is not None:
                wandb.log({"metrics/mean_priority": np.mean(priority), "metrics/max_priority": np.max(priority),
                           "metrics/min_priority": np.min(priority)}, commit=False)
            wandb.log({"losses/critic_loss": self._last_losses[0].item(), "losses/policy_loss": float(self._last_losses[1]),
                       "global_step": self.global_step})

    @th.no_grad()
    def eval(self, obs: Union[np.ndarray, th.Tensor], w: Union[np.ndarray, th.Tensor], torch_action=False) -> Union[np.ndarray, th.Tensor]:
        """Policy action; with ``use_gpi`` the GPI choice argmax_i max_a w . Q_0(s, pi(s, M_a), M_i) over the support (:454-485)."""
        if isinstance(obs, np.ndarray):
            obs = th.tensor(obs).float().to(self.device)
            w = th.tensor(w).float().to(self.device)
        if self.use_gpi:
            M = len(self.weight_support)
            obs_m = obs.reshape(1, -1).repeat(M, 1)
            actions_original = self.policy(obs_m, self.stacked_weight_support)  # action a = pi(s, M_a)
            # values[p, a] = Q_0(s, action_a, M_p): one batched critic call on the M*M pairs
            obs_mm = obs_m.repeat(M, 1, 1)
            actions = actions_original.repeat(M, 1, 1)
            stacked_m = self.stacked_weight_support.repeat_interleave(M, dim=0).view(M, M, self.reward_dim)
            values = self.q_nets[0](obs_mm, actions, stacked_m)  # [M, M, D]
            # max over a, argmax over p (first occurrence), fused: q[n=1, B=1, P=M, A=M, D]
            _, _, act = ops.gpi_envelope(values.reshape(1, 1, M, M, self.reward_dim).contiguous(), w.reshape(1, -1))
            action = actions_original[int(act[0])]
        else:
            action = self.policy(obs, w)
        if not torch_action:
            action = action.detach().cpu().numpy()
        return action

    @th.no_grad()
    def eval_batch(self, obs: np.ndarray, w: np.ndarray) -> np.ndarray:
        """Actions of ``eval`` for N (observation, weight) rows at once (common/evaluation.policy_evaluation_mo_batched).  With
        ``use_gpi``: one policy call gives the N x |M| candidate actions pi(s_n, M_a), one critic call covers the N x |M| x |M|
        (conditioning weight, candidate action) rows, and one GPI kernel over [1, N, |M|, |M|, d] picks each row's action."""
        obs_t = th.as_tensor(np.asarray(obs)).float().to(self.device).reshape(-1, self.observation_dim)
        w_t = th.as_tensor(np.asarray(w)).float().to(self.device).reshape(-1, self.reward_dim)
        if not self.use_gpi:
            return self.policy(obs_t, w_t).detach().cpu().numpy()
        N, M, O, D = obs_t.shape[0], len(self.weight_support), self.observation_dim, self.reward_dim
        Ms = self.stacked_weight_support
        cand = self.policy(obs_t.unsqueeze(1).expand(N, M, O).reshape(N * M, O), Ms.repeat(N, 1)).view(N, M, -1)  # [n, a] = pi(s_n, M_a)
        # values[n, p, a] = Q_0(s_n, cand[n, a], M_p)
        values = self.q_nets[0](obs_t.view(N, 1, 1, O).expand(N, M, M, O), cand.unsqueeze(1).expand(N, M, M, cand.shape[-1]),
                                Ms.view(1, M, 1, D).expand(N, M, M, D))
        _, _, act = ops.gpi_envelope(values.reshape(1, N, M, M, D).contiguous(), w_t)
        return cand[th.arange(N, device=self.device), act.long()].detach().cpu().numpy()

    def set_weight_support(self, weight_list: List[np.ndarray]):
        """Set the weight support set (duplicates within tolerance removed, reference :487-492)."""
        weights_no_repeat = unique_tol(weight_list)
        self.weight_support = [th.tensor(w).float().to(self.device) for w in weights_no_repeat]
        if len(self.weight_support) > 0:
            self.stacked_weight_support = th.stack(self.weight_support)
        self._graphs.clear()  # captured graphs read the previous support matrix

    def train_iteration(self, total_timesteps: int, weight: np.ndarray, weight_support: List[np.ndarray],
                        change_weight_every_episode: bool = False, eval_env=None, eval_freq: int = 1000, reset_num_timesteps: bool = False):
        """Collect ``total_timesteps`` transitions with the given weight and update after every step (reference :494-585)."""
        weight_support = unique_tol(weight_support)
        self.set_weight_support(weight_support)
        tensor_w = th.tensor(weight).float().to(self.device)
        self.global_step = 0 if reset_num_timesteps else self.global_step
        self.num_episodes = 0 if reset_num_timesteps else self.num_episodes
        obs, info = self.env.reset()
        for _ in range(1, total_timesteps + 1):
            self.global_step += 1
            if self.global_step < self.learning_starts:
                action = self.env.action_space.sample()
            else:
                with th.no_grad():
                    action = self.policy(th.tensor(obs).float().to(self.device), tensor_w, noise=self.policy_noise,
                                         noise_clip=self.noise_clip).detach().cpu().numpy()
            next_obs, vector_reward, terminated, truncated, info = self.env.step(action)
            self.replay_buffer.add(obs, action, vector_reward, next_obs, terminated)
            if self.global_step >= self.learning_starts:
                if self.dyna:
                    if self.global_step % self.dynamics_train_freq == 0:
                        self._train_dynamics()
                    if self.global_step >= self.dynamics_rollout_starts and self.global_step % self.dynamics_rollout_freq == 0:
                        self._rollout_dynamics(tensor_w)
                self.update(tensor_w)
            if eval_env is not None and self.log and self.global_step % eval_freq == 0:
                self.policy_eval(eval_env, weights=weight, log=self.log)
            if terminated or truncated:
                obs, _ = self.env.reset()
                self.num_episodes += 1
                if self.log and "episode" in info.keys():
                    from ...common.evaluation import log_episode_info

                    log_episode_info(info["episode"], np.dot, weight, self.global_step)
                if change_weight_every_episode:
                    weight = random.choice(weight_support)
                    tensor_w = th.tensor(weight).float().to(self.device)
            else:
                obs = next_obs

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              num_eval_weights_for_front: int = 100, num_eval_episodes_for_front: int = 5, num_eval_weights_for_eval: int = 50,
              weight_selection_algo: str = "gpi-ls", timesteps_per_iter: int = 10000, eval_freq: int = 1000, eval_mo_freq: int = 10000,
              checkpoints: bool = True, linear_support=None):
        """Outer loop of reference :587-702.  The weight selector is this package's ``LinearSupport`` (multi_policy/linear_support),
        built as the reference builds it (epsilon 0 for OLS, None for GPI-LS).  A caller-supplied ``linear_support`` -- any object with
        next_weight / get_weight_support / get_corner_weights / add_solution -- is used instead."""
        from ...common.evaluation import log_all_multi_policy_metrics, policy_evaluation_mo
        from ..linear_support.linear_support import LinearSupport

        if linear_support is None:
            linear_support = LinearSupport(num_objectives=self.reward_dim, epsilon=0.0 if weight_selection_algo == "ols" else None)

        if self.log:
            self.register_additional_config({"total_timesteps": total_timesteps, "ref_point": ref_point.tolist(), "known_front": known_pareto_front,
                                             "num_eval_weights_for_front": num_eval_weights_for_front,
                                             "num_eval_episodes_for_front": num_eval_episodes_for_front,
                                             "num_eval_weights_for_eval": num_eval_weights_for_eval,
                                             "weight_selection_algo": weight_selection_algo, "timesteps_per_iter": timesteps_per_iter,
                                             "eval_freq": eval_freq, "eval_mo_freq": eval_mo_freq})
        max_iter = total_timesteps // timesteps_per_iter
        eval_weights = equally_spaced_weights(self.reward_dim, n=num_eval_weights_for_front)
        for it in range(1, max_iter + 1):
            if weight_selection_algo == "gpi-ls":
                self.set_weight_support(linear_support.get_weight_support())
                use_gpi, self.use_gpi = self.use_gpi, True
                w = linear_support.next_weight(algo="gpi-ls", gpi_agent=self, env=eval_env, rep_eval=num_eval_episodes_for_front)
                self.use_gpi = use_gpi
            elif weight_selection_algo == "ols":
                w = linear_support.next_weight(algo="ols")
            else:
                raise ValueError(f"Unknown algorithm {weight_selection_algo}.")
            if w is None:
                break
            if weight_selection_algo == "gpi-ls":
                M = linear_support.get_weight_support() + linear_support.get_corner_weights(top_k=4) + [w]
            else:
                M = linear_support.get_weight_support() + [w]
            self.train_iteration(total_timesteps=timesteps_per_iter, weight=w, weight_support=M,
                                 change_weight_every_episode=weight_selection_algo == "gpi-ls", eval_env=eval_env, eval_freq=eval_freq)
            if weight_selection_algo == "ols":
                linear_support.add_solution(policy_evaluation_mo(self, eval_env, w, rep=num_eval_episodes_for_front)[3], w)
            else:
                for wcw in M:
                    linear_support.add_solution(policy_evaluation_mo(self, eval_env, wcw, rep=num_eval_episodes_for_front)[3], wcw)
            if self.log and self.global_step % eval_mo_freq == 0:
                returns = [policy_evaluation_mo(self, eval_env, ew, rep=num_eval_episodes_for_front)[3] for ew in eval_weights]
                log_all_multi_policy_metrics(current_front=returns, hv_ref_point=ref_point, reward_dim=self.reward_dim,
                                             global_step=self.global_step, n_sample_weights=num_eval_weights_for_eval,
                                             ref_front=known_pareto_front)
                import wandb

                mean_gpi = np.mean([np.dot(ew, q) for ew, q in zip(eval_weights, returns)], axis=0)
                wandb.log({"eval/Mean Utility - GPI": mean_gpi, "iteration": it})
            if checkpoints:
                self.save(filename=f"GPI-PD {weight_selection_algo} iter={it}", save_replay_buffer=False)
        if self.log:
            self.close_wandb()


class GPILSContinuousAction(GPIPDContinuousAction):
    """Model-free version of GPI-PD with continuous actions (reference :705-713)."""

    def __init__(self, *args, **kwargs):
        kwargs.setdefault("experiment_name", "GPI-LS Continuous Action")
        kwargs.pop("dyna", None)
        super().__init__(*args, dyna=False, **kwargs)
