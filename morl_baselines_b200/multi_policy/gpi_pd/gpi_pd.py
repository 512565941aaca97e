"""GPI-LS / GPI-PD (discrete actions) on the CUDA update engine -- drop-in for reference
morl_baselines/multi_policy/gpi_pd/gpi_pd.py (same constructor incl. the Dyna arguments, ``update / gpi_action / eval / max_action /
_envelope_target / _reset_priorities / _rollout_dynamics / _sample_batch_experiences / set_weight_support / train_iteration / save / load``).

Hot-path rows of SURVEY.md section 8 covered here: a7 (``_envelope_target``), a8 (update target + Huber loss + priorities),
a9 (``gpi_action``), a10 (``_reset_priorities``).  Under the API:
  * stack -> einsum -> argmin -> gather -> einsum -> argmax -> gather -> Bellman (gpi_pd.py:445-463) is ONE kernel
    (morl_critic_min_td_f32); the GPI envelope over the support set (gpi_pd.py:662-690) is ONE kernel
    (morl_gpi_envelope_f32) fed by a pairwise forward sf(s_b) * wf(M_p) that never materialises the repeated inputs;
  * per-net gather + huber + |td| stacks + max + einsum priorities (gpi_pd.py:469-487, 507-520) is ONE kernel
    (morl_td_huber_priority_f32);
  * gpi_action (gpi_pd.py:564-582) = one pairwise forward + ONE kernel.
  * the Dyna path (``dyna=True``, the reference's default; SURVEY 8(f)3): probabilistic ensemble trained from an HBM-resident data set
    (common/model_based/probabilistic_ensemble.py), model rollouts that never leave the device -- batched GPI action, ONE fused
    sampling / uncertainty kernel (morl_ensemble_sample_f32), masked bulk insert of the imagined transitions (gpi_pd.py:367-414).
``train()`` selects weights with this package's LinearSupport (multi_policy/linear_support: corner weights on the device), and
``eval_batch`` gives the batched GPI evaluation that selector's GPI-LS priority runs on.
"""

from __future__ import annotations

import os
import random
from itertools import chain
from typing import Callable, List, Optional, Union

import numpy as np
import torch as th
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.buffer import ReplayBuffer
from ...common.model_based.probabilistic_ensemble import ProbabilisticEnsemble
from ...common.model_based.utils import ModelEnv
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.networks import NatureCNN, layer_init, mlp, polyak_update
from ...common.prioritized_buffer import PrioritizedReplayBuffer
from ...common.utils import linearly_decaying_value, unique_tol
from ...common.weights import equally_spaced_weights
from ...tc_mlp import TCProductMlp


class QNet(nn.Module):
    """Conditioned vector Q-network relu(L(s)) * relu(L(w)) -> MLP (Dropout + LayerNorm); parameter names as in the
    reference (gpi_pd.py:41-76)."""

    def __init__(self, obs_shape, action_dim, rew_dim, net_arch, drop_rate=0.01, layer_norm=True):
        super().__init__()
        self.obs_shape = obs_shape
        self.action_dim = action_dim
        self.phi_dim = rew_dim
        self.weights_features = mlp(rew_dim, -1, net_arch[:1])
        if len(obs_shape) == 1:
            self.state_features = mlp(obs_shape[0], -1, net_arch[:1])
        else:
            self.state_features = NatureCNN(self.obs_shape, features_dim=net_arch[0])
        self.net = mlp(net_arch[0], action_dim * rew_dim, net_arch[1:], drop_rate=drop_rate, layer_norm=layer_norm)
        self.apply(layer_init)

    def forward(self, obs, w):
        sf = self.state_features(obs)
        wf = self.weights_features(w)
        return self.net(sf * wf).view(-1, self.action_dim, self.phi_dim)

    def forward_pairs(self, obs, M):
        """Q(s_b, M_p) for every pair: obs [B, ...], M [P, D] -> [B, P, A, D]; the two feature maps run on B and P rows."""
        sf = self.state_features(obs)
        wf = self.weights_features(M)
        h = (sf.unsqueeze(1) * wf.unsqueeze(0)).view(sf.shape[0] * wf.shape[0], -1)
        return self.net(h).view(sf.shape[0], wf.shape[0], self.action_dim, self.phi_dim)


class _FusedHuberLoss(th.autograd.Function):
    """(1/n) sum_n huber(|psi_n - target|) of gpi_pd.py:469-487 as one kernel (+ raw priorities into ``prio_out``)."""

    @staticmethod
    def forward(ctx, q_values, action, target_q, target_gpi, w, min_priority, p_rows, holder):
        loss, grad, prio = ops.td_huber_priority(q_values.detach(), action, target_q, target_gpi, w, min_priority, p_rows, want_grad=True)
        holder["prio"] = prio
        ctx.save_for_backward(grad)
        return loss.squeeze(0)

    @staticmethod
    def backward(ctx, grad_out):
        (grad,) = ctx.saved_tensors
        return grad * grad_out, None, None, None, None, None, None, None


class GPIPD(MOPolicy, MOAgent):
    """GPI-PD / GPI-LS (Alegre et al., AAMAS 2023), model-free path.  One gradient step (gather from the HBM replay mirror, weight
    tiling, critic-min target, GPI envelope target, Huber loss, backward, Adam, raw priorities) is captured in a CUDA graph over static
    index / weight buffers (``use_cuda_graph``, common/graphed.py): per step the host walks the PER tree, replays one graph and writes
    the priorities back."""

    def __init__(
        self,
        env,
        learning_rate: float = 3e-4,
        initial_epsilon: float = 0.01,
        final_epsilon: float = 0.01,
        epsilon_decay_steps: int = None,
        tau: float = 1.0,
        target_net_update_freq: int = 1000,
        buffer_size: int = int(1e6),
        net_arch: List = [256, 256, 256, 256],
        num_nets: int = 2,
        batch_size: int = 128,
        learning_starts: int = 100,
        gradient_updates: int = 20,
        gamma: float = 0.99,
        max_grad_norm: Optional[float] = None,
        use_gpi: bool = True,
        dyna: bool = True,
        per: bool = True,
        gpi_pd: bool = True,
        alpha_per: float = 0.6,
        min_priority: float = 0.01,
        drop_rate: float = 0.01,
        layer_norm: bool = True,
        dynamics_normalize_inputs: bool = False,
        dynamics_uncertainty_threshold: float = 1.5,
        dynamics_train_freq: Callable = lambda timestep: 250,
        dynamics_rollout_len: int = 1,
        dynamics_rollout_starts: int = 5000,
        dynamics_rollout_freq: int = 250,
        dynamics_rollout_batch_size: int = 25000,
        dynamics_buffer_size: int = 100000,
        dynamics_net_arch: List = [256, 256, 256],
        dynamics_ensemble_size: int = 5,
        dynamics_num_elites: int = 2,
        real_ratio: float = 0.5,
        project_name: str = "MORL-Baselines",
        experiment_name: str = "GPI-PD",
        wandb_entity: Optional[str] = None,
        log: bool = True,
        seed: Optional[int] = None,
        device: Union[th.device, str] = "auto",
        use_cuda_graph: bool = True,
        use_tensor_cores: bool = False,
        tensor_core_format: Optional[str] = None,
    ):
        MOAgent.__init__(self, env, device=device, seed=seed)
        MOPolicy.__init__(self, device=device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.GPIPD needs a CUDA device: the update path is CUDA-only (no CPU fallback)")
        ops._lib.load()
        self.learning_rate = learning_rate
        self.initial_epsilon = initial_epsilon
        self.epsilon = initial_epsilon
        self.epsilon_decay_steps = epsilon_decay_steps
        self.final_epsilon = final_epsilon
        self.tau = tau
        self.target_net_update_freq = target_net_update_freq
        self.gamma = gamma
        self.max_grad_norm = max_grad_norm
        self.use_gpi = use_gpi
        self.buffer_size = buffer_size
        self.net_arch = net_arch
        self.learning_starts = learning_starts
        self.batch_size = batch_size
        self.gradient_updates = gradient_updates
        self.num_nets = num_nets
        self.drop_rate = drop_rate
        self.layer_norm = layer_norm
        mk = lambda: QNet(self.observation_shape, self.action_dim, self.reward_dim, net_arch=net_arch, drop_rate=drop_rate,  # noqa: E731
                          layer_norm=layer_norm).to(self.device)
        self.q_nets = [mk() for _ in range(num_nets)]
        self.target_q_nets = [mk() for _ in range(num_nets)]
        for q, tq in zip(self.q_nets, self.target_q_nets):
            tq.load_state_dict(q.state_dict())
            for p in tq.parameters():
                p.requires_grad = False
        # a torch.optim.Adam subclass with the reference's arithmetic and state_dict layout, two launches per step, capture-safe
        self.q_optim = FusedClipAdam(chain(*[net.parameters() for net in self.q_nets]), lr=self.learning_rate)
        self.use_cuda_graph = use_cuda_graph
        # no-grad policy-set evaluations (_envelope_target, _reset_priorities, _rollout_dynamics) on the tensor cores (tc_mlp.TCProductMlp:
        # LayerNorm and dropout in the GEMM epilogue); the row-paired training pass and gpi_action stay on autograd.  Dropout masks then come
        # from the engine's Philox stream, not torch's generator: statistically equivalent, not bit-equal.
        fmt_name = tensor_core_format or os.environ.get("MORL_TC_FMT", "f16x2")
        if fmt_name not in ("f16x2", "bf16x3"):
            raise ValueError(f"tensor_core_format must be 'f16x2' or 'bf16x3', got {fmt_name!r}")
        self.tensor_core_format = fmt_name
        self._tc_fmt = ops.FMT_F16X2 if fmt_name == "f16x2" else ops.FMT_BF16X3
        if use_tensor_cores and not TCProductMlp.supported(self.q_nets[0], self._tc_fmt):
            raise ops._lib.MorlB200Error(
                "morl_baselines_b200.GPIPD: the tensor-core policy-set evaluation needs a flat observation and equal widths that are multiples "
                f"of 64 (f16x2) or 32 (bf16x3) and <= 256 (got obs {self.observation_shape}, net_arch {net_arch}, format {fmt_name}); "
                "pass use_tensor_cores=False to evaluate with library GEMMs")
        self.use_tensor_cores = bool(use_tensor_cores)
        self._tc_plans = None  # (plan of q_nets[0], plans of the target nets), activation buffers shared, sized for self._tc_rows pair rows
        self._tc_rows = 0
        if self.use_tensor_cores:
            # made once here, so their dropout seeds are drawn from torch's CPU generator at a fixed point (th.manual_seed reproduces them)
            tg = [TCProductMlp(self.target_q_nets[0], 128, self._tc_fmt)]
            tg += [TCProductMlp(n, 128, self._tc_fmt, share_buffers_with=tg[0]) for n in self.target_q_nets[1:]]
            self._tc_plans = (TCProductMlp(self.q_nets[0], 128, self._tc_fmt, share_buffers_with=tg[0]), tg)
            self._tc_rows = 128
        self._graphs = GraphCache()
        self._support_cache = None
        self.per = per
        self.gpi_pd = gpi_pd
        buf_cls = PrioritizedReplayBuffer if per else ReplayBuffer
        self.replay_buffer = buf_cls(self.observation_shape, 1, rew_dim=self.reward_dim, max_size=buffer_size, action_dtype=np.uint8,
                                     device=self.device)
        self.min_priority = min_priority
        self.alpha = alpha_per
        # model-based part (reference gpi_pd.py:240-268): probabilistic ensemble + imagined-transition buffer
        self.dyna = dyna
        self.dynamics_net_arch = dynamics_net_arch
        self.dynamics = None
        self.dynamics_buffer = None
        if self.dyna:
            self.dynamics = ProbabilisticEnsemble(input_dim=self.observation_dim + self.action_dim, output_dim=self.observation_dim + self.reward_dim,
                                                  arch=self.dynamics_net_arch, normalize_inputs=dynamics_normalize_inputs,
                                                  ensemble_size=dynamics_ensemble_size, num_elites=dynamics_num_elites, device=self.device)
            self.dynamics_buffer = ReplayBuffer(self.observation_shape, 1, rew_dim=self.reward_dim, max_size=dynamics_buffer_size, action_dtype=np.uint8,
                                                device=self.device)
        self.dynamics_train_freq = dynamics_train_freq
        self.dynamics_buffer_size = dynamics_buffer_size
        self.dynamics_normalize_inputs = dynamics_normalize_inputs
        self.dynamics_num_elites = dynamics_num_elites
        self.dynamics_ensemble_size = dynamics_ensemble_size
        self.dynamics_rollout_len = dynamics_rollout_len
        self.dynamics_rollout_starts = dynamics_rollout_starts if self.dyna else 0
        self.dynamics_rollout_freq = dynamics_rollout_freq
        self.dynamics_rollout_batch_size = dynamics_rollout_batch_size
        self.dynamics_uncertainty_threshold = dynamics_uncertainty_threshold
        self.real_ratio = real_ratio
        self.weight_support: List[th.Tensor] = []
        self.police_indices = []
        self.dot_mode = ops.DOT_UNFUSED
        self._last_loss = None
        self.log = log
        if self.log:
            self.setup_wandb(project_name, experiment_name, wandb_entity)

    # ------------------------------------------------------------------------------------------ config / io
    def get_config(self):
        return {
            "env_id": self.env.unwrapped.spec.id, "learning_rate": self.learning_rate, "initial_epsilon": self.initial_epsilon,
            "epsilon_decay_steps:": self.epsilon_decay_steps, "batch_size": self.batch_size, "per": self.per, "gpi_pd": self.gpi_pd,
            "alpha_per": self.alpha, "min_priority": self.min_priority, "tau": self.tau, "num_nets": self.num_nets,
            "clip_grand_norm": self.max_grad_norm, "target_net_update_freq": self.target_net_update_freq, "gamma": self.gamma,
            "net_arch": self.net_arch, "gradient_updates": self.gradient_updates, "buffer_size": self.buffer_size,
            "learning_starts": self.learning_starts, "dyna": self.dyna, "drop_rate": self.drop_rate, "layer_norm": self.layer_norm,
            "dynamics_model_arch": self.dynamics_net_arch, "dynamics_rollout_len": self.dynamics_rollout_len,
            "dynamics_uncertainty_threshold": self.dynamics_uncertainty_threshold, "dynamics_rollout_starts": self.dynamics_rollout_starts,
            "dynamics_rollout_freq": self.dynamics_rollout_freq, "dynamics_rollout_batch_size": self.dynamics_rollout_batch_size,
            "dynamics_buffer_size": self.dynamics_buffer_size, "dynamics_normalize_inputs": self.dynamics_normalize_inputs,
            "dynamics_ensemble_size": self.dynamics_ensemble_size, "dynamics_num_elites": self.dynamics_num_elites, "real_ratio": self.real_ratio,
            "seed": self.seed,
        }

    def save(self, save_replay_buffer=True, save_dir="weights/", filename=None):
        """Checkpoint with the reference's keys (gpi_pd.py:314-328)."""
        os.makedirs(save_dir, exist_ok=True)
        params = {f"psi_net_{i}_state_dict": net.state_dict() for i, net in enumerate(self.q_nets)}
        params["psi_nets_optimizer_state_dict"] = self.q_optim.state_dict()
        params["M"] = self.weight_support
        if self.dyna:
            params["dynamics_state_dict"] = self.dynamics.state_dict()
        if save_replay_buffer:
            params["replay_buffer"] = self.replay_buffer
        filename = getattr(self, "experiment_name", "GPI-PD") if filename is None else filename
        th.save(params, save_dir + "/" + filename + ".tar")

    def load(self, path, load_replay_buffer=True):
        params = th.load(path, map_location=self.device, weights_only=False)
        for i, (net, tnet) in enumerate(zip(self.q_nets, self.target_q_nets)):
            net.load_state_dict(params[f"psi_net_{i}_state_dict"])
            tnet.load_state_dict(params[f"psi_net_{i}_state_dict"])
        self.q_optim.load_state_dict(params["psi_nets_optimizer_state_dict"])
        self.weight_support = params["M"]
        if self.dyna:
            self.dynamics.load_state_dict(params["dynamics_state_dict"])
        if load_replay_buffer and "replay_buffer" in params:
            self.replay_buffer = params["replay_buffer"]
            if hasattr(self.replay_buffer, "to"):
                self.replay_buffer.to(self.device)
        self._graphs.clear()  # optimiser state / buffer / support may have been replaced
        self._support_cache = None

    # ------------------------------------------------------------------------------------------ the update
    def _uses_model_samples(self) -> bool:
        return self.dyna and self.global_step >= self.dynamics_rollout_starts and len(self.dynamics_buffer) > 0

    def _sample_batch_experiences(self):
        """Minibatch of real transitions, or -- once the model is rolled out -- ``real_ratio`` real + the rest imagined ones
        (reference gpi_pd.py:343-365).  Always returns the 6-tuple; only the real rows carry replay indices."""
        if not self._uses_model_samples():
            return self.replay_buffer.sample(self.batch_size, to_tensor=True, device=self.device)
        num_real = int(self.batch_size * self.real_ratio)
        s_obs, s_act, s_rew, s_nobs, s_done, idxes = self.replay_buffer.sample(num_real, to_tensor=True, device=self.device)
        m_obs, m_act, m_rew, m_nobs, m_done, _ = self.dynamics_buffer.sample(self.batch_size - num_real, to_tensor=True, device=self.device)
        return (th.cat([s_obs, m_obs], dim=0), th.cat([s_act, m_act], dim=0), th.cat([s_rew, m_rew], dim=0), th.cat([s_nobs, m_nobs], dim=0),
                th.cat([s_done, m_done], dim=0), idxes)

    @th.no_grad()
    def _rollout_dynamics(self, w: th.Tensor):
        """Dyna planning (reference gpi_pd.py:367-414): roll the learned model out from replayed states under the GPI policy and keep the
        imagined transitions whose ensemble uncertainty is below the threshold.  Everything stays on the device: one pairwise forward +
        one GPI kernel per step for all 10,000 x |M| rows, one batched ensemble forward + one fused sampling kernel
        (morl_ensemble_sample_f32), a masked BULK insert into the dynamics buffer (the reference appends row by row in python)."""
        num_times = int(np.ceil(self.dynamics_rollout_batch_size / 10000))
        batch_size = min(self.dynamics_rollout_batch_size, 10000)
        num_added_imagined_transitions = 0
        uncertainties = None
        model_env = None
        for _ in range(num_times):
            obs = self.replay_buffer.sample_obs(batch_size, to_tensor=True, device=self.device)
            model_env = ModelEnv(self.dynamics, self.env.unwrapped.spec.id, rew_dim=len(w))
            for _h in range(self.dynamics_rollout_len):
                M = self._support_matrix()
                if self.use_tensor_cores:
                    q0, _ = self._tc(obs.shape[0] * M.shape[0])
                    q = q0.forward_pairs(obs, M).view(obs.shape[0], M.shape[0], self.action_dim, self.reward_dim)
                else:
                    q = self.q_nets[0].forward_pairs(obs, M)  # [N, P, A, D] (module mode as the caller left it: dropout as in the reference)
                _, _, actions = ops.gpi_envelope(q.unsqueeze(0), w.reshape(1, -1), dot_mode=self.dot_mode)  # argmax_i max_a w . Q(s, a, M_i)
                actions_one_hot = F.one_hot(actions.long(), num_classes=self.action_dim)
                next_obs_pred, r_pred, dones, info = model_env.step_device(obs, actions_one_hot, deterministic=False)
                uncertainties = info["uncertainty"]
                keep = uncertainties < self.dynamics_uncertainty_threshold
                n_keep = int(keep.sum())  # (the only host round trip of the step: the bulk insert needs the count)
                if n_keep:
                    self.dynamics_buffer.add_batch(obs[keep], actions[keep].to(th.uint8).reshape(-1, 1), r_pred[keep], next_obs_pred[keep],
                                                   dones[keep].float())
                    num_added_imagined_transitions += n_keep
                nonterm_mask = ~dones.squeeze(-1)
                if int(nonterm_mask.sum()) == 0:
                    break
                obs = next_obs_pred[nonterm_mask]
        if self.log and uncertainties is not None:
            import wandb

            u = uncertainties.cpu().numpy()
            wandb.log({"dynamics/uncertainty_mean": u.mean(), "dynamics/uncertainty_max": u.max(), "dynamics/uncertainty_min": u.min(),
                       "dynamics/model_buffer_size": len(self.dynamics_buffer), "dynamics/imagined_transitions": num_added_imagined_transitions,
                       "global_step": self.global_step})
        return num_added_imagined_transitions

    def _train_dynamics(self):
        """Fit the ensemble on every stored transition: X = [s | one_hot(a)], Y = [r | s' - s] (reference gpi_pd.py:749-754)."""
        m_obs, m_actions, m_rewards, m_next_obs, _ = self.replay_buffer.get_all_data()
        one_hot = np.zeros((len(m_obs), self.action_dim))
        one_hot[np.arange(len(m_obs)), m_actions.astype(int).reshape(len(m_obs))] = 1
        X = np.hstack((m_obs, one_hot))
        Y = np.hstack((m_rewards, m_next_obs - m_obs))
        return self.dynamics.fit(X, Y)

    def _tc_reserve(self, rows: int):
        """Give the tensor-core plans room for ``rows`` pair rows.  Growing the shared activation buffers drops the captured update graphs,
        which hold the old ones; ``update`` reserves its rows before it looks a graph up, so no growth happens inside a capture."""
        if rows <= self._tc_rows:
            return
        q0, tg = self._tc_plans
        cap = max(rows, 2 * self._tc_rows)
        tg[0].reserve(cap)
        for p in tg[1:] + [q0]:
            p.reserve(cap, share_buffers_with=tg[0])
        self._tc_rows = cap
        self._graphs.clear()

    def _tc(self, rows: int):
        """(plan of q_nets[0], plans of the target nets) with room for ``rows`` pair rows."""
        self._tc_reserve(rows)
        return self._tc_plans

    def _support_matrix(self) -> th.Tensor:
        """[P, D] matrix of the support set, cached per support list (captured graphs read it)."""
        c = self._support_cache
        if c is None or c[0] is not self.weight_support or c[1].shape[0] != len(self.weight_support):
            self._support_cache = c = (self.weight_support, th.stack(self.weight_support))
            self._graphs.clear()
        return c[1]

    def _device_update(self, s_obs, s_actions, s_rewards, s_next_obs, s_dones, weight, picks, sampled_idx, p_rows: int, prio_out=None):
        """The device side of one gradient step (reference gpi_pd.py:425-505) on a gathered minibatch of B0 transitions.
        picks: int64 [B0] support indices of the doubled half (None: no doubling); sampled_idx: int64 [4] support indices of the
        sampled GPI weights (None: the whole support, or ``weight`` alone when the support is empty)."""
        B0, D = s_obs.shape[0], self.reward_dim
        P = len(self.weight_support)
        if picks is not None:
            # half of the effective batch uses `weight`, the other half weights drawn from the support set (gpi_pd.py:425-436)
            M = self._support_matrix()
            w = th.cat([weight.reshape(1, D).expand(B0, D), M.index_select(0, picks)], dim=0).contiguous()
            rep = (2,) + tuple(1 for _ in range(s_obs.dim() - 1))
            obs, nobs = s_obs.repeat(*rep), s_next_obs.repeat(*rep)
        else:
            w = weight.reshape(1, D).expand(B0, D).contiguous()
            obs, nobs = s_obs, s_next_obs
        if sampled_idx is not None:
            sampled_w = th.cat([weight.reshape(1, D), self._support_matrix().index_select(0, sampled_idx)], dim=0)
        else:
            sampled_w = self._support_matrix() if P > 0 else weight.reshape(1, D)
        with th.no_grad():
            # min_i Q_i(s', a, w) . w, greedy action, Bellman (gpi_pd.py:445-463) -- rewards / dones stay un-tiled (TILE map)
            next_q = th.stack([tn(nobs, w) for tn in self.target_q_nets])  # [n, N, A, D]
            target_q, _ = ops.critic_min_td(next_q, w, s_rewards, s_dones, self.gamma, self.dot_mode, ops.MAP_BLOCK, ops.MAP_TILE)
            target_gpi = None
            if self.gpi_pd:
                target_gpi, _ = self._envelope_target(nobs, w, sampled_w, rewards=s_rewards, dones=s_dones)
        psi = th.stack([net(obs, w) for net in self.q_nets])  # [n, N, A, D], train mode (dropout active as in the reference)
        holder = {}
        loss = _FusedHuberLoss.apply(psi, s_actions, target_q, target_gpi, w, float(self.min_priority), p_rows, holder)
        self.q_optim.zero_grad(set_to_none=True)
        loss.backward()
        if self.max_grad_norm is not None:
            for net in self.q_nets:
                th.nn.utils.clip_grad_norm_(net.parameters(), self.max_grad_norm)
        self.q_optim.step_fused(None)
        self._last_loss = loss.detach()
        if p_rows > 0 and prio_out is not None:
            prio_out.copy_(holder["prio"].reshape(-1))
        return holder.get("prio")

    def _mutated_tensors(self):
        return [p for m in self.q_nets for p in m.parameters()] + optimizer_tensors(self.q_optim)

    def update(self, weight: th.Tensor):
        """``gradient_updates`` gradient steps for the given weight vector (reference gpi_pd.py:416-562)."""
        critic_losses = []
        B0, D, rb = self.batch_size, self.reward_dim, self.replay_buffer
        # (mixed real / imagined minibatches come from two stores: they take the eager path)
        graphable = self.use_cuda_graph and getattr(rb, "_dev", None) is not None and self.max_grad_norm is None and not self._uses_model_samples()
        for _ in range(self.gradient_updates if self.global_step >= self.dynamics_rollout_starts else 1):
            P = len(self.weight_support)
            want_prio = self.per or self.gpi_pd
            if self.use_tensor_cores and self.gpi_pd:
                # pair rows of this step's envelope target (_device_update): doubled batch x sampled support weights
                self._tc_reserve((2 * B0 if P > 1 else B0) * (5 if P > 5 else max(P, 1)))
            if not graphable:
                s_obs, s_actions, s_rewards, s_next_obs, s_dones, idxes = self._sample_batch_experiences()
                s_actions = s_actions.to(th.int32).reshape(-1)
                # random.choices / random.sample on range(P) consume python's RNG exactly like the reference's calls on the weight list
                picks = th.tensor(random.choices(range(P), k=B0), device=self.device) if P > 1 else None
                sampled_idx = th.tensor(random.sample(range(P), k=4), device=self.device) if P > 5 else None
                prio = self._device_update(s_obs, s_actions, s_rewards, s_next_obs, s_dones, weight, picks, sampled_idx, len(idxes) if want_prio else 0)
                pr = prio.cpu().numpy().flatten() if want_prio else None
            else:
                # graph path: the host walks the PER tree and draws the support indices (same RNG consumption and order as the
                # reference), fills the static buffers, replays one graph, and reads the raw priorities back
                M = self._support_matrix() if P > 0 else None
                key = (P > 1, P > 5, P, id(rb), id(M))

                def build(doubled=P > 1, sampled=P > 5, want_prio=want_prio):
                    inds = Staging(2 * B0 + 4, th.int64, self.device)  # replay indices, support picks, sampled support indices
                    w, prio = th.zeros(D, device=self.device), Staging(B0, th.float32, self.device)

                    def step():
                        obs_s, nobs_s, act_s, rew_s, done_s = rb._dev
                        obs, act, rew, nobs, done = ops.replay_gather(obs_s, nobs_s, act_s, rew_s, done_s, inds.dev[:B0])
                        self._device_update(obs, act.reshape(-1), rew, nobs, done, w, inds.dev[B0:2 * B0] if doubled else None,
                                            inds.dev[2 * B0:] if sampled else None, B0 if want_prio else 0, prio.dev)

                    return Variant(key, step, self._mutated_tensors, inds=inds, w=w, prio=prio)

                v = self._graphs.get_or_build(key, build)
                hostv = v.inds.host()
                idxes = rb.tree.sample(B0) if self.per else rb._draw(B0)
                hostv[:B0] = idxes
                if P > 1:
                    hostv[B0:2 * B0] = random.choices(range(P), k=B0)
                if P > 5:
                    hostv[2 * B0:] = random.sample(range(P), k=4)
                v.inds.upload()
                v.w.copy_(weight.reshape(-1))
                rb.flush()
                v.graph()
                pr = v.prio.fetch() if want_prio else None
            critic_losses.append(self._last_loss)
            if want_prio:
                # priorities: |w . max_n err_n| of the first len(idxes) rows, clip(min)^alpha on the host (gpi_pd.py:507-525)
                priority = pr.clip(min=self.min_priority) ** self.alpha
                if self.per:
                    self.replay_buffer.update_priorities(np.asarray(idxes), priority)

        if self.tau != 1 or self.global_step % self.target_net_update_freq == 0:
            for net, tnet in zip(self.q_nets, self.target_q_nets):
                polyak_update(net.parameters(), tnet.parameters(), self.tau)
        if self.epsilon_decay_steps is not None:
            self.epsilon = linearly_decaying_value(self.initial_epsilon, self.epsilon_decay_steps, self.global_step, self.learning_starts,
                                                   self.final_epsilon)
        self._last_loss = critic_losses[-1] if critic_losses else None
        if self.log and self.global_step % 100 == 0:
            import wandb

            wandb.log({"losses/critic_loss": float(th.stack(critic_losses).mean()), "metrics/epsilon": self.epsilon,
                       "global_step": self.global_step})

    @th.no_grad()
    def _envelope_target(self, obs: th.Tensor, w: th.Tensor, sampled_w: th.Tensor, rewards=None, dones=None):
        """GPI envelope target over ``sampled_w`` with the critic-min over the target nets (reference gpi_pd.py:662-690).
        Returns (max_next_q [B, D], None); with rewards/dones the Bellman line is fused in (TILE map for a doubled batch)."""
        if self.use_tensor_cores:
            B, P = obs.shape[0], sampled_w.shape[0]
            _, plans = self._tc(B * P)
            q = th.empty((len(plans), B, P, self.action_dim, self.reward_dim), device=obs.device, dtype=th.float32)
            for i, plan in enumerate(plans):
                plan.forward_pairs(obs, sampled_w, out=q[i].view(B * P, -1))
        else:
            q = th.stack([tn.forward_pairs(obs, sampled_w) for tn in self.target_q_nets])  # [n, B, P, A, D]
        out, _, _ = ops.gpi_envelope(q, w, rewards, dones, self.gamma if rewards is not None else 0.0, self.dot_mode, ops.MAP_BLOCK, ops.MAP_TILE)
        return out, None

    @th.no_grad()
    def gpi_action(self, obs: th.Tensor, w: th.Tensor, return_policy_index=False, include_w=False):
        """argmax_i max_a w . Q_0(s, a, M_i) (reference gpi_pd.py:564-582): one pairwise forward + one kernel."""
        M = th.stack(self.weight_support + [w]) if include_w else self._support_matrix()
        q = self.q_nets[0].forward_pairs(obs.reshape(1, *self.observation_shape), M)  # [1, P, A, D]
        _, pol, act = ops.gpi_envelope(q.unsqueeze(0), w.reshape(1, -1), dot_mode=self.dot_mode)
        pa = th.stack([pol, act]).cpu()
        if return_policy_index:
            return int(pa[1, 0]), int(pa[0, 0])
        return int(pa[1, 0])

    @th.no_grad()
    def eval(self, obs: np.ndarray, w: np.ndarray) -> int:
        obs = th.as_tensor(obs).float().to(self.device)
        w = th.as_tensor(w).float().to(self.device)
        for net in self.q_nets:
            net.eval()
        action = self.gpi_action(obs, w, include_w=False) if self.use_gpi else self.max_action(obs, w)
        for net in self.q_nets:
            net.train()
        return action

    @th.no_grad()
    def eval_batch(self, obs: np.ndarray, w: np.ndarray) -> np.ndarray:
        """Actions of ``eval`` for N (observation, weight) rows at once -- the batched form used by the lockstep evaluation round
        (common/evaluation.policy_evaluation_mo_batched).  With ``use_gpi``: one pairwise forward over the N x |M| (state, support weight)
        pairs and one GPI kernel with per-row weights; otherwise the per-objective minimum over the nets and one greedy kernel.  The
        nets are in eval mode during the call, as in ``eval``."""
        obs_t = th.as_tensor(np.asarray(obs)).float().to(self.device).reshape(-1, *self.observation_shape)
        w_t = th.as_tensor(np.asarray(w)).float().to(self.device).reshape(-1, self.reward_dim)
        n = obs_t.shape[0]
        for net in self.q_nets:
            net.eval()
        if self.use_gpi:
            q = self.q_nets[0].forward_pairs(obs_t, self._support_matrix())  # [N, P, A, D]
            _, _, act = ops.gpi_envelope(q.unsqueeze(0), w_t, dot_mode=self.dot_mode)
        else:
            psi = th.min(th.stack([net(obs_t, w_t) for net in self.q_nets]), dim=0)[0]  # [N, A, D]
            _, _, act = ops.gpi_envelope(psi.view(1, n, 1, self.action_dim, self.reward_dim), w_t, dot_mode=self.dot_mode)
        for net in self.q_nets:
            net.train()
        return act.cpu().numpy()

    def _act(self, obs: th.Tensor, w: th.Tensor) -> int:
        if self.np_random.random() < self.epsilon:
            return self.env.action_space.sample()
        if self.use_gpi:
            action, policy_index = self.gpi_action(obs, w, return_policy_index=True)
            self.police_indices.append(policy_index)
            return action
        return self.max_action(obs, w)

    @th.no_grad()
    def max_action(self, obs: th.Tensor, w: th.Tensor) -> int:
        """Greedy action of the per-objective minimum over the nets (reference gpi_pd.py:609-616)."""
        psi = th.min(th.stack([net(obs.reshape(1, *self.observation_shape), w.reshape(1, -1)) for net in self.q_nets]), dim=0)[0]
        _, _, act = ops.gpi_envelope(psi.view(1, 1, 1, self.action_dim, self.reward_dim), w.reshape(1, -1), dot_mode=self.dot_mode)
        return int(act.item())

    @th.no_grad()
    def _reset_priorities(self, w: th.Tensor, chunk: int = 16384):
        """Recompute the priority of every stored transition for weight ``w`` (reference gpi_pd.py:619-660; the reference walks
        the buffer in 1000-row host chunks, here the device-resident store is swept in 16384-row slices)."""
        rb = self.replay_buffer
        n = rb.size
        priorities = np.repeat(0.1, n)
        obs_s, nobs_s, act_s, rew_s, done_s = rb.device_stores()
        D = self.reward_dim
        M = self._support_matrix()
        if self.use_tensor_cores:
            self._tc_reserve(min(n, chunk) * max(M.shape[0], 1))
        for b in range(0, n, chunk):
            e = min(b + chunk, n)
            obs, nobs, rew, done = obs_s[b:e], nobs_s[b:e], rew_s[b:e], done_s[b:e]
            act = act_s[b:e].long().reshape(-1, 1, 1).expand(-1, 1, D)
            wrow = w.reshape(1, D)
            if self.use_tensor_cores:  # the chunk against the single weight: a P = 1 pair batch
                q0, _ = self._tc(e - b)
                q_a = q0.forward_pairs(obs, wrow).view(e - b, self.action_dim, D).gather(1, act).squeeze(1)
            else:
                q_a = self.q_nets[0](obs, wrow.expand(e - b, D)).gather(1, act).squeeze(1)
            if self.gpi_pd:
                max_next_q, _ = self._envelope_target(nobs, wrow, M)
            else:
                q_sel = self.q_nets[0](nobs, wrow.expand(e - b, D))
                q_evl = self.target_q_nets[0](nobs, wrow.expand(e - b, D))
                max_next_q, _ = ops.greedy_td(q_sel, q_evl, wrow, dot_mode=self.dot_mode)
            gtd = th.einsum("r,br->b", w, (rew + (1 - done) * self.gamma * max_next_q - q_a)).abs()
            priorities[b:e] = gtd.clamp(min=self.min_priority).pow(self.alpha).cpu().numpy().flatten()
        rb.update_priorities(np.arange(n), priorities)

    def set_weight_support(self, weight_list: List[np.ndarray]):
        """Set the weight support set, de-duplicated within tolerance (reference gpi_pd.py:692-695)."""
        self.weight_support = [th.tensor(w).float().to(self.device) for w in unique_tol(weight_list)]

    # ------------------------------------------------------------------------------------------ training loops
    def train_iteration(self, total_timesteps: int, weight: np.ndarray, weight_support: List[np.ndarray], change_w_every_episode: bool = True,
                        reset_num_timesteps: bool = True, eval_env=None, eval_freq: int = 1000, reset_learning_starts: bool = False):
        """One training iteration for a weight vector and a support set (reference gpi_pd.py:697-788, model-free branch)."""
        weight_support = unique_tol(weight_support)
        self.set_weight_support(weight_support)
        tensor_w = th.tensor(weight).float().to(self.device)
        self.police_indices = []
        self.global_step = 0 if reset_num_timesteps else self.global_step
        self.num_episodes = 0 if reset_num_timesteps else self.num_episodes
        if reset_learning_starts:
            self.learning_starts = self.global_step
        if self.per and len(self.replay_buffer) > 0:
            self._reset_priorities(tensor_w)
        obs, info = self.env.reset()
        for _ in range(1, total_timesteps + 1):
            self.global_step += 1
            if self.global_step < self.learning_starts:
                action = self.env.action_space.sample()
            else:
                action = self._act(th.as_tensor(obs).float().to(self.device), tensor_w)
            next_obs, vec_reward, terminated, truncated, info = self.env.step(action)
            self.replay_buffer.add(obs, action, vec_reward, next_obs, terminated)
            if self.global_step >= self.learning_starts:
                if self.dyna:
                    if self.global_step % self.dynamics_train_freq(self.global_step) == 0:
                        mean_holdout_loss = self._train_dynamics()
                        if self.log:
                            import wandb

                            wandb.log({"dynamics/mean_holdout_loss": mean_holdout_loss, "global_step": self.global_step})
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
                    self.police_indices = []
                if change_w_every_episode:
                    weight = random.choice(weight_support)
                    tensor_w = th.tensor(weight).float().to(self.device)
            else:
                obs = next_obs

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              num_eval_weights_for_front: int = 100, num_eval_episodes_for_front: int = 5, num_eval_weights_for_eval: int = 50,
              timesteps_per_iter: int = 10000, weight_selection_algo: str = "gpi-ls", eval_freq: int = 1000, eval_mo_freq: int = 10000,
              checkpoints: bool = True, linear_support=None):
        """Outer loop of reference gpi_pd.py:790-911.  The weight selector is this package's ``LinearSupport``
        (multi_policy/linear_support: corner weights on the device, GPI-LS's expanded set in one batched evaluation round per call),
        built as the reference builds it (epsilon 0 for OLS, None for GPI-LS).  A caller-supplied ``linear_support`` -- any object
        with next_weight / get_weight_support / get_corner_weights / add_solution -- is used instead."""
        from ...common.evaluation import policy_evaluation_mo
        from ..linear_support.linear_support import LinearSupport

        if linear_support is None:
            linear_support = LinearSupport(num_objectives=self.reward_dim, epsilon=0.0 if weight_selection_algo == "ols" else None)

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
                                 change_w_every_episode=weight_selection_algo == "gpi-ls", eval_env=eval_env, eval_freq=eval_freq,
                                 reset_num_timesteps=False, reset_learning_starts=False)
            if weight_selection_algo == "ols":
                linear_support.add_solution(policy_evaluation_mo(self, eval_env, w, rep=num_eval_episodes_for_front)[3], w)
            else:
                for wcw in M:
                    linear_support.add_solution(policy_evaluation_mo(self, eval_env, wcw, rep=num_eval_episodes_for_front)[3], wcw)
            if self.log and self.global_step % eval_mo_freq == 0:
                from ...common.evaluation import log_all_multi_policy_metrics

                returns = [policy_evaluation_mo(self, eval_env, ew, rep=num_eval_episodes_for_front)[3] for ew in eval_weights]
                log_all_multi_policy_metrics(current_front=returns, hv_ref_point=ref_point, reward_dim=self.reward_dim,
                                             global_step=self.global_step, n_sample_weights=num_eval_weights_for_eval,
                                             ref_front=known_pareto_front)
            if checkpoints:
                self.save(filename=f"GPI-PD {weight_selection_algo} iter={it}", save_replay_buffer=False)
        if self.log:
            self.close_wandb()


class GPILS(GPIPD):
    """Model-free GPI-LS (reference gpi_pd.py:914-921)."""

    def __init__(self, *args, **kwargs):
        kwargs.setdefault("experiment_name", "GPI-LS")
        kwargs.pop("dyna", None)
        kwargs.pop("gpi_pd", None)
        super().__init__(*args, dyna=False, gpi_pd=False, **kwargs)
