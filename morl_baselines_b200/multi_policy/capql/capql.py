"""CAPQL on the CUDA update engine -- drop-in for reference morl_baselines/multi_policy/capql/capql.py (same classes
``ReplayMemory / WeightSamplerAngle / Policy / QNetwork / CAPQL`` and method names).

Hot-path row a12 of SURVEY.md section 8: the SAC vector target with the per-objective minimum over the critics and the
entropy term, stack -> min -> (alpha * logp) broadcast -> Bellman (capql.py:326-331), is ONE kernel
(morl_actor_critic_td_f32, variant ELEMENTWISE_MIN); the target sync of all critics is one multi-tensor launch per net.
The transition store keeps the reference's semantics (python ``random.sample`` over the stored tuples, capql.py:51-58) but
lives in preallocated arrays mirrored in HBM, so a minibatch is one index gather instead of six np.stack + six copies.
The reference's update is ~200 tiny tensor operations (launch bound): the device side
of one gradient update -- gather, target, critic step, policy step, target syncs -- is captured in a CUDA graph over static index /
noise buffers (``use_cuda_graph``, common/graphed.py) and replayed with one host call per update.
"""

from __future__ import annotations

import math
import os
import random
from itertools import chain
from typing import List, Optional, Union

import numpy as np
import torch as th
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.networks import layer_init, mlp, polyak_update
from ...common.weights import equally_spaced_weights

LOG_SIG_MAX = 2
LOG_SIG_MIN = -20
EPSILON = 1e-6


class ReplayMemory:
    """Transition memory holding the weight vector each transition was collected with (reference capql.py:32-66).

    ``sample`` draws ``random.sample(range(len), batch_size)`` -- the same python-RNG consumption as the reference's
    ``random.sample(self.buffer, batch_size)`` -- and gathers the rows from one packed float32 array (device mirror if
    a CUDA device was given)."""

    def __init__(self, capacity: int, device: Optional[th.device] = None):
        self.capacity = capacity
        self.position = 0
        self._len = 0
        self._packed = None  # [capacity, obs + act + d + d + obs + 1] float32, allocated at the first push
        self._dev = None
        self._dirty = []
        self.device = th.device(device) if device is not None else None
        self._dims = None

    def _alloc(self, dims):
        self._dims = dims
        width = sum(dims)
        t = th.zeros((self.capacity, width), dtype=th.float32)
        if self.device is not None and self.device.type == "cuda":
            t = t.pin_memory()
            self._dev = th.zeros((self.capacity, width), dtype=th.float32, device=self.device)
        self._packed_t = t
        self._packed = t.numpy()

    def push(self, state, action, weights, reward, next_state, done):
        parts = [np.asarray(x, dtype=np.float32).reshape(-1) for x in (state, action, weights, reward, next_state, done)]
        if self._packed is None:
            self._alloc([p.size for p in parts])
        self._packed[self.position] = np.concatenate(parts)
        if self._dev is not None:
            if self._dirty and self._dirty[-1][1] == self.position:
                self._dirty[-1] = (self._dirty[-1][0], self.position + 1)
            else:
                self._dirty.append((self.position, self.position + 1))
        self._len = min(self._len + 1, self.capacity)
        self.position = (self.position + 1) % self.capacity

    def _split(self, rows):
        out, o = [], 0
        for n in self._dims:
            out.append(rows[:, o : o + n])
            o += n
        out[5] = out[5].reshape(-1)  # the reference stacks 0-d `done`s into a [B] vector
        return tuple(out)

    def flush(self):
        """Copy the rows pushed since the last call to the HBM mirror."""
        if self._dev is not None:
            for a, b in self._dirty:
                self._dev[a:b].copy_(self._packed_t[a:b], non_blocking=True)
            self._dirty = []

    def draw(self, batch_size):
        """The reference's sampling rule (capql.py:51-58): ``random.sample`` without replacement over the stored transitions."""
        return random.sample(range(self._len), batch_size)

    def sample(self, batch_size, to_tensor=True, device=None):
        idx = self.draw(batch_size)
        if to_tensor and self._dev is not None:
            self.flush()
            rows = self._dev.index_select(0, th.tensor(idx, device=self.device))
            return self._split(rows)
        rows = self._packed[np.asarray(idx)]
        parts = self._split(rows)
        if to_tensor:
            return tuple(th.tensor(p, dtype=th.float32).to(device) for p in parts)
        return parts

    def __len__(self):
        return self._len


class WeightSamplerAngle:
    """Sample weight vectors within an angle of a direction (reference capql.py:69-99)."""

    def __init__(self, rwd_dim, angle, w=None):
        self.rwd_dim = rwd_dim
        self.angle = angle
        w = th.ones(rwd_dim) if w is None else w
        self.w = w / th.norm(w)

    def sample(self, n_sample):
        s = th.normal(th.zeros(n_sample, self.rwd_dim))
        s = s - (s @ self.w).view(-1, 1) * self.w.view(1, -1)
        s = s / th.norm(s, dim=1, keepdim=True)
        s_angle = th.rand(n_sample, 1) * self.angle
        w_sample = th.tan(s_angle) * s + self.w.view(1, -1)
        w_sample = w_sample / th.norm(w_sample, dim=1, keepdim=True, p=1)
        return w_sample.float()


class Policy(nn.Module):
    """Weight-conditioned Gaussian policy with tanh squashing (reference capql.py:102-158)."""

    def __init__(self, obs_dim, rew_dim, output_dim, action_space, net_arch=[256, 256]):
        super().__init__()
        self.action_space = action_space
        self.latent_pi = mlp(obs_dim + rew_dim, -1, net_arch)
        self.mean = nn.Linear(net_arch[-1], output_dim)
        self.log_std_linear = nn.Linear(net_arch[-1], output_dim)
        self.register_buffer("action_scale", th.tensor((action_space.high - action_space.low) / 2.0, dtype=th.float32))
        self.register_buffer("action_bias", th.tensor((action_space.high + action_space.low) / 2.0, dtype=th.float32))
        self.apply(layer_init)

    def forward(self, obs, w):
        h = self.latent_pi(th.concat((obs, w), dim=obs.dim() - 1))
        return self.mean(h), th.clamp(self.log_std_linear(h), min=LOG_SIG_MIN, max=LOG_SIG_MAX)

    def get_action(self, obs, w):
        mean, _ = self.forward(obs, w)
        return th.tanh(mean) * self.action_scale + self.action_bias

    def sample(self, obs, w, noise: Optional[th.Tensor] = None):
        """Reparameterised sample; ``noise`` (standard normal, same shape as the mean) may be injected for parity tests.  The Gaussian is
        written out with the arithmetic of ``torch.distributions.Normal`` (rsample: loc + eps * scale; log_prob: -((v - loc)^2) /
        (2 var) - log(scale) - log(sqrt(2 pi))) without the distribution object, whose argument validation synchronises with the host
        (illegal under CUDA-graph capture)."""
        mean, log_std = self.forward(obs, w)
        std = log_std.exp()
        eps = th.randn_like(mean) if noise is None else noise
        x_t = mean + eps * std
        y_t = th.tanh(x_t)
        action = y_t * self.action_scale + self.action_bias
        var = std**2
        log_prob = (-((x_t - mean) ** 2) / (2 * var) - std.log() - math.log(math.sqrt(2 * math.pi))).sum(dim=1)
        log_prob = log_prob - th.log(self.action_scale * (1 - y_t.pow(2)) + EPSILON).sum(dim=1)
        log_prob = log_prob.clamp(-1e3, 1e3)
        return action, log_prob, th.tanh(mean) * self.action_scale + self.action_bias


class QNetwork(nn.Module):
    """Vector critic Q(s, a, w) -> R^d (reference capql.py:161-171)."""

    def __init__(self, obs_dim, action_dim, rew_dim, net_arch=[256, 256]):
        super().__init__()
        self.net = mlp(obs_dim + action_dim + rew_dim, rew_dim, net_arch)
        self.apply(layer_init)

    def forward(self, obs, action, w):
        return self.net(th.cat((obs, action, w), dim=obs.dim() - 1))


class CAPQL(MOAgent, MOPolicy):
    """CAPQL (Lu, Herman, Yu, ICLR 2023): SAC with weight-conditioned vector critics."""

    def __init__(
        self,
        env,
        learning_rate: float = 3e-4,
        gamma: float = 0.99,
        tau: float = 0.005,
        buffer_size: int = 1000000,
        net_arch: List = [256, 256],
        batch_size: int = 128,
        num_q_nets: int = 2,
        alpha: float = 0.2,
        learning_starts: int = 1000,
        gradient_updates: int = 1,
        project_name: str = "MORL-Baselines",
        experiment_name: str = "CAPQL",
        wandb_entity: Optional[str] = None,
        log: bool = True,
        seed: Optional[int] = None,
        device: Union[th.device, str] = "auto",
        use_cuda_graph: bool = True,
    ):
        MOAgent.__init__(self, env, device=device, seed=seed)
        MOPolicy.__init__(self, device=device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.CAPQL needs a CUDA device: the update path is CUDA-only (no CPU fallback)")
        ops._lib.load()
        self.learning_rate = learning_rate
        self.tau = tau
        self.gamma = gamma
        self.buffer_size = buffer_size
        self.num_q_nets = num_q_nets
        self.net_arch = net_arch
        self.learning_starts = learning_starts
        self.batch_size = batch_size
        self.gradient_updates = gradient_updates
        self.alpha = alpha
        self.replay_buffer = ReplayMemory(self.buffer_size, device=self.device)
        mk = lambda: QNetwork(self.observation_dim, self.action_dim, self.reward_dim, net_arch=net_arch).to(self.device)  # noqa: E731
        self.q_nets = [mk() for _ in range(num_q_nets)]
        self.target_q_nets = [mk() for _ in range(num_q_nets)]
        for q, tq in zip(self.q_nets, self.target_q_nets):
            tq.load_state_dict(q.state_dict())
            for p in tq.parameters():
                p.requires_grad = False
        self.policy = Policy(self.observation_dim, self.reward_dim, self.action_dim, self.env.action_space, net_arch=net_arch).to(self.device)
        # torch.optim.Adam subclasses with the reference's arithmetic and state_dict layout, two launches per step, capture-safe
        self.q_optim = FusedClipAdam(chain(*[net.parameters() for net in self.q_nets]), lr=self.learning_rate)
        self.policy_optim = FusedClipAdam(list(self.policy.parameters()), lr=self.learning_rate)
        self._n_updates = 0
        self._noise_hook = None  # tests may set a callable(shape) -> standard-normal tensor to make rsample reproducible
        self.use_cuda_graph = use_cuda_graph
        self._graphs = GraphCache()
        self.log = log
        if self.log:
            self.setup_wandb(project_name, experiment_name, wandb_entity)

    def get_config(self):
        return {"env_id": self.env.unwrapped.spec.id, "learning_rate": self.learning_rate, "num_q_nets": self.num_q_nets,
                "batch_size": self.batch_size, "tau": self.tau, "gamma": self.gamma, "net_arch": self.net_arch,
                "gradient_updates": self.gradient_updates, "alpha": self.alpha, "buffer_size": self.buffer_size,
                "learning_starts": self.learning_starts, "seed": self.seed}

    def save(self, save_dir="weights/", filename=None, save_replay_buffer=True):
        """Checkpoint with the reference's keys (capql.py:288-305)."""
        os.makedirs(save_dir, exist_ok=True)
        params = {"policy_state_dict": self.policy.state_dict(), "policy_optimizer_state_dict": self.policy_optim.state_dict()}
        for i, (q, tq) in enumerate(zip(self.q_nets, self.target_q_nets)):
            params[f"q_net_{i}_state_dict"] = q.state_dict()
            params[f"target_q_net_{i}_state_dict"] = tq.state_dict()
        params["q_nets_optimizer_state_dict"] = self.q_optim.state_dict()
        if save_replay_buffer:
            params["replay_buffer"] = self.replay_buffer
        filename = getattr(self, "experiment_name", "CAPQL") if filename is None else filename
        th.save(params, save_dir + "/" + filename + ".tar")

    def load(self, path, load_replay_buffer=True):
        params = th.load(path, map_location=self.device, weights_only=False)
        self.policy.load_state_dict(params["policy_state_dict"])
        self.policy_optim.load_state_dict(params["policy_optimizer_state_dict"])
        for i, (q, tq) in enumerate(zip(self.q_nets, self.target_q_nets)):
            q.load_state_dict(params[f"q_net_{i}_state_dict"])
            tq.load_state_dict(params[f"target_q_net_{i}_state_dict"])
        self.q_optim.load_state_dict(params["q_nets_optimizer_state_dict"])
        if load_replay_buffer and "replay_buffer" in params:
            self.replay_buffer = params["replay_buffer"]
        self._graphs.clear()  # optimiser state tensors / the buffer may have been replaced

    def _sample_batch_experiences(self):
        return self.replay_buffer.sample(self.batch_size, to_tensor=True, device=self.device)

    def _device_update(self, s_obs, s_actions, w, s_rewards, s_next_obs, s_dones, noise):
        """The device side of one gradient update (reference capql.py:323-362) on an already gathered minibatch."""
        with th.no_grad():
            next_actions, log_pi, _ = self.policy.sample(s_next_obs, w, noise(0))
            q_targets = th.stack([tq(s_next_obs, next_actions, w) for tq in self.target_q_nets])  # [n, B, D]
            # per-objective min over critics - alpha * logp, vector Bellman: one kernel (capql.py:329-331)
            target_q = ops.actor_critic_td(q_targets, None, s_rewards, s_dones, log_pi, self.alpha, self.gamma, ops.AC_ELEMENTWISE_MIN)
        q_values = [q(s_obs, s_actions, w) for q in self.q_nets]
        critic_loss = (1 / self.num_q_nets) * sum([F.mse_loss(qv, target_q) for qv in q_values])
        self.q_optim.zero_grad(set_to_none=True)
        critic_loss.backward()
        self.q_optim.step_fused(None)

        pi, log_pi, _ = self.policy.sample(s_obs, w, noise(1))
        q_pi = th.stack([q(s_obs, pi, w) for q in self.q_nets])
        min_q = (th.min(q_pi, dim=0)[0] * w).sum(dim=-1, keepdim=True)
        policy_loss = ((self.alpha * log_pi) - min_q).mean()
        self.policy_optim.zero_grad(set_to_none=True)
        policy_loss.backward()
        self.policy_optim.step_fused(None)
        for q, tq in zip(self.q_nets, self.target_q_nets):
            polyak_update(q.parameters(), tq.parameters(), self.tau)
        self._last_losses = (critic_loss.detach(), policy_loss.detach())

    def _mutated_tensors(self):
        ts = [p for m in [self.policy] + self.q_nets + self.target_q_nets for p in m.parameters()]
        return ts + optimizer_tensors(self.q_optim) + optimizer_tensors(self.policy_optim)

    def update(self):
        """Critic and policy update (reference capql.py:321-362)."""
        B, hook = self.batch_size, self._noise_hook
        rb = self.replay_buffer
        graphable = self.use_cuda_graph and getattr(rb, "_dev", None) is not None
        for _ in range(self.gradient_updates):
            if not graphable:
                s_obs, s_actions, w, s_rewards, s_next_obs, s_dones = self._sample_batch_experiences()
                self._device_update(s_obs, s_actions, w, s_rewards, s_next_obs, s_dones,
                                    (lambda k: hook((B, self.action_dim))) if hook is not None else (lambda k: None))
            else:
                key = (hook is not None, id(rb))

                def build():
                    idx = Staging(B, th.int64, self.device)
                    noise = [th.zeros(B, self.action_dim, device=self.device) for _ in range(2)] if hook is not None else None

                    def step():
                        parts = rb._split(rb._dev.index_select(0, idx.dev))
                        self._device_update(*parts, (lambda k: noise[k]) if noise is not None else (lambda k: None))

                    return Variant(key, step, self._mutated_tensors, idx=idx, noise=noise)

                v = self._graphs.get_or_build(key, build)
                v.idx.host()[:] = rb.draw(B)  # python `random`, as the reference's random.sample(self.buffer, batch_size)
                v.idx.upload()
                if hook is not None:
                    for t in v.noise:
                        t.copy_(hook((B, self.action_dim)))
                rb.flush()
                v.graph()
            self._n_updates += 1
        if self.log and self.global_step % 100 == 0:
            import wandb

            wandb.log({"losses/critic_loss": self._last_losses[0].item(), "losses/policy_loss": self._last_losses[1].item(),
                       "global_step": self.global_step})

    @th.no_grad()
    def eval(self, obs, w, torch_action=False):
        """Deterministic action for the observation and weight vector (reference capql.py:364-377)."""
        if isinstance(obs, np.ndarray):
            obs = th.tensor(obs).float().to(self.device)
            w = th.tensor(w).float().to(self.device)
        action = self.policy.get_action(obs, w)
        return action if torch_action else action.detach().cpu().numpy()

    def train(self, total_timesteps: int, eval_env, ref_point: np.ndarray, known_pareto_front: Optional[List[np.ndarray]] = None,
              num_eval_weights_for_front: int = 100, num_eval_episodes_for_front: int = 5, num_eval_weights_for_eval: int = 50,
              eval_freq: int = 10000, reset_num_timesteps: bool = False, checkpoints: bool = False, save_freq: int = 10000):
        """Training loop (reference capql.py:379-484): a fresh weight within 22.5 degrees of the all-ones direction every step."""
        if self.log:
            self.register_additional_config({"total_timesteps": total_timesteps, "ref_point": ref_point.tolist(),
                                             "known_front": known_pareto_front, "num_eval_weights_for_front": num_eval_weights_for_front,
                                             "num_eval_episodes_for_front": num_eval_episodes_for_front,
                                             "num_eval_weights_for_eval": num_eval_weights_for_eval, "eval_freq": eval_freq,
                                             "reset_num_timesteps": reset_num_timesteps})
        eval_weights = equally_spaced_weights(self.reward_dim, n=num_eval_weights_for_front) if self.log else None
        weight_sampler = WeightSamplerAngle(self.env.unwrapped.reward_dim, th.pi * (22.5 / 180))
        self.global_step = 0 if reset_num_timesteps else self.global_step
        self.num_episodes = 0 if reset_num_timesteps else self.num_episodes
        obs, info = self.env.reset()
        for _ in range(1, total_timesteps + 1):
            self.global_step += 1
            tensor_w = weight_sampler.sample(1).view(-1).to(self.device)
            w = tensor_w.detach().cpu().numpy()
            if self.global_step < self.learning_starts:
                action = self.env.action_space.sample()
            else:
                with th.no_grad():
                    action = self.policy.get_action(th.tensor(obs).float().to(self.device), tensor_w).detach().cpu().numpy()
            next_obs, vector_reward, terminated, truncated, info = self.env.step(action)
            self.replay_buffer.push(obs, action, w, vector_reward, next_obs, terminated)
            if self.global_step >= self.learning_starts:
                self.update()
            if terminated or truncated:
                obs, _ = self.env.reset()
                self.num_episodes += 1
                if self.log and "episode" in info.keys():
                    from ...common.evaluation import log_episode_info

                    log_episode_info(info["episode"], np.dot, w, self.global_step)
            else:
                obs = next_obs
            if self.log and self.global_step % eval_freq == 0:
                from ...common.evaluation import log_all_multi_policy_metrics, policy_evaluation_mo

                returns = [policy_evaluation_mo(self, eval_env, ew, rep=num_eval_episodes_for_front)[3] for ew in eval_weights]
                log_all_multi_policy_metrics(current_front=returns, hv_ref_point=ref_point, reward_dim=self.reward_dim,
                                             global_step=self.global_step, n_sample_weights=num_eval_weights_for_eval,
                                             ref_front=known_pareto_front)
            if checkpoints and self.global_step % save_freq == 0:
                self.save(filename=f"CAPQL step={self.global_step}", save_replay_buffer=False)
        if self.log:
            self.close_wandb()
