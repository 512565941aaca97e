"""Multi-objective SAC (continuous actions) on the CUDA update engine -- drop-in for reference
morl_baselines/single_policy/ser/mosac_continuous_action.py (``MOSoftQNetwork / MOSACActor / MOSAC`` with the same
constructor, ``update / eval / train / get_buffer / set_buffer / set_weights / get_policy_net / get_save_dict / load``).
MOSAC is the inner learner of MORL/D (reference multi_policy/morld/morld.py:30-34).

Hot-path row a13 of SURVEY.md section 8: scalarise both target critics, min, - alpha * logp, scalarise the reward, Bellman
(mosac_continuous_action.py:435-442) is ONE kernel (morl_actor_critic_td_f32, variant SCALAR_MIN); the minibatch comes from
the HBM-resident replay mirror with one gather kernel; both target syncs are multi-tensor launches; clip-free Adam steps are the fused
two-launch optimiser.  The reference's update is ~250 tiny tensor operations (launch
bound); here the whole device side of ``update()`` -- gather, critic step, ``policy_freq`` actor / temperature steps, target syncs --
is captured in CUDA graphs over static index / noise buffers (``use_cuda_graph``, common/graphed.py) and replayed with one host call.
"""

from __future__ import annotations

import math
import time
from copy import deepcopy
from typing import Optional, Tuple, Union

import numpy as np
import torch as th
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...common.buffer import ReplayBuffer
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.morl_algorithm import MOPolicy
from ...common.networks import layer_init, mlp, polyak_update

LOG_STD_MAX = 2
LOG_STD_MIN = -5


class MOSoftQNetwork(nn.Module):
    """Vector soft critic Q(s, a) -> R^d (reference mosac_continuous_action.py:28-58)."""

    def __init__(self, obs_shape, action_shape, reward_dim, net_arch=[256, 256]):
        super().__init__()
        self.obs_shape, self.action_shape, self.reward_dim, self.net_arch = obs_shape, action_shape, reward_dim, net_arch
        self.critic = mlp(input_dim=int(np.array(obs_shape).prod() + np.prod(action_shape)), output_dim=reward_dim, net_arch=net_arch,
                          activation_fn=nn.ReLU)
        self.apply(layer_init)

    def forward(self, x, a):
        return self.critic(th.cat([x, a], dim=-1))


class MOSACActor(nn.Module):
    """Squashed-Gaussian actor (reference mosac_continuous_action.py:65-123)."""

    def __init__(self, obs_shape: Tuple, action_shape: Tuple, reward_dim: int, action_lower_bound, action_upper_bound, net_arch=[256, 256]):
        super().__init__()
        self.obs_shape, self.action_shape, self.reward_dim, self.net_arch = obs_shape, action_shape, reward_dim, net_arch
        self.latent_pi = mlp(int(np.array(obs_shape).prod()), -1, net_arch)
        self.fc_mean = nn.Linear(net_arch[-1], int(np.prod(action_shape)))
        self.fc_logstd = nn.Linear(net_arch[-1], int(np.prod(action_shape)))
        self.apply(layer_init)
        self.register_buffer("action_scale", th.tensor((action_upper_bound - action_lower_bound) / 2.0, dtype=th.float32))
        self.register_buffer("action_bias", th.tensor((action_upper_bound + action_lower_bound) / 2.0, dtype=th.float32))

    def forward(self, x):
        x = self.latent_pi(x)
        mean = self.fc_mean(x)
        log_std = th.tanh(self.fc_logstd(x))
        log_std = LOG_STD_MIN + 0.5 * (LOG_STD_MAX - LOG_STD_MIN) * (log_std + 1)
        return mean, log_std

    def get_action(self, x, noise: Optional[th.Tensor] = None):
        """(action, log_prob [B, 1], squashed mean); ``noise`` may be injected for reproducible parity tests.  The Gaussian is written
        out with the arithmetic of ``torch.distributions.Normal`` (rsample: loc + eps * scale; log_prob: -((v - loc)^2) / (2 var) -
        log(scale) - log(sqrt(2 pi))), without the distribution object: its argument validation synchronises with the host, which is
        illegal under CUDA-graph capture."""
        mean, log_std = self(x)
        std = log_std.exp()
        eps = th.randn_like(mean) if noise is None else noise
        x_t = mean + eps * std
        y_t = th.tanh(x_t)
        action = y_t * self.action_scale + self.action_bias
        var = std**2
        log_prob = -((x_t - mean) ** 2) / (2 * var) - std.log() - math.log(math.sqrt(2 * math.pi))
        log_prob = log_prob - th.log(self.action_scale * (1 - y_t.pow(2)) + 1e-6)
        log_prob = log_prob.sum(1, keepdim=True)
        return action, log_prob, th.tanh(mean) * self.action_scale + self.action_bias


class MOSAC(MOPolicy):
    """SAC with vector critics scalarised by a fixed weight vector (reference mosac_continuous_action.py:126-572)."""

    def __init__(self, env, weights: np.ndarray, scalarization=th.matmul, buffer_size: int = int(1e6), gamma: float = 0.99,
                 tau: float = 0.005, batch_size: int = 128, learning_starts: int = int(1e3), net_arch=[256, 256], policy_lr: float = 3e-4,
                 q_lr: float = 1e-3, policy_freq: int = 2, target_net_freq: int = 1, alpha: float = 0.2, autotune: bool = True,
                 id: Optional[int] = None, device: Union[th.device, str] = "auto", log: bool = True, seed: int = 42,
                 parent_rng: Optional[np.random.Generator] = None, use_cuda_graph: bool = True):
        super().__init__(id, device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.MOSAC needs a CUDA device: the update path is CUDA-only (no CPU fallback)")
        ops._lib.load()
        self.seed = seed
        self.parent_rng = parent_rng
        self.np_random = parent_rng if parent_rng is not None else np.random.default_rng(self.seed)
        self.env = env
        assert hasattr(env.action_space, "low") and hasattr(env.action_space, "high"), "only continuous action space is supported"
        self.obs_shape = tuple(env.observation_space.shape)
        self.action_shape = tuple(env.action_space.shape)
        self.reward_dim = env.unwrapped.reward_space.shape[0]
        self.weights = weights
        self.weights_tensor = th.from_numpy(np.asarray(self.weights)).float().to(self.device)
        self.batch_size = batch_size
        self.scalarization = scalarization
        self.buffer_size, self.gamma, self.tau, self.learning_starts, self.net_arch = buffer_size, gamma, tau, learning_starts, net_arch
        self.policy_lr, self.q_lr, self.policy_freq, self.target_net_freq = policy_lr, q_lr, policy_freq, target_net_freq
        lo, hi = env.action_space.low, env.action_space.high
        self.actor = MOSACActor(self.obs_shape, self.action_shape, self.reward_dim, lo, hi, net_arch).to(self.device)
        mkq = lambda: MOSoftQNetwork(self.obs_shape, self.action_shape, self.reward_dim, net_arch).to(self.device)  # noqa: E731
        self.qf1, self.qf2, self.qf1_target, self.qf2_target = mkq(), mkq(), mkq(), mkq()
        self.qf1_target.requires_grad_(False)
        self.qf2_target.requires_grad_(False)
        self.qf1_target.load_state_dict(self.qf1.state_dict())
        self.qf2_target.load_state_dict(self.qf2.state_dict())
        # torch.optim.Adam subclasses with the reference's arithmetic and state_dict layout, two launches per step, capture-safe
        self.q_optimizer = FusedClipAdam(list(self.qf1.parameters()) + list(self.qf2.parameters()), lr=self.q_lr)
        self.actor_optimizer = FusedClipAdam(list(self.actor.parameters()), lr=self.policy_lr)
        self.autotune = autotune
        if self.autotune:
            self.target_entropy = -float(np.prod(self.action_shape))
            self.log_alpha = th.zeros(1, requires_grad=True, device=self.device)
            alpha0 = self.log_alpha.exp().item()
            self.a_optimizer = FusedClipAdam([self.log_alpha], lr=self.q_lr)
        else:
            alpha0 = alpha
        self.alpha_tensor = th.scalar_tensor(alpha0).to(self.device)  # updated IN PLACE (captured graphs read it)
        self.use_cuda_graph = use_cuda_graph
        self._graphs = GraphCache()
        self.buffer = ReplayBuffer(obs_shape=self.obs_shape, action_dim=self.action_shape[0], rew_dim=self.reward_dim, max_size=self.buffer_size,
                                   device=self.device)
        self._linear = scalarization is th.matmul
        self._noise_hook = None
        self.log = log

    @property
    def alpha(self) -> float:
        """Entropy temperature as a python float (read lazily from the device scalar: no host sync inside ``update``)."""
        return float(self.alpha_tensor)

    @alpha.setter
    def alpha(self, value):
        with th.no_grad():
            self.alpha_tensor.fill_(float(value))

    def get_config(self) -> dict:
        return {"env_id": self.env.unwrapped.spec.id, "buffer_size": self.buffer_size, "gamma": self.gamma, "tau": self.tau,
                "batch_size": self.batch_size, "learning_starts": self.learning_starts, "net_arch": self.net_arch, "policy_lr": self.policy_lr,
                "q_lr": self.q_lr, "policy_freq": self.policy_freq, "target_net_freq": self.target_net_freq, "alpha": self.alpha,
                "autotune": self.autotune, "seed": self.seed}

    def __deepcopy__(self, memo):
        """Deep copy sharing nothing but the environment (reference mosac_continuous_action.py:295-340)."""
        c = type(self)(env=self.env, weights=self.weights, scalarization=self.scalarization, buffer_size=self.buffer_size, gamma=self.gamma,
                       tau=self.tau, batch_size=self.batch_size, learning_starts=self.learning_starts, net_arch=self.net_arch,
                       policy_lr=self.policy_lr, q_lr=self.q_lr, policy_freq=self.policy_freq, target_net_freq=self.target_net_freq,
                       alpha=self.alpha, autotune=self.autotune, id=self.id, device=self.device, log=self.log, seed=self.seed,
                       parent_rng=self.parent_rng)
        for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
            getattr(c, name).load_state_dict(getattr(self, name).state_dict())
        c.global_step = self.global_step
        c.actor_optimizer = FusedClipAdam(c.actor.parameters(), lr=self.policy_lr, eps=1e-5)
        c.q_optimizer = FusedClipAdam(list(c.qf1.parameters()) + list(c.qf2.parameters()), lr=self.q_lr)
        if self.autotune:
            with th.no_grad():
                c.log_alpha.copy_(self.log_alpha)
            c.a_optimizer = FusedClipAdam([c.log_alpha], lr=self.q_lr)
        with th.no_grad():
            c.alpha_tensor.copy_(self.alpha_tensor)
        c._graphs.clear()
        c.buffer = self.buffer if memo.get("share_buffer") else deepcopy(self.buffer)
        return c

    def get_buffer(self):
        return self.buffer

    def set_buffer(self, buffer):
        self.buffer = buffer
        self._graphs.clear()  # captured graphs read the previous buffer's device stores

    def get_policy_net(self) -> th.nn.Module:
        return self.actor

    def set_weights(self, weights: np.ndarray):
        self.weights = weights
        new = th.from_numpy(np.asarray(self.weights)).float().to(self.device)
        if hasattr(self, "weights_tensor") and self.weights_tensor.shape == new.shape:
            self.weights_tensor.copy_(new)  # in place: captured graphs read this tensor
        else:
            self.weights_tensor = new

    def get_save_dict(self, save_replay_buffer: bool = False) -> dict:
        d = {"actor_state_dict": self.actor.state_dict(), "qf1_state_dict": self.qf1.state_dict(), "qf2_state_dict": self.qf2.state_dict(),
             "qf1_target_state_dict": self.qf1_target.state_dict(), "qf2_target_state_dict": self.qf2_target.state_dict(),
             "actor_optimizer_state_dict": self.actor_optimizer.state_dict(), "q_optimizer_state_dict": self.q_optimizer.state_dict(),
             "weights": self.weights, "alpha": self.alpha}
        if save_replay_buffer:
            d["buffer"] = self.buffer
        if self.autotune:
            d["log_alpha"] = self.log_alpha
            d["a_optimizer_state_dict"] = self.a_optimizer.state_dict()
        return d

    def load(self, save_dict: Optional[dict] = None, path: Optional[str] = None, load_replay_buffer: bool = True):
        if save_dict is None:
            assert path is not None, "Either save_dict or path should be provided."
            save_dict = th.load(path, map_location=self.device, weights_only=False)
        for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
            getattr(self, name).load_state_dict(save_dict[f"{name}_state_dict"])
        self.actor_optimizer.load_state_dict(save_dict["actor_optimizer_state_dict"])
        self.q_optimizer.load_state_dict(save_dict["q_optimizer_state_dict"])
        if "log_alpha" in save_dict and self.autotune:
            with th.no_grad():
                self.log_alpha.copy_(save_dict["log_alpha"].to(self.device))
            self.a_optimizer.load_state_dict(save_dict["a_optimizer_state_dict"])
        if load_replay_buffer and "buffer" in save_dict:
            self.buffer = save_dict["buffer"]
            if hasattr(self.buffer, "to"):
                self.buffer.to(self.device)
        self.set_weights(save_dict["weights"])
        self.alpha = save_dict["alpha"]
        self._graphs.clear()  # optimiser state tensors may have been replaced

    def eval(self, obs: np.ndarray, w: Optional[np.ndarray] = None):
        obs = th.as_tensor(obs).float().to(self.device).unsqueeze(0)
        with th.no_grad():
            action, _, _ = self.actor.get_action(obs)
        return action[0].detach().cpu().numpy()

    def _scal(self, q):
        return self.scalarization(q, self.weights_tensor)

    def _device_update(self, mb_obs, mb_act, mb_rewards, mb_next_obs, mb_dones, with_actor: bool, with_target: bool, noise):
        """The device side of one SAC update (reference mosac_continuous_action.py:432-507) on an already gathered minibatch.
        ``noise(k)`` returns the injected standard-normal tensor of the k-th sampling site or None (torch RNG)."""
        with th.no_grad():
            next_a, next_logp, _ = self.actor.get_action(mb_next_obs, noise(0))
            q_next = th.stack([self.qf1_target(mb_next_obs, next_a), self.qf2_target(mb_next_obs, next_a)])  # [2, B, D]
            if self._linear:
                # scalarise, min over critics, - alpha * logp, scalarised reward, Bellman: one kernel (:438-442).  alpha * logp is
                # formed on the device (fl(alpha * logp), as the reference) so that no host value of alpha is baked into a graph.
                next_q_value = ops.actor_critic_td(q_next, self.weights_tensor, mb_rewards, mb_dones, self.alpha_tensor * next_logp, 1.0, self.gamma,
                                                   ops.AC_SCALAR_MIN)
            else:  # non-linear scalarisation (Tchebycheff): outside the fused path, evaluated with the user's callable
                mn = th.min(self._scal(q_next[0]), self._scal(q_next[1])) - (self.alpha_tensor * next_logp).flatten()
                next_q_value = self._scal(mb_rewards).flatten() + (1 - mb_dones.flatten()) * self.gamma * mn
        qf1_a = self._scal(self.qf1(mb_obs, mb_act)).flatten()
        qf2_a = self._scal(self.qf2(mb_obs, mb_act)).flatten()
        qf_loss = F.mse_loss(qf1_a, next_q_value) + F.mse_loss(qf2_a, next_q_value)
        self.q_optimizer.zero_grad(set_to_none=True)
        qf_loss.backward()
        self.q_optimizer.step_fused(None)
        self._last_qf_loss = qf_loss.detach()

        if with_actor:
            k = 1
            for _ in range(self.policy_freq):
                pi, log_pi, _ = self.actor.get_action(mb_obs, noise(k))
                k += 1
                min_qf_pi = th.min(self._scal(self.qf1(mb_obs, pi)), self._scal(self.qf2(mb_obs, pi))).view(-1)
                actor_loss = ((self.alpha_tensor * log_pi) - min_qf_pi).mean()
                self.actor_optimizer.zero_grad(set_to_none=True)
                actor_loss.backward()
                self.actor_optimizer.step_fused(None)
                if self.autotune:
                    with th.no_grad():
                        _, log_pi, _ = self.actor.get_action(mb_obs, noise(k))
                    k += 1
                    alpha_loss = (-self.log_alpha * (log_pi + self.target_entropy)).mean()
                    self.a_optimizer.zero_grad(set_to_none=True)
                    alpha_loss.backward()
                    self.a_optimizer.step_fused(None)
                    with th.no_grad():
                        self.alpha_tensor.copy_(self.log_alpha.exp().detach().reshape(()))
        if with_target:
            polyak_update(self.qf1.parameters(), self.qf1_target.parameters(), self.tau)
            polyak_update(self.qf2.parameters(), self.qf2_target.parameters(), self.tau)

    def _mutated_tensors(self):
        ts = [p for m in (self.actor, self.qf1, self.qf2, self.qf1_target, self.qf2_target) for p in m.parameters()] + [self.alpha_tensor]
        opts = [self.q_optimizer, self.actor_optimizer]
        if self.autotune:
            ts.append(self.log_alpha)
            opts.append(self.a_optimizer)
        for o in opts:
            ts += optimizer_tensors(o)
        return ts

    def _n_noise_sites(self, with_actor: bool) -> int:
        return 1 + (self.policy_freq * (2 if self.autotune else 1) if with_actor else 0)

    def update(self):
        """One SAC update (reference mosac_continuous_action.py:429-507)."""
        with_actor = self.global_step % self.policy_freq == 0
        with_target = self.global_step % self.target_net_freq == 0
        B, act_dim = self.batch_size, int(np.prod(self.action_shape))
        hook = self._noise_hook
        if not self.graph_update_ready():
            smp = self.buffer.sample(B, to_tensor=True, device=self.device)
            self._device_update(smp[0], smp[1], smp[2], smp[3], smp[4], with_actor, with_target,
                                (lambda k: hook((B, act_dim))) if hook is not None else (lambda k: None))
            return
        self._prepare_graph_update().graph()

    def graph_update_ready(self) -> bool:
        """True when ``update()`` takes the CUDA-graph path (so a population of learners can be replayed as ONE graph, morld.py)."""
        return bool(self.use_cuda_graph and getattr(self.buffer, "_dev", None) is not None)

    def _prepare_graph_update(self):
        """Host half of one graph-path update: draw the replay indices (global numpy RNG, as the reference's buffer.sample), stage them and
        any injected noise into the static device buffers, flush new transitions to the HBM mirror.  Returns the variant whose ``step``
        closure is the device half (captured by its ``graph`` for this learner alone, or by a PopulationGraph for many)."""
        with_actor = self.global_step % self.policy_freq == 0
        with_target = self.global_step % self.target_net_freq == 0
        B, act_dim = self.batch_size, int(np.prod(self.action_shape))
        hook = self._noise_hook
        key = (with_actor, with_target, hook is not None, id(self.buffer))

        def build():
            idx = Staging(B, th.int64, self.device)
            noise = [th.zeros(B, act_dim, device=self.device) for _ in range(self._n_noise_sites(with_actor))] if hook is not None else None

            def step():
                obs_s, nobs_s, act_s, rew_s, done_s = self.buffer._dev
                obs, act, rew, nobs, done = ops.replay_gather(obs_s, nobs_s, act_s, rew_s, done_s, idx.dev)
                self._device_update(obs, act, rew, nobs, done, with_actor, with_target, (lambda k: noise[k]) if noise is not None else (lambda k: None))

            return Variant(key, step, self._mutated_tensors, idx=idx, noise=noise)

        v = self._graphs.get_or_build(key, build)
        inds = self.buffer._draw(B)
        v.idx.host()[:] = inds
        v.idx.upload()
        if hook is not None:
            for t in v.noise:
                t.copy_(hook((B, act_dim)))
        self.buffer.flush()
        return v

    def train(self, total_timesteps: int, eval_env=None, start_time=None):
        """Interaction loop (reference mosac_continuous_action.py:509-572)."""
        if start_time is None:
            start_time = time.time()
        obs, _ = self.env.reset()
        for _ in range(total_timesteps):
            if self.global_step < self.learning_starts:
                actions = self.env.action_space.sample()
            else:
                with th.no_grad():
                    actions, _, _ = self.actor.get_action(th.as_tensor(obs).float().to(self.device).unsqueeze(0))
                actions = actions[0].detach().cpu().numpy()
            next_obs, rewards, terminated, truncated, infos = self.env.step(actions)
            real_next_obs = infos["final_observation"] if "final_observation" in infos else next_obs
            self.buffer.add(obs=obs, next_obs=real_next_obs, action=actions, reward=rewards, done=terminated)
            obs = next_obs
            if terminated or truncated:
                obs, _ = self.env.reset()
                if self.log and "episode" in infos.keys():
                    from ...common.evaluation import log_episode_info

                    log_episode_info(infos["episode"], np.dot, self.weights, self.global_step, self.id)
            if self.global_step > self.learning_starts:
                self.update()
                if self.log and self.global_step % 100 == 0:
                    import wandb

                    wandb.log({"charts/SPS": int(self.global_step / (time.time() - start_time)), "global_step": self.global_step})
            self.global_step += 1
