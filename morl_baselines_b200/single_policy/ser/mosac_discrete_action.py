"""Multi-objective SAC for discrete actions on the CUDA update engine -- drop-in for reference
morl_baselines/single_policy/ser/mosac_discrete_action.py (``MODiscreteSoftQNetwork / MOSACDiscreteActor / MOSACDiscrete`` with the same
constructor, ``update / eval / train / get_buffer / set_buffer / set_weights / get_policy_net / get_save_dict / load``).
MOSACDiscrete is an inner learner of MORL/D (reference multi_policy/morld/morld.py:30-34), e.g. on mo-lunar-lander.

The soft target is an expectation under the actor's softmax over all actions (mosac_discrete_action.py:452-464): ONE kernel
(morl_discrete_sac_target_f32).  The actor and temperature losses of :478-498 are ONE kernel (morl_discrete_sac_actor_loss_f32) that also
writes d loss / d logits in closed form and d alpha_loss / d log_alpha; two autograd Functions hand those seeds upstream.  The minibatch
comes from the HBM-resident replay mirror, the Adam steps are the fused capture-safe optimiser, and the whole device side of ``update()``
is captured in one CUDA graph per (target-sync, buffer) variant (``use_cuda_graph``, common/graphed.py).

Differences from the reference, each deliberate:
  * ``update()`` draws no ``Categorical.sample()``: the reference draws twice per update and never uses the result;
  * an action whose logit is -inf leaves the expectation (the reference computes 0 * -inf = NaN), include/morl_b200.h;
  * ``load`` copies ``log_alpha`` into the live tensor, so the temperature optimiser keeps stepping the loaded value.
"""

from __future__ import annotations

import time
from copy import deepcopy
from typing import Optional, Tuple, Union

import numpy as np
import torch as th
import torch.nn as nn
import torch.nn.functional as F
from torch.distributions.categorical import Categorical

from ... import ops
from ...common.buffer import ReplayBuffer
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.morl_algorithm import MOPolicy
from ...common.networks import NatureCNN, layer_init, mlp, polyak_update


class MODiscreteSoftQNetwork(nn.Module):
    """Soft Q-network S -> |A| x |R| (reference mosac_discrete_action.py:36-76)."""

    def __init__(self, obs_shape, action_dim, reward_dim, net_arch):
        super().__init__()
        self.obs_shape, self.action_dim, self.reward_dim = obs_shape, action_dim, reward_dim
        if len(obs_shape) == 1:
            self.feature_extractor = mlp(input_dim=obs_shape[0], output_dim=-1, net_arch=net_arch[:1])
        elif len(obs_shape) > 1:  # image observation
            self.feature_extractor = NatureCNN(self.obs_shape, features_dim=net_arch[0])
        self.net = mlp(input_dim=net_arch[0], output_dim=action_dim * reward_dim, net_arch=net_arch[1:])
        self.apply(layer_init)

    def forward(self, obs):
        return self.net(self.feature_extractor(obs)).view(-1, self.action_dim, self.reward_dim)


class MOSACDiscreteActor(nn.Module):
    """Categorical actor S -> logits over A (reference mosac_discrete_action.py:79-119)."""

    def __init__(self, obs_shape: Tuple, action_dim: int, reward_dim: int, net_arch=[256, 256]):
        super().__init__()
        self.obs_shape, self.action_dim, self.reward_dim, self.net_arch = obs_shape, action_dim, reward_dim, net_arch
        if len(obs_shape) == 1:
            self.feature_extractor = mlp(obs_shape[0], -1, net_arch[:1])
        elif len(obs_shape) > 1:  # image observation
            self.feature_extractor = NatureCNN(self.obs_shape, features_dim=net_arch[0])
        self.net = mlp(net_arch[0], action_dim, net_arch[1:])
        self.apply(layer_init)

    def forward(self, x):
        return self.net(self.feature_extractor(x))

    def get_action(self, x):
        """(sampled action, log_softmax(logits), probabilities), as the reference."""
        logits = self(x)
        dist = Categorical(logits=logits)
        return dist.sample(), F.log_softmax(logits, dim=1), dist.probs


class _SeededLoss(th.autograd.Function):
    """A loss whose value and derivative w.r.t. ``x`` one kernel already computed: forward returns the loss, backward returns the
    saved derivative times grad_out (the pattern of Envelope's _FusedTDLoss)."""

    @staticmethod
    def forward(ctx, x, loss, seed):
        ctx.save_for_backward(seed)
        return loss.reshape(()).clone()

    @staticmethod
    def backward(ctx, grad_out):
        (seed,) = ctx.saved_tensors
        return seed * grad_out, None, None


class MOSACDiscrete(MOPolicy):
    """SAC for discrete actions with vector critics scalarised by a fixed weight vector (reference mosac_discrete_action.py:122-581)."""

    ADAM_EPS = 1e-4  # every optimiser of the reference's discrete SAC

    def __init__(self, env, weights: np.ndarray, scalarization=th.matmul, buffer_size: int = int(1e6), gamma: float = 0.99, tau: float = 1.0,
                 batch_size: int = 128, learning_starts: int = int(2e4), net_arch=[256, 256], policy_lr: float = 3e-4, q_lr: float = 3e-4,
                 update_frequency: int = 4, target_net_freq: int = 2000, alpha: float = 0.2, autotune: bool = True,
                 target_entropy_scale: float = 0.89, id: Optional[int] = None, device: Union[th.device, str] = "auto", log: bool = True,
                 seed: int = 42, parent_rng: Optional[np.random.Generator] = None, use_cuda_graph: bool = True):
        super().__init__(id, device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.MOSACDiscrete needs a CUDA device: the update path is CUDA-only (no CPU fallback)")
        ops._lib.load()
        self.seed = seed
        self.parent_rng = parent_rng
        self.np_random = parent_rng if parent_rng is not None else np.random.default_rng(self.seed)
        self.env = env
        assert hasattr(env.action_space, "n"), "only discrete action space is supported"
        self.obs_shape = tuple(env.observation_space.shape)
        self.action_dim = int(env.action_space.n)
        self.reward_dim = env.unwrapped.reward_space.shape[0]
        self.weights = weights
        self.weights_tensor = th.from_numpy(np.asarray(self.weights)).float().to(self.device)
        self.batch_size = batch_size
        self.scalarization = scalarization
        self.buffer_size, self.gamma, self.tau, self.learning_starts, self.net_arch = buffer_size, gamma, tau, learning_starts, net_arch
        self.policy_lr, self.q_lr, self.update_frequency, self.target_net_freq = policy_lr, q_lr, update_frequency, target_net_freq
        assert self.target_net_freq % self.update_frequency == 0, "target_net_freq should be divisible by update_frequency"
        self.target_entropy_scale = target_entropy_scale
        self.actor = MOSACDiscreteActor(self.obs_shape, self.action_dim, self.reward_dim, net_arch).to(self.device)
        mkq = lambda: MODiscreteSoftQNetwork(self.obs_shape, self.action_dim, self.reward_dim, net_arch).to(self.device)  # noqa: E731
        self.qf1, self.qf2, self.qf1_target, self.qf2_target = mkq(), mkq(), mkq(), mkq()
        self.qf1_target.requires_grad_(False)
        self.qf2_target.requires_grad_(False)
        self.qf1_target.load_state_dict(self.qf1.state_dict())
        self.qf2_target.load_state_dict(self.qf2.state_dict())
        self.q_optimizer = FusedClipAdam(list(self.qf1.parameters()) + list(self.qf2.parameters()), lr=self.q_lr, eps=self.ADAM_EPS)
        self.actor_optimizer = FusedClipAdam(list(self.actor.parameters()), lr=self.policy_lr, eps=self.ADAM_EPS)
        self.autotune = autotune
        if self.autotune:
            self.target_entropy = -self.target_entropy_scale * th.log(1 / th.tensor(self.action_dim))  # fp32, as the reference
            self.log_alpha = th.zeros(1, requires_grad=True, device=self.device)
            alpha0 = self.log_alpha.exp().item()
            self.a_optimizer = FusedClipAdam([self.log_alpha], lr=self.q_lr, eps=self.ADAM_EPS)
        else:
            alpha0 = alpha
        self.alpha_tensor = th.scalar_tensor(alpha0).to(self.device)  # updated IN PLACE (captured graphs read it)
        self.use_cuda_graph = use_cuda_graph
        self._graphs = GraphCache()
        env.observation_space.dtype = np.float32
        self.buffer = ReplayBuffer(obs_shape=self.obs_shape, action_dim=1, rew_dim=self.reward_dim, max_size=self.buffer_size, device=self.device)
        self._linear = scalarization is th.matmul
        # critic, actor and temperature loss of the latest update: written in place, so every captured graph variant updates the same views
        self._losses = th.zeros(3, device=self.device)
        self._last_qf_loss, self._last_actor_loss, self._last_alpha_loss = self._losses[0], self._losses[1], self._losses[2]
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
                "q_lr": self.q_lr, "update_frequency": self.update_frequency, "target_net_freq": self.target_net_freq, "alpha": self.alpha,
                "autotune": self.autotune, "target_entropy_scale": self.target_entropy_scale, "seed": self.seed}

    def __deepcopy__(self, memo):
        """The reference's deep copy (mosac_discrete_action.py:276-324), quirks included: the networks and the step count are copied, the
        optimisers are fresh, and with autotune ``log_alpha`` is NOT copied (the copy starts from log_alpha = 0, alpha = 1)."""
        c = type(self)(env=self.env, weights=self.weights, scalarization=self.scalarization, buffer_size=self.buffer_size, gamma=self.gamma,
                       tau=self.tau, batch_size=self.batch_size, learning_starts=self.learning_starts, net_arch=self.net_arch,
                       policy_lr=self.policy_lr, q_lr=self.q_lr, update_frequency=self.update_frequency, target_net_freq=self.target_net_freq,
                       alpha=self.alpha, autotune=self.autotune, target_entropy_scale=self.target_entropy_scale, id=self.id, device=self.device,
                       log=self.log, seed=self.seed, parent_rng=self.parent_rng, use_cuda_graph=self.use_cuda_graph)
        for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
            getattr(c, name).load_state_dict(getattr(self, name).state_dict())
        c.global_step = self.global_step
        c.actor_optimizer = FusedClipAdam(c.actor.parameters(), lr=self.policy_lr, eps=self.ADAM_EPS)
        c.q_optimizer = FusedClipAdam(list(c.qf1.parameters()) + list(c.qf2.parameters()), lr=self.q_lr, eps=self.ADAM_EPS)
        if self.autotune:
            c.a_optimizer = FusedClipAdam([c.log_alpha], lr=self.q_lr, eps=self.ADAM_EPS)
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
            d["target_entropy_scale"] = self.target_entropy_scale
        return d

    def load(self, save_dict: Optional[dict] = None, path: Optional[str] = None, load_replay_buffer: bool = True):
        if save_dict is None:
            assert path is not None, "Either save_dict or path should be provided."
            save_dict = th.load(path, map_location=self.device, weights_only=False)
        for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
            getattr(self, name).load_state_dict(save_dict[f"{name}_state_dict"])
        self.actor_optimizer.load_state_dict(save_dict["actor_optimizer_state_dict"])
        self.q_optimizer.load_state_dict(save_dict["q_optimizer_state_dict"])
        if "log_alpha" in save_dict and self.autotune:  # previously used autotune
            with th.no_grad():
                self.log_alpha.copy_(save_dict["log_alpha"].to(self.device))
            self.a_optimizer.load_state_dict(save_dict["a_optimizer_state_dict"])
            self.target_entropy_scale = save_dict["target_entropy_scale"]
            self.target_entropy = -self.target_entropy_scale * th.log(1 / th.tensor(self.action_dim))
        if load_replay_buffer and "buffer" in save_dict:
            self.buffer = save_dict["buffer"]
            if hasattr(self.buffer, "to"):
                self.buffer.to(self.device)
        self.set_weights(save_dict["weights"])
        self.alpha = save_dict["alpha"]
        self._graphs.clear()  # optimiser state tensors may have been replaced

    def eval(self, obs: np.ndarray, w: Optional[np.ndarray] = None, **kwargs):
        obs = th.as_tensor(obs).float().to(self.device).unsqueeze(0)
        with th.no_grad():
            action, _, _ = self.actor.get_action(obs)
        return action[0].detach().cpu().numpy()

    def _scal(self, q):
        return self.scalarization(q, self.weights_tensor)

    def _device_update(self, mb_obs, mb_act, mb_rewards, mb_next_obs, mb_dones, with_target: bool):
        """The device side of one update (reference mosac_discrete_action.py:445-513) on an already gathered minibatch."""
        with th.no_grad():
            next_logits = self.actor(mb_next_obs)
            q_next = th.stack([self.qf1_target(mb_next_obs), self.qf2_target(mb_next_obs)])  # [2, B, A, D]
            if self._linear:
                next_q_value = ops.discrete_sac_target(q_next, next_logits, self.weights_tensor, mb_rewards, mb_dones, self.alpha_tensor, self.gamma)
            else:  # non-linear scalarisation: outside the fused path, evaluated with the user's callable
                probs, logp = F.softmax(next_logits, dim=1), F.log_softmax(next_logits, dim=1)
                v = (probs * (th.min(self._scal(q_next[0]), self._scal(q_next[1])) - self.alpha_tensor * logp)).sum(dim=1)
                next_q_value = self._scal(mb_rewards).flatten() + (1 - mb_dones.flatten()) * self.gamma * v
        a = mb_act.long().view(-1, 1)
        qf1_a = self._scal(self.qf1(mb_obs)).gather(1, a).view(-1)
        qf2_a = self._scal(self.qf2(mb_obs)).gather(1, a).view(-1)
        qf_loss = F.mse_loss(qf1_a, next_q_value) + F.mse_loss(qf2_a, next_q_value)
        self.q_optimizer.zero_grad(set_to_none=True)
        qf_loss.backward()
        self.q_optimizer.step_fused(None)
        self._last_qf_loss.copy_(qf_loss.detach())

        logits = self.actor(mb_obs)
        with th.no_grad():
            q_now = th.stack([self.qf1(mb_obs), self.qf2(mb_obs)])  # after the critic step, as the reference
        H = float(self.target_entropy) if self.autotune else 0.0
        if self._linear:
            loss, dlogits, aloss, dla = ops.discrete_sac_actor_loss(logits.detach(), q_now, self.weights_tensor, self.alpha_tensor,
                                                                    self.log_alpha.detach() if self.autotune else None, H)
            actor_loss = _SeededLoss.apply(logits, loss, dlogits)
            alpha_loss = _SeededLoss.apply(self.log_alpha, aloss, dla) if self.autotune else None
        else:
            probs, logp = F.softmax(logits, dim=1), F.log_softmax(logits, dim=1)
            min_q = th.min(self._scal(q_now[0]), self._scal(q_now[1]))
            actor_loss = (probs * (self.alpha_tensor * logp - min_q)).mean()
            alpha_loss = (probs.detach() * (-self.log_alpha.exp() * (logp + H).detach())).mean() if self.autotune else None
        self.actor_optimizer.zero_grad(set_to_none=True)
        actor_loss.backward()
        self.actor_optimizer.step_fused(None)
        self._last_actor_loss.copy_(actor_loss.detach())
        if self.autotune:
            self.a_optimizer.zero_grad(set_to_none=True)
            alpha_loss.backward()
            self.a_optimizer.step_fused(None)
            self._last_alpha_loss.copy_(alpha_loss.detach())
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

    def update(self):
        """One SAC update (reference mosac_discrete_action.py:445-530)."""
        with_target = self.global_step % self.target_net_freq == 0
        if not self.graph_update_ready():
            smp = self.buffer.sample(self.batch_size, to_tensor=True, device=self.device)
            self._device_update(smp[0], smp[1], smp[2], smp[3], smp[4], with_target)
            return
        self._prepare_graph_update().graph()

    def graph_update_ready(self) -> bool:
        """True when ``update()`` takes the CUDA-graph path (so a population of learners can be replayed as ONE graph, morld.py)."""
        return bool(self.use_cuda_graph and getattr(self.buffer, "_dev", None) is not None)

    def _prepare_graph_update(self):
        """Host half of one graph-path update: draw the replay indices (global numpy RNG, as the reference's buffer.sample), stage them into
        the static device buffer, flush new transitions to the HBM mirror.  Returns the variant whose ``step`` closure is the device half
        (captured by its ``graph`` for this learner alone, or by a PopulationGraph for many)."""
        with_target = self.global_step % self.target_net_freq == 0
        B = self.batch_size
        key = (with_target, id(self.buffer))

        def build():
            idx = Staging(B, th.int64, self.device)

            def step():
                obs_s, nobs_s, act_s, rew_s, done_s = self.buffer._dev
                obs, act, rew, nobs, done = ops.replay_gather(obs_s, nobs_s, act_s, rew_s, done_s, idx.dev)
                self._device_update(obs, act, rew, nobs, done, with_target)

            return Variant(key, step, self._mutated_tensors, idx=idx)

        v = self._graphs.get_or_build(key, build)
        inds = self.buffer._draw(B)
        v.idx.host()[:] = inds
        v.idx.upload()
        self.buffer.flush()
        return v

    def train(self, total_timesteps: int, eval_env=None, start_time=None, verbose: bool = False):
        """Interaction loop (reference mosac_discrete_action.py:531-611)."""
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

                    log_episode_info(infos["episode"], np.dot, self.weights, self.global_step, self.id, verbose=verbose)
            if self.global_step > self.learning_starts:
                if self.global_step % self.update_frequency == 0:
                    self.update()
                if self.log and self.global_step % 100 == 0:
                    import wandb

                    wandb.log({"charts/SPS": int(self.global_step / (time.time() - start_time)), "global_step": self.global_step})
            self.global_step += 1
