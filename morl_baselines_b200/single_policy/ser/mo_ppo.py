"""Multi-objective PPO on the CUDA update engine -- drop-in for reference morl_baselines/single_policy/ser/mo_ppo.py
(``PPOReplayBuffer``, ``make_env``, ``MOPPONet`` and ``MOPPO`` with the same constructor arguments, attributes and methods).
MOPPO is the learner of PGMORL (multi_policy/pgmorl/pgmorl.py).

The critic regresses a vector value onto vector GAE returns; the policy is a diagonal Gaussian trained on the weighted sum of the
advantages.  On the device:
  * the reverse GAE recursion of a whole rollout is ONE kernel (morl_vector_gae_f32), bit-exact against the reference's returns;
  * each minibatch's clipped loss, its gradients w.r.t. the actor mean, actor_logstd and the value head, and the logged statistics are
    ONE kernel (morl_ppo_loss_f32); an autograd Function hands the gradients to the dense layers, which keep torch autograd;
  * clip + Adam is ``FusedClipAdam`` (eps 1e-5) reading the learning rate from a device scalar, so ``anneal_lr`` never re-captures;
  * ``update()`` is ONE CUDA graph replay over every epoch and minibatch (``use_cuda_graph``).  The epoch permutations are drawn on the
    host with ``self.np_random.shuffle`` exactly as the reference draws them and uploaded once per update.  With ``target_kl`` set, one
    single-epoch graph is replayed per epoch and ``approx_kl`` is read once per epoch, so early stopping consumes the same shuffles.

Differences from the reference, each deliberate:
  * the clip fraction and the other logged losses stay on the device; ``explained_var`` and the wandb values are computed only with
    ``log=True`` (the reference computes ``explained_var`` on every update and discards it);
  * the scalarised advantages are a dot product summed in double and rounded once, which may differ from the reference's matmul in the
    last bit.
"""

from __future__ import annotations

import time
from copy import deepcopy
from typing import List, Optional, Union

import numpy as np
import torch as th
from torch import nn
from torch.distributions import Normal

from ... import ops
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.morl_algorithm import MOPolicy
from ...common.networks import layer_init, mlp

DEFAULT_SEED = 42  # MOPPO's default seed: also the seed of a deep copy, which the reference builds without passing one
ADAM_EPS = 1e-5


class PPOReplayBuffer:
    """Rollout storage of ``size`` steps of ``num_envs`` environments, on the device (reference mo_ppo.py:22-104)."""

    def __init__(self, size: int, num_envs: int, obs_shape: tuple, action_shape: tuple, reward_dim: int, device: Union[th.device, str]):
        self.size, self.ptr, self.num_envs, self.device = size, 0, num_envs, device
        self.obs = th.zeros((size, num_envs) + tuple(obs_shape), device=device)
        self.actions = th.zeros((size, num_envs) + tuple(action_shape), device=device)
        self.logprobs = th.zeros((size, num_envs), device=device)
        self.rewards = th.zeros((size, num_envs, reward_dim), dtype=th.float32, device=device)
        self.dones = th.zeros((size, num_envs), device=device)
        self.values = th.zeros((size, num_envs, reward_dim), dtype=th.float32, device=device)

    FIELDS = ("obs", "actions", "logprobs", "rewards", "dones", "values")

    def add(self, obs, actions, logprobs, rewards, dones, values):
        """Store one vector-env step at ``ptr`` (in place) and advance it."""
        for name, v in zip(self.FIELDS, (obs, actions, logprobs, rewards, dones, values)):
            getattr(self, name)[self.ptr] = v
        self.ptr = (self.ptr + 1) % self.size

    def get(self, step: int):
        """(obs, actions, logprobs, rewards, dones, values) of one step."""
        return tuple(getattr(self, name)[step] for name in self.FIELDS)

    def get_all(self):
        """(obs, actions, logprobs, rewards, dones, values) of the whole rollout."""
        return tuple(getattr(self, name) for name in self.FIELDS)


def make_env(env_id, seed, idx, run_name, gamma):
    """Thunk building one mo-gymnasium environment with PPO's wrappers: action clipping, observation normalisation clipped to
    [-10, 10], per-objective reward normalisation clipped to [-10, 10], and episode statistics (reference mo_ppo.py:107-145)."""

    def thunk():
        import gymnasium as gym
        import mo_gymnasium as mo_gym

        env = mo_gym.make(env_id, render_mode="rgb_array") if idx == 0 else mo_gym.make(env_id)
        reward_dim = env.unwrapped.reward_space.shape[0]
        env = gym.wrappers.ClipAction(env)
        env = gym.wrappers.NormalizeObservation(env)
        env = gym.wrappers.TransformObservation(env, lambda obs: np.clip(obs, -10, 10), env.observation_space)
        for o in range(reward_dim):
            env = mo_gym.wrappers.MONormalizeReward(env, idx=o, gamma=gamma)
            env = mo_gym.wrappers.MOClipReward(env, idx=o, min_r=-10, max_r=10)
        env = mo_gym.wrappers.MORecordEpisodeStatistics(env, gamma=gamma)
        env.reset(seed=seed)
        env.action_space.seed(seed)
        env.observation_space.seed(seed)
        return env

    return thunk


class MOPPONet(nn.Module):
    """Tanh actor-critic: critic S -> R^d, Gaussian actor S -> mean, state-independent ``actor_logstd`` (reference mo_ppo.py:160-235).
    Same state_dict keys and the same orthogonal initialisation (hidden gain sqrt 2, critic head 1.0, mean head 0.01)."""

    def __init__(self, obs_shape: tuple, action_shape: tuple, reward_dim: int, net_arch: List = [64, 64]):
        super().__init__()
        self.obs_shape, self.action_shape, self.reward_dim, self.net_arch = obs_shape, action_shape, reward_dim, net_arch
        n_in, n_act = int(np.prod(obs_shape)), int(np.prod(action_shape))
        hidden = lambda m: layer_init(m, weight_gain=np.sqrt(2), bias_const=0.0)  # noqa: E731
        self.critic = mlp(input_dim=n_in, output_dim=reward_dim, net_arch=net_arch, activation_fn=nn.Tanh)
        self.critic.apply(hidden)
        layer_init(list(self.critic.modules())[-1], weight_gain=1.0)
        self.actor_mean = mlp(input_dim=n_in, output_dim=n_act, net_arch=net_arch, activation_fn=nn.Tanh)
        self.actor_mean.apply(hidden)
        layer_init(list(self.actor_mean.modules())[-1], weight_gain=0.01)
        self.actor_logstd = nn.Parameter(th.zeros(1, n_act))

    def get_value(self, obs):
        return self.critic(obs)

    def get_action_and_value(self, obs, action=None):
        """(action, log-prob summed over action dims, entropy summed over action dims, vector value); samples when ``action`` is None."""
        mean = self.actor_mean(obs)
        probs = Normal(mean, th.exp(self.actor_logstd.expand_as(mean)))
        if action is None:
            action = probs.sample()
        return action, probs.log_prob(action).sum(1), probs.entropy().sum(1), self.critic(obs)


class _PPOLoss(th.autograd.Function):
    """The minibatch loss whose gradients w.r.t. the actor mean, actor_logstd and the value head one kernel already computed."""

    @staticmethod
    def forward(ctx, mean, logstd, value, loss, dmean, dlogstd, dvalue):
        ctx.save_for_backward(dmean, dlogstd, dvalue)
        ctx.logstd_shape = logstd.shape
        return loss.reshape(()).clone()

    @staticmethod
    def backward(ctx, g):
        dmean, dlogstd, dvalue = ctx.saved_tensors
        return dmean * g, (dlogstd * g).reshape(ctx.logstd_shape), dvalue * g, None, None, None, None


STAT_NAMES = ("policy_loss", "value_loss", "entropy", "old_approx_kl", "approx_kl", "clipfrac")


class MOPPO(MOPolicy):
    """PPO with a vector critic and weighted-sum scalarised advantages (reference mo_ppo.py:238-613)."""

    def __init__(self, id: int, networks: MOPPONet, weights: np.ndarray, envs, log: bool = False, steps_per_iteration: int = 2048,
                 num_minibatches: int = 32, update_epochs: int = 10, learning_rate: float = 3e-4, gamma: float = 0.995, anneal_lr: bool = False,
                 clip_coef: float = 0.2, ent_coef: float = 0.0, vf_coef: float = 0.5, clip_vloss: bool = True, max_grad_norm: float = 0.5,
                 norm_adv: bool = True, target_kl: Optional[float] = None, gae: bool = True, gae_lambda: float = 0.95,
                 device: Union[th.device, str] = "auto", seed: int = DEFAULT_SEED, rng: Optional[np.random.Generator] = None,
                 use_cuda_graph: bool = True):
        super().__init__(id, device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.MOPPO needs a CUDA device: the update path is CUDA-only (no CPU fallback)")
        ops._lib.load()
        self.id, self.envs, self.num_envs, self.networks, self.seed = id, envs, envs.num_envs, networks, seed
        self.np_random = rng if rng is not None else np.random.default_rng(self.seed)
        self.steps_per_iteration = steps_per_iteration
        self.np_weights = weights
        self.weights = th.from_numpy(weights).to(self.device)
        self.batch_size = int(self.num_envs * self.steps_per_iteration)
        self.num_minibatches = num_minibatches
        self.minibatch_size = int(self.batch_size // num_minibatches)
        self.update_epochs, self.learning_rate, self.gamma, self.anneal_lr = update_epochs, learning_rate, gamma, anneal_lr
        self.clip_coef, self.vf_coef, self.ent_coef, self.max_grad_norm = clip_coef, vf_coef, ent_coef, max_grad_norm
        self.norm_adv, self.target_kl, self.clip_vloss, self.gae_lambda, self.log, self.gae = norm_adv, target_kl, clip_vloss, gae_lambda, log, gae
        self.use_cuda_graph = use_cuda_graph

        self.optimizer = FusedClipAdam(networks.parameters(), lr=self.learning_rate, eps=ADAM_EPS)
        self._lr = th.full((1,), float(self.learning_rate), dtype=th.float64, device=self.device)  # written in place by anneal_lr
        self.optimizer.lr_device = self._lr
        self.batch = PPOReplayBuffer(self.steps_per_iteration, self.num_envs, self.networks.obs_shape, self.networks.action_shape,
                                     self.networks.reward_dim, self.device)
        self._w32 = self.weights.float().reshape(-1).clone()
        # GAE outputs, written in place so captured graphs keep reading the same storage
        self.returns = th.zeros_like(self.batch.rewards)
        self.advantages = th.zeros((self.steps_per_iteration, self.num_envs), device=self.device)
        self._stats = th.zeros(6, device=self.device)
        self._perm = Staging((self.update_epochs, self.batch_size), th.int64, self.device)
        self._graphs = GraphCache()

    def __deepcopy__(self, memo):
        """The reference's deep copy (mo_ppo.py:343-376): an independent network, a FRESH Adam, a deep-copied batch, the step count; the
        copy is built without ``seed`` or ``rng``, so it draws its shuffles from its own generator seeded with the default seed."""
        copied_net = deepcopy(self.networks, memo)
        c = type(self)(self.id, copied_net, self.weights.detach().cpu().numpy(), self.envs, self.log, self.steps_per_iteration, self.num_minibatches,
                       self.update_epochs, self.learning_rate, self.gamma, self.anneal_lr, self.clip_coef, self.ent_coef, self.vf_coef, self.clip_vloss,
                       self.max_grad_norm, self.norm_adv, self.target_kl, self.gae, self.gae_lambda, self.device, use_cuda_graph=self.use_cuda_graph)
        c.global_step = self.global_step
        c.batch = deepcopy(self.batch, memo)
        return c

    @th.no_grad()
    def become_copy_of(self, src: "MOPPO"):
        """Make this learner what ``deepcopy(src)`` would be, writing into its existing tensors: parameters, a zeroed (fresh) Adam state,
        the batch, the step count, the weights and a generator seeded with the default seed.  Graphs captured on this learner stay valid."""
        for p, q in zip(self.networks.parameters(), src.networks.parameters()):
            p.copy_(q)
        self.optimizer._ensure_state()
        for st in self.optimizer.state.values():
            for k in ("step", "exp_avg", "exp_avg_sq"):
                st[k].zero_()
        self.optimizer.param_groups[0]["lr"] = self.learning_rate
        self._lr.fill_(float(self.learning_rate))
        for name in PPOReplayBuffer.FIELDS:
            getattr(self.batch, name).copy_(getattr(src.batch, name))
        self.batch.ptr = src.batch.ptr
        self.id, self.global_step = src.id, src.global_step
        self.np_weights = src.weights.detach().cpu().numpy()
        self.change_weights(self.np_weights)
        self.seed = DEFAULT_SEED
        self.np_random = np.random.default_rng(self.seed)

    def change_weights(self, new_weights: np.ndarray):
        """Scalarisation weights of the advantages."""
        self.weights = th.from_numpy(deepcopy(new_weights)).to(self.device)
        self._w32.copy_(self.weights.float().reshape(-1))

    def __collect_samples(self, obs: th.Tensor, done: th.Tensor):
        """Fill the batch with ``steps_per_iteration`` vector-env steps (reference mo_ppo.py:390-431)."""
        for _ in range(self.steps_per_iteration):
            self.global_step += 1 * self.num_envs
            with th.no_grad():
                action, logprob, _, value = self.networks.get_action_and_value(obs)
                value = value.view(self.num_envs, self.networks.reward_dim)
            next_obs, reward, next_terminated, next_truncated, info = self.envs.step(action.cpu().numpy())
            reward = th.tensor(reward).to(self.device).view(self.num_envs, self.networks.reward_dim)
            self.batch.add(obs, action, logprob, reward, done, value)
            obs, done = th.Tensor(next_obs).to(self.device), th.Tensor(next_terminated).to(self.device)
            if self.log and "episode" in info.keys():
                from ...common.evaluation import log_episode_info

                for idx in np.where(next_terminated | next_truncated)[0]:
                    log_episode_info({k: v[idx] for k, v in info["episode"].items()}, scalarization=np.dot, weights=self.weights,
                                     global_timestep=self.global_step, id=self.id)
        return obs, done

    def __compute_advantages(self, next_obs, next_done):
        """(vector returns [T, E, d], scalarised advantages [T, E]) of the batch: one kernel (reference mo_ppo.py:433-476)."""
        with th.no_grad():
            next_value = self.networks.get_value(next_obs).reshape(self.num_envs, -1)
            return ops.vector_gae(self.batch.rewards, self.batch.values, self.batch.dones, next_value.contiguous(), next_done.float().contiguous(),
                                  self._w32, self.gamma, self.gae_lambda, self.gae, returns_out=self.returns, adv_out=self.advantages)

    def eval(self, obs: np.ndarray, w=None):
        """A sampled action for one observation (reference mo_ppo.py:478-490)."""
        obs = th.as_tensor(obs).float().to(self.device).unsqueeze(0).repeat(self.num_envs, 1)
        with th.no_grad():
            action, _, _, _ = self.networks.get_action_and_value(obs)
        return action[0].detach().cpu().numpy()

    # ---- update ------------------------------------------------------------------------------------------------------------------
    def _epochs(self, epochs):
        """Device half of ``len(epochs)`` epochs: minibatch gathers, forward, loss kernel, backward, clip + Adam (reference
        mo_ppo.py:507-554).  Row ``e`` of the uploaded permutations orders epoch ``e``."""
        net = self.networks
        obs_shape, act_shape, d = tuple(net.obs_shape), tuple(net.action_shape), net.reward_dim
        b_obs = self.batch.obs.reshape((-1,) + obs_shape)
        b_actions = self.batch.actions.reshape((-1,) + act_shape)
        b_logprobs, b_values = self.batch.logprobs.reshape(-1), self.batch.values.reshape(-1, d)
        b_advantages, b_returns = self.advantages.reshape(-1), self.returns.reshape(-1, d)
        for e in epochs:
            for start in range(0, self.batch_size, self.minibatch_size):
                idx = self._perm.dev[e, start:start + self.minibatch_size]
                mb_obs = b_obs.index_select(0, idx)
                mean = net.actor_mean(mb_obs)
                value = net.critic(mb_obs).view(-1, d)
                loss, dmean, dlogstd, dvalue = ops.ppo_loss(mean.detach(), net.actor_logstd.detach(), value.detach(), b_actions.index_select(0, idx),
                                                            b_logprobs.index_select(0, idx), b_advantages.index_select(0, idx),
                                                            b_returns.index_select(0, idx), b_values.index_select(0, idx), self.clip_coef,
                                                            self.ent_coef, self.vf_coef, self.norm_adv, self.clip_vloss, self._stats)
                total = _PPOLoss.apply(mean, net.actor_logstd, value, loss, dmean, dlogstd, dvalue)
                self.optimizer.zero_grad(set_to_none=True)
                total.backward()
                self.optimizer.step_fused(self.max_grad_norm)

    def _mutated_tensors(self):
        return list(self.networks.parameters()) + optimizer_tensors(self.optimizer) + [self._stats]

    def _variant(self, key):
        """Per-variant device step: "all" runs every epoch (zeroing the clip-fraction sum first), "epoch" runs one epoch from row 0."""
        def build():
            if key == "all":
                def step():
                    self._stats[5].zero_()
                    self._epochs(range(self.update_epochs))
            else:
                def step():
                    self._epochs([0])
            return Variant(key, step, self._mutated_tensors)

        return self._graphs.get_or_build(key, build)

    def _upload_permutations(self, n_epochs: int):
        """Draw ``n_epochs`` shuffles of the running index order (in place, as the reference does) and copy them to the device."""
        rows = self._perm.host()
        for e in range(n_epochs):
            self.np_random.shuffle(self._b_inds)
            rows[e] = self._b_inds
        self._perm.upload(n_epochs)

    def prepare_update(self):
        """Host half of a full update without early stopping: draws and uploads every epoch's shuffle; returns the device step."""
        self._b_inds = np.arange(self.batch_size)
        self._upload_permutations(self.update_epochs)
        return self._variant("all")

    def _run(self, st):
        if self.use_cuda_graph:
            st.graph()
        else:
            st.step()

    def update(self):
        if self.target_kl is None:
            self._run(self.prepare_update())
        else:
            self._b_inds = np.arange(self.batch_size)
            self._stats.zero_()
            st = self._variant("epoch")
            for _ in range(self.update_epochs):
                self._upload_permutations(1)
                self._run(st)
                if np.float32(self._stats[4].item()) > np.float32(self.target_kl):
                    break
        if self.log:
            self._log_update()

    def _log_update(self):
        import wandb

        y_pred = self.batch.values.reshape(-1, self.networks.reward_dim).cpu().numpy()
        y_true = self.returns.reshape(-1, self.networks.reward_dim).cpu().numpy()
        var_y = np.var(y_true)
        explained_var = np.nan if var_y == 0 else 1 - np.var(y_true - y_pred) / var_y
        s = self._stats.cpu().numpy()
        n_minibatches = len(range(0, self.batch_size, self.minibatch_size))
        vals = {f"losses_{self.id}/{k}": float(v) for k, v in zip(STAT_NAMES[:5], s[:5])}
        vals[f"losses_{self.id}/clipfrac"] = float(s[5]) / (n_minibatches * self.update_epochs) if self.target_kl is None else float("nan")
        vals.update({f"charts_{self.id}/learning_rate": float(self._lr.item()), f"losses_{self.id}/explained_variance": explained_var,
                     "global_step": self.global_step})
        wandb.log(vals)

    def set_learning_rate(self, lr: float):
        """Learning rate of the next updates (a device write: captured graphs read it at replay)."""
        self.optimizer.param_groups[0]["lr"] = lr
        self._lr.fill_(float(lr))

    def rollout(self, current_iteration: int, max_iterations: int):
        """The host half of ``train``: reset, learning-rate schedule, rollout and GAE (reference mo_ppo.py:588-602)."""
        next_obs, _ = self.envs.reset(seed=self.seed)
        next_obs = th.Tensor(next_obs).to(self.device)
        next_done = th.zeros(self.num_envs).to(self.device)
        if self.anneal_lr:
            self.set_learning_rate((1.0 - (current_iteration - 1.0) / max_iterations) * self.learning_rate)
        next_obs, next_done = self.__collect_samples(next_obs, next_done)
        self.__compute_advantages(next_obs, next_done)

    def train(self, start_time, current_iteration: int, max_iterations: int):
        """One iteration: ``steps_per_iteration * num_envs`` environment steps, then one update (reference mo_ppo.py:580-613)."""
        self.rollout(current_iteration, max_iterations)
        self.update()
        print("SPS:", int(self.global_step / (time.time() - start_time)))
        if self.log:
            import wandb

            print(f"Worker {self.id} - Global step: {self.global_step}")
            wandb.log({"charts/SPS": int(self.global_step / (time.time() - start_time)), "global_step": self.global_step})
