"""Non-linear multi-objective PPO on the CUDA update engine -- drop-in for reference morl_baselines/single_policy/ser/nl_mo_ppo.py
(``layer_init``, ``Agent`` and ``NLMOPPO`` with the same constructor arguments, attributes and methods).  NLMOPPO is the learner IPRO's
outer loop calls once per referent.

The policy is a Categorical actor and the critic a vector value head, both on the observation augmented with the accrued discounted
reward and a preference vector.  The surrogate is clipped per objective and weighted by ``w = du/dv(s0)``, the gradient of the user's
utility ``u`` at the mean value of the initial observations.  What runs where, for shapes of ``nl_ppo_ops.nl_ppo_supported``:
  * Rollout, per vector-env step: the forward kernel on the carried observations (values written straight into the step's storage row),
    ``Categorical(logits).sample()`` on the CUDA generator as the reference samples, one device-to-host copy of the actions and one sync,
    then the environment outputs go up in one pinned copy and one commit kernel stores the step and advances the accrued reward and the
    timestep, bit-identical to the reference's device expression.
  * GAE: one kernel writing the per-objective advantages and returns, bit-identical to the reference's float32 loop.
  * ``update()``: the host evaluates the loss weights (the forward kernel on ``init_obs``, ``.mean(0)``, ``autograd.grad`` of ``u_func``)
    and draws the epoch shuffles with ``self.rng.shuffle`` in place, as the reference does.  The device then replays ONE CUDA graph of
    every epoch and minibatch: the fused update pair (``morl_nl_ppo_update_f32``) and ``FusedClipAdam.step_fused(max_grad_norm)``.  With
    ``target_kl`` one single-epoch graph is replayed per epoch and ``approx_kl`` read once per epoch, so early stopping draws the
    reference's shuffles.  ``anneal_lr``, the loss weights and the preference are device writes, read at replay: no recapture.
  * ``policy_evaluate``: the forward kernel on one pinned row; ``deterministic=True`` reads its argmax, the stochastic path samples from
    its logits with ``Categorical`` on the device.

Other shapes run the reference's expressions through torch autograd on the same device storages; the choice depends on the shape alone.

Differences from the reference, each deliberate:
  * ``update()`` returns the last minibatch's losses and KL estimates as CPU scalars read once per update, and the clip fraction as the
    float32 sum of the minibatch fractions over their count;
  * ``eval`` (one sampled action for a given preference) runs the Agent's torch forward: its preference is an argument of the call,
    not the learner's.
"""

from __future__ import annotations

import time
from math import ceil
from typing import Callable, Literal, Optional, Union

import numpy as np
import torch
import torch.nn as nn
from torch.distributions.categorical import Categorical

from ... import nl_ppo_ops, ops
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import GraphCache, Staging, Variant, optimizer_tensors
from ...common.morl_algorithm import MOPolicy

ADAM_EPS = 1e-5


def layer_init(layer, std=np.sqrt(2), bias_const=0.0):
    """Orthogonal weights with gain ``std`` and constant biases."""
    torch.nn.init.orthogonal_(layer.weight, std)
    torch.nn.init.constant_(layer.bias, bias_const)
    return layer


class Agent(nn.Module):
    """Tanh actor-critic on [obs || accrued reward || pref] (reference nl_mo_ppo.py:26-108).  The pref columns are zeros when no
    preference is given, so the input width is fixed; ``pref_dim`` may be 0."""

    def __init__(self, envs, num_objectives: int, pref_dim: int):
        super().__init__()
        self.num_objectives, self.pref_dim = num_objectives, pref_dim
        in_dim = int(np.array(envs.single_observation_space.shape).prod()) + num_objectives + pref_dim

        def net(n_out, head_std):
            return nn.Sequential(layer_init(nn.Linear(in_dim, 64)), nn.Tanh(), layer_init(nn.Linear(64, 64)), nn.Tanh(),
                                 layer_init(nn.Linear(64, n_out), std=head_std))

        # critic first, then actor: a seeded construction draws the reference's initial parameters
        self.critic = net(num_objectives, 1.0)
        self.actor = net(envs.single_action_space.n, 0.01)

    def _build_aug_obs(self, x, acc_reward, pref):
        x = x.float()
        acc_reward = acc_reward.float().to(x.device)
        if x.ndim < 2:
            parts = [x, acc_reward]
            if self.pref_dim > 0:
                parts.append(torch.zeros(self.pref_dim, device=x.device, dtype=x.dtype) if pref is None else pref.float().to(x.device).view(-1))
            return torch.cat(parts, dim=-1)
        B = x.shape[0]
        parts = [x, acc_reward.expand(B, -1) if acc_reward.ndim == 1 else acc_reward]
        if self.pref_dim > 0:
            if pref is None:
                parts.append(torch.zeros((B, self.pref_dim), device=x.device, dtype=x.dtype))
            else:
                pref = pref.float().to(x.device)
                parts.append(pref.expand(B, -1) if pref.ndim == 1 or pref.shape[0] != B else pref)
        return torch.cat(parts, dim=-1)

    def get_value(self, x, acc_reward, pref=None):
        """Vector value [B, d]."""
        return self.critic(self._build_aug_obs(x, acc_reward, pref))

    def get_action_and_value(self, x, acc_reward, action=None, pref=None):
        """(action, log-probability, entropy, vector value); samples when ``action`` is None."""
        aug = self._build_aug_obs(x, acc_reward, pref)
        probs = Categorical(logits=self.actor(aug))
        if action is None:
            action = probs.sample()
        return action, probs.log_prob(action), probs.entropy(), self.critic(aug)

    def get_greedy_action(self, x, acc_reward, pref=None):
        """Argmax of the logits."""
        return torch.argmax(self.actor(self._build_aug_obs(x, acc_reward, pref)), dim=-1)


def agent_tensors(agent: Agent):
    """The 12 parameters in the kernels' order (the Agent's parameter order)."""
    return list(agent.parameters())


class NLMOPPO(MOPolicy):
    """Non-linear multi-objective PPO (reference nl_mo_ppo.py:111-490)."""

    def __init__(
        self,
        id: int,
        envs,
        log: bool = False,
        experiment_name: Optional[str] = "NLMOPPO",
        wandb_project_name: str = "MORL-Baselines",
        wandb_entity: str = None,
        wandb_mode: Literal["online", "offline", "disabled"] = "online",
        total_timesteps: int = 500000,
        learning_rate: float = 2.5e-4,
        num_steps: int = 128,
        anneal_lr: bool = True,
        gamma: float = 0.99,
        gae_lambda: float = 0.95,
        num_minibatches: int = 4,
        update_epochs: int = 4,
        norm_adv: bool = True,
        clip_coef: float = 0.2,
        clip_vloss: bool = True,
        ent_coef: float = 0.01,
        vf_coef: float = 0.5,
        max_grad_norm: float = 0.5,
        target_kl: float = None,
        mc_k: int = 32,
        device: Union[torch.device, str] = "auto",
        seed: int = 1,
        rng: Union[np.random.Generator, None] = None,
        use_cuda_graph: bool = True,
    ):
        super().__init__(id, device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.NLMOPPO needs a CUDA device: the update path is CUDA-only (no CPU fallback)")
        ops._lib.load()
        self.envs = envs
        self.seed = seed
        self.rng = rng or np.random.default_rng(seed)
        self.log = log
        self.experiment_name = experiment_name
        self.wandb_project_name = wandb_project_name
        self.wandb_entity = wandb_entity
        self.wandb_mode = wandb_mode
        self.total_timesteps = total_timesteps
        self.learning_rate = learning_rate
        self.num_envs = self.envs.num_envs
        self.num_steps = num_steps
        self.anneal_lr = anneal_lr
        self.gamma = gamma
        self.gae_lambda = gae_lambda
        self.num_minibatches = num_minibatches
        self.update_epochs = update_epochs
        self.norm_adv = norm_adv
        self.clip_coef = clip_coef
        self.clip_vloss = clip_vloss
        self.ent_coef = ent_coef
        self.vf_coef = vf_coef
        self.max_grad_norm = max_grad_norm
        self.target_kl = target_kl
        self.use_cuda_graph = use_cuda_graph

        self.num_objectives = self.envs.reward_space.shape[0]
        self.batch_size = int(self.num_envs * self.num_steps)
        self.minibatch_size = int(self.batch_size // self.num_minibatches)
        self.num_iterations = self.total_timesteps // self.batch_size
        self.obs_dim = int(np.array(envs.single_observation_space.shape).prod())
        self.n_actions = int(envs.single_action_space.n)

        # initial observations of the utility-gradient evaluation: ceil(mc_k / num_envs) seeded resets, as the reference draws them
        self.init_obs = torch.as_tensor(
            np.concatenate([envs.reset(seed=self.seed + i)[0] for i in range(ceil(mc_k / self.num_envs))])[:mc_k],
            device=self.device, dtype=torch.float32,
        )
        self.pref: Union[torch.Tensor, None] = None
        self._graphs = GraphCache()
        self.agent = None
        self.reset_agent(pref_dim=self.num_objectives)
        self._setup_storage()

    # ---- networks and kernel state ---------------------------------------------------------------------------------------------------
    def reset_agent(self, pref_dim: int):
        """A fresh Agent and Adam, built as the reference builds them; the utility and the preference are forgotten.  With an unchanged
        ``pref_dim`` the fresh parameters are copied into the existing storages and the Adam state is zeroed in place, so captured graphs
        stay valid."""
        fresh = Agent(self.envs, self.num_objectives, pref_dim=pref_dim).to(self.device)
        if self.agent is not None and self.agent.pref_dim == pref_dim:
            with torch.no_grad():
                for p, q in zip(self.agent.parameters(), fresh.parameters()):
                    p.copy_(q)
                self.optimizer._ensure_state()
                for st in self.optimizer.state.values():
                    for k in ("step", "exp_avg", "exp_avg_sq"):
                        st[k].zero_()
            self.set_learning_rate(self.learning_rate)
        else:
            self.agent = fresh
            self.optimizer = FusedClipAdam(self.agent.parameters(), lr=self.learning_rate, eps=ADAM_EPS)
            self._lr = torch.full((1,), float(self.learning_rate), dtype=torch.float64, device=self.device)
            self.optimizer.lr_device = self._lr
            self._bind_kernels()
        self.u_func = None
        self.pref = None
        if self._pref is not None:
            self._pref.zero_()

    def _bind_kernels(self):
        """Persistent ``.grad`` storages, the device preference and loss-weight vectors, and the kernels' tables and workspace."""
        S, d, A, Dp = self.obs_dim, self.num_objectives, self.n_actions, self.agent.pref_dim
        self._graphs.clear()
        self._params = agent_tensors(self.agent)
        self._grads = [torch.zeros_like(p) for p in self._params]
        for p, g in zip(self._params, self._grads):
            p.grad = g
        self._pref = torch.zeros(Dp, device=self.device) if Dp else None
        self._w = torch.zeros(d, device=self.device)
        self._stats = torch.zeros(nl_ppo_ops.N_STATS, device=self.device)
        mb_sizes = {min(self.minibatch_size, self.batch_size - s) for s in range(0, self.batch_size, max(1, self.minibatch_size))}
        self.fused = all(nl_ppo_ops.nl_ppo_supported(S, d, Dp, A, m) and (m >= 2 or not self.norm_adv) for m in mb_sizes) and self.minibatch_size > 0
        if self.fused:
            self._net = nl_ppo_ops.NlPpoNet(S, d, Dp, A, self._params, self._grads, self._pref)
            self._ws = self._net.workspace(self.device)
            self._row_obs = torch.zeros((1, S)).pin_memory()
            self._row_acc = torch.zeros((1, d)).pin_memory()
            self._row_arg = torch.zeros(1, dtype=torch.int32).pin_memory()
            self._row_logits = torch.zeros((1, A), device=self.device)

    def _setup_storage(self):
        T, E, S, d, A = self.num_steps, self.num_envs, self.obs_dim, self.num_objectives, self.n_actions
        dev = self.device
        self.obs = torch.zeros((T, E) + self.envs.single_observation_space.shape, device=dev, dtype=torch.float32)
        self.acc_rewards = torch.zeros((T, E, d), device=dev, dtype=torch.float32)
        self.actions = torch.zeros((T, E) + self.envs.single_action_space.shape, device=dev, dtype=torch.long)
        self.logprobs = torch.zeros((T, E), device=dev, dtype=torch.float32)
        self.rewards = torch.zeros((T, E, d), device=dev, dtype=torch.float32)
        self.dones = torch.zeros((T, E), device=dev, dtype=torch.float32)
        self.values = torch.zeros((T, E, d), device=dev, dtype=torch.float32)
        # GAE outputs, written in place so captured graphs keep reading the same storage
        self.returns = torch.zeros((T, E, d), device=dev)
        self.advantages = torch.zeros((T, E, d), device=dev)
        # the state carried from one step to the next, and the step's staging
        self._next_obs = torch.zeros((E, S), device=dev)
        self._next_acc = torch.zeros((E, d), device=dev)
        self._next_done = torch.zeros(E, device=dev)
        self._timestep = torch.zeros(E, dtype=torch.int32, device=dev)
        self._next_value = torch.zeros((E, d), device=dev)
        self._logits = torch.zeros((E, A), device=dev)
        self._env_out = Staging((E, S + d + 2), torch.float32, dev)
        self._act_host = torch.zeros(E, dtype=torch.long).pin_memory()
        self._perm = Staging((self.update_epochs, self.batch_size), torch.int64, dev)
        self._zero_acc = torch.zeros((self.init_obs.shape[0], d), device=dev)
        self._v0 = torch.zeros((self.init_obs.shape[0], d), device=dev)

    def set_learning_rate(self, lr: float):
        """Learning rate of the next updates (a device write: captured graphs read it at replay)."""
        self.optimizer.param_groups[0]["lr"] = lr
        self._lr.fill_(float(lr))

    def _set_pref(self, pref):
        self.pref = None if pref is None else torch.as_tensor(pref, device=self.device, dtype=torch.float32)
        if self._pref is not None:
            if self.pref is None:
                self._pref.zero_()
            else:
                self._pref.copy_(self.pref.reshape(-1))

    # ---- rollout -----------------------------------------------------------------------------------------------------------------------
    def _collect_rollouts(self, global_step: int) -> int:
        """``num_steps`` vector-env steps from the carried state (reference nl_mo_ppo.py:248-288)."""
        E, S, d = self.num_envs, self.obs_dim, self.num_objectives
        for step in range(self.num_steps):
            global_step += E
            if self.fused:
                nl_ppo_ops.nl_ppo_forward(self._net, self._next_obs, self._next_acc, logits_out=self._logits, values_out=self.values[step])
            else:
                with torch.no_grad():
                    aug = self.agent._build_aug_obs(self._next_obs, self._next_acc, self.pref)
                    self._logits.copy_(self.agent.actor(aug))
                    self.values[step] = self.agent.critic(aug)
            action = Categorical(logits=self._logits).sample()
            self._act_host.copy_(action, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            next_obs_np, reward_np, term_np, trunc_np, infos = self.envs.step(self._act_host.numpy().copy())
            host = self._env_out.host()
            host[:, :S] = np.asarray(next_obs_np).reshape(E, S)
            host[:, S:S + d] = reward_np
            host[:, S + d] = term_np
            host[:, S + d + 1] = trunc_np
            self._env_out.upload()
            nl_ppo_ops.nl_ppo_commit(self._env_out.dev, self._logits, action, step, self.gamma, self.obs.view(-1, E, S), self.acc_rewards,
                                     self.dones, self.rewards, self.actions.view(-1, E), self.logprobs, self._next_obs, self._next_acc,
                                     self._next_done, self._timestep)
            if self.log and "final_info" in infos:
                import wandb

                for info in infos["final_info"]:
                    if info and "episode" in info:
                        wandb.log({"charts/episodic_return": info["episode"]["r"], "charts/episodic_length": info["episode"]["l"]}, step=global_step)
        return global_step

    def _compute_advantages_and_returns(self):
        """Per-objective GAE of the rollout (reference nl_mo_ppo.py:290-308), into ``self.advantages`` / ``self.returns``."""
        if self.fused:
            nl_ppo_ops.nl_ppo_forward(self._net, self._next_obs, self._next_acc, values_out=self._next_value)
            nl_ppo_ops.vector_gae_objectives(self.rewards, self.values, self.dones, self._next_value, self._next_done, self.gamma, self.gae_lambda,
                                             returns_out=self.returns, adv_out=self.advantages)
            return self.advantages, self.returns
        with torch.no_grad():
            next_value = self.agent.get_value(self._next_obs, self._next_acc, self.pref)
            lastgaelam = torch.zeros((self.num_envs, self.num_objectives), device=self.device)
            for t in reversed(range(self.num_steps)):
                if t == self.num_steps - 1:
                    nextnonterminal, nextvalues = (1.0 - self._next_done).unsqueeze(-1), next_value
                else:
                    nextnonterminal, nextvalues = (1.0 - self.dones[t + 1]).unsqueeze(-1), self.values[t + 1]
                delta = self.rewards[t] + self.gamma * nextvalues * nextnonterminal - self.values[t]
                lastgaelam = delta + self.gamma * self.gae_lambda * nextnonterminal * lastgaelam
                self.advantages[t] = lastgaelam
            self.returns.copy_(self.advantages + self.values)
        return self.advantages, self.returns

    # ---- update ------------------------------------------------------------------------------------------------------------------------
    def _compute_loss_weights(self) -> torch.Tensor:
        """w = du/dv at the mean value of ``init_obs`` with zero accrued reward (reference nl_mo_ppo.py:310-323), written into the
        device vector the update reads."""
        if self.fused:
            nl_ppo_ops.nl_ppo_forward(self._net, self.init_obs, self._zero_acc, values_out=self._v0)
            v = self._v0
        else:
            with torch.no_grad():
                v = self.agent.get_value(self.init_obs, acc_reward=self._zero_acc, pref=self.pref)
        v0 = v.mean(0).detach().requires_grad_(True)
        (w,) = torch.autograd.grad(self.u_func(v0), v0, retain_graph=False, create_graph=False)
        self._w.copy_(w.detach())
        return w.detach()

    def _batch(self):
        d = self.num_objectives
        return (self.obs.reshape(self.batch_size, self.obs_dim), self.acc_rewards.reshape(-1, d), self.actions.reshape(-1), self.logprobs.reshape(-1),
                self.advantages.reshape(-1, d), self.returns.reshape(-1, d), self.values.reshape(-1, d))

    def _epochs(self, epochs):
        """Device half of the given epochs: every minibatch's fused update and clip + Adam step.  Row ``e`` of the uploaded
        permutations orders epoch ``e``."""
        b = self._batch()
        for e in epochs:
            for start in range(0, self.batch_size, self.minibatch_size):
                nl_ppo_ops.nl_ppo_update(self._net, *b, self._perm.dev[e, start:start + self.minibatch_size], self._w, self.clip_coef, self.ent_coef,
                                         self.vf_coef, self.norm_adv, self.clip_vloss, self._stats, self._ws)
                self.optimizer.step_fused(self.max_grad_norm)

    def _variant(self, key):
        """"all" runs every epoch (zeroing the clip-fraction sum first), "epoch" runs one epoch from row 0."""
        def build():
            if key == "all":
                def step():
                    self._stats[5].zero_()
                    self._epochs(range(self.update_epochs))
            else:
                def step():
                    self._epochs([0])
            return Variant(key, step, lambda: self._params + optimizer_tensors(self.optimizer) + [self._stats])

        return self._graphs.get_or_build(key, build)

    def _run(self, st):
        if self.use_cuda_graph:
            st.graph()
        else:
            st.step()

    def _upload_permutations(self, b_inds: np.ndarray, n_epochs: int):
        """Draw ``n_epochs`` shuffles of the running index order (in place, as the reference does) and copy them to the device."""
        rows = self._perm.host()
        for e in range(n_epochs):
            self.rng.shuffle(b_inds)
            rows[e] = b_inds
        self._perm.upload(n_epochs)

    def update(self):
        """One PPO update (reference nl_mo_ppo.py:325-398).  Returns (v_loss, pg_loss, entropy_loss, old_approx_kl, approx_kl, clipfrac)."""
        self._compute_loss_weights()
        if not self.fused:
            return self._update_eager()
        b_inds = np.arange(self.batch_size)
        n_minibatches = len(range(0, self.batch_size, self.minibatch_size))
        epochs = self.update_epochs
        if self.target_kl is None:
            self._upload_permutations(b_inds, self.update_epochs)
            self._run(self._variant("all"))
        else:
            self._stats.zero_()
            st = self._variant("epoch")
            for epoch in range(self.update_epochs):
                self._upload_permutations(b_inds, 1)
                self._run(st)
                if np.float32(self._stats[4].item()) > np.float32(self.target_kl):
                    epochs = epoch + 1
                    break
        s = self._stats.cpu().numpy()
        pg, v, ent, okl, kl = (torch.tensor(x) for x in s[:5])
        return v, pg, ent, okl, kl, float(s[5]) / (n_minibatches * epochs)

    def _update_eager(self):
        """The reference's update loop through torch autograd (shapes the kernels do not cover); gradients go through the persistent
        ``.grad`` storages into the same fused clip + Adam step."""
        b_obs, b_acc, b_actions, b_logprobs, b_adv, b_ret, b_values = self._batch()
        b_inds = np.arange(self.batch_size)
        clipfracs = []
        for epoch in range(self.update_epochs):
            self.rng.shuffle(b_inds)
            for start in range(0, self.batch_size, self.minibatch_size):
                mb = torch.as_tensor(b_inds[start:start + self.minibatch_size], device=self.device)
                _, newlogprob, entropy, newvalue = self.agent.get_action_and_value(b_obs[mb], acc_reward=b_acc[mb], action=b_actions[mb], pref=self.pref)
                logratio = newlogprob - b_logprobs[mb]
                ratio = logratio.exp()
                with torch.no_grad():
                    old_approx_kl = (-logratio).mean()
                    approx_kl = ((ratio - 1) - logratio).mean()
                    clipfracs.append(((ratio - 1.0).abs() > self.clip_coef).float().mean().item())
                adv = b_adv[mb]
                if self.norm_adv:
                    adv = (adv - adv.mean(dim=0, keepdim=True)) / (adv.std(dim=0, keepdim=True) + 1e-8)
                pg1 = -adv * ratio.unsqueeze(-1)
                pg2 = -adv * torch.clamp(ratio, 1 - self.clip_coef, 1 + self.clip_coef).unsqueeze(-1)
                pg_loss = (torch.max(pg1, pg2).mean(dim=0) * self._w).sum()
                if self.clip_vloss:
                    v_unclipped = (newvalue - b_ret[mb]) ** 2
                    v_clipped = b_values[mb] + torch.clamp(newvalue - b_values[mb], -self.clip_coef, self.clip_coef)
                    v_loss = 0.5 * torch.max(v_unclipped, (v_clipped - b_ret[mb]) ** 2).mean()
                else:
                    v_loss = 0.5 * ((newvalue - b_ret[mb]) ** 2).mean()
                entropy_loss = entropy.mean()
                loss = pg_loss - self.ent_coef * entropy_loss + self.vf_coef * v_loss
                for g, new in zip(self._grads, torch.autograd.grad(loss, self._params)):
                    g.copy_(new)
                self.optimizer.step_fused(self.max_grad_norm)
            if self.target_kl is not None and approx_kl > self.target_kl:
                break
        return (v_loss.detach(), pg_loss.detach(), entropy_loss.detach(), old_approx_kl, approx_kl, float(np.mean(clipfracs) if clipfracs else 0.0))

    # ---- evaluation --------------------------------------------------------------------------------------------------------------------
    def eval(self, obs, disc_vec_return, pref=None):
        """An action sampled for one observation, accrued reward and preference (reference nl_mo_ppo.py:400-405)."""
        obs = torch.as_tensor(obs, device=self.device, dtype=torch.float32)
        disc_vec_return = torch.as_tensor(disc_vec_return, device=self.device, dtype=torch.float32)
        pref = None if pref is None else torch.as_tensor(pref, device=self.device, dtype=torch.float32)
        with torch.no_grad():
            return self.agent.get_action_and_value(obs, acc_reward=disc_vec_return, pref=pref)[0]

    def _act(self, obs, accrued_reward, deterministic: bool) -> int:
        if not self.fused:
            o = torch.as_tensor(obs, device=self.device, dtype=torch.float32)
            a = torch.as_tensor(accrued_reward, device=self.device, dtype=torch.float32)
            with torch.no_grad():
                if deterministic:
                    return self.agent.get_greedy_action(o, acc_reward=a, pref=self.pref).item()
                return self.agent.get_action_and_value(o, acc_reward=a, pref=self.pref)[0].item()
        self._row_obs.numpy()[0] = np.asarray(obs, dtype=np.float32).reshape(-1)
        self._row_acc.numpy()[0] = accrued_reward
        if deterministic:
            nl_ppo_ops.nl_ppo_forward(self._net, self._row_obs, self._row_acc, argmax_out=self._row_arg)
            torch.cuda.current_stream().synchronize()
            return int(self._row_arg[0])
        nl_ppo_ops.nl_ppo_forward(self._net, self._row_obs, self._row_acc, logits_out=self._row_logits)
        return Categorical(logits=self._row_logits[0]).sample().item()

    def policy_evaluate(self, eval_env, eval_episodes=100, deterministic=False):
        """Mean discounted vector return over ``eval_episodes`` episodes, each reset with ``seed=self.seed`` (reference
        nl_mo_ppo.py:407-442)."""
        pareto_point = np.zeros(self.num_objectives)
        for _ in range(eval_episodes):
            obs, _ = eval_env.reset(seed=self.seed)
            terminated = truncated = False
            accrued_reward = np.zeros(self.num_objectives, dtype=np.float32)
            timestep = 0
            while not (terminated or truncated):
                action = self._act(obs, accrued_reward, deterministic)
                obs, reward, terminated, truncated, _ = eval_env.step(action)
                accrued_reward += (self.gamma**timestep) * reward
                timestep += 1
            pareto_point += accrued_reward
        return pareto_point / eval_episodes

    # ---- training ----------------------------------------------------------------------------------------------------------------------
    def train(self, eval_env, u_func: Callable[[torch.Tensor], torch.Tensor], pref: torch.Tensor = None, deterministic: bool = False) -> np.ndarray:
        """Train on the utility ``u_func`` (and preference ``pref``), then evaluate (reference nl_mo_ppo.py:444-490)."""
        self.u_func = u_func
        self._set_pref(pref)
        global_step = 0
        start_time = time.time()
        next_obs, _ = self.envs.reset(seed=self.seed)
        self._next_obs.copy_(torch.as_tensor(np.asarray(next_obs, dtype=np.float32).reshape(self.num_envs, self.obs_dim)))
        self._next_acc.zero_()
        self._next_done.zero_()
        self._timestep.zero_()
        for iteration in range(1, self.num_iterations + 1):
            if self.anneal_lr:
                self.set_learning_rate((1.0 - (iteration - 1.0) / self.num_iterations) * self.learning_rate)
            global_step = self._collect_rollouts(global_step)
            self._compute_advantages_and_returns()
            v_loss, pg_loss, entropy_loss, old_approx_kl, approx_kl, clipfrac = self.update()
            if self.log:
                import wandb

                wandb.log({"charts/learning_rate": self.optimizer.param_groups[0]["lr"], "losses/value_loss": float(v_loss.item()),
                           "losses/policy_loss": float(pg_loss.item()), "losses/entropy": float(entropy_loss.item()),
                           "losses/old_approx_kl": float(old_approx_kl.item()), "losses/approx_kl": float(approx_kl.item()),
                           "losses/clipfrac": clipfrac, "charts/SPS": int(global_step / (time.time() - start_time))}, step=global_step)
        return self.policy_evaluate(eval_env, deterministic=deterministic)
