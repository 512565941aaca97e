"""Expected Utility Policy Gradient on the CUDA update engine -- drop-in for reference morl_baselines/single_policy/esr/eupg.py
(``PolicyNet`` and ``EUPG`` with the same constructor arguments, public methods, state-dict, checkpoint and wandb keys).

EUPG is an ESR learner: the policy is conditioned on the reward accrued so far and maximises the expected utility of each episode's
return.  What runs where:
  * Acting: the forward kernel (``morl_eupg_probs_f32``) runs on one row through pinned host memory, and the action is drawn on the host
    by ``Categorical(probs).sample()`` from a CPU tensor holding the kernel's probabilities.
  * The accrued reward stays on the host as a float32 tensor, accumulated with torch's in-place promotion rule (float64 rewards are
    added in float64 and rounded to float32), as the reference does on its device.
  * At the end of an episode, the buffer's rows ``[0, size)`` (int32 observations, accrued rewards, int32 actions, rewards) are packed
    into one pinned staging block and copied to the device at once.  The update is then one launch for the discounted forward returns
    (``morl_eupg_returns_f32``, bit-identical to the reference's loop), the user's scalarisation, one fused forward + loss + backward
    (``morl_eupg_update_f32``, two launches, gradients written into the ``.grad`` storages) and one fused Adam step.  No host sync: the
    loss is read back only when logging.  There is no CUDA graph: T changes every episode and the user's callable runs between kernels.

The kernels cover the networks of ``ops.eupg_supported``.  A network outside that range, or a scalarisation whose output the kernel does
not take (anything but a float32 device tensor of T elements or of zero dimensions), runs the reference's update expression through torch autograd
on the same staged device rows.

Differences from the reference, each deliberate:
  * On CUDA the reference samples actions from the CUDA generator; this port samples from torch's CPU generator, so a seeded run draws
    the actions of the reference run with ``device="cpu"``.
  * The reference's ``__deepcopy__`` deep-copies ``self.net``, builds the copy (a fresh network) and then builds the copy's optimiser on
    the deep-copied network, which the copy never uses: the copy's ``net`` keeps its fresh initialisation and is never stepped.  Here the
    copy is constructed the same way (so the torch RNG is consumed identically), then the source's parameters are loaded into
    ``copied.net`` and the optimiser is built on that net.
"""

from __future__ import annotations

import time
from copy import deepcopy
from typing import Callable, List, Optional, Union

import numpy as np
import torch as th
import torch.nn as nn
from torch.distributions import Categorical

from ... import ops
from ...common.accrued_reward_buffer import AccruedRewardReplayBuffer
from ...common.evaluation import log_episode_info
from ...common.fused_adam import FusedClipAdam
from ...common.graphed import Staging
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.networks import layer_init, mlp


class PolicyNet(nn.Module):
    """Policy network (reference eupg.py:22-75): [obs || accrued reward] -> Linear/Tanh stack -> normalised sigmoid over the actions."""

    def __init__(self, obs_shape, action_dim, rew_dim, net_arch):
        super().__init__()
        self.obs_shape = obs_shape
        self.action_dim = action_dim
        self.rew_dim = rew_dim
        input_dim = obs_shape[0] + rew_dim
        self.net = mlp(input_dim, action_dim, net_arch, activation_fn=nn.Tanh)
        self.apply(layer_init)

    def forward(self, obs: th.Tensor, acc_reward: th.Tensor):
        """Probability of each action, [batch, |A|]."""
        x = th.cat((obs, acc_reward), dim=acc_reward.dim() - 1)  # an int observation is promoted to float32 here
        gates = th.sigmoid(self.net(x))
        # the division by the sum over the whole batch is the reference's; Categorical renormalises every row afterwards
        return (gates / th.sum(gates)).view(-1, self.action_dim)

    def distribution(self, obs: th.Tensor, acc_reward: th.Tensor):
        """``Categorical`` over the actions, built from ``forward``."""
        return Categorical(self.forward(obs, acc_reward))


def policy_tensors(net: PolicyNet) -> List[th.Tensor]:
    """The Linear layers' weights and biases in state-dict order (the kernels' order)."""
    out = []
    for m in net.net:
        if isinstance(m, nn.Linear):
            out += [m.weight, m.bias]
    return out


def accrue(accrued_reward: th.Tensor, vec_reward: np.ndarray) -> th.Tensor:
    """``accrued_reward`` (float32, host) += ``vec_reward`` in place with torch's promotion rule, as the reference accumulates on its
    device (eupg.py:350): float64 rewards are added in float64 and the sum rounded to float32."""
    accrued_reward += th.from_numpy(vec_reward)
    return accrued_reward


def kernel_takes(v, T: int, device: th.device) -> bool:
    """Whether the fused update takes this scalarisation output as it is: a float32 tensor on the device with T elements in one
    dimension, or one element in zero dimensions, that needs no gradient."""
    if not isinstance(v, th.Tensor) or v.device != device or v.dtype != th.float32 or v.requires_grad:
        return False
    return v.dim() == 0 or (v.dim() == 1 and v.shape[0] == T)


class EUPG(MOPolicy, MOAgent):
    """Expected Utility Policy Gradient (Roijers, Steckelmacher & Nowé, 2018) on the CUDA update engine (reference eupg.py:78-398)."""

    def __init__(
        self,
        env,
        scalarization: Callable[[np.ndarray, np.ndarray], float],
        weights: np.ndarray = np.ones(2),
        id: Optional[int] = None,
        buffer_size: int = int(1e5),
        net_arch: List = [50],
        gamma: float = 0.99,
        learning_rate: float = 1e-3,
        project_name: str = "MORL-Baselines",
        experiment_name: str = "EUPG",
        wandb_entity: Optional[str] = None,
        log: bool = True,
        log_every: int = 1000,
        device: Union[th.device, str] = "auto",
        seed: Optional[int] = None,
        parent_rng: Optional[np.random.Generator] = None,
    ):
        MOAgent.__init__(self, env, device, seed=seed)
        MOPolicy.__init__(self, None, device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error(f"morl_baselines_b200.{type(self).__name__} needs a CUDA device: the update path is CUDA-only")
        if self.device.index is None:  # "cuda" names the current device; the tensors the scalarisation returns carry its index
            self.device = th.device("cuda", th.cuda.current_device())
        ops._lib.load()

        self.seed = seed
        self.parent_rng = parent_rng
        if parent_rng is not None:
            self.np_random = parent_rng
        else:
            self.np_random = np.random.default_rng(self.seed)

        self.env = env
        self.id = id
        self.scalarization = scalarization
        self.weights = weights
        self.gamma = gamma

        self.buffer_size = buffer_size
        self.net_arch = net_arch
        self.learning_rate = learning_rate
        self.buffer = AccruedRewardReplayBuffer(
            obs_shape=self.observation_shape,
            action_shape=self.action_shape,
            rew_dim=self.reward_dim,
            max_size=self.buffer_size,
            obs_dtype=np.int32,
            action_dtype=np.int32,
        )
        self.net = PolicyNet(
            obs_shape=self.observation_shape,
            rew_dim=self.reward_dim,
            action_dim=self.action_dim,
            net_arch=self.net_arch,
        ).to(self.device)
        self.optimizer = FusedClipAdam(self.net.parameters(), lr=self.learning_rate)
        self._bind_kernels()

        self.project_name = project_name
        self.experiment_name = experiment_name
        self.log = log
        self.log_every = log_every
        if log and parent_rng is None:
            self.setup_wandb(self.project_name, self.experiment_name, wandb_entity)

    # ---- kernel state ----------------------------------------------------------------------------------------------------------------
    def _bind_kernels(self):
        """Persistent ``.grad`` storages (both update paths write into them), the kernels' pointer tables and workspace, and the pinned
        row of the action path."""
        S, d, A = self.observation_shape[0], self.reward_dim, self.action_dim
        self._params = policy_tensors(self.net)
        self._grads = [th.zeros_like(p) for p in self._params]
        for p, g in zip(self._params, self._grads):
            p.grad = g
        self.fused = ops.eupg_supported(S, d, self.net_arch, A)
        if self.fused:
            self._knet = ops.EupgNet(S, d, self.net_arch, A, self._params, self._grads)
            self._ws = self._knet.workspace(self.device)
            self._act_in = th.zeros((1, S + d), dtype=th.float32).pin_memory()
            self._act_out = th.zeros((1, A), dtype=th.float32).pin_memory()
        self._loss = th.zeros(1, dtype=th.float32, device=self.device)
        self._stage: Optional[Staging] = None
        self.last_update_fused = False  # which path the latest update() took

    def _restore_grads(self):
        # the kernels and the optimiser's tables hold these storages: undo a zero_grad(set_to_none=True) or a replaced .grad
        for p, g in zip(self._params, self._grads):
            if p.grad is not g:
                p.grad = g

    def _staging(self, T: int) -> Staging:
        """Pinned block [rows, S + 2d + 1]: obs (int32 bits) | accrued reward | action (int32 bits) | reward.  Grows to the longest episode."""
        if self._stage is None or self._stage.pin.shape[0] < T:
            rows = max(T, 256 if self._stage is None else min(self.buffer.max_size, 2 * self._stage.pin.shape[0]))
            self._stage = Staging((rows, self.observation_shape[0] + 2 * self.reward_dim + 1), th.float32, self.device)
        return self._stage

    def __deepcopy__(self, memo):
        """Deep copy the policy (see the module docstring for how the copy's network and optimiser differ from the reference's)."""
        copied_net = deepcopy(self.net)
        copied = type(self)(
            self.env,
            self.scalarization,
            self.weights,
            self.id,
            self.buffer_size,
            self.net_arch,
            self.gamma,
            self.learning_rate,
            self.project_name,
            self.experiment_name,
            log=self.log,
            device=self.device,
            parent_rng=self.parent_rng,
        )

        copied.global_step = self.global_step
        copied.net.load_state_dict(copied_net.state_dict())
        copied.optimizer = FusedClipAdam(copied.net.parameters(), lr=self.learning_rate)
        copied.buffer = deepcopy(self.buffer)
        return copied

    def get_policy_net(self) -> nn.Module:
        return self.net

    def get_buffer(self):
        return self.buffer

    def set_buffer(self, buffer):
        raise Exception("EUPG learns on-policy from its own episodes: its buffer cannot be replaced by a shared one.")

    def set_weights(self, weights: np.ndarray):
        self.weights = weights

    # ---- acting ----------------------------------------------------------------------------------------------------------------------
    def _probs(self, obs: np.ndarray, accrued_reward: np.ndarray) -> th.Tensor:
        """Action probabilities [1, A] of one row as a CPU tensor; obs and accrued reward as float32."""
        S = self.observation_shape[0]
        if self.fused:
            x = self._act_in.numpy()
            x[0, :S] = obs
            x[0, S:] = accrued_reward
            ops.eupg_probs(self._knet, self._act_in, self._act_out)
            th.cuda.current_stream().synchronize()
            return self._act_out
        with th.no_grad():
            return self.net(th.from_numpy(obs).to(self.device), th.from_numpy(accrued_reward).to(self.device)).cpu()

    def _choose_action(self, obs: np.ndarray, accrued_reward: np.ndarray) -> int:
        return Categorical(self._probs(obs, accrued_reward)).sample().item()

    def eval(self, obs: np.ndarray, accrued_reward: Optional[np.ndarray]) -> Union[int, np.ndarray]:
        """Action sampled by the policy for the observation and the reward accrued so far."""
        if type(obs) is int:
            obs = [obs]
        obs = np.asarray(obs, dtype=np.float32).reshape(-1)
        return self._choose_action(obs, np.asarray(accrued_reward, dtype=np.float32).reshape(-1))

    # ---- update ----------------------------------------------------------------------------------------------------------------------
    def _stage_episode(self) -> th.Tensor:
        """Packs the buffer's rows [0, size) into the pinned block and queues one copy; returns the device rows."""
        T = self.buffer.size
        S, d = self.observation_shape[0], self.reward_dim
        stage = self._staging(T)
        host = stage.host()[:T]
        bits = host.view(np.int32)
        bits[:, :S] = self.buffer.obs[:T].reshape(T, S)
        host[:, S:S + d] = self.buffer.accrued_rewards[:T]
        bits[:, S + d] = self.buffer.actions[:T].reshape(T)
        host[:, S + d + 1:] = self.buffer.rewards[:T]
        stage.upload(T)
        return stage.dev[:T]

    def update(self):
        """One policy-gradient step on the episode in the buffer (reference eupg.py:226-261)."""
        T = self.buffer.size
        S, d = self.observation_shape[0], self.reward_dim
        # the episode's total reward, summed on the host in float32 as the reference sums its CPU tensor (no device sync)
        utility = self.scalarization(th.sum(th.from_numpy(self.buffer.rewards[:T]), dim=0).numpy(), self.weights)

        rows = self._stage_episode()
        obs, accrued_rewards = rows[:, :S].view(th.int32), rows[:, S:S + d]
        actions = rows[:, S + d].view(th.int32)
        # the callable sees the [T, d] returns alone, once, after the episodic-return call
        v = self.scalarization(ops.eupg_returns(rows[:, S + d + 1:], self.gamma))

        self._restore_grads()
        self.last_update_fused = self.fused and kernel_takes(v, T, self.device)
        if self.last_update_fused:
            ops.eupg_update(self._knet, obs, accrued_rewards, actions, v, self._loss, self._ws)
        else:
            self._eager_update(obs, accrued_rewards, actions, v)
        self.optimizer.step_fused(None)

        if self.log:
            import wandb

            log_str = f"_{self.id}" if self.id is not None else ""
            wandb.log(
                {
                    f"losses{log_str}/loss": self._loss.item(),
                    f"metrics{log_str}/scalarized_episodic_return": utility,
                    "global_step": self.global_step,
                },
            )

    def _eager_update(self, obs: th.Tensor, accrued_rewards: th.Tensor, actions: th.Tensor, v):
        """The reference's update expression (eupg.py:244-251) through torch autograd on the staged rows; the gradients go into the
        persistent ``.grad`` storages."""
        # [T, 1] squeezed as the buffer's action column is: a 0-d action when T = 1, so broadcasting follows the reference's
        logp = self.net.distribution(obs, accrued_rewards).log_prob(actions.reshape(-1, 1).squeeze())
        loss = -th.mean(logp * v)
        grads = th.autograd.grad(loss, self._params)
        for g, new in zip(self._grads, grads):
            g.copy_(new)
        self._loss.copy_(loss.detach().reshape(1))

    def _forward_cumulative_rewards(self, rewards: th.Tensor) -> th.Tensor:
        """Discounted forward returns of rewards [T, d] (reference eupg.py:263-270), on the device kernel."""
        return ops.eupg_returns(rewards.to(device=self.device, dtype=th.float32).contiguous(), self.gamma)

    # ---- checkpoints -----------------------------------------------------------------------------------------------------------------
    def get_save_dict(self, save_replay_buffer=True):
        """Checkpoint contents: network and optimiser state dicts, the scalarisation weights and, optionally, the buffer."""
        save_dict = {
            "policy_net_state_dict": self.net.state_dict(),
            "optimizer_state_dict": self.optimizer.state_dict(),
            "policy_weights": self.weights,
        }
        if save_replay_buffer:
            save_dict["replay_buffer"] = self.get_buffer()
        return save_dict

    def load(self, save_dict: Optional[dict] = None, path: Optional[str] = None, load_replay_buffer: bool = True):
        """Restore a checkpoint of ``get_save_dict`` given as a dict or a path; the buffer only when it was saved and asked for."""
        if save_dict is None:
            assert path is not None, "Either save_dict or path must be provided."
            save_dict = th.load(path, weights_only=False)
        self.net.load_state_dict(save_dict["policy_net_state_dict"])
        self.optimizer.load_state_dict(save_dict["optimizer_state_dict"])
        self.weights = save_dict["policy_weights"]
        if load_replay_buffer and "replay_buffer" in save_dict:
            self.buffer = save_dict["replay_buffer"]

    # ---- training --------------------------------------------------------------------------------------------------------------------
    def train(self, total_timesteps: int, eval_env=None, eval_freq: int = 1000, start_time=None):
        """Train the agent: one update at the end of every episode (reference eupg.py:305-387)."""
        if start_time is None:
            start_time = time.time()
        obs, _ = self.env.reset()
        accrued = th.zeros(self.reward_dim, dtype=th.float32)  # reward accrued before the current step, on the host

        for _ in range(total_timesteps):
            self.global_step += 1
            obs = [obs] if type(obs) is int else obs  # a Discrete observation is one column

            action = self._choose_action(np.asarray(obs, dtype=np.float32).reshape(-1), accrued.numpy())
            next_obs, vec_reward, terminated, truncated, info = self.env.step(action)
            self.buffer.add(obs, accrued.numpy(), action, vec_reward, next_obs, terminated)  # the value from before this step
            accrue(accrued, vec_reward)

            if eval_env is not None and self.log and self.global_step % eval_freq == 0:
                self.policy_eval_esr(eval_env, scalarization=self.scalarization, weights=self.weights, log=self.log)

            if not (terminated or truncated):
                obs = next_obs
            else:  # one update per episode, then a fresh episode with nothing accrued
                self.update()
                self.buffer.cleanup()
                obs, _ = self.env.reset()
                self.num_episodes += 1
                accrued = th.zeros(self.reward_dim, dtype=th.float32)
                if self.log and self.num_episodes % self.log_every == 0 and "episode" in info.keys():
                    log_episode_info(info=info["episode"], scalarization=self.scalarization, weights=self.weights, id=self.id,
                                     global_timestep=self.global_step)

            if self.log and self.global_step % 1000 == 0:
                import wandb

                sps = int(self.global_step / (time.time() - start_time))
                print("SPS:", sps)
                wandb.log({"charts/SPS": sps, "global_step": self.global_step})

    def get_config(self) -> dict:
        return {
            "env_id": self.env.unwrapped.spec.id,
            "learning_rate": self.learning_rate,
            "buffer_size": self.buffer_size,
            "gamma": self.gamma,
            "net_arch": self.net_arch,
            "seed": self.seed,
        }
