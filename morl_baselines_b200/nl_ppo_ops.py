"""Bindings of non-linear MO-PPO's kernels (csrc/nl_ppo.cu and the objective GAE of csrc/ppo.cu).

They follow the argument contract of :mod:`ops` (``ops._Args``) and launch through ``ops._launch``, so ``ops.launch_count`` counts them.
The 12 parameter tensors are those of the reference ``Agent`` in its parameter order: critic.0, critic.2, critic.4, actor.0, actor.2,
actor.4, weight then bias each.
"""

from __future__ import annotations

from typing import Optional

import torch as th

from . import _lib
from .ops import _Args, _launch, _param_table, _workspace

N_TENSORS = 12
N_STATS = 6  # pg_loss, v_loss, entropy, old_approx_kl, approx_kl, clip-fraction sum


def nl_ppo_supported(obs_dim: int, d: int, pref_dim: int, n_actions: int, batch: int) -> bool:
    """Whether the kernels cover this Agent and minibatch: 1 <= obs_dim, 1 <= d <= 8, pref_dim in {0, d}, obs_dim + d + pref_dim <= 256,
    1 <= n_actions <= 32, 1 <= batch <= 4096 (include/morl_b200.h).  Needs no device."""
    return bool(_lib.load().morl_nl_ppo_supported(int(obs_dim), int(d), int(pref_dim), int(n_actions), int(batch)))


class NlPpoNet:
    """What the kernels need about one Agent: its shape, the pointer tables of its parameters and gradients, and the device ``pref``
    vector [pref_dim] (read in place at run time).  Build it once per set of storages (the tables hold raw device pointers)."""

    def __init__(self, obs_dim: int, d: int, pref_dim: int, n_actions: int, params, grads=None, pref: Optional[th.Tensor] = None):
        self.obs_dim, self.d, self.pref_dim, self.n_actions = int(obs_dim), int(d), int(pref_dim), int(n_actions)
        a = _Args("NlPpoNet")
        if not nl_ppo_supported(self.obs_dim, self.d, self.pref_dim, self.n_actions, 1):
            a.fail("shape", f"is unsupported: obs_dim={obs_dim} d={d} pref_dim={pref_dim} n_actions={n_actions}")
        K, H = self.obs_dim + self.d + self.pref_dim, 64
        self.shapes = [(H, K), (H,), (H, H), (H,), (self.d, H), (self.d,), (H, K), (H,), (H, H), (H,), (self.n_actions, H), (self.n_actions,)]
        self.params = _param_table(a, params, "params", N_TENSORS, "tensors of the Agent", self.shapes)
        self.grads = None if grads is None else _param_table(a, grads, "grads", N_TENSORS, "tensors of the Agent", self.shapes)
        self.pref = a.inp(pref, "pref", (self.pref_dim,), inplace=True) if self.pref_dim else None

    @property
    def workspace_bytes(self) -> int:
        return int(_lib.load().morl_nl_ppo_workspace_bytes(self.obs_dim, self.d, self.pref_dim, self.n_actions))

    def workspace(self, device) -> th.Tensor:
        return _workspace(self.workspace_bytes, device)


def vector_gae_objectives(rewards, values, dones, next_value, next_done, gamma: float, gae_lambda: float,
                          returns_out: Optional[th.Tensor] = None, adv_out: Optional[th.Tensor] = None):
    """Per-objective GAE (reference nl_mo_ppo.py:290-308) in one launch: rewards / values [T, E, D], dones [T, E], next_value [E, D],
    next_done [E].  Returns (returns [T, E, D], advantages [T, E, D]), written into ``returns_out`` / ``adv_out`` when given."""
    a = _Args("vector_gae_objectives")
    rewards = a.inp(rewards, "rewards", (None,) * 3)
    T, E, D = rewards.shape
    values, dones = a.inp(values, "values", (T, E, D)), a.inp(dones, "dones", (T, E))
    next_value, next_done = a.inp(next_value, "next_value", reshape=(E * D,)), a.inp(next_done, "next_done", reshape=(E,))
    ret, adv = a.out(returns_out, "returns_out", (T, E, D)), a.out(adv_out, "adv_out", (T, E, D))
    _launch("morl_vector_gae_objectives_f32", rewards, values, dones, next_value, next_done, T, E, D, float(gamma), float(gae_lambda), ret, adv)
    return ret, adv


def nl_ppo_update(net: NlPpoNet, obs, acc, actions, old_logprob, advantages, returns, old_values, perm, loss_weights, clip_coef: float,
                  ent_coef: float, vf_coef: float, norm_adv: bool, clip_vloss: bool, stats: th.Tensor, workspace: th.Tensor,
                  loss_out: Optional[th.Tensor] = None):
    """One minibatch (reference nl_mo_ppo.py:349-391) in two launches: rows ``perm`` int64 [M] of the batch obs [B, S], acc [B, d], actions
    int64 [B], old_logprob [B], advantages / returns / old_values [B, d]; ``loss_weights`` [d].  Overwrites ``net.grads``, writes stats
    [6] (clip fraction added to stats[5]) and, when given, ``loss_out`` [1].  Every input is read in place."""
    a = _Args("nl_ppo_update")
    if net.grads is None:
        a.fail("net", "was built without gradient tensors")
    S, d = net.obs_dim, net.d
    obs = a.inp(obs, "obs", (None, S), inplace=True)
    B = obs.shape[0]
    acc = a.inp(acc, "acc", (B, d), inplace=True)
    actions = a.inp(actions, "actions", (B,), th.int64, inplace=True)
    old_logprob = a.inp(old_logprob, "old_logprob", (B,), inplace=True)
    advantages, returns = a.inp(advantages, "advantages", (B, d), inplace=True), a.inp(returns, "returns", (B, d), inplace=True)
    old_values = a.inp(old_values, "old_values", (B, d), inplace=True, opt=not clip_vloss)
    perm = a.inp(perm, "perm", (None,), th.int64, inplace=True)
    M = perm.shape[0]
    if not nl_ppo_supported(S, d, net.pref_dim, net.n_actions, M):
        a.fail("perm", f"has {M} rows: a minibatch must hold 1 to 4096")
    loss_weights = a.inp(loss_weights, "loss_weights", (d,), inplace=True)
    stats = a.out(stats, "stats", (N_STATS,))
    loss_out = a.out(loss_out, "loss_out", (1,), alloc=False)
    workspace = a.ws(workspace, "workspace", net.workspace_bytes)
    if net.pref is not None:
        a.inp(net.pref, "pref", (net.pref_dim,), inplace=True)
    _launch("morl_nl_ppo_update_f32", net.params, net.grads, obs, acc, actions, old_logprob, advantages, returns, old_values, perm, int(M), S, d,
            net.pref_dim, net.n_actions, net.pref, loss_weights, float(clip_coef), float(ent_coef), float(vf_coef), int(bool(norm_adv)),
            int(bool(clip_vloss)), loss_out, stats, workspace, launches=2)


def nl_ppo_forward(net: NlPpoNet, obs, acc, logits_out: Optional[th.Tensor] = None, values_out: Optional[th.Tensor] = None,
                   argmax_out: Optional[th.Tensor] = None):
    """Both networks (or the one asked for) on N rows obs [N, S], acc [N, d] with the net's pref (reference nl_mo_ppo.py:90-108): logits
    [N, A], values [N, d], first-occurrence argmax int32 [N], each written when given.  Rows and outputs may be CUDA tensors or pinned host
    tensors; with pinned outputs the caller synchronises the stream before reading them."""
    a = _Args("nl_ppo_forward")
    obs = a.inp(obs, "obs", (None, net.obs_dim), inplace=True, pinned=True)
    N = obs.shape[0]
    if N < 1:
        a.fail("obs", "must have at least one row")
    acc = a.inp(acc, "acc", (N, net.d), inplace=True, pinned=True)
    logits_out = a.out(logits_out, "logits_out", (N, net.n_actions), alloc=False, pinned=True)
    values_out = a.out(values_out, "values_out", (N, net.d), alloc=False, pinned=True)
    argmax_out = a.out(argmax_out, "argmax_out", (N,), th.int32, alloc=False, pinned=True)
    if logits_out is None and values_out is None and argmax_out is None:
        a.fail("logits_out", "or values_out or argmax_out must be given")
    if net.pref is not None:
        a.inp(net.pref, "pref", (net.pref_dim,), inplace=True)
    _launch("morl_nl_ppo_forward_f32", net.params, obs, acc, int(N), net.obs_dim, net.d, net.pref_dim, net.n_actions, net.pref, logits_out, values_out,
            argmax_out)


def nl_ppo_commit(staged, logits, action, step: int, gamma: float, obs_store, acc_store, done_store, rew_store, act_store, logp_store, next_obs,
                  next_acc, next_done, timestep):
    """One rollout step's bookkeeping (reference nl_mo_ppo.py:251-275) in one launch: ``staged`` [E, S + d + 2] (obs | reward | terminated
    | truncated of the environment step), the step's ``logits`` [E, A] and sampled ``action`` int64 [E]; the stores [T, E, ...] get row
    ``step``; the carried next_obs [E, S], next_acc [E, d], next_done [E] and int32 ``timestep`` [E] are advanced in place."""
    a = _Args("nl_ppo_commit")
    obs_store = a.out(obs_store, "obs_store", (None, None, None))
    T, E, S = obs_store.shape
    rew_store = a.out(rew_store, "rew_store", (T, E, None))
    d = rew_store.shape[2]
    logits = a.inp(logits, "logits", (E, None), inplace=True)
    A = logits.shape[1]
    staged = a.inp(staged, "staged", (E, S + d + 2), inplace=True)
    action = a.inp(action, "action", (E,), th.int64, inplace=True)
    if not 0 <= step < T:
        a.fail("step", f"must be in [0, {T}), got {step}")
    acc_store, done_store = a.out(acc_store, "acc_store", (T, E, d)), a.out(done_store, "done_store", (T, E))
    act_store, logp_store = a.out(act_store, "act_store", (T, E), th.int64), a.out(logp_store, "logp_store", (T, E))
    next_obs, next_acc = a.out(next_obs, "next_obs", (E, S)), a.out(next_acc, "next_acc", (E, d))
    next_done, timestep = a.out(next_done, "next_done", (E,)), a.out(timestep, "timestep", (E,), th.int32)
    _launch("morl_nl_ppo_commit_f32", staged, logits, action, int(step), int(E), int(S), int(d), int(A), float(gamma), obs_store, acc_store, done_store,
            rew_store, act_store, logp_store, next_obs, next_acc, next_done, timestep)
