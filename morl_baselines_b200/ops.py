"""Thin PyTorch-facing wrappers over the C-ABI (include/morl_b200.h).

PyTorch is plumbing here: it owns the device buffers and the stream; every operator below is one (or two) launches of a
hand-written sm_90a kernel from libmorl_b200.so.  All wrappers require CUDA tensors and raise otherwise -- there is
no CPU / eager fallback (the CPU restatement lives in oracle/ and is test-only).
"""

from __future__ import annotations

from typing import Optional, Tuple

import torch as th

from . import _lib
from ._lib import (  # noqa: F401  (re-exported constants)
    AC_ARGMIN_GATHER,
    AC_ELEMENTWISE_MIN,
    AC_SCALAR_MIN,
    DOT_FMA,
    DOT_PAIRFMA,
    DOT_UNFUSED,
    MAP_BLOCK,
    MAP_TILE,
    ROWS_BMAJOR,
    ROWS_REFERENCE,
)

# number of kernels launched through this module (bench.py reports it as `gpu_launches`)
launch_count = 0


def _count(n=1):
    global launch_count
    launch_count += n


def _dev(t: th.Tensor, name: str, dtype=th.float32) -> th.Tensor:
    if not isinstance(t, th.Tensor) or not t.is_cuda:
        raise _lib.MorlB200Error(f"{name} must be a CUDA tensor (morl_baselines_b200 has no CPU fallback)")
    if t.dtype != dtype:
        raise _lib.MorlB200Error(f"{name} must have dtype {dtype}, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _ptr(t: Optional[th.Tensor]):
    return None if t is None else t.data_ptr()


def _stream():
    return th.cuda.current_stream().cuda_stream


def envelope_td(q_online, q_target, wset, reward, done, gamma: float, dot_mode: int = DOT_UNFUSED, row_order: int = ROWS_REFERENCE,
                want_indices: bool = True, out: Optional[th.Tensor] = None, pref_out=None, act_out=None):
    """Fused envelope-max TD target (reference envelope.py:404-440 + :298).  q_*: [B, W, A, D]; returns
    (target [W*B, D], pref [W*B] int32, act [W*B] int32)."""
    q_online, q_target = _dev(q_online, "q_online"), _dev(q_target, "q_target")
    B, W, A, D = q_online.shape
    if q_target.shape != q_online.shape:
        raise _lib.MorlB200Error("q_online / q_target shape mismatch")
    wset, reward, done = _dev(wset, "wset"), _dev(reward, "reward"), _dev(done, "done")
    if wset.shape != (W, D) or reward.shape != (B, D) or done.numel() != B:
        raise _lib.MorlB200Error(f"bad shapes: wset {tuple(wset.shape)}, reward {tuple(reward.shape)}, done {tuple(done.shape)}")
    if out is None:
        out = th.empty((W * B, D), device=q_online.device, dtype=th.float32)
    if want_indices:
        pref_out = th.empty(W * B, device=q_online.device, dtype=th.int32) if pref_out is None else pref_out
        act_out = th.empty(W * B, device=q_online.device, dtype=th.int32) if act_out is None else act_out
    rc = _lib.load().morl_envelope_td_f32(_ptr(q_online), _ptr(q_target), _ptr(wset), _ptr(reward), _ptr(done), float(gamma), B, W, A, D,
                                          dot_mode, row_order, _ptr(out), _ptr(pref_out), _ptr(act_out), _stream())
    _lib.check(rc, "morl_envelope_td_f32")
    _count()
    return out, pref_out, act_out


def _rows(t, D, name):
    t = _dev(t, name)
    return t.reshape(-1, D)


def greedy_td(q_select, q_eval, w, reward=None, done=None, gamma: float = 0.0, dot_mode: int = DOT_UNFUSED, w_map: int = MAP_BLOCK,
              r_map: int = MAP_TILE):
    """Double-DQN target with per-row weights (reference envelope.py:442-463).  q_*: [N, A, D]."""
    q_select, q_eval = _dev(q_select, "q_select"), _dev(q_eval, "q_eval")
    N, A, D = q_select.shape
    w = _rows(w, D, "w")
    if reward is not None:
        reward, done = _rows(reward, D, "reward"), _dev(done, "done").reshape(-1)
    out = th.empty((N, D), device=q_select.device, dtype=th.float32)
    act = th.empty(N, device=q_select.device, dtype=th.int32)
    rc = _lib.load().morl_greedy_td_f32(_ptr(q_select), _ptr(q_eval), _ptr(w), w.shape[0], w_map, _ptr(reward), _ptr(done),
                                        N if reward is None else reward.shape[0], r_map, float(gamma), N, A, D, dot_mode, _ptr(out),
                                        _ptr(act), _stream())
    _lib.check(rc, "morl_greedy_td_f32")
    _count()
    return out, act


def critic_min_td(q_nets, w, reward=None, done=None, gamma: float = 0.0, dot_mode: int = DOT_UNFUSED, w_map: int = MAP_BLOCK,
                  r_map: int = MAP_TILE):
    """GPI-PD critic-min greedy target (reference gpi_pd.py:445-463).  q_nets: [n_nets, N, A, D]."""
    q_nets = _dev(q_nets, "q_nets")
    n_nets, N, A, D = q_nets.shape
    w = _rows(w, D, "w")
    if reward is not None:
        reward, done = _rows(reward, D, "reward"), _dev(done, "done").reshape(-1)
    out = th.empty((N, D), device=q_nets.device, dtype=th.float32)
    act = th.empty(N, device=q_nets.device, dtype=th.int32)
    rc = _lib.load().morl_critic_min_td_f32(_ptr(q_nets), n_nets, _ptr(w), w.shape[0], w_map, _ptr(reward), _ptr(done),
                                            N if reward is None else reward.shape[0], r_map, float(gamma), N, A, D, dot_mode, _ptr(out),
                                            _ptr(act), _stream())
    _lib.check(rc, "morl_critic_min_td_f32")
    _count()
    return out, act


def gpi_envelope(q_nets, w, reward=None, done=None, gamma: float = 0.0, dot_mode: int = DOT_UNFUSED, w_map: int = MAP_BLOCK,
                 r_map: int = MAP_TILE):
    """GPI envelope / policy-set evaluation (reference gpi_pd.py:662-690, 564-582).  q_nets: [n_nets, B, P, A, D];
    returns (out [B, D], policy [B] int32, action [B] int32)."""
    q_nets = _dev(q_nets, "q_nets")
    n_nets, B, P, A, D = q_nets.shape
    w = _rows(w, D, "w")
    if reward is not None:
        reward, done = _rows(reward, D, "reward"), _dev(done, "done").reshape(-1)
    out = th.empty((B, D), device=q_nets.device, dtype=th.float32)
    pol = th.empty(B, device=q_nets.device, dtype=th.int32)
    act = th.empty(B, device=q_nets.device, dtype=th.int32)
    rc = _lib.load().morl_gpi_envelope_f32(_ptr(q_nets), n_nets, _ptr(w), w.shape[0], w_map, _ptr(reward), _ptr(done),
                                           B if reward is None else reward.shape[0], r_map, float(gamma), B, P, A, D, dot_mode, _ptr(out),
                                           _ptr(pol), _ptr(act), _stream())
    _lib.check(rc, "morl_gpi_envelope_f32")
    _count()
    return out, pol, act


def actor_critic_td(q_nets, w, reward, done, logp, alpha: float, gamma: float, variant: int, w_map: int = MAP_BLOCK):
    """Continuous-action vector targets (CAPQL / MOSAC / TD3-style GPI-PD; SURVEY Appendix A.4).  q_nets: [n_nets, N, D]."""
    q_nets = _dev(q_nets, "q_nets")
    n_nets, N, D = q_nets.shape
    reward, done = _dev(reward, "reward").reshape(N, D), _dev(done, "done").reshape(-1)
    if w is not None:
        w = _rows(w, D, "w")
    if logp is not None:
        logp = _dev(logp, "logp").reshape(-1)
    out = th.empty((N,) if variant == AC_SCALAR_MIN else (N, D), device=q_nets.device, dtype=th.float32)
    rc = _lib.load().morl_actor_critic_td_f32(_ptr(q_nets), n_nets, _ptr(w), 0 if w is None else w.shape[0], w_map, _ptr(reward), _ptr(done),
                                              _ptr(logp), float(alpha), float(gamma), N, D, variant, _ptr(out), _stream())
    _lib.check(rc, "morl_actor_critic_td_f32")
    _count()
    return out


def _discrete_sac_args(q_nets, logits, w, alpha):
    q_nets, logits = _dev(q_nets, "q_nets"), _dev(logits, "logits")
    if q_nets.dim() != 4 or logits.dim() != 2:
        raise _lib.MorlB200Error(f"q_nets must be [n_nets, N, A, D] and logits [N, A], got {tuple(q_nets.shape)} and {tuple(logits.shape)}")
    n_nets, N, A, D = q_nets.shape
    if tuple(logits.shape) != (N, A):
        raise _lib.MorlB200Error(f"logits {tuple(logits.shape)} do not match q_nets {tuple(q_nets.shape)}")
    w = _rows(w, D, "w")
    alpha = _dev(alpha, "alpha").reshape(-1)
    if alpha.numel() != 1:
        raise _lib.MorlB200Error("alpha must be a device tensor with one element")
    return q_nets, logits, w, alpha, (n_nets, N, A, D)


def discrete_sac_target(q_nets, logits, w, reward, done, alpha: th.Tensor, gamma: float, w_map: int = MAP_BLOCK, out: Optional[th.Tensor] = None):
    """Discrete-action MOSAC soft target (reference mosac_discrete_action.py:452-464): q_nets [n_nets, N, A, D] target critics at s',
    logits [N, A] actor at s', ``alpha`` a device scalar read at run time.  Returns target [N]."""
    q_nets, logits, w, alpha, (n_nets, N, A, D) = _discrete_sac_args(q_nets, logits, w, alpha)
    reward, done = _dev(reward, "reward").reshape(-1, D), _dev(done, "done").reshape(-1)
    if reward.shape[0] != N or done.shape[0] != N:
        raise _lib.MorlB200Error(f"reward / done must have {N} rows, got {reward.shape[0]} / {done.shape[0]}")
    out = th.empty(N, device=q_nets.device, dtype=th.float32) if out is None else out
    rc = _lib.load().morl_discrete_sac_target_f32(_ptr(q_nets), n_nets, _ptr(logits), _ptr(w), w.shape[0], w_map, _ptr(reward), _ptr(done),
                                                  _ptr(alpha), float(gamma), N, A, D, _ptr(out), _stream())
    _lib.check(rc, "morl_discrete_sac_target_f32")
    _count()
    return out


def discrete_sac_actor_loss(logits, q_nets, w, alpha: th.Tensor, log_alpha: Optional[th.Tensor] = None, target_entropy: float = 0.0,
                            w_map: int = MAP_BLOCK, want_grad: bool = True, workspace: Optional[th.Tensor] = None):
    """Discrete-action MOSAC actor loss, d loss / d logits and, with ``log_alpha``, the temperature loss and its derivative w.r.t.
    log_alpha (reference mosac_discrete_action.py:478-498).  Returns (actor_loss [1], dlogits [N, A] or None, alpha_loss [1] or None,
    dlog_alpha [1] or None)."""
    q_nets, logits, w, alpha, (n_nets, N, A, D) = _discrete_sac_args(q_nets, logits, w, alpha)
    if log_alpha is not None:
        log_alpha = _dev(log_alpha, "log_alpha").reshape(-1)
        if log_alpha.numel() != 1:
            raise _lib.MorlB200Error("log_alpha must be a device tensor with one element")
    dev = logits.device
    loss = th.empty(1, device=dev, dtype=th.float32)
    grad = th.empty_like(logits) if want_grad else None
    aloss = th.empty(1, device=dev, dtype=th.float32) if log_alpha is not None else None
    dla = th.empty(1, device=dev, dtype=th.float32) if log_alpha is not None else None
    if workspace is None:
        nbytes = _lib.load().morl_discrete_sac_workspace_bytes(N)
        workspace = th.empty((nbytes + 3) // 4, device=dev, dtype=th.float32)
    rc = _lib.load().morl_discrete_sac_actor_loss_f32(_ptr(logits), _ptr(q_nets), n_nets, _ptr(w), w.shape[0], w_map, _ptr(alpha), _ptr(log_alpha),
                                                      float(target_entropy), N, A, D, _ptr(loss), _ptr(grad), _ptr(aloss), _ptr(dla), _ptr(workspace),
                                                      _stream())
    _lib.check(rc, "morl_discrete_sac_actor_loss_f32")
    _count(2)
    return loss, grad, aloss, dla


def vector_gae(rewards, values, dones, next_value, next_done, weights, gamma: float, gae_lambda: float, gae: bool = True,
               returns_out: Optional[th.Tensor] = None, adv_out: Optional[th.Tensor] = None):
    """MO-PPO's reverse GAE recursion (reference mo_ppo.py:439-476) in one launch.  rewards / values [T, E, D], dones [T, E],
    next_value [E, D], next_done [E], weights [D]; ``gae=False`` gives the plain discounted returns.  Returns (returns [T, E, D],
    scalarised advantages [T, E]), written into ``returns_out`` / ``adv_out`` when given."""
    rewards, values, dones = _dev(rewards, "rewards"), _dev(values, "values"), _dev(dones, "dones")
    if rewards.dim() != 3 or values.shape != rewards.shape:
        raise _lib.MorlB200Error(f"rewards / values must both be [T, E, D], got {tuple(rewards.shape)} and {tuple(values.shape)}")
    T, E, D = rewards.shape
    if tuple(dones.shape) != (T, E):
        raise _lib.MorlB200Error(f"dones must be [{T}, {E}], got {tuple(dones.shape)}")
    next_value, next_done, weights = _dev(next_value, "next_value").reshape(-1), _dev(next_done, "next_done").reshape(-1), _dev(weights, "weights").reshape(-1)
    if next_value.numel() != E * D or next_done.numel() != E or weights.numel() != D:
        raise _lib.MorlB200Error(f"next_value / next_done / weights must have {E * D} / {E} / {D} elements")
    ret = th.empty_like(rewards) if returns_out is None else returns_out
    adv = th.empty((T, E), device=rewards.device, dtype=th.float32) if adv_out is None else adv_out
    for t, shape, name in ((ret, (T, E, D), "returns_out"), (adv, (T, E), "adv_out")):
        if t.dtype != th.float32 or not t.is_cuda or not t.is_contiguous() or t.numel() != T * E * (D if name == "returns_out" else 1):
            raise _lib.MorlB200Error(f"{name} must be a contiguous float32 CUDA tensor of shape {shape}")
    rc = _lib.load().morl_vector_gae_f32(_ptr(rewards), _ptr(values), _ptr(dones), _ptr(next_value), _ptr(next_done), _ptr(weights), T, E, D,
                                         float(gamma), float(gae_lambda), int(bool(gae)), _ptr(ret), _ptr(adv), _stream())
    _lib.check(rc, "morl_vector_gae_f32")
    _count()
    return ret, adv


def ppo_loss(mean, logstd, value, actions, old_logprob, advantages, returns, old_values, clip_coef: float, ent_coef: float, vf_coef: float,
             norm_adv: bool, clip_vloss: bool, stats: th.Tensor, out: Optional[Tuple[th.Tensor, th.Tensor, th.Tensor, th.Tensor]] = None):
    """One minibatch's MO-PPO loss and its gradients (reference mo_ppo.py:514-549) in one launch.  mean [M, A], logstd [A] (or [1, A]),
    value [M, D], actions [M, A], old_logprob [M], advantages [M], returns / old_values [M, D]; ``stats`` a float32 device vector of 6
    (pg_loss, v_loss, entropy, old_approx_kl, approx_kl written; clip fraction added).  Returns (loss [1], dmean [M, A], dlogstd [A],
    dvalue [M, D]), written into ``out`` when given."""
    mean, value, actions = _dev(mean, "mean"), _dev(value, "value"), _dev(actions, "actions")
    M, A = mean.shape
    D = value.shape[-1]
    logstd = _dev(logstd, "logstd").reshape(-1)
    value = value.reshape(-1, D)
    old_logprob, advantages = _dev(old_logprob, "old_logprob").reshape(-1), _dev(advantages, "advantages").reshape(-1)
    returns = _dev(returns, "returns").reshape(-1, D)
    old_values = _dev(old_values, "old_values").reshape(-1, D) if old_values is not None else None
    if (tuple(actions.shape) != (M, A) or logstd.numel() != A or value.shape[0] != M or old_logprob.numel() != M or advantages.numel() != M
            or returns.shape[0] != M or (old_values is not None and old_values.shape[0] != M)):
        raise _lib.MorlB200Error("ppo_loss: inconsistent shapes")
    stats = _dev(stats, "stats")
    if stats.numel() != 6:
        raise _lib.MorlB200Error("ppo_loss: stats must have 6 elements")
    dev = mean.device
    if out is None:
        out = (th.empty(1, device=dev), th.empty_like(mean), th.empty(A, device=dev), th.empty((M, D), device=dev))
    loss, dmean, dlogstd, dvalue = out
    rc = _lib.load().morl_ppo_loss_f32(_ptr(mean), _ptr(logstd), _ptr(value), _ptr(actions), _ptr(old_logprob), _ptr(advantages), _ptr(returns),
                                       _ptr(old_values), M, A, D, float(clip_coef), float(ent_coef), float(vf_coef), int(bool(norm_adv)),
                                       int(bool(clip_vloss)), _ptr(loss), _ptr(dmean), _ptr(dlogstd), _ptr(dvalue), _ptr(stats), _stream())
    _lib.check(rc, "morl_ppo_loss_f32")
    _count()
    return loss, dmean, dlogstd, dvalue


def td_workspace(n_rows: int, device) -> th.Tensor:
    nbytes = _lib.load().morl_td_workspace_bytes(int(n_rows))
    return th.empty((nbytes + 3) // 4, device=device, dtype=th.float32)


def td_mse_priority(q_values, action, target_q, wset, homotopy_lambda: float, B: int, W: int, row_order: int = ROWS_REFERENCE,
                    want_grad: bool = True, want_prio: bool = True, workspace: Optional[th.Tensor] = None, loss_out=None, grad_out=None,
                    prio_out=None, q_taken_out=None, lambda_dev=None):
    """Fused Envelope TD loss + d loss / d q_values + priorities (reference envelope.py:301-313, 329-331).  ``lambda_dev`` (device f32 [1])
    overrides ``homotopy_lambda`` and is read by the kernels at run time (graph-replay safe)."""
    q_values = _dev(q_values, "q_values")
    N, A, D = q_values.shape
    if N != B * W:
        raise _lib.MorlB200Error(f"q_values has {N} rows, expected B*W = {B * W}")
    action = _dev(action, "action", th.int32).reshape(-1)
    target_q, wset = _dev(target_q, "target_q"), _dev(wset, "wset")
    dev = q_values.device
    loss = th.empty(1, device=dev, dtype=th.float32) if loss_out is None else loss_out
    grad = (th.empty_like(q_values) if grad_out is None else grad_out) if want_grad else None
    prio = (th.empty(B, device=dev, dtype=th.float32) if prio_out is None else prio_out) if want_prio else None
    ws = td_workspace(N, dev) if workspace is None else workspace
    rc = _lib.load().morl_td_mse_priority_f32(_ptr(q_values), _ptr(action), _ptr(target_q), _ptr(wset), float(homotopy_lambda), _ptr(lambda_dev), B, W, A, D,
                                              row_order, _ptr(loss), _ptr(grad), _ptr(q_taken_out), _ptr(prio), _ptr(ws), _stream())
    _lib.check(rc, "morl_td_mse_priority_f32")
    _count(2)
    return loss, grad, prio


def td_huber_priority(q_values, action, target_q, target_q_gpi, w, min_priority: float, p_rows: int, w_map: int = MAP_BLOCK,
                      want_grad: bool = True, workspace: Optional[th.Tensor] = None):
    """GPI-PD Huber-style loss, gradient seed and raw priorities (reference gpi_pd.py:469-487, 507-520)."""
    q_values = _dev(q_values, "q_values")
    n_nets, N, A, D = q_values.shape
    action = _dev(action, "action", th.int32).reshape(-1)
    target_q = _dev(target_q, "target_q")
    if target_q_gpi is not None:
        target_q_gpi = _dev(target_q_gpi, "target_q_gpi")
    w = _rows(w, D, "w")
    dev = q_values.device
    loss = th.empty(1, device=dev, dtype=th.float32)
    grad = th.empty_like(q_values) if want_grad else None
    prio = th.empty(p_rows, device=dev, dtype=th.float32) if p_rows > 0 else None
    ws = td_workspace(N, dev) if workspace is None else workspace
    rc = _lib.load().morl_td_huber_priority_f32(_ptr(q_values), n_nets, _ptr(action), action.shape[0], _ptr(target_q), _ptr(target_q_gpi),
                                                _ptr(w), w.shape[0], w_map, float(min_priority), N, A, D, p_rows, _ptr(loss), _ptr(grad),
                                                _ptr(prio), _ptr(ws), _stream())
    _lib.check(rc, "morl_td_huber_priority_f32")
    _count(2)
    return loss, grad, prio


def replay_gather(obs_store, next_obs_store, act_store, rew_store, done_store, idx, outs=None):
    """Gather a minibatch from device-resident stores (reference buffer.py:82-94).  Returns
    (obs, actions, rewards, next_obs, dones); uint8 actions come back as int32."""
    obs_store, next_obs_store = _dev(obs_store, "obs_store"), _dev(next_obs_store, "next_obs_store")
    rew_store, done_store = _dev(rew_store, "rew_store"), _dev(done_store, "done_store")
    idx = _dev(idx, "idx", th.int64).reshape(-1)
    cap, obs_dim = obs_store.shape[0], obs_store[0].numel()
    is_u8 = act_store.dtype == th.uint8
    act_store = _dev(act_store, "act_store", th.uint8 if is_u8 else th.float32)
    act_dim, rew_dim = act_store[0].numel(), rew_store[0].numel()
    B = idx.shape[0]
    dev = obs_store.device
    if outs is None:
        obs = th.empty((B,) + tuple(obs_store.shape[1:]), device=dev, dtype=th.float32)
        nobs = th.empty_like(obs)
        act = th.empty((B, act_dim), device=dev, dtype=th.int32 if is_u8 else th.float32)
        rew = th.empty((B, rew_dim), device=dev, dtype=th.float32)
        done = th.empty((B, 1), device=dev, dtype=th.float32)
    else:
        obs, act, rew, nobs, done = outs
    rc = _lib.load().morl_replay_gather(_ptr(obs_store), _ptr(next_obs_store), _ptr(act_store), _ptr(rew_store), _ptr(done_store), _ptr(idx),
                                        B, obs_dim, act_dim, rew_dim, int(is_u8), cap, _ptr(obs), _ptr(nobs), _ptr(act), _ptr(rew), _ptr(done),
                                        _stream())
    _lib.check(rc, "morl_replay_gather")
    _count()
    return obs, act, rew, nobs, done


def pareto_mask(points: th.Tensor, remove_duplicates: bool = True, raw: bool = False, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Non-dominated mask (reference pareto.py:34-57) of an [N, D] fp32 / fp64 CUDA tensor -> bool [N] (``raw``: the kernel's uint8 [N],
    optionally written into ``out``: no further launch)."""
    if not points.is_cuda:
        raise _lib.MorlB200Error("points must be a CUDA tensor (morl_baselines_b200 has no CPU fallback)")
    if points.dtype not in (th.float32, th.float64):
        raise _lib.MorlB200Error(f"points must be float32 or float64, got {points.dtype}")
    points = points.contiguous()
    N, D = points.shape
    keep = th.empty(N, device=points.device, dtype=th.uint8) if out is None else out
    if N == 0:
        return keep if raw else keep.bool()
    fn = _lib.load().morl_pareto_mask_f32 if points.dtype == th.float32 else _lib.load().morl_pareto_mask_f64
    rc = fn(_ptr(points), N, D, int(bool(remove_duplicates)), _ptr(keep), _stream())
    _lib.check(rc, "morl_pareto_mask")
    _count(2)
    return keep if raw else keep.bool()


def front_pack(points: th.Tensor, keep: Optional[th.Tensor], cap: int, rec: th.Tensor, extras: Optional[th.Tensor] = None) -> th.Tensor:
    """rec (float64 [1 + cap*d + n_extra]) = [count | first cap kept rows of points [n, d] (float64), -inf padded | extras]; one launch,
    no host sync (the count stays on the device)."""
    n, d = points.shape
    n_extra = 0 if extras is None else extras.numel()
    if points.dtype != th.float64 or not points.is_contiguous() or rec.numel() != 1 + cap * d + n_extra:
        raise _lib.MorlB200Error("front_pack: points must be contiguous float64 [n, d] and rec float64 [1 + cap*d + n_extra]")
    rc = _lib.load().morl_front_pack_f64(_ptr(points), _ptr(keep), n, d, cap, _ptr(extras), n_extra, _ptr(rec), _stream())
    _lib.check(rc, "morl_front_pack_f64")
    _count()
    return rec


def front_unpack(gathered: th.Tensor, world: int, d: int, cap: int, n_extra: int, pts_out: th.Tensor, meta_out: th.Tensor):
    """gathered records [world, 1 + cap*d + n_extra] -> pts_out [world*cap, d], meta_out [world, 1 + n_extra] (count, extras); one launch."""
    rc = _lib.load().morl_front_unpack_f64(_ptr(gathered), world, d, cap, n_extra, _ptr(pts_out), _ptr(meta_out), _stream())
    _lib.check(rc, "morl_front_unpack_f64")
    _count()
    return pts_out, meta_out


def hypervolume(points: th.Tensor, ref_point: th.Tensor, keep: Optional[th.Tensor] = None, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Exact hypervolume (maximisation, d <= 3, n <= 2048) of float64 CUDA points [n, d] above ``ref_point`` [d]; returns a device float64
    scalar tensor [1] (no host sync).  ``keep`` (uint8 [n]) restricts the set, e.g. to the output of ``pareto_mask(..., raw=True)``."""
    if not points.is_cuda or points.dtype != th.float64 or not points.is_contiguous():
        raise _lib.MorlB200Error("hypervolume: points must be a contiguous float64 CUDA tensor [n, d]")
    n, d = points.shape
    ref_point = ref_point.to(device=points.device, dtype=th.float64).contiguous()
    out = th.empty(1, dtype=th.float64, device=points.device) if out is None else out
    rc = _lib.load().morl_hypervolume_f64(_ptr(points), _ptr(keep), n, d, _ptr(ref_point), _ptr(out), _stream())
    _lib.check(rc, "morl_hypervolume_f64")
    _count()
    return out


def corner_weights(V: th.Tensor, cap: int = 256) -> th.Tensor:
    """Vertices (w, u) of { V w <= u, w >= 0, sum w = 1 } for a float64 CUDA tensor V [n, d] (reference linear_support.py:295-349;
    the caller rounds V).  Returns float64 [K, d+1] in no particular order; one launch, plus a second one with a buffer of the exact size
    when more than ``cap`` vertices exist (the count is read back: one host sync)."""
    if not V.is_cuda or V.dtype != th.float64 or V.dim() != 2:
        raise _lib.MorlB200Error("corner_weights: V must be a float64 CUDA tensor [n, d]")
    V = V.contiguous()
    n, d = V.shape
    count = th.empty(1, dtype=th.int32, device=V.device)
    while True:
        verts = th.empty((cap, d + 1), dtype=th.float64, device=V.device)
        rc = _lib.load().morl_corner_weights_f64(_ptr(V), n, d, _ptr(verts) if cap > 0 else None, cap, _ptr(count), _stream())
        _lib.check(rc, "morl_corner_weights_f64")
        _count()
        k = int(count.item())
        if k <= cap:
            return verts[:k]
        cap = k


class PolyakPlan:
    """Device-side (param, target, size) table for morl_polyak_f32; build once per pair of networks."""

    def __init__(self, params, targets):
        params, targets = list(params), list(targets)
        assert len(params) == len(targets) and len(params) > 0
        for p, t in zip(params, targets):
            if not (p.is_cuda and t.is_cuda and p.dtype == th.float32 and t.dtype == th.float32 and p.is_contiguous() and t.is_contiguous()):
                raise _lib.MorlB200Error("polyak: parameters must be contiguous float32 CUDA tensors")
            assert p.numel() == t.numel()
        dev = params[0].device
        self.keepalive = (params, targets)
        self.p_tab = th.tensor([p.data_ptr() for p in params], dtype=th.int64, device=dev)
        self.t_tab = th.tensor([t.data_ptr() for t in targets], dtype=th.int64, device=dev)
        self.sizes = th.tensor([p.numel() for p in params], dtype=th.int64, device=dev)
        self.n = len(params)
        self.max_size = max(p.numel() for p in params)

    def run(self, tau: float):
        rc = _lib.load().morl_polyak_f32(_ptr(self.p_tab), _ptr(self.t_tab), _ptr(self.sizes), self.n, self.max_size, float(tau), _stream())
        _lib.check(rc, "morl_polyak_f32")
        _count()


def sm_count() -> int:
    n = _lib.load().morl_device_sm_count()
    if n < 0:
        _lib.check(n, "morl_device_sm_count")
    return n


# ------------------------------------------------------------------------------------------------ wgmma dense layers
def _pad(n: int, m: int) -> int:
    return (n + m - 1) // m * m


FMT_BF16X3, FMT_F16X2 = _lib.FMT_BF16X3, _lib.FMT_F16X2
_FMT_DTYPE = {FMT_BF16X3: th.bfloat16, FMT_F16X2: th.float16}
_FMT_PLANES = {FMT_BF16X3: 3, FMT_F16X2: 2}


def fmt_of(planes: th.Tensor) -> int:
    """Plane format of a plane tensor: bf16 [3, rows, ld] = bf16x3, fp16 [2, rows, ld] = f16x2."""
    if planes.dtype == th.bfloat16 and planes.shape[0] == 3:
        return FMT_BF16X3
    if planes.dtype == th.float16 and planes.shape[0] == 2:
        return FMT_F16X2
    raise _lib.MorlB200Error(f"not a plane tensor: dtype {planes.dtype}, leading dimension {planes.shape[0]}")


def empty_planes(fmt: int, rows: int, ld: int, device) -> th.Tensor:
    return th.empty((_FMT_PLANES[fmt], rows, ld), device=device, dtype=_FMT_DTYPE[fmt])


def scale_tensor(value: float, device) -> th.Tensor:
    """A device-resident power-of-two scale (float32 [1])."""
    return th.full((1,), float(value), device=device, dtype=th.float32)


def plane_overflow_count(reset: bool = False) -> int:
    """Number of f16x2 range violations (|scale * x| > 65504) the plane-producing kernels saw since the last reset (synchronises)."""
    n = _lib.load().morl_plane_overflow_count(int(reset))
    if n < 0:
        _lib.check(n, "morl_plane_overflow_count")
    return n


def amax_scale(x: th.Tensor, target_exp: int, scale_out: th.Tensor, workspace: th.Tensor) -> th.Tensor:
    """scale_out[0] = 2^(target_exp - e) with max|x| < 2^e (one launch; workspace: 2 zeroed int32, left zeroed)."""
    x = _dev(x, "x")
    rc = _lib.load().morl_amax_scale_f32(_ptr(x), x.numel(), int(target_exp), _ptr(scale_out), _ptr(workspace), _stream())
    _lib.check(rc, "morl_amax_scale_f32")
    _count()
    return scale_out


def split_planes(x: th.Tensor, fmt: int = FMT_F16X2, rows_pad: Optional[int] = None, ldp: Optional[int] = None, transpose: bool = False,
                 out: Optional[th.Tensor] = None, scale: Optional[th.Tensor] = None) -> th.Tensor:
    """fp32 [rows, cols] -> planes [P, rows_pad, ldp] of scale * x (zero padded); with ``transpose`` the planes hold x^T."""
    x = _dev(x, "x")
    r, c = (x.shape[1], x.shape[0]) if transpose else (x.shape[0], x.shape[1])
    rows_pad = r if rows_pad is None else rows_pad
    ldp = _pad(c, 64 if fmt == FMT_F16X2 else 32) if ldp is None else ldp
    if out is None:
        out = empty_planes(fmt, rows_pad, ldp, x.device)
    rc = _lib.load().morl_split_planes(fmt, _ptr(x), r, c, x.shape[1], int(transpose), _ptr(out), rows_pad, ldp, out.stride(0), _ptr(scale), _stream())
    _lib.check(rc, "morl_split_planes")
    _count()
    return out


def split_planes_multi(jobs, fmt: int = FMT_F16X2) -> None:
    """One launch for several splits.  jobs: iterable of (src [rows, cols] fp32 CUDA, out planes [P, rows_pad, ldp], transpose, scale, target_exp):
    ``scale`` is a device float [1] or None; ``target_exp`` None = use the scale as given, an int = derive it from the matrix's amax and store it."""
    jobs = list(jobs)
    if not jobs:
        return
    if len(jobs) > _lib.SPLIT_MAX_JOBS:
        raise _lib.MorlB200Error(f"split_planes_multi: at most {_lib.SPLIT_MAX_JOBS} jobs per call")
    arr = (_lib.SplitJob * len(jobs))()
    for k, job in enumerate(jobs):
        src, out, transpose = job[0], job[1], job[2]
        scale = job[3] if len(job) > 3 else None
        target_exp = job[4] if len(job) > 4 else None
        src = _dev(src, "src")
        rows, cols = (src.shape[1], src.shape[0]) if transpose else (src.shape[0], src.shape[1])
        arr[k].src, arr[k].dst_planes, arr[k].plane_stride = src.data_ptr(), out.data_ptr(), out.stride(0)
        arr[k].scale = None if scale is None else scale.data_ptr()
        arr[k].rows, arr[k].cols, arr[k].ld_src, arr[k].transpose = rows, cols, src.stride(0), int(bool(transpose))
        arr[k].rows_pad, arr[k].ldp = out.shape[1], out.shape[2]
        arr[k].auto_scale, arr[k].target_exp = (0, 0) if target_exp is None else (1, int(target_exp))
    rc = _lib.load().morl_split_planes_multi(fmt, arr, len(jobs), _stream())
    _lib.check(rc, "morl_split_planes_multi")
    _count(2 if any(a.auto_scale for a in arr) else 1)


def gemm_planes(a_planes: th.Tensor, b_planes: th.Tensor, n_out: int, bias: Optional[th.Tensor] = None, relu: bool = False,
                relu_mask: Optional[th.Tensor] = None, out_f32: bool = True, out_planes: bool = False, c_f32: Optional[th.Tensor] = None,
                c_planes: Optional[th.Tensor] = None, reverse_tiles: bool = False, a_scale: Optional[th.Tensor] = None,
                b_scale: Optional[th.Tensor] = None, c_scale: Optional[th.Tensor] = None, split_acc: bool = False,
                relu_bits_in: Optional[th.Tensor] = None, relu_bits_out: Optional[th.Tensor] = None):
    """C = act(A . B^T + bias) on the tensor cores (wgmma) with split operands (fp32-accurate).
    a_planes [P, M, K], b_planes [P, N_pad, K]; the scales are device floats the planes were multiplied by (None = 1);
    ``split_acc``: leading and correction products in separate accumulators (the tensor cores truncate their fp32 accumulation; ~2.5x
    smaller systematic error, ~20 % slower per launch); False (default): one double-buffered accumulator.
    ``relu_bits_out`` / ``relu_bits_in`` (:func:`empty_relu_bits`): the forward call records [C > 0] as one bit per column, the backward
    call zeroes the outputs whose bit is clear (ReLU backward from 32 bytes per row instead of the activation planes; ``relu_mask`` is the
    plane-based form of the same mask).  Their width is the padded output width N_pad = b_planes.shape[1]
    (``empty_relu_bits(M, device, N_pad)``): 8 words per row up to 256, 16 above.
    returns (c_f32 [M, n_out] or None, c_planes [P, M, ldp] holding c_scale * C, or None)."""
    fmt = fmt_of(a_planes)
    if fmt_of(b_planes) != fmt or not a_planes.is_cuda:
        raise _lib.MorlB200Error("gemm_planes: operands must be CUDA plane tensors of the same format")
    _, M, K = a_planes.shape
    _, n_pad, Kb = b_planes.shape
    if Kb != K or a_planes.stride(1) != K or b_planes.stride(1) != K:
        raise _lib.MorlB200Error("gemm_planes: operand planes must be K-major with equal K")
    dev = a_planes.device
    if out_f32 and c_f32 is None:
        c_f32 = th.empty((M, n_out), device=dev, dtype=th.float32)
    if out_planes and c_planes is None:
        c_planes = empty_planes(fmt, M, _pad(n_out, 32), dev)
    mask0 = None if relu_mask is None else relu_mask[0]
    words = relu_bits_words(n_pad)  # one word per 32-column chunk of the padded output (the kernel visits them all)
    for bits in (relu_bits_in, relu_bits_out):
        if bits is not None and (bits.dtype != th.int32 or tuple(bits.shape) != (M, words) or not bits.is_contiguous() or bits.device != dev):
            raise _lib.MorlB200Error(f"gemm_planes: ReLU bit masks must be contiguous int32 [{M}, {words}] on {dev}")
    rc = _lib.load().morl_gemm_planes_f32(fmt, _ptr(a_planes), a_planes.stride(0), _ptr(a_scale), _ptr(b_planes), b_planes.stride(0), _ptr(b_scale), M,
                                          n_out, n_pad, K, _ptr(bias), int(relu), _ptr(mask0), 0 if mask0 is None else mask0.stride(0), _ptr(c_f32),
                                          0 if c_f32 is None else c_f32.stride(0), _ptr(c_planes), 0 if c_planes is None else c_planes.shape[2],
                                          0 if c_planes is None else c_planes.stride(0), _ptr(c_scale), int(reverse_tiles), int(bool(split_acc)),
                                          _ptr(relu_bits_in), _ptr(relu_bits_out), _stream())
    _lib.check(rc, "morl_gemm_planes_f32")
    _count()
    return c_f32, c_planes


def gemm_planes_ln(a_planes: th.Tensor, b_planes: th.Tensor, n_out: int, bias: Optional[th.Tensor] = None, ln_weight: Optional[th.Tensor] = None,
                   ln_bias: Optional[th.Tensor] = None, ln_eps: Optional[float] = None, drop_p: float = 0.0, drop_seed: Optional[th.Tensor] = None,
                   drop_offset: Optional[th.Tensor] = None, drop_salt: int = 0, out_f32: bool = False, out_planes: bool = True,
                   c_f32: Optional[th.Tensor] = None, c_planes: Optional[th.Tensor] = None, reverse_tiles: bool = False,
                   a_scale: Optional[th.Tensor] = None, b_scale: Optional[th.Tensor] = None, c_scale: Optional[th.Tensor] = None,
                   drop_bits_out: Optional[th.Tensor] = None):
    """Hidden layer Linear -> Dropout -> LayerNorm -> ReLU in one tensor-core GEMM: C = relu(LN(dropout(A . B^T + bias))).
    a_planes [P, M, K], b_planes [P, n_out, K] (n_out % 32 == 0, <= 256).  ``ln_eps`` None: no LayerNorm (``ln_weight`` / ``ln_bias``
    [n_out] fp32, None = 1 / 0).  Dropout runs when ``drop_seed`` (int64 [1]) and ``drop_offset`` (int32 [1], the pass counter, see
    :func:`philox_advance`) are given: element kept iff its Philox4x32-10 draw >= round(drop_p 2^32), kept values scaled by 1 / (1 - drop_p);
    ``drop_salt`` separates the layers of one pass.  ``drop_bits_out`` ([M, 8] int32) receives the keep mask in the ReLU-bit layout.
    Returns (c_f32 [M, n_out] or None, c_planes [P, M, n_out] holding c_scale * C, or None)."""
    fmt = fmt_of(a_planes)
    if fmt_of(b_planes) != fmt or not a_planes.is_cuda:
        raise _lib.MorlB200Error("gemm_planes_ln: operands must be CUDA plane tensors of the same format")
    _, M, K = a_planes.shape
    _, n_pad, Kb = b_planes.shape
    if Kb != K or a_planes.stride(1) != K or b_planes.stride(1) != K:
        raise _lib.MorlB200Error("gemm_planes_ln: operand planes must be K-major with equal K")
    if n_pad != n_out or n_out % 32 or n_out > 256:
        raise _lib.MorlB200Error(f"gemm_planes_ln: need weight planes [P, n_out, K] with n_out % 32 == 0 and n_out <= 256 (got {tuple(b_planes.shape)}, n_out={n_out})")
    if not 0.0 <= drop_p < 1.0:
        raise _lib.MorlB200Error(f"gemm_planes_ln: dropout probability {drop_p} outside [0, 1)")
    if (drop_seed is None) != (drop_offset is None):
        raise _lib.MorlB200Error("gemm_planes_ln: dropout needs both drop_seed and drop_offset")
    if drop_seed is not None and (drop_seed.dtype != th.int64 or drop_offset.dtype != th.int32 or not drop_seed.is_cuda or not drop_offset.is_cuda):
        raise _lib.MorlB200Error("gemm_planes_ln: drop_seed must be a CUDA int64 [1] tensor and drop_offset a CUDA int32 [1] tensor")
    for name, t in (("bias", bias), ("ln_weight", ln_weight), ("ln_bias", ln_bias)):
        if t is not None and (t.dtype != th.float32 or t.numel() != n_out or not t.is_contiguous() or not t.is_cuda):
            raise _lib.MorlB200Error(f"gemm_planes_ln: {name} must be a contiguous CUDA float32 vector of {n_out}")
    dev = a_planes.device
    if out_f32 and c_f32 is None:
        c_f32 = th.empty((M, n_out), device=dev, dtype=th.float32)
    if out_planes and c_planes is None:
        c_planes = empty_planes(fmt, M, n_out, dev)
    if c_f32 is None and c_planes is None:
        raise _lib.MorlB200Error("gemm_planes_ln: no output requested")
    if drop_bits_out is not None and (drop_bits_out.dtype != th.int32 or tuple(drop_bits_out.shape) != (M, relu_bits_words(n_out))
                                      or not drop_bits_out.is_contiguous()):
        raise _lib.MorlB200Error(f"gemm_planes_ln: the keep mask must be contiguous int32 [{M}, {relu_bits_words(n_out)}]")
    rc = _lib.load().morl_gemm_planes_ln_f32(fmt, _ptr(a_planes), a_planes.stride(0), _ptr(a_scale), _ptr(b_planes), b_planes.stride(0), _ptr(b_scale), M,
                                             n_out, K, _ptr(None if bias is None else bias.detach()), int(ln_eps is not None),
                                             _ptr(None if ln_weight is None else ln_weight.detach()), _ptr(None if ln_bias is None else ln_bias.detach()),
                                             float(ln_eps or 0.0), float(drop_p), _ptr(drop_seed), _ptr(drop_offset), int(drop_salt) & 0xFFFFFFFF,
                                             _ptr(c_f32), 0 if c_f32 is None else c_f32.stride(0), _ptr(c_planes),
                                             0 if c_planes is None else c_planes.shape[2], 0 if c_planes is None else c_planes.stride(0), _ptr(c_scale),
                                             int(reverse_tiles), _ptr(drop_bits_out), _stream())
    _lib.check(rc, "morl_gemm_planes_ln_f32")
    _count()
    return c_f32, c_planes


def philox_advance(offset: th.Tensor, inc: int = 1) -> th.Tensor:
    """offset[0] += inc (int32 [1] CUDA tensor, wrapping) as one stream-ordered launch: the dropout pass counter of :func:`gemm_planes_ln`."""
    if not isinstance(offset, th.Tensor) or not offset.is_cuda or offset.dtype != th.int32 or offset.numel() != 1:
        raise _lib.MorlB200Error("philox_advance: offset must be a CUDA int32 [1] tensor")
    rc = _lib.load().morl_philox_advance(_ptr(offset), int(inc) & 0xFFFFFFFF, _stream())
    _lib.check(rc, "morl_philox_advance")
    _count()
    return offset


def ensemble_sample(out: th.Tensor, max_logvar: th.Tensor, min_logvar: th.Tensor, model_idx: th.Tensor, noise: Optional[th.Tensor] = None,
                    obs: Optional[th.Tensor] = None, rew_dim: int = 0):
    """Probabilistic-ensemble sampling + ensemble uncertainty in one pass (reference probabilistic_ensemble.py:115-154, utils.py:165).
    out [E, N, 2*O] raw last-layer output, model_idx [N] int32, noise [E, N, O] or None (deterministic), obs [N, O - rew_dim] or None.
    Returns (sample [N, O], var [N, O], uncertainty [N])."""
    out = _dev(out, "out")
    E, N, O2 = out.shape
    O = O2 // 2
    max_logvar, min_logvar = _dev(max_logvar, "max_logvar").reshape(-1), _dev(min_logvar, "min_logvar").reshape(-1)
    model_idx = _dev(model_idx, "model_idx", th.int32)
    if O2 != 2 * O or max_logvar.numel() != O or min_logvar.numel() != O or model_idx.numel() != N:
        raise _lib.MorlB200Error(f"ensemble_sample: bad shapes out {tuple(out.shape)}, logvar bounds {max_logvar.numel()}, model_idx {tuple(model_idx.shape)} {model_idx.dtype}")
    if noise is not None:
        noise = _dev(noise, "noise")
        if tuple(noise.shape) != (E, N, O):
            raise _lib.MorlB200Error(f"ensemble_sample: noise must be [{E}, {N}, {O}]")
    if obs is not None:
        obs = _dev(obs, "obs")
        if tuple(obs.shape) != (N, O - rew_dim):
            raise _lib.MorlB200Error(f"ensemble_sample: obs must be [{N}, {O - rew_dim}]")
    sample = th.empty((N, O), device=out.device, dtype=th.float32)
    var = th.empty((N, O), device=out.device, dtype=th.float32)
    unc = th.empty(N, device=out.device, dtype=th.float32)
    rc = _lib.load().morl_ensemble_sample_f32(_ptr(out), _ptr(max_logvar), _ptr(min_logvar), _ptr(model_idx), _ptr(noise), _ptr(obs), int(rew_dim), E, N, O,
                                              _ptr(sample), _ptr(var), _ptr(unc), _stream())
    _lib.check(rc, "morl_ensemble_sample_f32")
    _count()
    return sample, var, unc


TERM_NONE, TERM_HOPPER, TERM_HUMANOID, TERM_MOUNTAINCAR, TERM_LUNARLANDER = 0, 1, 2, 3, 4  # MORL_TERM_* of include/morl_b200.h


def dyna_commit_workspace(n_rows: int, device) -> th.Tensor:
    nbytes = _lib.load().morl_dyna_commit_workspace_bytes(int(n_rows))
    return th.empty((nbytes + 3) // 4, device=device, dtype=th.int32)


def dyna_commit(out: th.Tensor, max_logvar: th.Tensor, min_logvar: th.Tensor, model_idx: th.Tensor, noise: Optional[th.Tensor], obs: th.Tensor,
                act: th.Tensor, rew_dim: int, rule: int, max_uncertainty: float, stores, ptr: int, next_alive: th.Tensor, uncertainty_out: th.Tensor,
                counts_out: th.Tensor, workspace: Optional[th.Tensor] = None):
    """One imagined Dyna step (``morl_dyna_commit_f32``, two launches, no host synchronisation): ensemble sample + uncertainty (as
    :func:`ensemble_sample`, with ``obs`` added), termination ``rule`` (``TERM_*``), the gate ``uncertainty < max_uncertainty``, the ring append
    of the kept rows into ``stores`` = (obs [C, S], next_obs [C, S], act [C, A], rew [C, rew_dim], done [C, 1]) from slot ``ptr``, and the
    alive rows' s' compacted into ``next_alive`` [N, S].  ``counts_out`` (int32 [2]) receives {kept, alive} on the device."""
    out = _dev(out, "out")
    E, N, O2 = out.shape
    O = O2 // 2
    S = O - int(rew_dim)
    max_logvar, min_logvar = _dev(max_logvar, "max_logvar").reshape(-1), _dev(min_logvar, "min_logvar").reshape(-1)
    model_idx = _dev(model_idx, "model_idx", th.int32)
    obs, act = _dev(obs, "obs"), _dev(act, "act")
    if (O2 != 2 * O or max_logvar.numel() != O or min_logvar.numel() != O or model_idx.numel() != N or obs.dim() != 2 or tuple(obs.shape) != (N, S)
            or act.dim() != 2 or act.shape[0] != N):
        raise _lib.MorlB200Error(f"dyna_commit: bad shapes out {tuple(out.shape)}, logvar bounds {max_logvar.numel()}, model_idx {tuple(model_idx.shape)}, "
                                 f"obs {tuple(obs.shape)} (want [{N}, {S}]), act {tuple(act.shape)}")
    A = act.shape[1]
    if noise is not None:
        noise = _dev(noise, "noise")
        if tuple(noise.shape) != (E, N, O):
            raise _lib.MorlB200Error(f"dyna_commit: noise must be [{E}, {N}, {O}]")
    st_obs, st_nobs, st_act, st_rew, st_done = stores
    C = st_obs.shape[0]
    for name, t, cols in (("obs", st_obs, S), ("next_obs", st_nobs, S), ("actions", st_act, A), ("rewards", st_rew, rew_dim), ("dones", st_done, 1)):
        if not (isinstance(t, th.Tensor) and t.is_cuda and t.dtype == th.float32 and t.is_contiguous() and t.dim() == 2 and tuple(t.shape) == (C, cols)):
            raise _lib.MorlB200Error(f"dyna_commit: store {name} must be a contiguous float32 CUDA tensor [{C}, {cols}]")
    for name, t, shape, dt in (("next_alive", next_alive, (N, S), th.float32), ("uncertainty_out", uncertainty_out, (N,), th.float32),
                               ("counts_out", counts_out, (2,), th.int32)):
        if not (isinstance(t, th.Tensor) and t.is_cuda and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == shape):
            raise _lib.MorlB200Error(f"dyna_commit: {name} must be a contiguous {dt} CUDA tensor {list(shape)}")
    ws = dyna_commit_workspace(N, out.device) if workspace is None else workspace
    if ws.numel() * ws.element_size() < _lib.load().morl_dyna_commit_workspace_bytes(N):
        raise _lib.MorlB200Error("dyna_commit: workspace too small")
    rc = _lib.load().morl_dyna_commit_f32(_ptr(out), _ptr(max_logvar), _ptr(min_logvar), _ptr(model_idx), _ptr(noise), _ptr(obs), _ptr(act), int(rew_dim), E, N,
                                          O, A, int(rule), float(max_uncertainty), _ptr(st_obs), _ptr(st_nobs), _ptr(st_act), _ptr(st_rew), _ptr(st_done), C,
                                          int(ptr), _ptr(next_alive), _ptr(uncertainty_out), _ptr(counts_out), _ptr(ws), _stream())
    _lib.check(rc, "morl_dyna_commit_f32")
    _count(2)
    return counts_out


def qhead_envelope_supported(fmt: int, B: int, W: int, A: int, D: int, K: int) -> bool:
    """True if :func:`qhead_envelope_td` covers the configuration (else use gemm_planes x 2 + envelope_td)."""
    return bool(_lib.load().morl_qhead_envelope_supported(int(fmt), int(B), int(W), int(A), int(D), int(K)))


def qhead_envelope_td(a_on: th.Tensor, a_tg: th.Tensor, w_on: th.Tensor, w_tg: th.Tensor, bias_on: th.Tensor, bias_tg: th.Tensor, wset, reward,
                      done, gamma: float, B: int, W: int, A: int, D: int, dot_mode: int = DOT_UNFUSED, row_order: int = ROWS_REFERENCE,
                      a_scale_on=None, a_scale_tg=None, w_scale_on=None, w_scale_tg=None, want_indices: bool = False, out=None, pref_out=None,
                      act_out=None, q_on_out=None, q_tg_out=None, reverse_tiles: bool = False):
    """Output layer of both Q-networks + envelope operator + Bellman line in ONE kernel (reference envelope.py:420-440, :298): the Q
    tensors never reach HBM.  a_on / a_tg: last hidden activation planes [2, B*W, K] (row b*W + j) of the online / target net on s';
    w_on / w_tg: output-layer weight planes [2, 32, K]; the rest as :func:`envelope_td`.  ``q_on_out`` / ``q_tg_out`` ([B*W, A*D] fp32)
    optionally receive the Q tiles (validation).  Returns (target [W*B, D], pref, act)."""
    fmt = fmt_of(a_on)
    if fmt_of(a_tg) != fmt or fmt_of(w_on) != fmt or fmt_of(w_tg) != fmt or not a_on.is_cuda:
        raise _lib.MorlB200Error("qhead_envelope_td: operands must be CUDA plane tensors of one format")
    _, M, K = a_on.shape
    if M != B * W or tuple(a_tg.shape) != tuple(a_on.shape) or a_on.stride(1) != K or a_tg.stride(1) != K or a_tg.stride(0) != a_on.stride(0):
        raise _lib.MorlB200Error(f"qhead_envelope_td: activation planes must both be [P, {B * W}, K], K-major, equal plane strides")
    if tuple(w_on.shape) != tuple(w_tg.shape) or w_on.shape[1] != 32 or w_on.shape[2] != K or w_on.stride(1) != K or w_tg.stride(0) != w_on.stride(0):
        raise _lib.MorlB200Error(f"qhead_envelope_td: weight planes must both be [P, 32, {K}], K-major")
    wset, reward, done = _dev(wset, "wset"), _dev(reward, "reward"), _dev(done, "done")
    if wset.shape != (W, D) or reward.shape != (B, D) or done.numel() != B or bias_on.numel() != A * D or bias_tg.numel() != A * D:
        raise _lib.MorlB200Error(f"bad shapes: wset {tuple(wset.shape)}, reward {tuple(reward.shape)}, done {tuple(done.shape)}, bias {tuple(bias_on.shape)}")
    dev = a_on.device
    if out is None:
        out = th.empty((W * B, D), device=dev, dtype=th.float32)
    if want_indices:
        pref_out = th.empty(W * B, device=dev, dtype=th.int32) if pref_out is None else pref_out
        act_out = th.empty(W * B, device=dev, dtype=th.int32) if act_out is None else act_out
    rc = _lib.load().morl_qhead_envelope_td_f32(fmt, _ptr(a_on), _ptr(a_tg), a_on.stride(0), _ptr(a_scale_on), _ptr(a_scale_tg), _ptr(w_on), _ptr(w_tg),
                                                w_on.stride(0), _ptr(w_scale_on), _ptr(w_scale_tg), _ptr(bias_on), _ptr(bias_tg), K, _ptr(wset),
                                                _ptr(reward), _ptr(done), float(gamma), B, W, A, D, dot_mode, row_order, int(reverse_tiles), _ptr(out),
                                                _ptr(pref_out), _ptr(act_out), _ptr(q_on_out), _ptr(q_tg_out), _stream())
    _lib.check(rc, "morl_qhead_envelope_td_f32")
    _count()
    return out, pref_out, act_out


def gemm_chain_supported(fmt: int, M: int, K: int) -> bool:
    return bool(_lib.load().morl_gemm_chain_supported(int(fmt), int(M), int(K)))


class GemmChain:
    """Static plan of a chained launch (:func:`gemm_chain`): the pointer tables are built once, a call is one launch.
    ``acts[c]``: the n_layers + 1 plane tensors [P, M, 256] of chain c (input, then every layer's output); ``weights[c]`` / ``w_scales[c]`` /
    ``biases[c]`` / ``bits[c]`` (ReLU masks recorded) / ``bits_in[c]`` (ReLU-backward masks applied): per layer, all optional.  ``relu``: ReLU on every
    output (forward chains); False for the dX chains of the backward pass."""

    def __init__(self, acts, weights, biases=None, w_scales=None, bits=None, act_scale=None, relu: bool = True, bits_in=None, k_first: int = 0):
        import ctypes as C

        self.n_chains, self.n_layers = len(acts), len(weights[0])
        a0 = acts[0][1]  # (the first OUTPUT: the chain's input may be narrower, see k_first)
        self.fmt = fmt_of(a0)
        _, self.M, self.K = a0.shape  # (square layers: the output width of every layer is also the reduction length)
        self.N = a0.shape[2]  # output width of every layer: the width of its ReLU bit masks
        self.k_first = int(k_first) if k_first else self.K
        flat_a = [t for ch in acts for t in ch]
        flat_w = [t for ch in weights for t in ch]
        flat_b = [None] * len(flat_w) if biases is None else [t.detach() for ch in biases for t in ch]
        flat_i = [None] * len(flat_w) if bits_in is None else [t for ch in bits_in for t in ch]
        flat_s = [None] * len(flat_w) if w_scales is None else [t for ch in w_scales for t in ch]
        flat_m = [None] * len(flat_w) if bits is None else [t for ch in bits for t in ch]
        if len(flat_a) != self.n_chains * (self.n_layers + 1) or any(len(w) != self.n_layers for w in weights):
            raise _lib.MorlB200Error("GemmChain: every chain needs n_layers + 1 activation tensors and n_layers weight tensors")
        for i, t in enumerate(flat_a):
            kk = self.k_first if i % (self.n_layers + 1) == 0 else self.K
            if fmt_of(t) != self.fmt or tuple(t.shape[1:]) != (self.M, kk) or not t.is_contiguous() or not t.is_cuda:
                raise _lib.MorlB200Error(f"GemmChain: activation planes must be contiguous CUDA plane tensors [P, {self.M}, {kk}] (input {self.k_first} wide, outputs 256)")
        for i, t in enumerate(flat_w):
            kk = self.k_first if i % self.n_layers == 0 else self.K
            if fmt_of(t) != self.fmt or tuple(t.shape[1:]) != (256, kk) or not t.is_contiguous():
                raise _lib.MorlB200Error(f"GemmChain: weight planes must be contiguous [P, 256, {kk}]")
        for t in flat_m + flat_i:
            if t is not None and (t.dtype != th.int32 or tuple(t.shape) != (self.M, relu_bits_words(self.N)) or not t.is_contiguous()):
                raise _lib.MorlB200Error(f"GemmChain: ReLU bit masks must be contiguous int32 [{self.M}, {relu_bits_words(self.N)}]")
        self._keep = (flat_a, flat_w, flat_b, flat_s, flat_m, flat_i, act_scale)
        self.relu = bool(relu)
        arr = lambda ts: (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])  # noqa: E731
        self._pa, self._pw, self._pb, self._ps, self._pm, self._pi = arr(flat_a), arr(flat_w), arr(flat_b), arr(flat_s), arr(flat_m), arr(flat_i)
        self._a_stride, self._w_stride, self._act_scale = a0.stride(0), 256 * self.K, act_scale

    def __call__(self):
        rc = _lib.load().morl_gemm_chain_f32(self.fmt, self.n_chains, self.n_layers, self._pa, self._a_stride, _ptr(self._act_scale), self._pw, self._w_stride,
                                             self._ps, self._pb, int(self.relu), self._pi, self._pm, self.M, self.K, self.k_first, _stream())
        _lib.check(rc, "morl_gemm_chain_f32")
        _count()


class GemmChainPairs:
    """Static plan of a chained launch that starts from the separable first layer (f16x2): the input of chain c is
    relu(u[c][b] + v[c][j]) * act_scale for row b*W + j, built in shared memory (the planes :func:`pairs_relu_split` would write), then the
    hidden layers as :class:`GemmChain`.  ``outs[c]``: per layer, the output plane tensor [P, B*W, 256], or None when that output is not
    needed -- only the others are written to memory; ``weights`` / ``biases`` / ``w_scales`` / ``bits`` as :class:`GemmChain`.  A call takes
    the per-chain u [B, 256] and v [W, 256] (fp32, contiguous) of that pass."""

    def __init__(self, outs, weights, B: int, W: int, biases=None, w_scales=None, bits=None, act_scale=None):
        import ctypes as C

        self.n_chains, self.n_layers = len(outs), len(weights[0])
        self.B, self.W, self.M = int(B), int(W), int(B) * int(W)
        flat_o = [t for ch in outs for t in ch]
        flat_w = [t for ch in weights for t in ch]
        flat_b = [None] * len(flat_w) if biases is None else [t.detach() for ch in biases for t in ch]
        flat_s = [None] * len(flat_w) if w_scales is None else [t for ch in w_scales for t in ch]
        flat_m = [None] * len(flat_w) if bits is None else [t for ch in bits for t in ch]
        if len(flat_o) != len(flat_w) or any(len(w) != self.n_layers for w in weights) or any(len(o) != self.n_layers for o in outs):
            raise _lib.MorlB200Error("GemmChainPairs: every chain needs n_layers outputs (or None) and n_layers weight tensors")
        for t in flat_w:
            if fmt_of(t) != FMT_F16X2 or tuple(t.shape[1:]) != (256, 256) or not t.is_contiguous():
                raise _lib.MorlB200Error("GemmChainPairs: weight planes must be contiguous f16x2 [2, 256, 256]")
        stored = [t for t in flat_o if t is not None]
        for t in stored:
            if fmt_of(t) != FMT_F16X2 or tuple(t.shape[1:]) != (self.M, 256) or not t.is_contiguous() or not t.is_cuda:
                raise _lib.MorlB200Error(f"GemmChainPairs: output planes must be contiguous CUDA f16x2 tensors [2, {self.M}, 256]")
        if any(t.stride(0) != stored[0].stride(0) for t in stored):
            raise _lib.MorlB200Error("GemmChainPairs: output planes need one plane stride")
        for t in flat_m:
            if t is not None and (t.dtype != th.int32 or tuple(t.shape) != (self.M, relu_bits_words(256)) or not t.is_contiguous()):
                raise _lib.MorlB200Error(f"GemmChainPairs: ReLU bit masks must be contiguous int32 [{self.M}, {relu_bits_words(256)}]")
        self.store = sum(1 << i for i, t in enumerate(flat_o) if t is not None)
        self._keep = (flat_o, flat_w, flat_b, flat_s, flat_m, act_scale)
        arr = lambda ts: (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])  # noqa: E731
        self._po, self._pw, self._pb, self._ps, self._pm = arr(flat_o), arr(flat_w), arr(flat_b), arr(flat_s), arr(flat_m)
        self._o_stride = stored[0].stride(0) if stored else 0
        self._w_stride, self._act_scale = flat_w[0].stride(0), act_scale

    def __call__(self, us, vs):
        import ctypes as C

        if len(us) != self.n_chains or len(vs) != self.n_chains:
            raise _lib.MorlB200Error(f"GemmChainPairs: need u and v of {self.n_chains} chains")
        for u, v in zip(us, vs):
            if (u.dtype != th.float32 or v.dtype != th.float32 or tuple(u.shape) != (self.B, 256) or tuple(v.shape) != (self.W, 256)
                    or not u.is_contiguous() or not v.is_contiguous() or not u.is_cuda or not v.is_cuda):
                raise _lib.MorlB200Error(f"GemmChainPairs: u / v must be contiguous CUDA float32 [{self.B}, 256] / [{self.W}, 256]")
        pu = (C.c_void_p * self.n_chains)(*[u.data_ptr() for u in us])
        pv = (C.c_void_p * self.n_chains)(*[v.data_ptr() for v in vs])
        rc = _lib.load().morl_gemm_chain_pairs_f32(self.n_chains, self.n_layers, pu, pv, self.B, self.W, self._po, self._o_stride, _ptr(self._act_scale),
                                                   self._pw, self._w_stride, self._ps, self._pb, self._pm, self.store, _stream())
        _lib.check(rc, "morl_gemm_chain_pairs_f32")
        _count()


def qhead_gemm_supported(fmt: int, M: int, N: int, K: int) -> bool:
    return bool(_lib.load().morl_qhead_gemm_supported(int(fmt), int(M), int(N), int(K)))


def qhead_gemm(a_planes: th.Tensor, w_planes: th.Tensor, n_out: int, bias: th.Tensor, out: Optional[th.Tensor] = None, a_scale=None, w_scale=None,
               reverse_tiles: bool = False) -> th.Tensor:
    """Output layer Q = A . W^T + bias (n_out <= 32) as fp32 [M, n_out]: the narrow form of :func:`gemm_planes` (bit-identical) with the weight
    planes resident in shared memory (csrc/qhead_envelope.cu without its operator half)."""
    fmt = fmt_of(a_planes)
    _, M, K = a_planes.shape
    if fmt_of(w_planes) != fmt or tuple(w_planes.shape[1:]) != (32, K) or a_planes.stride(1) != K or w_planes.stride(1) != K:
        raise _lib.MorlB200Error(f"qhead_gemm: need K-major planes A [P, M, K] and W [P, 32, K] of one format (got {tuple(a_planes.shape)}, {tuple(w_planes.shape)})")
    if out is None:
        out = th.empty((M, n_out), device=a_planes.device, dtype=th.float32)
    rc = _lib.load().morl_qhead_gemm_f32(fmt, _ptr(a_planes), a_planes.stride(0), _ptr(a_scale), _ptr(w_planes), w_planes.stride(0), _ptr(w_scale), _ptr(bias), M,
                                         n_out, K, int(reverse_tiles), _ptr(out), _stream())
    _lib.check(rc, "morl_qhead_gemm_f32")
    _count()
    return out


def relu_bits_words(width: int) -> int:
    """int32 words per row of the ReLU bit mask of an activation ``width`` columns wide: 8 up to 256 columns, 16 up to 512."""
    return 16 if width > 256 else 8


def relu_bits_word(chunk):
    """Word of a bit-mask row holding columns [32 chunk, 32 chunk + 32) (int or integer tensor): within each 256-column half
    (chunk & 1) * 4 + ((chunk >> 1) & 3), the second half's eight words after the first's (include/morl_b200.h)."""
    return 8 * (chunk >> 3) + (chunk & 1) * 4 + ((chunk >> 1) & 3)


def empty_relu_bits(rows: int, device, width: int = 256) -> th.Tensor:
    """ReLU bit-mask tensor [rows, relu_bits_words(width)] int32 (layout: include/morl_b200.h, morl_gemm_planes_f32)."""
    return th.empty((rows, relu_bits_words(width)), device=device, dtype=th.int32)


def unpack_relu_bits(bits: th.Tensor, n_cols: int) -> th.Tensor:
    """[rows, n_cols] bool from a ReLU bit-mask tensor (tests / diagnostics)."""
    c = th.arange((n_cols + 31) // 32, device=bits.device)
    words = bits[:, relu_bits_word(c)].to(th.int64) & 0xFFFFFFFF  # [rows, chunks]
    j = th.arange(32, device=bits.device)
    return (((words[:, :, None] >> j) & 1) != 0).reshape(bits.shape[0], -1)[:, :n_cols]


def pairs_relu_split(u: th.Tensor, v: th.Tensor, out: Optional[th.Tensor] = None, fmt: int = FMT_F16X2, scale: Optional[th.Tensor] = None,
                     relu_bits_out: Optional[th.Tensor] = None) -> th.Tensor:
    """relu(u[b] + v[j]) for every pair, written as planes [P, B*W, H] of scale * h (row b*W + j); ``relu_bits_out``
    ([B*W, relu_bits_words(H)] int32) additionally receives [h > 0] as bits (the ReLU-backward mask of :func:`gemm_planes`)."""
    u, v = _dev(u, "u"), _dev(v, "v")
    B, H = u.shape
    W = v.shape[0]
    if out is None:
        out = empty_planes(fmt, B * W, H, u.device)
    else:
        fmt = fmt_of(out)
    if relu_bits_out is not None and (relu_bits_out.dtype != th.int32 or tuple(relu_bits_out.shape) != (B * W, relu_bits_words(H))
                                      or not relu_bits_out.is_contiguous()):
        raise _lib.MorlB200Error(f"pairs_relu_split: ReLU bit masks must be contiguous int32 [{B * W}, {relu_bits_words(H)}]")
    rc = _lib.load().morl_pairs_relu_split_planes(fmt, _ptr(u), _ptr(v), B, W, H, _ptr(out), out.stride(0), _ptr(scale), _ptr(relu_bits_out), _stream())
    _lib.check(rc, "morl_pairs_relu_split_planes")
    _count()
    return out


def pairs_product_split(u: th.Tensor, v: th.Tensor, out: Optional[th.Tensor] = None, fmt: int = FMT_F16X2, scale: Optional[th.Tensor] = None) -> th.Tensor:
    """u[b] * v[p] for every pair (one fp32 multiply), written as planes [P_fmt, B*P, H] of scale * h (row b*P + p): the product-conditioned
    first layer of GPI-PD's Q-network."""
    u, v = _dev(u, "u"), _dev(v, "v")
    B, H = u.shape
    P = v.shape[0]
    if v.shape[1] != H or H % 8:
        raise _lib.MorlB200Error(f"pairs_product_split: u {tuple(u.shape)} and v {tuple(v.shape)} need equal widths, a multiple of 8")
    if out is None:
        out = empty_planes(fmt, B * P, H, u.device)
    else:
        fmt = fmt_of(out)
        if out.shape[1] < B * P or out.shape[2] != H or out.stride(1) != H:
            raise _lib.MorlB200Error(f"pairs_product_split: out must be planes [P, >= {B * P}, {H}] with rows of {H}")
    rc = _lib.load().morl_pairs_product_split_planes(fmt, _ptr(u), _ptr(v), B, P, H, _ptr(out), out.stride(0), _ptr(scale), _stream())
    _lib.check(rc, "morl_pairs_product_split_planes")
    _count()
    return out


def product_layer1_uv(s: th.Tensor, s_weight: th.Tensor, s_bias: th.Tensor, m: th.Tensor, w_weight: th.Tensor, w_bias: th.Tensor,
                      u: Optional[th.Tensor] = None, v: Optional[th.Tensor] = None):
    """u = relu(s @ Ls^T + bs) [B, H] and v = relu(m @ Lw^T + bw) [P, H] in one launch (the two feature maps of GPI-PD's Q-network)."""
    s, m = _dev(s, "s"), _dev(m, "m")
    s_weight, s_bias, w_weight, w_bias = _dev(s_weight.detach(), "s_weight"), _dev(s_bias.detach(), "s_bias"), _dev(w_weight.detach(), "w_weight"), _dev(w_bias.detach(), "w_bias")
    B, F = s.shape
    P, D = m.shape
    H = s_weight.shape[0]
    if s_weight.shape[1] != F or tuple(w_weight.shape) != (H, D) or s_bias.numel() != H or w_bias.numel() != H:
        raise _lib.MorlB200Error(f"product_layer1_uv: weights {tuple(s_weight.shape)} / {tuple(w_weight.shape)} do not match s {tuple(s.shape)}, m {tuple(m.shape)}")
    u = th.empty((B, H), device=s.device, dtype=th.float32) if u is None else u
    v = th.empty((P, H), device=s.device, dtype=th.float32) if v is None else v
    rc = _lib.load().morl_product_layer1_uv_f32(_ptr(s), _ptr(s_weight), _ptr(s_bias), B, F, _ptr(m), _ptr(w_weight), _ptr(w_bias), P, D, H, _ptr(u),
                                                _ptr(v), _stream())
    _lib.check(rc, "morl_product_layer1_uv_f32")
    _count()
    return u, v


def pair_layer1_uv(feats: th.Tensor, wset: th.Tensor, weight: th.Tensor, bias: th.Tensor, u: Optional[th.Tensor] = None,
                   v: Optional[th.Tensor] = None):
    """u = feats @ W1[:, :F]^T [B, H] and v = wset @ W1[:, F:]^T + b1 [W, H] in one launch (separable first layer of the pair batch)."""
    feats, wset, weight, bias = _dev(feats, "feats"), _dev(wset, "wset"), _dev(weight, "weight"), _dev(bias, "bias")
    B, F = feats.shape
    W, D = wset.shape
    H = weight.shape[0]
    if weight.shape[1] != F + D or bias.numel() != H:
        raise _lib.MorlB200Error(f"pair_layer1_uv: weight {tuple(weight.shape)} does not match F={F}, D={D}")
    u = th.empty((B, H), device=feats.device, dtype=th.float32) if u is None else u
    v = th.empty((W, H), device=feats.device, dtype=th.float32) if v is None else v
    rc = _lib.load().morl_pair_layer1_uv_f32(_ptr(feats), _ptr(wset), _ptr(weight), _ptr(bias), B, W, F, D, H, _ptr(u), _ptr(v), _stream())
    _lib.check(rc, "morl_pair_layer1_uv_f32")
    _count()
    return u, v


def pair_layer1_grad_workspace(F: int, D: int, H: int, device) -> th.Tensor:
    nbytes = _lib.load().morl_pair_layer1_grad_workspace_bytes(int(F), int(D), int(H))
    return th.zeros((nbytes + 3) // 4, device=device, dtype=th.float32)  # arrival counters start at zero (self-resetting afterwards)


def pair_layer1_grad(dU: th.Tensor, dV: th.Tensor, feats: th.Tensor, wset: th.Tensor, dW1: Optional[th.Tensor] = None, db1: Optional[th.Tensor] = None,
                     workspace: Optional[th.Tensor] = None):
    """dW1 [H, F + D] = [dU^T feats | dV^T wset] and db1 [H] = colsum(dV) in one launch (backward of the separable first layer)."""
    dU, dV, feats, wset = _dev(dU, "dU"), _dev(dV, "dV"), _dev(feats, "feats"), _dev(wset, "wset")
    B, H = dU.shape
    W, D = wset.shape
    F = feats.shape[1]
    if dV.shape != (W, H) or feats.shape[0] != B:
        raise _lib.MorlB200Error(f"pair_layer1_grad: dU {tuple(dU.shape)}, dV {tuple(dV.shape)}, feats {tuple(feats.shape)}, wset {tuple(wset.shape)} disagree")
    dW1 = th.empty((H, F + D), device=dU.device, dtype=th.float32) if dW1 is None else dW1
    db1 = th.empty(H, device=dU.device, dtype=th.float32) if db1 is None else db1
    ws = pair_layer1_grad_workspace(F, D, H, dU.device) if workspace is None else workspace
    rc = _lib.load().morl_pair_layer1_grad_f32(_ptr(dU), _ptr(dV), _ptr(feats), _ptr(wset), B, W, F, D, H, _ptr(dW1), _ptr(db1), _ptr(ws), _stream())
    _lib.check(rc, "morl_pair_layer1_grad_f32")
    _count()
    return dW1, db1


def gemm_mn_workspace_bytes(M: int, g_cols: int, h_cols: int) -> int:
    return int(_lib.load().morl_gemm_mn_workspace_bytes(int(M), int(g_cols), int(h_cols)))


def gemm_mn_workspace(M: int, g_cols: int, h_cols: int, device) -> th.Tensor:
    nbytes = gemm_mn_workspace_bytes(M, g_cols, h_cols)
    return th.empty((nbytes + 3) // 4, device=device, dtype=th.float32)


def gemm_planes_mn(g_planes: th.Tensor, g_cols: int, h_planes: th.Tensor, h_cols: int, transpose_out: bool = False,
                   out: Optional[th.Tensor] = None, workspace: Optional[th.Tensor] = None, colsum: Optional[th.Tensor] = None,
                   g_scale: Optional[th.Tensor] = None, h_scale: Optional[th.Tensor] = None) -> th.Tensor:
    """out[n, k] = sum_m G[m, n] H[m, k] (weight gradient; reduction over the rows) from plane tensors [P, M, ld] (scales removed).
    ``colsum`` ([g_cols] fp32, optional) additionally receives sum_m G[m, n] (the bias gradient) from the same pass."""
    fmt = fmt_of(g_planes)
    _, M, ldg = g_planes.shape
    _, M2, ldh = h_planes.shape
    if M != M2 or fmt_of(h_planes) != fmt:
        raise _lib.MorlB200Error("gemm_planes_mn: plane tensors must share format and number of rows")
    dev = g_planes.device
    if out is None:
        out = th.empty((h_cols, g_cols) if transpose_out else (g_cols, h_cols), device=dev, dtype=th.float32)
    ws = gemm_mn_workspace(M, g_cols, h_cols, dev) if workspace is None else workspace
    rc = _lib.load().morl_gemm_planes_mn_f32(fmt, _ptr(g_planes), g_planes.stride(0), ldg, g_cols, _ptr(g_scale), _ptr(h_planes), h_planes.stride(0), ldh,
                                             h_cols, _ptr(h_scale), M, int(transpose_out), _ptr(out), out.stride(0), _ptr(colsum), _ptr(ws), _stream())
    _lib.check(rc, "morl_gemm_planes_mn_f32")
    _count(2)
    return out


def colsum_planes(planes: th.Tensor, n_cols: int, out: Optional[th.Tensor] = None, workspace: Optional[th.Tensor] = None,
                  scale: Optional[th.Tensor] = None) -> th.Tensor:
    """Column sums over the rows and the planes, scale removed (bias gradients)."""
    fmt = fmt_of(planes)
    _, M, ld = planes.shape
    dev = planes.device
    out = th.empty(n_cols, device=dev, dtype=th.float32) if out is None else out
    ws = th.empty(296 * n_cols, device=dev, dtype=th.float32) if workspace is None else workspace
    rc = _lib.load().morl_colsum_planes(fmt, _ptr(planes), planes.stride(0), _ptr(scale), M, ld, n_cols, _ptr(out), _ptr(ws), _stream())
    _lib.check(rc, "morl_colsum_planes")
    _count(2)
    return out


def pairs_grad_reduce(planes: th.Tensor, B: int, W: int, workspace: Optional[th.Tensor] = None, dU: Optional[th.Tensor] = None,
                      dV: Optional[th.Tensor] = None, scale: Optional[th.Tensor] = None):
    """dU [B, H] and dV [W, H] from the planes of dL/dh1 [P, B*W, H] (gradient of relu(u[b] + v[j]) w.r.t. u and v), scale removed."""
    fmt = fmt_of(planes)
    _, M, H = planes.shape
    dev = planes.device
    dU = th.empty((B, H), device=dev, dtype=th.float32) if dU is None else dU
    dV = th.empty((W, H), device=dev, dtype=th.float32) if dV is None else dV
    ws = th.empty(296 * W * H, device=dev, dtype=th.float32) if workspace is None else workspace
    rc = _lib.load().morl_pairs_grad_reduce_planes(fmt, _ptr(planes), planes.stride(0), _ptr(scale), B, W, H, _ptr(dU), _ptr(dV), _ptr(ws), _stream())
    _lib.check(rc, "morl_pairs_grad_reduce_planes")
    _count(2)
    return dU, dV


# ---- PCN / LCN (csrc/pcn.cu) ---------------------------------------------------------------------------------------------------------
def pcn_supported(obs_dim: int, d: int, hidden: int, n_out: int, batch: int = 1) -> bool:
    """Whether the fused PCN kernels cover this model and batch: 1 <= obs_dim <= 256, 1 <= d <= 8, hidden in {32, 64, 128, 256},
    1 <= n_out <= 32, 1 <= batch <= 4096 (include/morl_b200.h)."""
    return bool(_lib.load().morl_pcn_supported(int(obs_dim), int(d), int(hidden), int(n_out), int(batch)))


def pcn_workspace(obs_dim: int, d: int, hidden: int, n_out: int, batch: int, device) -> th.Tensor:
    nbytes = int(_lib.load().morl_pcn_workspace_bytes(int(obs_dim), int(d), int(hidden), int(n_out), int(batch)))
    if nbytes == 0:
        raise _lib.MorlB200Error(f"pcn_workspace: unsupported configuration obs_dim={obs_dim} d={d} hidden={hidden} n_out={n_out} batch={batch}")
    return th.empty((nbytes + 7) // 8, device=device, dtype=th.float64)


def pcn_pointer_table(tensors) -> "ctypes.Array":
    """Host array of the 8 device pointers (Ls, bs, Lc, bc, W1, b1, W2, b2) the PCN kernels take; build it once per set of storages."""
    import ctypes

    ts = list(tensors)
    if len(ts) != 8:
        raise _lib.MorlB200Error(f"PCN kernels take 8 parameter tensors, got {len(ts)}")
    for i, t in enumerate(ts):
        _dev(t, f"pcn tensor {i}")
        if not t.is_contiguous():
            raise _lib.MorlB200Error(f"pcn tensor {i} must be contiguous")
    return (ctypes.c_void_p * 8)(*[t.data_ptr() for t in ts])


def pcn_update(params, grads, scaling: th.Tensor, store: th.Tensor, obs_dim: int, d: int, rows: th.Tensor, horizons: th.Tensor, batch: int,
               hidden: int, n_out: int, continuous: bool, loss_out: th.Tensor, entropy_out: Optional[th.Tensor], pred_out: Optional[th.Tensor],
               workspace: th.Tensor):
    """One PCN minibatch (reference pcn.py:202-236): gather ``rows`` [batch] int32 of the episode store f32 [N, ld] (columns obs | return-to-go
    | action, a discrete action as int32 bits) with ``horizons`` [batch] int32, forward, loss, backward.  ``params`` / ``grads``: pointer
    tables of ``pcn_pointer_table``; the gradients are overwritten.  ``loss_out`` / ``entropy_out`` / ``pred_out`` are device views written
    in place."""
    _dev(scaling, "scaling")
    _dev(store, "store")
    _dev(rows, "rows", th.int32)
    _dev(horizons, "horizons", th.int32)
    rc = _lib.load().morl_pcn_update_f32(params, grads, _ptr(scaling), _ptr(store), int(store.shape[1]), _ptr(rows), _ptr(horizons), int(batch),
                                         int(obs_dim), int(d), int(hidden), int(n_out), int(bool(continuous)), _ptr(loss_out), _ptr(entropy_out),
                                         _ptr(pred_out), _ptr(workspace), _stream())
    _lib.check(rc, "morl_pcn_update_f32")
    _count(2)


def _dev_or_pinned(t: th.Tensor, name: str, dtype=th.float32) -> th.Tensor:
    if not isinstance(t, th.Tensor) or not (t.is_cuda or t.is_pinned()) or t.dtype != dtype or not t.is_contiguous():
        raise _lib.MorlB200Error(f"{name} must be a contiguous {dtype} CUDA or pinned host tensor")
    return t


def pcn_forward(params, scaling: th.Tensor, obs: th.Tensor, ret: th.Tensor, hor: th.Tensor, hidden: int, log_softmax: bool, out: th.Tensor,
                argmax_out: Optional[th.Tensor] = None):
    """The PCN model on N rows with their own commands (reference pcn.py:309-322 on one row): obs [N, S], ret [N, d], hor [N] ->
    ``out`` [N, A] (log-probabilities or predictions), optionally the first-occurrence argmax into ``argmax_out`` int32 [N].  The row
    tensors and outputs may be CUDA tensors or pinned host tensors (the kernel reads and writes pinned memory directly); with pinned
    outputs the caller synchronises the stream before reading them."""
    _dev(scaling, "scaling")
    for t, n in ((obs, "obs"), (ret, "ret"), (hor, "hor"), (out, "out")):
        _dev_or_pinned(t, n)
    if argmax_out is not None:
        _dev_or_pinned(argmax_out, "argmax_out", th.int32)
    N, S = obs.shape
    rc = _lib.load().morl_pcn_forward_f32(params, _ptr(scaling), _ptr(obs), _ptr(ret), _ptr(hor), int(N), int(S), int(ret.shape[1]), int(hidden),
                                          int(out.shape[1]), int(bool(log_softmax)), _ptr(out), _ptr(argmax_out), _stream())
    _lib.check(rc, "morl_pcn_forward_f32")
    _count()


# ---- EUPG (csrc/eupg.cu) -------------------------------------------------------------------------------------------------------------
def _int_array(values):
    import ctypes

    vals = [int(x) for x in values]
    return (ctypes.c_int * max(1, len(vals)))(*vals), len(vals)


def eupg_supported(obs_dim: int, d: int, hidden, n_out: int) -> bool:
    """Whether the fused EUPG kernels cover this policy network: 1 <= obs_dim, 1 <= d <= 8, obs_dim + d <= 256, 1 to 4 hidden layers of
    widths 1 to 256, 1 <= n_out <= 32 (include/morl_b200.h).  Needs no device."""
    arr, n = _int_array(hidden)
    return bool(_lib.load().morl_eupg_supported(int(obs_dim), int(d), arr, n, int(n_out)))


class EupgNet:
    """What the EUPG kernels need about one network: its shape and the host pointer tables of its parameters and gradients.  Build it
    once per set of storages (the tables hold raw device pointers)."""

    def __init__(self, obs_dim: int, d: int, hidden, n_out: int, params, grads=None):
        self.obs_dim, self.d, self.n_out = int(obs_dim), int(d), int(n_out)
        self.hidden, self.n_hidden = _int_array(hidden)
        if not _lib.load().morl_eupg_supported(self.obs_dim, self.d, self.hidden, self.n_hidden, self.n_out):
            raise _lib.MorlB200Error(f"EupgNet: unsupported configuration obs_dim={obs_dim} d={d} hidden={list(hidden)} n_out={n_out}")
        self.params = self._table(params, "param")
        self.grads = None if grads is None else self._table(grads, "grad")

    def _table(self, tensors, what):
        import ctypes

        ts = list(tensors)
        if len(ts) != 2 * (self.n_hidden + 1):
            raise _lib.MorlB200Error(f"EUPG kernels take {2 * (self.n_hidden + 1)} {what} tensors, got {len(ts)}")
        for i, t in enumerate(ts):
            _dev_view(t, f"eupg {what} {i}")
            if not t.is_contiguous():
                raise _lib.MorlB200Error(f"eupg {what} {i} must be contiguous")
        return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])

    @property
    def workspace_bytes(self) -> int:
        return int(_lib.load().morl_eupg_workspace_bytes(self.obs_dim, self.d, self.hidden, self.n_hidden, self.n_out))

    def workspace(self, device) -> th.Tensor:
        return th.empty((self.workspace_bytes + 7) // 8, device=device, dtype=th.float64)


def eupg_workspace_bytes(obs_dim: int, d: int, hidden, n_out: int) -> int:
    arr, n = _int_array(hidden)
    return int(_lib.load().morl_eupg_workspace_bytes(int(obs_dim), int(d), arr, n, int(n_out)))


def _dev_view(t: th.Tensor, name: str, dtype=th.float32) -> th.Tensor:
    """A CUDA tensor of ``dtype``, checked without copying: the EUPG kernels read strided views of one staging block in place."""
    if not isinstance(t, th.Tensor) or not t.is_cuda:
        raise _lib.MorlB200Error(f"{name} must be a CUDA tensor (morl_baselines_b200 has no CPU fallback)")
    if t.dtype != dtype:
        raise _lib.MorlB200Error(f"{name} must have dtype {dtype}, got {t.dtype}")
    return t


def _eupg_rows(t: th.Tensor, name: str, cols: int, dtype=th.float32) -> th.Tensor:
    """[T, cols] with contiguous columns and a non-negative row stride."""
    _dev_view(t, name, dtype)
    if t.dim() != 2 or t.shape[1] != cols or (cols > 1 and t.stride(1) != 1) or t.stride(0) < 0:
        raise _lib.MorlB200Error(f"{name} must be [T, {cols}] with contiguous columns, got shape {tuple(t.shape)} strides {t.stride()}")
    return t


def eupg_returns(rewards: th.Tensor, gamma: float, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Discounted forward returns of an episode's rewards [T, d] (rows may be strided, columns contiguous), bit-identical to the
    reference's float32 loop ``c = gamma * c + r_t`` run backward (eupg.py:263-270), for any number of objectives.  ``out``: a
    contiguous float32 [T, d] CUDA tensor, allocated when not given."""
    if not isinstance(rewards, th.Tensor) or rewards.dim() != 2:
        raise _lib.MorlB200Error("eupg_returns: rewards must be a [T, d] tensor")
    T, d = rewards.shape
    _eupg_rows(rewards, "rewards", d)
    if out is None:
        out = th.empty((T, d), device=rewards.device, dtype=th.float32)
    elif not (isinstance(out, th.Tensor) and out.is_cuda and out.dtype == th.float32 and tuple(out.shape) == (T, d) and out.is_contiguous()):
        raise _lib.MorlB200Error(f"eupg_returns: out must be a contiguous float32 CUDA tensor of shape {(T, d)}")
    rc = _lib.load().morl_eupg_returns_f32(_ptr(rewards), int(rewards.stride(0)), int(T), int(d), float(gamma), _ptr(out), _stream())
    _lib.check(rc, "morl_eupg_returns_f32")
    _count()
    return out


def eupg_update(net: EupgNet, obs: th.Tensor, acc: th.Tensor, actions: th.Tensor, v: th.Tensor, loss_out: th.Tensor, workspace: th.Tensor):
    """One EUPG episode update (reference eupg.py:236-251): rows ``obs`` int32 [T, S], ``acc`` f32 [T, d] and ``actions`` int32 [T] are
    views with one common row stride (columns of one staging block), read in place; ``v`` f32 [T] or one element (broadcast).  Writes
    the loss into ``loss_out`` [>= 1] and overwrites the gradients of ``net.grads``."""
    if net.grads is None:
        raise _lib.MorlB200Error("eupg_update: the EupgNet was built without gradient tensors")
    _eupg_rows(obs, "obs", net.obs_dim, th.int32)
    _eupg_rows(acc, "acc", net.d)
    _dev_view(actions, "actions", th.int32)
    _dev_view(v, "v")
    _dev_view(loss_out, "loss_out")
    _dev_view(workspace, "workspace", workspace.dtype)
    T = obs.shape[0]
    ld = obs.stride(0)
    if actions.dim() != 1 or acc.stride(0) != ld or actions.stride(0) != ld or acc.shape[0] != T or actions.shape[0] != T:
        raise _lib.MorlB200Error("eupg_update: obs, acc and actions must be rows of one block with a common row stride")
    if loss_out.numel() < 1 or not loss_out.is_contiguous():
        raise _lib.MorlB200Error("eupg_update: loss_out must be a contiguous float32 CUDA tensor with at least one element")
    if not workspace.is_contiguous() or workspace.numel() * workspace.element_size() < net.workspace_bytes:
        raise _lib.MorlB200Error(f"eupg_update: workspace must be contiguous and hold {net.workspace_bytes} bytes")
    if v.numel() == 1:
        v_stride = 0
    elif v.dim() == 1 and v.shape[0] == T and v.stride(0) >= 0:
        v_stride = int(v.stride(0))
    else:
        raise _lib.MorlB200Error(f"eupg_update: v must have T={T} elements or one, got shape {tuple(v.shape)}")
    rc = _lib.load().morl_eupg_update_f32(net.params, net.grads, _ptr(obs), _ptr(acc), _ptr(actions), int(ld), _ptr(v), v_stride, int(T),
                                          net.obs_dim, net.d, net.hidden, net.n_hidden, net.n_out, _ptr(loss_out), _ptr(workspace), _stream())
    _lib.check(rc, "morl_eupg_update_f32")
    _count(2)


def eupg_probs(net: EupgNet, x: th.Tensor, out: th.Tensor):
    """Action probabilities [N, A] of rows ``x`` [N, S + d] (reference eupg.py:46-61 after Categorical's renormalisation).  ``x`` and
    ``out`` may be contiguous CUDA tensors or pinned host tensors; with a pinned output the caller synchronises the stream before reading
    it."""
    _dev_or_pinned(x, "x")
    _dev_or_pinned(out, "out")
    N = x.shape[0] if x.dim() == 2 else 0
    if x.dim() != 2 or N < 1 or x.shape[1] != net.obs_dim + net.d:
        raise _lib.MorlB200Error(f"eupg_probs: x must be [N, {net.obs_dim + net.d}], got {tuple(x.shape)}")
    if tuple(out.shape) != (N, net.n_out):
        raise _lib.MorlB200Error(f"eupg_probs: out must be {(N, net.n_out)}, got {tuple(out.shape)}")
    rc = _lib.load().morl_eupg_probs_f32(net.params, _ptr(x), int(N), net.obs_dim, net.d, net.hidden, net.n_hidden, net.n_out, _ptr(out),
                                         _stream())
    _lib.check(rc, "morl_eupg_probs_f32")
    _count()
