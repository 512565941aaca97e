"""Thin PyTorch-facing wrappers over the C-ABI (include/morl_b200.h).

PyTorch is plumbing here: it owns the device buffers and the stream; every operator below is one (or two) launches of a
hand-written sm_90a kernel from libmorl_b200.so.  All wrappers require CUDA tensors and raise otherwise -- there is
no CPU / eager fallback (the CPU restatement lives in oracle/ and is test-only).

The kernels trust the pointers they are given, so every tensor a binding hands to the library passes one argument contract
(:class:`_Args`) before anything is launched, and every launch goes through :func:`_launch`.
"""

from __future__ import annotations

import ctypes
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


def _stream():
    return th.cuda.current_stream().cuda_stream


def _launch(entry: str, *args, launches: int = 1):
    """Call the library entry point ``entry`` with ``args`` (tensors become their device pointers) and the current stream, raise on a
    non-zero return code, and count the binding's ``launches`` kernels."""
    rc = getattr(_lib.load(), entry)(*[a.data_ptr() if isinstance(a, th.Tensor) else a for a in args], _stream())
    _lib.check(rc, entry)
    _count(launches)


def _pointer_table(tensors):
    """Host array of device pointers (None = NULL) for the entry points that take per-layer tables."""
    return (ctypes.c_void_p * max(1, len(tensors)))(*[None if t is None else t.data_ptr() for t in tensors])


def _param_table(a, tensors, what: str, count: int, holds: str, shapes=None):
    """Pointer table of the ``count`` parameter (or gradient) tensors of one network, each checked as an in-place input ``what[i]`` of
    ``shapes[i]`` (any shape when None); ``holds`` names them in the error for a wrong count."""
    ts = list(tensors)
    if len(ts) != count:
        a.fail(what, f"must hold the {count} {holds}, got {len(ts)}")
    return _pointer_table([a.inp(t, f"{what}[{i}]", None if shapes is None else shapes[i], inplace=True) for i, t in enumerate(ts)])


def _workspace(nbytes: int, device) -> th.Tensor:
    """A workspace of ``nbytes`` (the library's count) on ``device``, 8-byte aligned for the double partials the kernels keep in it."""
    return th.empty((nbytes + 7) // 8, device=device, dtype=th.float64)


class _Args:
    """The argument contract of one binding call.  Each check raises MorlB200Error naming the binding and the argument:

    - ``inp``: an input of the given dtype and shape (None = any extent) on the call's CUDA device; ``reshape`` views it first (checked by
      element count).  A non-contiguous input is copied to a contiguous one, unless ``inplace`` (the library keeps or writes through the
      pointer), which refuses it instead.  ``pinned`` also accepts a contiguous pinned host tensor, read in place.
    - ``out``: an output, allocated when None (and ``alloc``); when given, exactly that dtype, device and shape, contiguous (``ld``: rows
      may be padded, the library takes the row stride), written in place -- never copied, which would drop the result.
    - ``ws``: a workspace of at least ``nbytes`` (the library's count), contiguous; allocated (zeroed if ``zero``) when None.
    - ``scalar``: a device scalar with exactly one element (None passes when ``opt``).
    - ``planes``: a plane tensor [P, rows, ld] (:func:`fmt_of`) read or written in place: K-major rows, any plane stride of at least
      rows * ld (or a contiguous one).  Returns its format.

    All CUDA tensors of one call must be on one device."""

    def __init__(self, binding: str):
        self.binding, self.device = binding, None

    def fail(self, name: str, msg: str):
        raise _lib.MorlB200Error(f"{self.binding}: {name} {msg}")

    def _tensor(self, t, name, dtype, pinned=False):
        if not isinstance(t, th.Tensor) or not (t.is_cuda or (pinned and t.is_pinned())):
            self.fail(name, f"must be a CUDA{' or pinned host' if pinned else ''} tensor (morl_baselines_b200 has no CPU fallback)")
        if t.is_cuda:
            if self.device is None:
                self.device = t.device
            elif t.device != self.device:
                self.fail(name, f"is on {t.device}, the other arguments on {self.device}")
        if dtype is not None and t.dtype not in (dtype if isinstance(dtype, tuple) else (dtype,)):
            self.fail(name, f"must have dtype {dtype}, got {t.dtype}")

    def _shape(self, t, name, shape):
        if shape is not None and (t.dim() != len(shape) or any(s is not None and s != n for s, n in zip(shape, t.shape))):
            self.fail(name, f"must have shape {tuple('*' if s is None else s for s in shape)}, got {tuple(t.shape)}")

    def inp(self, t, name, shape=None, dtype=th.float32, reshape=None, inplace=False, pinned=False, opt=False):
        if t is None and opt:
            return None
        self._tensor(t, name, dtype, pinned)
        if not t.is_contiguous():
            if inplace or not t.is_cuda:
                self.fail(name, "must be contiguous")
            t = t.contiguous()
        if reshape is not None and t.shape != reshape:
            try:
                t = t.reshape(reshape)
            except RuntimeError:
                self.fail(name, f"has {t.numel()} elements, cannot be viewed as {tuple(reshape)}")
        self._shape(t, name, shape)
        return t

    def out(self, t, name, shape, dtype=th.float32, alloc=True, ld=False, pinned=False):
        if t is None:
            return th.empty(shape, device=self.device, dtype=dtype) if alloc else None
        self._tensor(t, name, dtype, pinned)
        self._shape(t, name, shape)
        if not (t.is_contiguous() or (ld and t.dim() == 2 and t.stride(1) == 1 and t.stride(0) >= t.shape[1])):
            self.fail(name, "must be contiguous" + (" (row stride >= columns, unit column stride)" if ld else ""))
        return t

    def ws(self, t, name, nbytes, zero=False):
        nbytes = int(nbytes)
        if t is None:
            return (th.zeros if zero else th.empty)((nbytes + 3) // 4, device=self.device, dtype=th.float32)
        self._tensor(t, name, None)
        if not t.is_contiguous() or t.numel() * t.element_size() < nbytes:
            self.fail(name, f"must be a contiguous CUDA tensor of at least {nbytes} bytes, got {t.numel() * t.element_size()}")
        return t

    def scalar(self, t, name, dtype=th.float32, opt=True):
        if t is None and opt:
            return None
        self._tensor(t, name, dtype)
        if t.numel() != 1:
            self.fail(name, f"must be a device scalar with one element, got shape {tuple(t.shape)}")
        return t

    def planes(self, t, name, fmt=None, rows=None, ld=None, contiguous=False) -> int:
        self._tensor(t, name, (th.bfloat16, th.float16))
        if t.dim() != 3 or t.shape[0] != (3 if t.dtype == th.bfloat16 else 2):
            self.fail(name, f"must be a plane tensor (bf16 [3, rows, ld] or fp16 [2, rows, ld]), got {t.dtype} {tuple(t.shape)}")
        f = fmt_of(t)
        if fmt is not None and f != fmt:
            self.fail(name, "must have the plane format of the other operands")
        self._shape(t, name, (None, rows, ld))
        if not (t.is_contiguous() if contiguous else t.stride(2) == 1 and t.stride(1) == t.shape[2] and t.stride(0) >= t.shape[1] * t.shape[2]):
            self.fail(name, "must be contiguous" if contiguous else f"must be K-major planes (row stride {t.shape[2]}), got strides {t.stride()}")
        return f


def envelope_td(q_online, q_target, wset, reward, done, gamma: float, dot_mode: int = DOT_UNFUSED, row_order: int = ROWS_REFERENCE,
                want_indices: bool = True, out: Optional[th.Tensor] = None, pref_out=None, act_out=None):
    """Fused envelope-max TD target (reference envelope.py:404-440 + :298).  q_*: [B, W, A, D]; returns
    (target [W*B, D], pref [W*B] int32, act [W*B] int32)."""
    a = _Args("envelope_td")
    q_online = a.inp(q_online, "q_online", (None,) * 4)
    B, W, A, D = q_online.shape
    q_target = a.inp(q_target, "q_target", (B, W, A, D))
    wset, reward, done = a.inp(wset, "wset", (W, D)), a.inp(reward, "reward", (B, D)), a.inp(done, "done", reshape=(B,))
    out = a.out(out, "out", (W * B, D))
    pref_out = a.out(pref_out, "pref_out", (W * B,), th.int32, alloc=want_indices)
    act_out = a.out(act_out, "act_out", (W * B,), th.int32, alloc=want_indices)
    _launch("morl_envelope_td_f32", q_online, q_target, wset, reward, done, float(gamma), B, W, A, D, dot_mode, row_order, out, pref_out, act_out)
    return out, pref_out, act_out


def _rewards(a, reward, done, D):
    """Optional reward rows [R, D] and done [R] of the greedy targets (R rows, tiled or blocked over the batch)."""
    if reward is None:
        return None, None
    reward = a.inp(reward, "reward", reshape=(-1, D))
    return reward, a.inp(done, "done", reshape=(reward.shape[0],))


def greedy_td(q_select, q_eval, w, reward=None, done=None, gamma: float = 0.0, dot_mode: int = DOT_UNFUSED, w_map: int = MAP_BLOCK,
              r_map: int = MAP_TILE):
    """Double-DQN target with per-row weights (reference envelope.py:442-463).  q_*: [N, A, D]."""
    a = _Args("greedy_td")
    q_select = a.inp(q_select, "q_select", (None,) * 3)
    N, A, D = q_select.shape
    q_eval, w = a.inp(q_eval, "q_eval", (N, A, D)), a.inp(w, "w", reshape=(-1, D))
    reward, done = _rewards(a, reward, done, D)
    out, act = a.out(None, "out", (N, D)), a.out(None, "act", (N,), th.int32)
    _launch("morl_greedy_td_f32", q_select, q_eval, w, w.shape[0], w_map, reward, done, N if reward is None else reward.shape[0], r_map, float(gamma), N,
            A, D, dot_mode, out, act)
    return out, act


def critic_min_td(q_nets, w, reward=None, done=None, gamma: float = 0.0, dot_mode: int = DOT_UNFUSED, w_map: int = MAP_BLOCK,
                  r_map: int = MAP_TILE):
    """GPI-PD critic-min greedy target (reference gpi_pd.py:445-463).  q_nets: [n_nets, N, A, D]."""
    a = _Args("critic_min_td")
    q_nets = a.inp(q_nets, "q_nets", (None,) * 4)
    n_nets, N, A, D = q_nets.shape
    w = a.inp(w, "w", reshape=(-1, D))
    reward, done = _rewards(a, reward, done, D)
    out, act = a.out(None, "out", (N, D)), a.out(None, "act", (N,), th.int32)
    _launch("morl_critic_min_td_f32", q_nets, n_nets, w, w.shape[0], w_map, reward, done, N if reward is None else reward.shape[0], r_map, float(gamma),
            N, A, D, dot_mode, out, act)
    return out, act


def gpi_envelope(q_nets, w, reward=None, done=None, gamma: float = 0.0, dot_mode: int = DOT_UNFUSED, w_map: int = MAP_BLOCK,
                 r_map: int = MAP_TILE):
    """GPI envelope / policy-set evaluation (reference gpi_pd.py:662-690, 564-582).  q_nets: [n_nets, B, P, A, D];
    returns (out [B, D], policy [B] int32, action [B] int32)."""
    a = _Args("gpi_envelope")
    q_nets = a.inp(q_nets, "q_nets", (None,) * 5)
    n_nets, B, P, A, D = q_nets.shape
    w = a.inp(w, "w", reshape=(-1, D))
    reward, done = _rewards(a, reward, done, D)
    out, pol, act = a.out(None, "out", (B, D)), a.out(None, "pol", (B,), th.int32), a.out(None, "act", (B,), th.int32)
    _launch("morl_gpi_envelope_f32", q_nets, n_nets, w, w.shape[0], w_map, reward, done, B if reward is None else reward.shape[0], r_map, float(gamma),
            B, P, A, D, dot_mode, out, pol, act)
    return out, pol, act


def actor_critic_td(q_nets, w, reward, done, logp, alpha: float, gamma: float, variant: int, w_map: int = MAP_BLOCK):
    """Continuous-action vector targets (CAPQL / MOSAC / TD3-style GPI-PD; SURVEY Appendix A.4).  q_nets: [n_nets, N, D]."""
    a = _Args("actor_critic_td")
    q_nets = a.inp(q_nets, "q_nets", (None,) * 3)
    n_nets, N, D = q_nets.shape
    reward, done = a.inp(reward, "reward", reshape=(N, D)), a.inp(done, "done", reshape=(N,))
    w, logp = a.inp(w, "w", reshape=(-1, D), opt=True), a.inp(logp, "logp", reshape=(N,), opt=True)
    out = a.out(None, "out", (N,) if variant == AC_SCALAR_MIN else (N, D))
    _launch("morl_actor_critic_td_f32", q_nets, n_nets, w, 0 if w is None else w.shape[0], w_map, reward, done, logp, float(alpha), float(gamma), N, D,
            variant, out)
    return out


def _discrete_sac_args(a, q_nets, logits, w, alpha):
    q_nets = a.inp(q_nets, "q_nets", (None,) * 4)
    n_nets, N, A, D = q_nets.shape
    logits, w = a.inp(logits, "logits", (N, A)), a.inp(w, "w", reshape=(-1, D))
    return q_nets, logits, w, a.scalar(alpha, "alpha", opt=False), (n_nets, N, A, D)


def discrete_sac_target(q_nets, logits, w, reward, done, alpha: th.Tensor, gamma: float, w_map: int = MAP_BLOCK, out: Optional[th.Tensor] = None):
    """Discrete-action MOSAC soft target (reference mosac_discrete_action.py:452-464): q_nets [n_nets, N, A, D] target critics at s',
    logits [N, A] actor at s', ``alpha`` a device scalar read at run time.  Returns target [N]."""
    a = _Args("discrete_sac_target")
    q_nets, logits, w, alpha, (n_nets, N, A, D) = _discrete_sac_args(a, q_nets, logits, w, alpha)
    reward, done = a.inp(reward, "reward", reshape=(N, D)), a.inp(done, "done", reshape=(N,))
    out = a.out(out, "out", (N,))
    _launch("morl_discrete_sac_target_f32", q_nets, n_nets, logits, w, w.shape[0], w_map, reward, done, alpha, float(gamma), N, A, D, out)
    return out


def discrete_sac_actor_loss(logits, q_nets, w, alpha: th.Tensor, log_alpha: Optional[th.Tensor] = None, target_entropy: float = 0.0,
                            w_map: int = MAP_BLOCK, want_grad: bool = True, workspace: Optional[th.Tensor] = None):
    """Discrete-action MOSAC actor loss, d loss / d logits and, with ``log_alpha``, the temperature loss and its derivative w.r.t.
    log_alpha (reference mosac_discrete_action.py:478-498).  Returns (actor_loss [1], dlogits [N, A] or None, alpha_loss [1] or None,
    dlog_alpha [1] or None)."""
    a = _Args("discrete_sac_actor_loss")
    q_nets, logits, w, alpha, (n_nets, N, A, D) = _discrete_sac_args(a, q_nets, logits, w, alpha)
    log_alpha = a.scalar(log_alpha, "log_alpha")
    loss, grad = a.out(None, "loss", (1,)), a.out(None, "grad", (N, A), alloc=want_grad)
    aloss, dla = a.out(None, "aloss", (1,), alloc=log_alpha is not None), a.out(None, "dla", (1,), alloc=log_alpha is not None)
    workspace = a.ws(workspace, "workspace", _lib.load().morl_discrete_sac_workspace_bytes(N))
    _launch("morl_discrete_sac_actor_loss_f32", logits, q_nets, n_nets, w, w.shape[0], w_map, alpha, log_alpha, float(target_entropy), N, A, D, loss, grad,
            aloss, dla, workspace, launches=2)
    return loss, grad, aloss, dla


def vector_gae(rewards, values, dones, next_value, next_done, weights, gamma: float, gae_lambda: float, gae: bool = True,
               returns_out: Optional[th.Tensor] = None, adv_out: Optional[th.Tensor] = None):
    """MO-PPO's reverse GAE recursion (reference mo_ppo.py:439-476) in one launch.  rewards / values [T, E, D], dones [T, E],
    next_value [E, D], next_done [E], weights [D]; ``gae=False`` gives the plain discounted returns.  Returns (returns [T, E, D],
    scalarised advantages [T, E]), written into ``returns_out`` / ``adv_out`` when given."""
    a = _Args("vector_gae")
    rewards = a.inp(rewards, "rewards", (None,) * 3)
    T, E, D = rewards.shape
    values, dones = a.inp(values, "values", (T, E, D)), a.inp(dones, "dones", (T, E))
    next_value, next_done = a.inp(next_value, "next_value", reshape=(E * D,)), a.inp(next_done, "next_done", reshape=(E,))
    weights = a.inp(weights, "weights", reshape=(D,))
    ret, adv = a.out(returns_out, "returns_out", (T, E, D)), a.out(adv_out, "adv_out", (T, E))
    _launch("morl_vector_gae_f32", rewards, values, dones, next_value, next_done, weights, T, E, D, float(gamma), float(gae_lambda), int(bool(gae)), ret, adv)
    return ret, adv


def ppo_loss(mean, logstd, value, actions, old_logprob, advantages, returns, old_values, clip_coef: float, ent_coef: float, vf_coef: float,
             norm_adv: bool, clip_vloss: bool, stats: th.Tensor, out: Optional[Tuple[th.Tensor, th.Tensor, th.Tensor, th.Tensor]] = None):
    """One minibatch's MO-PPO loss and its gradients (reference mo_ppo.py:514-549) in one launch.  mean [M, A], logstd [A] (or [1, A]),
    value [M, D], actions [M, A], old_logprob [M], advantages [M], returns / old_values [M, D]; ``stats`` a float32 device vector of 6
    (pg_loss, v_loss, entropy, old_approx_kl, approx_kl written; clip fraction added).  Returns (loss [1], dmean [M, A], dlogstd [A],
    dvalue [M, D]), written into ``out`` when given."""
    a = _Args("ppo_loss")
    mean = a.inp(mean, "mean", (None, None))
    M, A = mean.shape
    if not isinstance(value, th.Tensor) or value.dim() == 0:
        a.fail("value", "must be a [M, D] tensor")
    D = value.shape[-1]
    value, actions = a.inp(value, "value", reshape=(M, D)), a.inp(actions, "actions", (M, A))
    logstd, old_logprob = a.inp(logstd, "logstd", reshape=(A,)), a.inp(old_logprob, "old_logprob", reshape=(M,))
    advantages, returns = a.inp(advantages, "advantages", reshape=(M,)), a.inp(returns, "returns", reshape=(M, D))
    old_values = a.inp(old_values, "old_values", reshape=(M, D), opt=True)
    stats = a.out(stats, "stats", (6,))
    out = (None,) * 4 if out is None else tuple(out)
    loss, dmean, dlogstd, dvalue = (a.out(out[0], "out[0]", (1,)), a.out(out[1], "out[1]", (M, A)), a.out(out[2], "out[2]", (A,)),
                                    a.out(out[3], "out[3]", (M, D)))
    _launch("morl_ppo_loss_f32", mean, logstd, value, actions, old_logprob, advantages, returns, old_values, M, A, D, float(clip_coef), float(ent_coef),
            float(vf_coef), int(bool(norm_adv)), int(bool(clip_vloss)), loss, dmean, dlogstd, dvalue, stats)
    return loss, dmean, dlogstd, dvalue


def td_workspace(n_rows: int, device) -> th.Tensor:
    nbytes = _lib.load().morl_td_workspace_bytes(int(n_rows))
    return th.empty((nbytes + 3) // 4, device=device, dtype=th.float32)


def td_mse_priority(q_values, action, target_q, wset, homotopy_lambda: float, B: int, W: int, row_order: int = ROWS_REFERENCE,
                    want_grad: bool = True, want_prio: bool = True, workspace: Optional[th.Tensor] = None, loss_out=None, grad_out=None,
                    prio_out=None, q_taken_out=None, lambda_dev=None):
    """Fused Envelope TD loss + d loss / d q_values + priorities (reference envelope.py:301-313, 329-331).  ``lambda_dev`` (device f32 [1])
    overrides ``homotopy_lambda`` and is read by the kernels at run time (graph-replay safe)."""
    a = _Args("td_mse_priority")
    q_values = a.inp(q_values, "q_values", (B * W, None, None))
    N, A, D = q_values.shape
    action, target_q = a.inp(action, "action", dtype=th.int32, reshape=(B,)), a.inp(target_q, "target_q", (N, D))
    wset, lambda_dev = a.inp(wset, "wset", (W, D)), a.scalar(lambda_dev, "lambda_dev")
    loss, grad = a.out(loss_out, "loss_out", (1,)), a.out(grad_out if want_grad else None, "grad_out", (N, A, D), alloc=want_grad)
    prio = a.out(prio_out if want_prio else None, "prio_out", (B,), alloc=want_prio)
    q_taken_out = a.out(q_taken_out, "q_taken_out", (N, D), alloc=False)
    workspace = a.ws(workspace, "workspace", _lib.load().morl_td_workspace_bytes(N))
    _launch("morl_td_mse_priority_f32", q_values, action, target_q, wset, float(homotopy_lambda), lambda_dev, B, W, A, D, row_order, loss, grad,
            q_taken_out, prio, workspace, launches=2)
    return loss, grad, prio


def td_huber_priority(q_values, action, target_q, target_q_gpi, w, min_priority: float, p_rows: int, w_map: int = MAP_BLOCK,
                      want_grad: bool = True, workspace: Optional[th.Tensor] = None):
    """GPI-PD Huber-style loss, gradient seed and raw priorities (reference gpi_pd.py:469-487, 507-520)."""
    a = _Args("td_huber_priority")
    q_values = a.inp(q_values, "q_values", (None,) * 4)
    n_nets, N, A, D = q_values.shape
    action, target_q = a.inp(action, "action", dtype=th.int32, reshape=(-1,)), a.inp(target_q, "target_q", (N, D))
    target_q_gpi, w = a.inp(target_q_gpi, "target_q_gpi", (N, D), opt=True), a.inp(w, "w", reshape=(-1, D))
    loss, grad = a.out(None, "loss", (1,)), a.out(None, "grad", (n_nets, N, A, D), alloc=want_grad)
    prio = a.out(None, "prio", (p_rows,), alloc=p_rows > 0)
    workspace = a.ws(workspace, "workspace", _lib.load().morl_td_workspace_bytes(N))
    _launch("morl_td_huber_priority_f32", q_values, n_nets, action, action.shape[0], target_q, target_q_gpi, w, w.shape[0], w_map, float(min_priority), N,
            A, D, p_rows, loss, grad, prio, workspace, launches=2)
    return loss, grad, prio


def replay_gather(obs_store, next_obs_store, act_store, rew_store, done_store, idx, outs=None):
    """Gather a minibatch from device-resident stores (reference buffer.py:82-94).  Returns
    (obs, actions, rewards, next_obs, dones); uint8 actions come back as int32."""
    a = _Args("replay_gather")
    obs_store = a.inp(obs_store, "obs_store")
    if obs_store.dim() < 2:
        a.fail("obs_store", f"must be [capacity, ...], got shape {tuple(obs_store.shape)}")
    cap, obs_dim = obs_store.shape[0], obs_store[0].numel()
    next_obs_store = a.inp(next_obs_store, "next_obs_store", tuple(obs_store.shape))
    act_store = a.inp(act_store, "act_store", dtype=(th.uint8, th.float32))
    rew_store, done_store = a.inp(rew_store, "rew_store"), a.inp(done_store, "done_store", reshape=(cap,))
    for name, t in (("act_store", act_store), ("rew_store", rew_store)):
        if t.dim() < 1 or t.shape[0] != cap:
            a.fail(name, f"must have {cap} rows, got shape {tuple(t.shape)}")
    idx = a.inp(idx, "idx", dtype=th.int64, reshape=(-1,))
    is_u8 = act_store.dtype == th.uint8
    act_dim, rew_dim = act_store[0].numel(), rew_store[0].numel()
    B = idx.shape[0]
    outs = (None,) * 5 if outs is None else tuple(outs)
    obs, act = a.out(outs[0], "outs[0]", (B,) + tuple(obs_store.shape[1:])), a.out(outs[1], "outs[1]", (B, act_dim), th.int32 if is_u8 else th.float32)
    rew, nobs, done = a.out(outs[2], "outs[2]", (B, rew_dim)), a.out(outs[3], "outs[3]", (B,) + tuple(obs_store.shape[1:])), a.out(outs[4], "outs[4]", (B, 1))
    _launch("morl_replay_gather", obs_store, next_obs_store, act_store, rew_store, done_store, idx, B, obs_dim, act_dim, rew_dim, int(is_u8), cap, obs,
            nobs, act, rew, done)
    return obs, act, rew, nobs, done


def pareto_mask(points: th.Tensor, remove_duplicates: bool = True, raw: bool = False, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Non-dominated mask (reference pareto.py:34-57) of an [N, D] fp32 / fp64 CUDA tensor -> bool [N] (``raw``: the kernel's uint8 [N],
    optionally written into ``out``: no further launch)."""
    a = _Args("pareto_mask")
    points = a.inp(points, "points", (None, None), dtype=(th.float32, th.float64))
    N, D = points.shape
    keep = a.out(out, "out", (N,), th.uint8)
    if N > 0:
        _launch("morl_pareto_mask_f32" if points.dtype == th.float32 else "morl_pareto_mask_f64", points, N, D, int(bool(remove_duplicates)), keep,
                launches=2)
    return keep if raw else keep.bool()


def front_pack(points: th.Tensor, keep: Optional[th.Tensor], cap: int, rec: th.Tensor, extras: Optional[th.Tensor] = None) -> th.Tensor:
    """rec (float64 [1 + cap*d + n_extra]) = [count | first cap kept rows of points [n, d] (float64), -inf padded | extras]; one launch,
    no host sync (the count stays on the device)."""
    a = _Args("front_pack")
    points = a.inp(points, "points", (None, None), th.float64)
    n, d = points.shape
    keep, extras = a.inp(keep, "keep", (n,), th.uint8, opt=True), a.inp(extras, "extras", dtype=th.float64, reshape=(-1,), opt=True)
    n_extra = 0 if extras is None else extras.numel()
    rec = a.out(rec, "rec", (1 + cap * d + n_extra,), th.float64)
    _launch("morl_front_pack_f64", points, keep, n, d, cap, extras, n_extra, rec)
    return rec


def front_unpack(gathered: th.Tensor, world: int, d: int, cap: int, n_extra: int, pts_out: th.Tensor, meta_out: th.Tensor):
    """gathered records [world, 1 + cap*d + n_extra] -> pts_out [world*cap, d], meta_out [world, 1 + n_extra] (count, extras); one launch."""
    a = _Args("front_unpack")
    gathered = a.inp(gathered, "gathered", dtype=th.float64, reshape=(world, 1 + cap * d + n_extra))
    pts_out, meta_out = a.out(pts_out, "pts_out", (world * cap, d), th.float64), a.out(meta_out, "meta_out", (world, 1 + n_extra), th.float64)
    _launch("morl_front_unpack_f64", gathered, world, d, cap, n_extra, pts_out, meta_out)
    return pts_out, meta_out


def hypervolume(points: th.Tensor, ref_point: th.Tensor, keep: Optional[th.Tensor] = None, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Exact hypervolume (maximisation, d <= 3, n <= 2048) of float64 CUDA points [n, d] above ``ref_point`` [d]; returns a device float64
    scalar tensor [1] (no host sync).  ``keep`` (uint8 [n]) restricts the set, e.g. to the output of ``pareto_mask(..., raw=True)``."""
    a = _Args("hypervolume")
    points = a.inp(points, "points", (None, None), th.float64)
    n, d = points.shape
    ref_point = a.inp(th.as_tensor(ref_point).to(device=points.device, dtype=th.float64), "ref_point", reshape=(d,), dtype=th.float64)
    keep, out = a.inp(keep, "keep", (n,), th.uint8, opt=True), a.out(out, "out", (1,), th.float64)
    _launch("morl_hypervolume_f64", points, keep, n, d, ref_point, out)
    return out


def corner_weights(V: th.Tensor, cap: int = 256) -> th.Tensor:
    """Vertices (w, u) of { V w <= u, w >= 0, sum w = 1 } for a float64 CUDA tensor V [n, d] (reference linear_support.py:295-349;
    the caller rounds V).  Returns float64 [K, d+1] in no particular order; one launch, plus a second one with a buffer of the exact size
    when more than ``cap`` vertices exist (the count is read back: one host sync)."""
    a = _Args("corner_weights")
    V = a.inp(V, "V", (None, None), th.float64)
    n, d = V.shape
    count = a.out(None, "count", (1,), th.int32)
    while True:
        verts = a.out(None, "verts", (cap, d + 1), th.float64)
        _launch("morl_corner_weights_f64", V, n, d, verts if cap > 0 else None, cap, count)
        k = int(count.item())
        if k <= cap:
            return verts[:k]
        cap = k


class PolyakPlan:
    """Device-side (param, target, size) table for morl_polyak_f32; build once per pair of networks."""

    def __init__(self, params, targets):
        params, targets = list(params), list(targets)
        a = _Args("PolyakPlan")
        if len(params) != len(targets) or not params:
            a.fail("params", f"and targets must be two non-empty lists of one length, got {len(params)} and {len(targets)}")
        for i, (p, t) in enumerate(zip(params, targets)):
            a.inp(p, f"params[{i}]", inplace=True)
            a.inp(t, f"targets[{i}]", inplace=True)
            if p.numel() != t.numel():
                a.fail(f"targets[{i}]", f"has {t.numel()} elements, params[{i}] {p.numel()}")
        dev = params[0].device
        self.keepalive = (params, targets)
        self.p_tab = th.tensor([p.data_ptr() for p in params], dtype=th.int64, device=dev)
        self.t_tab = th.tensor([t.data_ptr() for t in targets], dtype=th.int64, device=dev)
        self.sizes = th.tensor([p.numel() for p in params], dtype=th.int64, device=dev)
        self.n = len(params)
        self.max_size = max(p.numel() for p in params)

    def run(self, tau: float):
        _launch("morl_polyak_f32", self.p_tab, self.t_tab, self.sizes, self.n, self.max_size, float(tau))


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
    a = _Args("amax_scale")
    x = a.inp(x, "x")
    scale_out, workspace = a.scalar(scale_out, "scale_out", opt=False), a.ws(workspace, "workspace", 8, zero=True)
    _launch("morl_amax_scale_f32", x, x.numel(), int(target_exp), scale_out, workspace)
    return scale_out


def split_planes(x: th.Tensor, fmt: int = FMT_F16X2, rows_pad: Optional[int] = None, ldp: Optional[int] = None, transpose: bool = False,
                 out: Optional[th.Tensor] = None, scale: Optional[th.Tensor] = None) -> th.Tensor:
    """fp32 [rows, cols] -> planes [P, rows_pad, ldp] of scale * x (zero padded); with ``transpose`` the planes hold x^T."""
    a = _Args("split_planes")
    x = a.inp(x, "x", (None, None))
    r, c = (x.shape[1], x.shape[0]) if transpose else (x.shape[0], x.shape[1])
    rows_pad = r if rows_pad is None else rows_pad
    ldp = _pad(c, 64 if fmt == FMT_F16X2 else 32) if ldp is None else ldp
    if out is None:
        out = empty_planes(fmt, rows_pad, ldp, x.device)
    a.planes(out, "out", fmt, rows_pad, ldp)
    _launch("morl_split_planes", fmt, x, r, c, x.shape[1], int(transpose), out, rows_pad, ldp, out.stride(0), a.scalar(scale, "scale"))
    return out


def split_planes_multi(jobs, fmt: int = FMT_F16X2) -> None:
    """One launch for several splits.  jobs: iterable of (src [rows, cols] fp32 CUDA, out planes [P, rows_pad, ldp], transpose, scale, target_exp):
    ``scale`` is a device float [1] or None; ``target_exp`` None = use the scale as given, an int = derive it from the matrix's amax and store it."""
    jobs = list(jobs)
    if not jobs:
        return
    a = _Args("split_planes_multi")
    if len(jobs) > _lib.SPLIT_MAX_JOBS:
        a.fail("jobs", f"may hold at most {_lib.SPLIT_MAX_JOBS} jobs per call, got {len(jobs)}")
    arr = (_lib.SplitJob * len(jobs))()
    srcs = []  # contiguous copies live until the launch
    for k, job in enumerate(jobs):
        src, out, transpose = job[0], job[1], job[2]
        scale = a.scalar(job[3] if len(job) > 3 else None, f"jobs[{k}][3]")
        target_exp = job[4] if len(job) > 4 else None
        src = a.inp(src, f"jobs[{k}][0]", (None, None))
        a.planes(out, f"jobs[{k}][1]", fmt)
        srcs.append(src)
        rows, cols = (src.shape[1], src.shape[0]) if transpose else (src.shape[0], src.shape[1])
        arr[k].src, arr[k].dst_planes, arr[k].plane_stride = src.data_ptr(), out.data_ptr(), out.stride(0)
        arr[k].scale = None if scale is None else scale.data_ptr()
        arr[k].rows, arr[k].cols, arr[k].ld_src, arr[k].transpose = rows, cols, src.stride(0), int(bool(transpose))
        arr[k].rows_pad, arr[k].ldp = out.shape[1], out.shape[2]
        arr[k].auto_scale, arr[k].target_exp = (0, 0) if target_exp is None else (1, int(target_exp))
    _launch("morl_split_planes_multi", fmt, arr, len(jobs), launches=2 if any(j.auto_scale for j in arr) else 1)


def _relu_bits(a, t, name, rows, width, out=False):
    """A ReLU / dropout bit mask [rows, relu_bits_words(width)] int32 (read, or written when ``out``)."""
    shape = (rows, relu_bits_words(width))
    return a.out(t, name, shape, th.int32, alloc=False) if out else a.inp(t, name, shape, th.int32, inplace=True, opt=True)


def gemm_planes(a_planes: th.Tensor, b_planes: th.Tensor, n_out: int, bias: Optional[th.Tensor] = None, relu: bool = False,
                out_f32: bool = True, out_planes: bool = False, c_f32: Optional[th.Tensor] = None, c_planes: Optional[th.Tensor] = None,
                reverse_tiles: bool = False, a_scale: Optional[th.Tensor] = None, b_scale: Optional[th.Tensor] = None,
                c_scale: Optional[th.Tensor] = None, split_acc: bool = False, relu_bits_in: Optional[th.Tensor] = None,
                relu_bits_out: Optional[th.Tensor] = None):
    """C = act(A . B^T + bias) on the tensor cores (wgmma) with split operands (fp32-accurate).
    a_planes [P, M, K], b_planes [P, N_pad, K]; the scales are device floats the planes were multiplied by (None = 1);
    ``split_acc``: leading and correction products in separate accumulators (the tensor cores truncate their fp32 accumulation; ~2.5x
    smaller systematic error, ~20 % slower per launch); False (default): one double-buffered accumulator.
    ``relu_bits_out`` / ``relu_bits_in`` (:func:`empty_relu_bits`): the forward call records [C > 0] as one bit per column, the backward
    call zeroes the outputs whose bit is clear (ReLU backward from 32 bytes per row instead of the activation planes).  Their width is the
    padded output width N_pad = b_planes.shape[1]
    (``empty_relu_bits(M, device, N_pad)``): 8 words per row up to 256, 16 above.
    returns (c_f32 [M, n_out] or None, c_planes [P, M, ldp] holding c_scale * C, or None)."""
    a = _Args("gemm_planes")
    fmt = a.planes(a_planes, "a_planes")
    _, M, K = a_planes.shape
    a.planes(b_planes, "b_planes", fmt, ld=K)
    n_pad = b_planes.shape[1]
    bias = a.inp(bias, "bias", reshape=(n_out,), opt=True)
    c_f32 = a.out(c_f32, "c_f32", (M, n_out), alloc=out_f32, ld=True)
    if out_planes and c_planes is None:
        c_planes = empty_planes(fmt, M, _pad(n_out, 32), a.device)
    if c_planes is not None:
        a.planes(c_planes, "c_planes", fmt, M)
    # one bit-mask word per 32-column chunk of the padded output (the kernel visits them all)
    relu_bits_in, relu_bits_out = _relu_bits(a, relu_bits_in, "relu_bits_in", M, n_pad), _relu_bits(a, relu_bits_out, "relu_bits_out", M, n_pad, True)
    _launch("morl_gemm_planes_f32", fmt, a_planes, a_planes.stride(0), a.scalar(a_scale, "a_scale"), b_planes, b_planes.stride(0), a.scalar(b_scale, "b_scale"),
            M, n_out, n_pad, K, bias, int(relu), c_f32, 0 if c_f32 is None else c_f32.stride(0), c_planes, 0 if c_planes is None else c_planes.shape[2],
            0 if c_planes is None else c_planes.stride(0), a.scalar(c_scale, "c_scale"), int(reverse_tiles), int(bool(split_acc)), relu_bits_in, relu_bits_out)
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
    a = _Args("gemm_planes_ln")
    fmt = a.planes(a_planes, "a_planes")
    _, M, K = a_planes.shape
    a.planes(b_planes, "b_planes", fmt, ld=K)
    if b_planes.shape[1] != n_out or n_out % 32 or n_out > 256:
        a.fail("b_planes", f"must be [P, n_out, K] with n_out % 32 == 0 and n_out <= 256 (got {tuple(b_planes.shape)}, n_out={n_out})")
    if not 0.0 <= drop_p < 1.0:
        a.fail("drop_p", f"{drop_p} is outside [0, 1)")
    if (drop_seed is None) != (drop_offset is None):
        a.fail("drop_seed", "and drop_offset must be given together")
    drop_seed, drop_offset = a.scalar(drop_seed, "drop_seed", th.int64), a.scalar(drop_offset, "drop_offset", th.int32)
    bias, ln_weight, ln_bias = (a.inp(t, name, (n_out,), opt=True) for t, name in ((bias, "bias"), (ln_weight, "ln_weight"), (ln_bias, "ln_bias")))
    c_f32 = a.out(c_f32, "c_f32", (M, n_out), alloc=out_f32, ld=True)
    if out_planes and c_planes is None:
        c_planes = empty_planes(fmt, M, n_out, a.device)
    if c_planes is not None:
        a.planes(c_planes, "c_planes", fmt, M)
    if c_f32 is None and c_planes is None:
        a.fail("c_f32", "and c_planes are both absent: no output requested")
    drop_bits_out = _relu_bits(a, drop_bits_out, "drop_bits_out", M, n_out, True)
    _launch("morl_gemm_planes_ln_f32", fmt, a_planes, a_planes.stride(0), a.scalar(a_scale, "a_scale"), b_planes, b_planes.stride(0),
            a.scalar(b_scale, "b_scale"), M, n_out, K, bias, int(ln_eps is not None), ln_weight, ln_bias, float(ln_eps or 0.0), float(drop_p), drop_seed,
            drop_offset, int(drop_salt) & 0xFFFFFFFF, c_f32, 0 if c_f32 is None else c_f32.stride(0), c_planes, 0 if c_planes is None else c_planes.shape[2],
            0 if c_planes is None else c_planes.stride(0), a.scalar(c_scale, "c_scale"), int(reverse_tiles), drop_bits_out)
    return c_f32, c_planes


def philox_advance(offset: th.Tensor, inc: int = 1) -> th.Tensor:
    """offset[0] += inc (int32 [1] CUDA tensor, wrapping) as one stream-ordered launch: the dropout pass counter of :func:`gemm_planes_ln`."""
    offset = _Args("philox_advance").scalar(offset, "offset", th.int32, opt=False)
    _launch("morl_philox_advance", offset, int(inc) & 0xFFFFFFFF)
    return offset


def _ensemble_args(a, out, max_logvar, min_logvar, model_idx, noise, rew_dim):
    """The ensemble-sampling inputs shared by :func:`ensemble_sample` and :func:`dyna_commit`."""
    out = a.inp(out, "out", (None,) * 3)
    E, N, O2 = out.shape
    if O2 % 2:
        a.fail("out", f"must be [E, N, 2*O], got {tuple(out.shape)}")
    O = O2 // 2
    max_logvar, min_logvar = a.inp(max_logvar, "max_logvar", reshape=(O,)), a.inp(min_logvar, "min_logvar", reshape=(O,))
    model_idx = a.inp(model_idx, "model_idx", dtype=th.int32, reshape=(N,))
    noise = a.inp(noise, "noise", (E, N, O), opt=True)
    return out, max_logvar, min_logvar, model_idx, noise, (E, N, O, O - int(rew_dim))


def ensemble_sample(out: th.Tensor, max_logvar: th.Tensor, min_logvar: th.Tensor, model_idx: th.Tensor, noise: Optional[th.Tensor] = None,
                    obs: Optional[th.Tensor] = None, rew_dim: int = 0):
    """Probabilistic-ensemble sampling + ensemble uncertainty in one pass (reference probabilistic_ensemble.py:115-154, utils.py:165).
    out [E, N, 2*O] raw last-layer output, model_idx [N] int32, noise [E, N, O] or None (deterministic), obs [N, O - rew_dim] or None.
    Returns (sample [N, O], var [N, O], uncertainty [N])."""
    a = _Args("ensemble_sample")
    out, max_logvar, min_logvar, model_idx, noise, (E, N, O, S) = _ensemble_args(a, out, max_logvar, min_logvar, model_idx, noise, rew_dim)
    obs = a.inp(obs, "obs", (N, S), opt=True)
    sample, var, unc = a.out(None, "sample", (N, O)), a.out(None, "var", (N, O)), a.out(None, "uncertainty", (N,))
    _launch("morl_ensemble_sample_f32", out, max_logvar, min_logvar, model_idx, noise, obs, int(rew_dim), E, N, O, sample, var, unc)
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
    a = _Args("dyna_commit")
    out, max_logvar, min_logvar, model_idx, noise, (E, N, O, S) = _ensemble_args(a, out, max_logvar, min_logvar, model_idx, noise, rew_dim)
    obs, act = a.inp(obs, "obs", (N, S)), a.inp(act, "act", (N, None))
    A = act.shape[1]
    st_obs = a.out(stores[0], "stores[0]", (None, S))
    C = st_obs.shape[0]
    st_nobs, st_act = a.out(stores[1], "stores[1]", (C, S)), a.out(stores[2], "stores[2]", (C, A))
    st_rew, st_done = a.out(stores[3], "stores[3]", (C, int(rew_dim))), a.out(stores[4], "stores[4]", (C, 1))
    next_alive, uncertainty_out = a.out(next_alive, "next_alive", (N, S)), a.out(uncertainty_out, "uncertainty_out", (N,))
    counts_out = a.out(counts_out, "counts_out", (2,), th.int32)
    workspace = a.ws(workspace, "workspace", _lib.load().morl_dyna_commit_workspace_bytes(N))
    _launch("morl_dyna_commit_f32", out, max_logvar, min_logvar, model_idx, noise, obs, act, int(rew_dim), E, N, O, A, int(rule), float(max_uncertainty),
            st_obs, st_nobs, st_act, st_rew, st_done, C, int(ptr), next_alive, uncertainty_out, counts_out, workspace, launches=2)
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
    a = _Args("qhead_envelope_td")
    fmt = a.planes(a_on, "a_on", rows=B * W)
    K = a_on.shape[2]
    a.planes(a_tg, "a_tg", fmt, B * W, K)
    a.planes(w_on, "w_on", fmt, 32, K)
    a.planes(w_tg, "w_tg", fmt, 32, K)
    if a_tg.stride(0) != a_on.stride(0):
        a.fail("a_tg", "must have the plane stride of a_on")
    if w_tg.stride(0) != w_on.stride(0):
        a.fail("w_tg", "must have the plane stride of w_on")
    bias_on, bias_tg = a.inp(bias_on, "bias_on", reshape=(A * D,)), a.inp(bias_tg, "bias_tg", reshape=(A * D,))
    wset, reward, done = a.inp(wset, "wset", (W, D)), a.inp(reward, "reward", (B, D)), a.inp(done, "done", reshape=(B,))
    out = a.out(out, "out", (W * B, D))
    pref_out = a.out(pref_out, "pref_out", (W * B,), th.int32, alloc=want_indices)
    act_out = a.out(act_out, "act_out", (W * B,), th.int32, alloc=want_indices)
    q_on_out, q_tg_out = a.out(q_on_out, "q_on_out", (B * W, A * D), alloc=False), a.out(q_tg_out, "q_tg_out", (B * W, A * D), alloc=False)
    _launch("morl_qhead_envelope_td_f32", fmt, a_on, a_tg, a_on.stride(0), a.scalar(a_scale_on, "a_scale_on"), a.scalar(a_scale_tg, "a_scale_tg"), w_on,
            w_tg, w_on.stride(0), a.scalar(w_scale_on, "w_scale_on"), a.scalar(w_scale_tg, "w_scale_tg"), bias_on, bias_tg, K, wset, reward, done,
            float(gamma), B, W, A, D, dot_mode, row_order, int(reverse_tiles), out, pref_out, act_out, q_on_out, q_tg_out)
    return out, pref_out, act_out


def gemm_chain_supported(fmt: int, M: int, K: int) -> bool:
    return bool(_lib.load().morl_gemm_chain_supported(int(fmt), int(M), int(K)))


def _chain_layers(a, weights, biases, w_scales, bits, fmt, rows, width, k_first=None):
    """Flattened per-layer tables of a chained launch: weight planes [P, width, k] (k_first for each chain's first layer), biases
    [width], weight scales and ReLU bit masks [rows, relu_bits_words(width)], each optional but the weights."""
    n_layers = len(weights[0])
    if any(len(w) != n_layers for w in weights):
        a.fail("weights", f"must hold {n_layers} tensors per chain")
    flat = lambda ts: [None] * (len(weights) * n_layers) if ts is None else [t for ch in ts for t in ch]  # noqa: E731
    flat_w, flat_b, flat_s, flat_m = flat(weights), flat(biases), flat(w_scales), flat(bits)
    if not len(flat_w) == len(flat_b) == len(flat_s) == len(flat_m):
        a.fail("biases", "/ w_scales / bits must have one entry per layer of every chain")
    for i, t in enumerate(flat_w):
        a.planes(t, f"weights[{i // n_layers}][{i % n_layers}]", fmt, width, k_first if k_first and i % n_layers == 0 else width, contiguous=True)
    flat_b = [a.inp(t, f"biases[{i // n_layers}][{i % n_layers}]", reshape=(width,), inplace=True, opt=True)
              for i, t in enumerate(flat_b)]
    flat_s = [a.scalar(t, f"w_scales[{i // n_layers}][{i % n_layers}]") for i, t in enumerate(flat_s)]
    flat_m = [_relu_bits(a, t, f"bits[{i // n_layers}][{i % n_layers}]", rows, width, True) for i, t in enumerate(flat_m)]
    return n_layers, flat_w, flat_b, flat_s, flat_m


class GemmChain:
    """Static plan of a chained launch (:func:`gemm_chain`): the pointer tables are built once, a call is one launch.
    ``acts[c]``: the n_layers + 1 plane tensors [P, M, 256] of chain c (input, then every layer's output); ``weights[c]`` / ``w_scales[c]`` /
    ``biases[c]`` / ``bits[c]`` (ReLU masks recorded) / ``bits_in[c]`` (ReLU-backward masks applied): per layer, all optional.  ``relu``: ReLU on every
    output (forward chains); False for the dX chains of the backward pass."""

    def __init__(self, acts, weights, biases=None, w_scales=None, bits=None, act_scale=None, relu: bool = True, bits_in=None, k_first: int = 0):
        a = _Args("GemmChain")
        self.n_chains = len(acts)
        a0 = acts[0][1]  # (the first OUTPUT: the chain's input may be narrower, see k_first)
        self.fmt = a.planes(a0, "acts[0][1]", contiguous=True)
        _, self.M, self.K = a0.shape  # (square layers: the output width of every layer is also the reduction length)
        self.N = a0.shape[2]  # output width of every layer: the width of its ReLU bit masks
        self.k_first = int(k_first) if k_first else self.K
        self.n_layers, flat_w, flat_b, flat_s, flat_m = _chain_layers(a, weights, biases, w_scales, bits, self.fmt, self.M, 256, self.k_first)
        flat_a = [t for ch in acts for t in ch]
        flat_i = [None] * len(flat_w) if bits_in is None else [t for ch in bits_in for t in ch]
        if len(flat_a) != self.n_chains * (self.n_layers + 1) or len(flat_i) != len(flat_w):
            a.fail("acts", "must hold n_layers + 1 activation tensors per chain (and bits_in one mask per layer)")
        for i, t in enumerate(flat_a):
            kk = self.k_first if i % (self.n_layers + 1) == 0 else self.K
            a.planes(t, f"acts[{i // (self.n_layers + 1)}][{i % (self.n_layers + 1)}]", self.fmt, self.M, kk, contiguous=True)
        flat_i = [_relu_bits(a, t, f"bits_in[{i // self.n_layers}][{i % self.n_layers}]", self.M, self.N) for i, t in enumerate(flat_i)]
        self._act_scale = a.scalar(act_scale, "act_scale")
        self._keep = (flat_a, flat_w, flat_b, flat_s, flat_m, flat_i, act_scale)
        self.relu = bool(relu)
        self._pa, self._pw, self._pb = _pointer_table(flat_a), _pointer_table(flat_w), _pointer_table(flat_b)
        self._ps, self._pm, self._pi = _pointer_table(flat_s), _pointer_table(flat_m), _pointer_table(flat_i)
        self._a_stride, self._w_stride = a0.stride(0), 256 * self.K

    def __call__(self):
        _launch("morl_gemm_chain_f32", self.fmt, self.n_chains, self.n_layers, self._pa, self._a_stride, self._act_scale, self._pw, self._w_stride,
                self._ps, self._pb, int(self.relu), self._pi, self._pm, self.M, self.K, self.k_first)


class GemmChainPairs:
    """Static plan of a chained launch that starts from the separable first layer (f16x2): the input of chain c is
    relu(u[c][b] + v[c][j]) * act_scale for row b*W + j, built in shared memory (the planes :func:`pairs_relu_split` would write), then the
    hidden layers as :class:`GemmChain`.  ``outs[c]``: per layer, the output plane tensor [P, B*W, 256], or None when that output is not
    needed -- only the others are written to memory; ``weights`` / ``biases`` / ``w_scales`` / ``bits`` as :class:`GemmChain`.  A call takes
    the per-chain u [B, 256] and v [W, 256] (fp32, contiguous) of that pass."""

    def __init__(self, outs, weights, B: int, W: int, biases=None, w_scales=None, bits=None, act_scale=None):
        a = _Args("GemmChainPairs")
        self.n_chains = len(outs)
        self.B, self.W, self.M = int(B), int(W), int(B) * int(W)
        self.n_layers, flat_w, flat_b, flat_s, flat_m = _chain_layers(a, weights, biases, w_scales, bits, FMT_F16X2, self.M, 256)
        flat_o = [t for ch in outs for t in ch]
        if len(flat_o) != len(flat_w):
            a.fail("outs", "must hold n_layers outputs (or None) per chain")
        stored = [t for t in flat_o if t is not None]
        for i, t in enumerate(flat_o):
            if t is not None:
                a.planes(t, f"outs[{i // self.n_layers}][{i % self.n_layers}]", FMT_F16X2, self.M, 256, contiguous=True)
                if t.stride(0) != stored[0].stride(0):
                    a.fail(f"outs[{i // self.n_layers}][{i % self.n_layers}]", "must have the plane stride of the other outputs")
        self.store = sum(1 << i for i, t in enumerate(flat_o) if t is not None)
        self._act_scale = a.scalar(act_scale, "act_scale")
        self._keep = (flat_o, flat_w, flat_b, flat_s, flat_m, act_scale)
        self._po, self._pw, self._pb, self._ps, self._pm = (_pointer_table(t) for t in (flat_o, flat_w, flat_b, flat_s, flat_m))
        self._o_stride = stored[0].stride(0) if stored else 0
        self._w_stride = flat_w[0].stride(0)

    def __call__(self, us, vs):
        a = _Args("GemmChainPairs")
        if len(us) != self.n_chains or len(vs) != self.n_chains:
            a.fail("us", f"and vs must hold {self.n_chains} tensors, got {len(us)} and {len(vs)}")
        us = [a.inp(u, f"us[{c}]", (self.B, 256)) for c, u in enumerate(us)]
        vs = [a.inp(v, f"vs[{c}]", (self.W, 256)) for c, v in enumerate(vs)]
        _launch("morl_gemm_chain_pairs_f32", self.n_chains, self.n_layers, _pointer_table(us), _pointer_table(vs), self.B, self.W, self._po, self._o_stride,
                self._act_scale, self._pw, self._w_stride, self._ps, self._pb, self._pm, self.store)


def qhead_gemm_supported(fmt: int, M: int, N: int, K: int) -> bool:
    return bool(_lib.load().morl_qhead_gemm_supported(int(fmt), int(M), int(N), int(K)))


def qhead_gemm(a_planes: th.Tensor, w_planes: th.Tensor, n_out: int, bias: th.Tensor, out: Optional[th.Tensor] = None, a_scale=None, w_scale=None,
               reverse_tiles: bool = False) -> th.Tensor:
    """Output layer Q = A . W^T + bias (n_out <= 32) as fp32 [M, n_out]: the narrow form of :func:`gemm_planes` (bit-identical) with the weight
    planes resident in shared memory (csrc/qhead_envelope.cu without its operator half)."""
    a = _Args("qhead_gemm")
    fmt = a.planes(a_planes, "a_planes")
    _, M, K = a_planes.shape
    a.planes(w_planes, "w_planes", fmt, 32, K)
    bias, out = a.inp(bias, "bias", reshape=(n_out,)), a.out(out, "out", (M, n_out))
    _launch("morl_qhead_gemm_f32", fmt, a_planes, a_planes.stride(0), a.scalar(a_scale, "a_scale"), w_planes, w_planes.stride(0),
            a.scalar(w_scale, "w_scale"), bias, M, n_out, K, int(reverse_tiles), out)
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
    a = _Args("pairs_relu_split")
    u = a.inp(u, "u", (None, None))
    B, H = u.shape
    v = a.inp(v, "v", (None, H))
    W = v.shape[0]
    if out is None:
        out = empty_planes(fmt, B * W, H, u.device)
    fmt = a.planes(out, "out", rows=B * W, ld=H)
    relu_bits_out = _relu_bits(a, relu_bits_out, "relu_bits_out", B * W, H, True)
    _launch("morl_pairs_relu_split_planes", fmt, u, v, B, W, H, out, out.stride(0), a.scalar(scale, "scale"), relu_bits_out)
    return out


def pairs_product_split(u: th.Tensor, v: th.Tensor, out: Optional[th.Tensor] = None, fmt: int = FMT_F16X2, scale: Optional[th.Tensor] = None) -> th.Tensor:
    """u[b] * v[p] for every pair (one fp32 multiply), written as planes [P_fmt, B*P, H] of scale * h (row b*P + p): the product-conditioned
    first layer of GPI-PD's Q-network.  A given ``out`` may hold more rows than B*P (the first B*P are written)."""
    a = _Args("pairs_product_split")
    u = a.inp(u, "u", (None, None))
    B, H = u.shape
    v = a.inp(v, "v", (None, H))
    P = v.shape[0]
    if H % 8:
        a.fail("u", f"must be a multiple of 8 wide, got {H}")
    if out is None:
        out = empty_planes(fmt, B * P, H, u.device)
    fmt = a.planes(out, "out", ld=H)
    if out.shape[1] < B * P:
        a.fail("out", f"must hold at least {B * P} rows, got {out.shape[1]}")
    _launch("morl_pairs_product_split_planes", fmt, u, v, B, P, H, out, out.stride(0), a.scalar(scale, "scale"))
    return out


def product_layer1_uv(s: th.Tensor, s_weight: th.Tensor, s_bias: th.Tensor, m: th.Tensor, w_weight: th.Tensor, w_bias: th.Tensor,
                      u: Optional[th.Tensor] = None, v: Optional[th.Tensor] = None):
    """u = relu(s @ Ls^T + bs) [B, H] and v = relu(m @ Lw^T + bw) [P, H] in one launch (the two feature maps of GPI-PD's Q-network)."""
    a = _Args("product_layer1_uv")
    s, m = a.inp(s, "s", (None, None)), a.inp(m, "m", (None, None))
    (B, F), (P, D) = s.shape, m.shape
    s_weight = a.inp(s_weight, "s_weight", (None, F))
    H = s_weight.shape[0]
    s_bias, w_weight, w_bias = a.inp(s_bias, "s_bias", reshape=(H,)), a.inp(w_weight, "w_weight", (H, D)), a.inp(w_bias, "w_bias", reshape=(H,))
    u, v = a.out(u, "u", (B, H)), a.out(v, "v", (P, H))
    _launch("morl_product_layer1_uv_f32", s, s_weight, s_bias, B, F, m, w_weight, w_bias, P, D, H, u, v)
    return u, v


def pair_layer1_uv(feats: th.Tensor, wset: th.Tensor, weight: th.Tensor, bias: th.Tensor, u: Optional[th.Tensor] = None,
                   v: Optional[th.Tensor] = None):
    """u = feats @ W1[:, :F]^T [B, H] and v = wset @ W1[:, F:]^T + b1 [W, H] in one launch (separable first layer of the pair batch)."""
    a = _Args("pair_layer1_uv")
    feats, wset = a.inp(feats, "feats", (None, None)), a.inp(wset, "wset", (None, None))
    (B, F), (W, D) = feats.shape, wset.shape
    weight = a.inp(weight, "weight", (None, F + D))
    H = weight.shape[0]
    bias = a.inp(bias, "bias", reshape=(H,))
    u, v = a.out(u, "u", (B, H)), a.out(v, "v", (W, H))
    _launch("morl_pair_layer1_uv_f32", feats, wset, weight, bias, B, W, F, D, H, u, v)
    return u, v


def pair_layer1_grad_workspace(F: int, D: int, H: int, device) -> th.Tensor:
    nbytes = _lib.load().morl_pair_layer1_grad_workspace_bytes(int(F), int(D), int(H))
    return th.zeros((nbytes + 3) // 4, device=device, dtype=th.float32)  # arrival counters start at zero (self-resetting afterwards)


def pair_layer1_grad(dU: th.Tensor, dV: th.Tensor, feats: th.Tensor, wset: th.Tensor, dW1: Optional[th.Tensor] = None, db1: Optional[th.Tensor] = None,
                     workspace: Optional[th.Tensor] = None):
    """dW1 [H, F + D] = [dU^T feats | dV^T wset] and db1 [H] = colsum(dV) in one launch (backward of the separable first layer)."""
    a = _Args("pair_layer1_grad")
    dU, wset = a.inp(dU, "dU", (None, None)), a.inp(wset, "wset", (None, None))
    (B, H), (W, D) = dU.shape, wset.shape
    dV, feats = a.inp(dV, "dV", (W, H)), a.inp(feats, "feats", (B, None))
    F = feats.shape[1]
    dW1, db1 = a.out(dW1, "dW1", (H, F + D)), a.out(db1, "db1", (H,))
    workspace = a.ws(workspace, "workspace", _lib.load().morl_pair_layer1_grad_workspace_bytes(F, D, H), zero=True)
    _launch("morl_pair_layer1_grad_f32", dU, dV, feats, wset, B, W, F, D, H, dW1, db1, workspace)
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
    a = _Args("gemm_planes_mn")
    fmt = a.planes(g_planes, "g_planes")
    _, M, ldg = g_planes.shape
    a.planes(h_planes, "h_planes", fmt, M)
    ldh = h_planes.shape[2]
    out = a.out(out, "out", (h_cols, g_cols) if transpose_out else (g_cols, h_cols), ld=True)
    colsum = a.out(colsum, "colsum", (g_cols,), alloc=False)
    workspace = a.ws(workspace, "workspace", gemm_mn_workspace_bytes(M, g_cols, h_cols))
    _launch("morl_gemm_planes_mn_f32", fmt, g_planes, g_planes.stride(0), ldg, g_cols, a.scalar(g_scale, "g_scale"), h_planes, h_planes.stride(0), ldh,
            h_cols, a.scalar(h_scale, "h_scale"), M, int(transpose_out), out, out.stride(0), colsum, workspace, launches=2)
    return out


def pairs_grad_reduce_workspace(B: int, W: int, H: int, device) -> th.Tensor:
    nbytes = _lib.load().morl_pairs_grad_reduce_workspace_bytes(int(B), int(W), int(H))
    return th.empty((nbytes + 3) // 4, device=device, dtype=th.float32)


def pairs_grad_reduce(planes: th.Tensor, B: int, W: int, workspace: Optional[th.Tensor] = None, dU: Optional[th.Tensor] = None,
                      dV: Optional[th.Tensor] = None, scale: Optional[th.Tensor] = None):
    """dU [B, H] and dV [W, H] from the planes of dL/dh1 [P, B*W, H] (gradient of relu(u[b] + v[j]) w.r.t. u and v), scale removed."""
    a = _Args("pairs_grad_reduce")
    fmt = a.planes(planes, "planes", rows=B * W)
    H = planes.shape[2]
    dU, dV = a.out(dU, "dU", (B, H)), a.out(dV, "dV", (W, H))
    workspace = a.ws(workspace, "workspace", _lib.load().morl_pairs_grad_reduce_workspace_bytes(int(B), int(W), int(H)))
    _launch("morl_pairs_grad_reduce_planes", fmt, planes, planes.stride(0), a.scalar(scale, "scale"), B, W, H, dU, dV, workspace, launches=2)
    return dU, dV


# ---- PCN / LCN (csrc/pcn.cu) ---------------------------------------------------------------------------------------------------------
def pcn_supported(obs_dim: int, d: int, hidden: int, n_out: int, batch: int = 1) -> bool:
    """Whether the fused PCN kernels cover this model and batch: 1 <= obs_dim <= 256, 1 <= d <= 8, hidden in {32, 64, 128, 256},
    1 <= n_out <= 32, 1 <= batch <= 4096 (include/morl_b200.h)."""
    return bool(_lib.load().morl_pcn_supported(int(obs_dim), int(d), int(hidden), int(n_out), int(batch)))


def _pcn_workspace_bytes(obs_dim: int, d: int, hidden: int, n_out: int, batch: int) -> int:
    nbytes = int(_lib.load().morl_pcn_workspace_bytes(int(obs_dim), int(d), int(hidden), int(n_out), int(batch)))
    if nbytes == 0:
        raise _lib.MorlB200Error(f"pcn_workspace: unsupported configuration obs_dim={obs_dim} d={d} hidden={hidden} n_out={n_out} batch={batch}")
    return nbytes


def pcn_workspace(obs_dim: int, d: int, hidden: int, n_out: int, batch: int, device) -> th.Tensor:
    return _workspace(_pcn_workspace_bytes(obs_dim, d, hidden, n_out, batch), device)


def pcn_pointer_table(tensors) -> "ctypes.Array":
    """Host array of the 8 device pointers (Ls, bs, Lc, bc, W1, b1, W2, b2) the PCN kernels take; build it once per set of storages."""
    return _param_table(_Args("pcn_pointer_table"), tensors, "tensors", 8, "parameter tensors of the PCN kernels")


def pcn_update(params, grads, scaling: th.Tensor, store: th.Tensor, obs_dim: int, d: int, rows: th.Tensor, horizons: th.Tensor, batch: int,
               hidden: int, n_out: int, continuous: bool, loss_out: th.Tensor, entropy_out: Optional[th.Tensor], pred_out: Optional[th.Tensor],
               workspace: th.Tensor):
    """One PCN minibatch (reference pcn.py:202-236): gather ``rows`` [batch] int32 of the episode store f32 [N, ld] (columns obs | return-to-go
    | action, a discrete action as int32 bits) with ``horizons`` [batch] int32, forward, loss, backward.  ``params`` / ``grads``: pointer
    tables of ``pcn_pointer_table``; the gradients are overwritten.  ``loss_out`` / ``entropy_out`` / ``pred_out`` are device views written
    in place."""
    a = _Args("pcn_update")
    scaling, store = a.inp(scaling, "scaling", reshape=(d + 1,)), a.inp(store, "store", (None, None))
    rows, horizons = a.inp(rows, "rows", (batch,), th.int32), a.inp(horizons, "horizons", (batch,), th.int32)
    loss_out, entropy_out = a.out(loss_out, "loss_out", (1,)), a.out(entropy_out, "entropy_out", (1,), alloc=False)
    pred_out = a.out(pred_out, "pred_out", (batch, n_out), alloc=False)
    workspace = a.ws(workspace, "workspace", _pcn_workspace_bytes(obs_dim, d, hidden, n_out, batch))
    _launch("morl_pcn_update_f32", params, grads, scaling, store, int(store.shape[1]), rows, horizons, int(batch), int(obs_dim), int(d), int(hidden),
            int(n_out), int(bool(continuous)), loss_out, entropy_out, pred_out, workspace, launches=2)


def pcn_forward(params, scaling: th.Tensor, obs: th.Tensor, ret: th.Tensor, hor: th.Tensor, hidden: int, log_softmax: bool, out: th.Tensor,
                argmax_out: Optional[th.Tensor] = None):
    """The PCN model on N rows with their own commands (reference pcn.py:309-322 on one row): obs [N, S], ret [N, d], hor [N] ->
    ``out`` [N, A] (log-probabilities or predictions), optionally the first-occurrence argmax into ``argmax_out`` int32 [N].  The row
    tensors and outputs may be CUDA tensors or pinned host tensors (the kernel reads and writes pinned memory directly); with pinned
    outputs the caller synchronises the stream before reading them."""
    a = _Args("pcn_forward")
    obs, ret = a.inp(obs, "obs", (None, None), inplace=True, pinned=True), a.inp(ret, "ret", (None, None), inplace=True, pinned=True)
    (N, S), d = obs.shape, ret.shape[1]
    if ret.shape[0] != N:
        a.fail("ret", f"must have {N} rows, got shape {tuple(ret.shape)}")
    hor, scaling = a.inp(hor, "hor", reshape=(N,), inplace=True, pinned=True), a.inp(scaling, "scaling", reshape=(d + 1,))
    out = a.out(out, "out", (N, None), pinned=True)
    argmax_out = a.out(argmax_out, "argmax_out", (N,), th.int32, alloc=False, pinned=True)
    _launch("morl_pcn_forward_f32", params, scaling, obs, ret, hor, int(N), int(S), int(d), int(hidden), int(out.shape[1]), int(bool(log_softmax)), out,
            argmax_out)


# ---- EUPG (csrc/eupg.cu) -------------------------------------------------------------------------------------------------------------
def _int_array(values):
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
        a = _Args("EupgNet")
        if not _lib.load().morl_eupg_supported(self.obs_dim, self.d, self.hidden, self.n_hidden, self.n_out):
            a.fail("hidden", f"is an unsupported configuration obs_dim={obs_dim} d={d} hidden={list(hidden)} n_out={n_out}")
        n = 2 * (self.n_hidden + 1)
        self.params = _param_table(a, params, "params", n, "tensors of the EUPG kernels")
        self.grads = None if grads is None else _param_table(a, grads, "grads", n, "tensors of the EUPG kernels")

    @property
    def workspace_bytes(self) -> int:
        return int(_lib.load().morl_eupg_workspace_bytes(self.obs_dim, self.d, self.hidden, self.n_hidden, self.n_out))

    def workspace(self, device) -> th.Tensor:
        return _workspace(self.workspace_bytes, device)


def eupg_workspace_bytes(obs_dim: int, d: int, hidden, n_out: int) -> int:
    arr, n = _int_array(hidden)
    return int(_lib.load().morl_eupg_workspace_bytes(int(obs_dim), int(d), arr, n, int(n_out)))


def _eupg_rows(a, t, name, cols, dtype=th.float32):
    """EUPG's rows [T, cols], read in place from strided views of one staging block: contiguous columns, a non-negative row stride."""
    a._tensor(t, name, dtype)
    if t.dim() != 2 or t.shape[1] != cols or (cols > 1 and t.stride(1) != 1) or t.stride(0) < 0:
        a.fail(name, f"must be [T, {cols}] with contiguous columns, got shape {tuple(t.shape)} strides {t.stride()}")
    return t


def eupg_returns(rewards: th.Tensor, gamma: float, out: Optional[th.Tensor] = None) -> th.Tensor:
    """Discounted forward returns of an episode's rewards [T, d] (rows may be strided, columns contiguous), bit-identical to the
    reference's float32 loop ``c = gamma * c + r_t`` run backward (eupg.py:263-270), for any number of objectives.  ``out``: a
    contiguous float32 [T, d] CUDA tensor, allocated when not given."""
    a = _Args("eupg_returns")
    if not isinstance(rewards, th.Tensor) or rewards.dim() != 2:
        a.fail("rewards", "must be a [T, d] tensor")
    T, d = rewards.shape
    rewards = _eupg_rows(a, rewards, "rewards", d)
    out = a.out(out, "out", (T, d))
    _launch("morl_eupg_returns_f32", rewards, int(rewards.stride(0)), int(T), int(d), float(gamma), out)
    return out


def eupg_update(net: EupgNet, obs: th.Tensor, acc: th.Tensor, actions: th.Tensor, v: th.Tensor, loss_out: th.Tensor, workspace: th.Tensor):
    """One EUPG episode update (reference eupg.py:236-251): rows ``obs`` int32 [T, S], ``acc`` f32 [T, d] and ``actions`` int32 [T] are
    views with one common row stride (columns of one staging block), read in place; ``v`` f32 [T] or one element (broadcast).  Writes
    the loss into ``loss_out`` [>= 1] and overwrites the gradients of ``net.grads``."""
    a = _Args("eupg_update")
    if net.grads is None:
        a.fail("net", "was built without gradient tensors")
    obs, acc = _eupg_rows(a, obs, "obs", net.obs_dim, th.int32), _eupg_rows(a, acc, "acc", net.d)
    T, ld = obs.shape[0], obs.stride(0)
    a._tensor(actions, "actions", th.int32)
    a._tensor(v, "v", th.float32)
    if acc.shape[0] != T or acc.stride(0) != ld:
        a.fail("acc", "must be rows of the block of obs (same rows, same row stride)")
    if actions.dim() != 1 or actions.shape[0] != T or actions.stride(0) != ld:
        a.fail("actions", "must be rows of the block of obs (same rows, same row stride)")
    if v.numel() != 1 and (v.dim() != 1 or v.shape[0] != T or v.stride(0) < 0):
        a.fail("v", f"must have T={T} elements or one, got shape {tuple(v.shape)}")
    loss_out = a.out(loss_out, "loss_out", (None,))
    if loss_out.numel() < 1:
        a.fail("loss_out", "must have at least one element")
    workspace = a.ws(workspace, "workspace", net.workspace_bytes)
    _launch("morl_eupg_update_f32", net.params, net.grads, obs, acc, actions, int(ld), v, 0 if v.numel() == 1 else int(v.stride(0)), int(T), net.obs_dim,
            net.d, net.hidden, net.n_hidden, net.n_out, loss_out, workspace, launches=2)


def eupg_probs(net: EupgNet, x: th.Tensor, out: th.Tensor):
    """Action probabilities [N, A] of rows ``x`` [N, S + d] (reference eupg.py:46-61 after Categorical's renormalisation).  ``x`` and
    ``out`` may be contiguous CUDA tensors or pinned host tensors; with a pinned output the caller synchronises the stream before reading
    it."""
    a = _Args("eupg_probs")
    x = a.inp(x, "x", (None, net.obs_dim + net.d), inplace=True, pinned=True)
    N = x.shape[0]
    if N < 1:
        a.fail("x", "must have at least one row")
    out = a.out(out, "out", (N, net.n_out), pinned=True)
    _launch("morl_eupg_probs_f32", net.params, x, int(N), net.obs_dim, net.d, net.hidden, net.n_hidden, net.n_out, out)
