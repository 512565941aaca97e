"""Float64 restatement of one MO-PPO minibatch loss (reference single_policy/ser/mo_ppo.py:514-549) and its gradients w.r.t. the actor
mean, actor_logstd and the value head: the reference's formulas on float64 CPU tensors, differentiated by torch autograd (whose th.max
splits a tie half and half and whose clamp passes the gradient on its closed interval, the rules the kernel restates)."""

from __future__ import annotations

import math

import numpy as np
import torch as th


def ppo_loss_f64(mean, logstd, value, actions, old_logprob, advantages, returns, old_values, clip_coef, ent_coef, vf_coef, norm_adv, clip_vloss):
    """numpy in; returns dict(loss, dmean, dlogstd, dvalue, pg_loss, v_loss, entropy, old_approx_kl, approx_kl, clipfrac) in float64."""
    f = lambda x: th.tensor(np.asarray(x, np.float64))  # noqa: E731
    mu, ls, v = f(mean).requires_grad_(), f(logstd).reshape(-1).requires_grad_(), f(value).requires_grad_()
    act, old_lp, adv, R = f(actions), f(old_logprob), f(advantages), f(returns)
    std = th.exp(ls).expand_as(mu)
    logp = (-((act - mu) ** 2) / (2 * std**2) - ls - math.log(math.sqrt(2 * math.pi))).sum(1)
    entropy = (0.5 + 0.5 * math.log(2 * math.pi) + ls).expand_as(mu).sum(1)
    logratio = logp - old_lp
    ratio = logratio.exp()
    with th.no_grad():
        old_kl = (-logratio).mean()
        kl = ((ratio - 1) - logratio).mean()
        clipfrac = ((ratio - 1.0).abs() > clip_coef).double().mean()
    if norm_adv:
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    pg_loss = th.max(-adv * ratio, -adv * th.clamp(ratio, 1 - clip_coef, 1 + clip_coef)).mean()
    if clip_vloss:
        ov = f(old_values)
        v_unc = (v - R) ** 2
        v_clip = (ov + th.clamp(v - ov, -clip_coef, clip_coef) - R) ** 2
        v_loss = 0.5 * th.max(v_unc, v_clip).mean()
    else:
        v_loss = 0.5 * ((v - R) ** 2).mean()
    ent = entropy.mean()
    loss = pg_loss - ent_coef * ent + v_loss * vf_coef
    loss.backward()
    return dict(loss=loss.item(), dmean=mu.grad.numpy(), dlogstd=ls.grad.numpy(), dvalue=v.grad.numpy(), pg_loss=pg_loss.item(), v_loss=v_loss.item(),
                entropy=ent.item(), old_approx_kl=old_kl.item(), approx_kl=kl.item(), clipfrac=clipfrac.item())
