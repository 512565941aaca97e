"""Float64 restatement of one NLMOPPO minibatch (reference nl_mo_ppo.py:349-391) through torch autograd: the loss, its gradients
w.r.t. the 12 Agent parameters and the logged statistics, for inputs gathered by ``perm``."""

from __future__ import annotations

import torch as th


def agent_forward(params, x):
    """(values [M, d], logits [M, A]) of the Agent with parameters ``params`` (its parameter order) on rows x."""
    def mlp(p, h):
        h = th.tanh(h @ p[0].T + p[1])
        h = th.tanh(h @ p[2].T + p[3])
        return h @ p[4].T + p[5]

    return mlp(params[:6], x), mlp(params[6:], x)


def minibatch(params, obs, acc, actions, old_logp, adv, ret, old_v, perm, pref, w, clip_coef, ent_coef, vf_coef, norm_adv, clip_vloss,
              dtype=th.float64):
    """Returns (loss, grads [12], stats dict) computed in ``dtype``."""
    ps = [p.detach().to(dtype).requires_grad_(True) for p in params]
    idx = perm.long()
    M, d = idx.shape[0], acc.shape[1]
    cols = [obs[idx].to(dtype), acc[idx].to(dtype)]
    if pref is not None and pref.numel():
        cols.append(pref.to(dtype).reshape(1, -1).expand(M, -1))
    x = th.cat(cols, 1)
    value, logits = agent_forward(ps, x)
    logl = logits - th.logsumexp(logits, 1, keepdim=True)
    newlogprob = logl.gather(1, actions[idx].long().view(-1, 1)).squeeze(1)
    entropy = -(logl.exp() * logl).sum(1)
    logratio = newlogprob - old_logp[idx].to(dtype)
    ratio = logratio.exp()
    a = adv[idx].to(dtype)
    if norm_adv:
        a = (a - a.mean(0, keepdim=True)) / (a.std(0, keepdim=True) + 1e-8)
    pg1 = -a * ratio.unsqueeze(-1)
    pg2 = -a * th.clamp(ratio, 1 - clip_coef, 1 + clip_coef).unsqueeze(-1)
    pg_loss = (th.max(pg1, pg2).mean(0) * w.to(dtype)).sum()
    R = ret[idx].to(dtype)
    if clip_vloss:
        ov = old_v[idx].to(dtype)
        vc = ov + th.clamp(value - ov, -clip_coef, clip_coef)
        v_loss = 0.5 * th.max((value - R) ** 2, (vc - R) ** 2).mean()
    else:
        v_loss = 0.5 * ((value - R) ** 2).mean()
    ent = entropy.mean()
    loss = pg_loss - ent_coef * ent + vf_coef * v_loss
    grads = th.autograd.grad(loss, ps)
    with th.no_grad():
        stats = {"pg": pg_loss.item(), "v": v_loss.item(), "ent": ent.item(), "okl": (-logratio).mean().item(),
                 "kl": ((ratio - 1) - logratio).mean().item(), "clip": ((ratio - 1).abs() > clip_coef).to(dtype).mean().item()}
    return loss.detach(), [g.detach() for g in grads], stats
