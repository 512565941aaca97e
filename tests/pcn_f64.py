"""Float64 restatement of the default PCN model's forward, loss and backward (reference pcn.py:51-103, 213-234), for the kernel tests."""

from __future__ import annotations

import numpy as np

KEYS = ["s_emb.0.weight", "s_emb.0.bias", "c_emb.0.weight", "c_emb.0.bias", "fc.0.weight", "fc.0.bias", "fc.2.weight", "fc.2.bias"]


def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def forward(p: dict, scaling, obs, ret, hor, continuous: bool):
    """(pred, cache): log-probabilities (discrete) or predictions [N, A] in float64."""
    f = {k: np.asarray(v, np.float64) for k, v in p.items()}
    c = np.concatenate([np.asarray(ret, np.float64), np.asarray(hor, np.float64).reshape(-1, 1)], axis=1) * np.asarray(scaling, np.float64)
    obs = np.asarray(obs, np.float64)
    s = _sig(obs @ f["s_emb.0.weight"].T + f["s_emb.0.bias"])
    e = _sig(c @ f["c_emb.0.weight"].T + f["c_emb.0.bias"])
    x = s * e
    h = np.maximum(x @ f["fc.0.weight"].T + f["fc.0.bias"], 0.0)
    y = h @ f["fc.2.weight"].T + f["fc.2.bias"]
    if not continuous:
        z = y - y.max(axis=1, keepdims=True)
        y = z - np.log(np.exp(z).sum(axis=1, keepdims=True))
    return y, (f, obs, c, s, e, x, h)


def loss_and_grads(p: dict, scaling, obs, ret, hor, actions, continuous: bool):
    """(loss, entropy or None, pred, grads by state-dict key) of one minibatch."""
    y, (f, obs, c, s, e, x, h) = forward(p, scaling, obs, ret, hor, continuous)
    B, A = y.shape
    if continuous:
        diff = y - np.asarray(actions, np.float64)
        loss, ent = np.mean(diff * diff), None
        dy = 2.0 * diff / (B * A)
    else:
        a = np.asarray(actions).astype(np.int64).reshape(-1)
        loss = -np.mean(y[np.arange(B), a])
        prob = np.exp(y)
        ent = np.sum(-prob * y)
        onehot = np.zeros_like(y)
        onehot[np.arange(B), a] = 1.0
        dy = (prob - onehot) / B
    g = {"fc.2.weight": dy.T @ h, "fc.2.bias": dy.sum(0)}
    dh = (dy @ f["fc.2.weight"]) * (h > 0)
    g["fc.0.weight"], g["fc.0.bias"] = dh.T @ x, dh.sum(0)
    dx = dh @ f["fc.0.weight"]
    dzs, dze = dx * e * s * (1 - s), dx * s * e * (1 - e)
    g["s_emb.0.weight"], g["s_emb.0.bias"] = dzs.T @ obs, dzs.sum(0)
    g["c_emb.0.weight"], g["c_emb.0.bias"] = dze.T @ c, dze.sum(0)
    return loss, ent, y, g
