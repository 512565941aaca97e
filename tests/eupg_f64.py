"""EUPG's episode update restated in float64 numpy (reference eupg.py:236-251): forward through the Linear/Tanh stack, p = sigmoid(z) /
sum sigmoid(z) per row, log p of the taken action clamped to [eps, 1 - eps] with eps = 2^-23 (zero gradient where the clamp acts),
loss = -mean(logp * v) and the gradient of every parameter, written out by hand."""

from __future__ import annotations

import numpy as np

EPS = float(np.finfo(np.float32).eps)


def forward(params, x):
    """params: [W_0, b_0, ..., W_L, b_L]; x [T, S + d].  Returns the layer inputs, the sigmoids and p."""
    acts = [np.asarray(x, np.float64)]
    L = len(params) // 2
    for l in range(L):
        z = acts[-1] @ np.asarray(params[2 * l], np.float64).T + np.asarray(params[2 * l + 1], np.float64)
        if l < L - 1:
            acts.append(np.tanh(z))
    sg = 1.0 / (1.0 + np.exp(-z))
    return acts, sg, sg / sg.sum(axis=1, keepdims=True)


def probs(params, x) -> np.ndarray:
    return forward(params, x)[2]


def update(params, x, actions, v, eps: float = EPS):
    """Loss and gradients [dW_0, db_0, ...] of -mean(logp(actions) * v); v is [T] or a scalar.  ``eps`` is the clamp of the dtype the
    network runs in (torch.finfo(dtype).eps): float32 by default."""
    acts, sg, p = forward(params, x)
    T = x.shape[0]
    a = np.asarray(actions, np.int64).reshape(T)
    v = np.broadcast_to(np.asarray(v, np.float64), (T,))
    pa = p[np.arange(T), a]
    passes = (pa >= eps) & (pa <= 1.0 - eps)
    logp = np.log(np.clip(pa, eps, 1.0 - eps))
    loss = -np.mean(logp * v)
    g = np.where(passes, -v / T, 0.0)  # d loss / d log p_a
    onehot = np.zeros_like(p)
    onehot[np.arange(T), a] = 1.0
    dz = g[:, None] * (1.0 - sg) * (onehot - p)
    L = len(params) // 2
    grads = [None] * len(params)
    for l in range(L - 1, -1, -1):
        grads[2 * l] = dz.T @ acts[l]
        grads[2 * l + 1] = dz.sum(axis=0)
        if l > 0:
            dz = (dz @ np.asarray(params[2 * l], np.float64)) * (1.0 - acts[l] ** 2)
    return loss, grads


def returns(rewards: np.ndarray, gamma: float) -> np.ndarray:
    """The reference's loop c = gamma * c + r_t run backward, in float32 (product and sum rounded separately)."""
    r = np.asarray(rewards, np.float32)
    out = np.empty_like(r)
    c = np.zeros(r.shape[1], np.float32)
    g = np.float32(gamma)
    for t in range(len(r) - 1, -1, -1):
        c = (g * c).astype(np.float32) + r[t]
        out[t] = c
    return out
