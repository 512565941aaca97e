"""Evaluation utilities (mirrors reference morl_baselines/common/evaluation.py).  Rollouts stay on the host (env-bound);
the Pareto prune of the evaluated front runs on the GPU (common/pareto.py)."""

from __future__ import annotations

import os
import random
from typing import List, Optional, Tuple

import numpy as np
import torch as th


def eval_mo(agent, env, w: Optional[np.ndarray] = None, scalarization=np.dot, render: bool = False) -> Tuple[float, float, np.ndarray, np.ndarray]:
    """One evaluation episode: (scalarised return, scalarised discounted return, vector return, discounted vector return)
    (reference evaluation.py:23-67)."""
    obs, _ = env.reset()
    done = False
    vec_return, disc_vec_return = np.zeros_like(w), np.zeros_like(w)
    gamma = 1.0
    while not done:
        if render:
            env.render()
        obs, r, terminated, truncated, info = env.step(agent.eval(obs, w))
        done = terminated or truncated
        vec_return += r
        disc_vec_return += gamma * r
        gamma *= agent.gamma
    if w is None:
        return scalarization(vec_return), scalarization(disc_vec_return), vec_return, disc_vec_return
    return scalarization(w, vec_return), scalarization(w, disc_vec_return), vec_return, disc_vec_return


def eval_mo_reward_conditioned(agent, env, scalarization=np.dot, w: Optional[np.ndarray] = None, render: bool = False, **kwargs):
    """One episode of an accrued-reward-conditioned (ESR) agent (reference evaluation.py:70-115)."""
    obs, _ = env.reset()
    done = False
    d = env.unwrapped.reward_space.shape[0]
    vec_return, disc_vec_return = np.zeros(d), np.zeros(d)
    gamma = 1.0
    while not done:
        if render:
            env.render()
        obs, r, terminated, truncated, info = env.step(agent.eval(obs, disc_vec_return, **kwargs))
        done = terminated or truncated
        vec_return += r
        disc_vec_return += gamma * r
        gamma *= agent.gamma
    if w is None:
        return scalarization(vec_return), scalarization(disc_vec_return), vec_return, disc_vec_return
    return scalarization(vec_return, w), scalarization(disc_vec_return, w), vec_return, disc_vec_return


def policy_evaluation_mo(agent, env, w: np.ndarray, scalarization=np.dot, rep: int = 5):
    """Average of ``rep`` evaluation episodes (reference evaluation.py:118-144)."""
    evals = [eval_mo(agent=agent, env=env, w=w, scalarization=scalarization) for _ in range(rep)]
    return (np.mean([e[0] for e in evals]), np.mean([e[1] for e in evals]), np.mean([e[2] for e in evals], axis=0),
            np.mean([e[3] for e in evals], axis=0))


def policy_evaluation_mo_batched(agent, env, weights: List[np.ndarray], rep: int = 5, seeds: Optional[List[int]] = None, weight_dtype=np.float32):
    """All ``len(weights) * rep`` evaluation episodes of an evaluation round in LOCKSTEP on copies of ``env`` (SURVEY.md 8(f)4): the
    reference evaluates one (weight, episode) after the other, one single-row network call per environment step
    (evaluation.py:118-144 called from a python loop, e.g. envelope.py:545-557: 100 weights x 5 episodes); here every environment step
    of the whole round is ONE batched ``agent.eval_batch(obs [N, ...], w [N, d])`` call -- one device round trip per step instead of N.

    Returns, per weight, the tuple of ``policy_evaluation_mo``: (scalarised return, scalarised discounted return, vector return,
    discounted vector return), each averaged over the ``rep`` episodes (scalarisation: np.dot, as the default of the serial routine).
    Identical to the serial routine for deterministic environments; a stochastic environment's copies share the RNG state of ``env``
    unless ``seeds`` (one per episode, passed to ``reset``) is given.  The weights and the return accumulators have ``weight_dtype``
    (``np.zeros_like(w)`` of the serial routine): pass np.float64 to match serial calls made with float64 weights."""
    from copy import deepcopy

    if not hasattr(agent, "eval_batch"):
        raise NotImplementedError(f"{type(agent).__name__} has no eval_batch(obs, w): use policy_evaluation_mo")
    n_w = len(weights)
    N = n_w * rep
    envs = [deepcopy(env) for _ in range(N)]
    w_all = np.repeat(np.asarray(weights, dtype=weight_dtype), rep, axis=0)  # episode e of weight i sits at row i * rep + e
    obs = []
    for k, e in enumerate(envs):
        o, _ = e.reset(seed=None if seeds is None else seeds[k % rep])
        obs.append(np.asarray(o))
    # per-episode accumulators with the serial routine's dtypes and operation order (np.zeros_like(w); python-float discount)
    vec = [np.zeros_like(w_all[k]) for k in range(N)]
    disc = [np.zeros_like(w_all[k]) for k in range(N)]
    gamma = [1.0] * N
    alive = np.ones(N, dtype=bool)
    obs = np.stack(obs)
    while alive.any():
        idx = np.nonzero(alive)[0]
        acts = agent.eval_batch(obs[idx], w_all[idx])
        for a, k in zip(acts, idx):
            o, r, terminated, truncated, _ = envs[k].step(a)
            vec[k] += r
            disc[k] += gamma[k] * r
            gamma[k] *= agent.gamma
            obs[k] = o
            alive[k] = not (terminated or truncated)
    out = []
    for i in range(n_w):
        sl = slice(i * rep, (i + 1) * rep)
        w = np.asarray(weights[i])
        out.append((np.mean([np.dot(w, v) for v in vec[sl]]), np.mean([np.dot(w, v) for v in disc[sl]]), np.mean(vec[sl], axis=0),
                    np.mean(disc[sl], axis=0)))
    return out


def multi_policy_metrics(current_front: List[np.ndarray], hv_ref_point: np.ndarray, reward_dim: int, n_sample_weights: int = 50,
                         ref_front: Optional[List[np.ndarray]] = None) -> dict:
    """The metric values of ``log_all_multi_policy_metrics`` as a dictionary with the reference's wandb key names
    (reference evaluation.py:147-200): hypervolume, sparsity, EUM, cardinality (+ IGD / MUL with a known front)."""
    from .pareto import filter_pareto_dominated
    from .performance_indicators import cardinality, expected_utility, hypervolume, igd, maximum_utility_loss, sparsity
    from .weights import equally_spaced_weights

    filtered = list(filter_pareto_dominated(current_front))
    weights = equally_spaced_weights(reward_dim, n_sample_weights)
    out = {
        "eval/hypervolume": hypervolume(hv_ref_point, filtered),
        "eval/sparsity": sparsity(filtered),
        "eval/eum": expected_utility(filtered, weights_set=weights),
        "eval/cardinality": cardinality(filtered),
        "front": filtered,
    }
    if ref_front is not None:
        out["eval/igd"] = igd(known_front=ref_front, current_estimate=filtered)
        out["eval/mul"] = maximum_utility_loss(front=filtered, reference_set=ref_front, weights_set=np.array(weights))
    return out


def log_all_multi_policy_metrics(current_front: List[np.ndarray], hv_ref_point: np.ndarray, reward_dim: int, global_step: int,
                                 n_sample_weights: int = 50, ref_front: Optional[List[np.ndarray]] = None):
    """Compute the front metrics and log them to wandb under the reference's keys (reference evaluation.py:147-200)."""
    import wandb

    m = multi_policy_metrics(current_front, hv_ref_point, reward_dim, n_sample_weights, ref_front)
    front = m.pop("front")
    wandb.log({**m, "global_step": global_step}, commit=False)
    table = wandb.Table(columns=[f"objective_{i}" for i in range(1, reward_dim + 1)], data=[p.tolist() for p in front])
    wandb.log({"eval/front": table})


def seed_everything(seed: int):
    """Seed python, numpy and torch (reference evaluation.py:203-218)."""
    random.seed(seed)
    os.environ["PYTHONHASHSEED"] = str(seed)
    np.random.seed(seed)
    th.manual_seed(seed)
    th.cuda.manual_seed(seed)
    th.backends.cudnn.deterministic = True
    th.backends.cudnn.benchmark = True


def log_episode_info(info: dict, scalarization, weights: Optional[np.ndarray], global_timestep: int, id: Optional[int] = None,
                     verbose: bool = True):
    """Log the statistics of a finished episode (reference evaluation.py:221-277; keys r, dr, l, t of MORecordEpisodeStatistics)."""
    import wandb

    episode_ts, episode_time = info["l"], info["t"]
    episode_return, disc_episode_return = info["r"], info["dr"]
    if weights is None:
        scal_return, disc_scal_return = scalarization(episode_return), scalarization(disc_episode_return)
    else:
        scal_return, disc_scal_return = scalarization(episode_return, weights), scalarization(disc_episode_return, weights)
    if verbose:
        print(f"Episode infos:\nSteps: {episode_ts}, Time: {episode_time}\nTotal Reward: {episode_return}, Discounted: {disc_episode_return}")
        print(f"Scalarized Reward: {scal_return}, Discounted: {disc_scal_return}")
    idstr = "" if id is None else "_" + str(id)
    wandb.log({f"charts{idstr}/timesteps_per_episode": episode_ts, f"charts{idstr}/episode_time": episode_time,
               f"metrics{idstr}/scalarized_episode_return": scal_return,
               f"metrics{idstr}/discounted_scalarized_episode_return": disc_scal_return, "global_step": global_timestep}, commit=False)
    for i in range(episode_return.shape[0]):
        wandb.log({f"metrics{idstr}/episode_return_obj_{i}": episode_return[i],
                   f"metrics{idstr}/disc_episode_return_obj_{i}": disc_episode_return[i]})
