"""Golden cases of multi-policy MO Q-learning, run on the treasure grid stand-in (tests/pql_standin.py) by the reference's MPMOQLearning
and by this package's, and the per-iteration record both sides produce.

d = 2 is deterministic; d = 3 slips with probability 0.2 and burns extra fuel, so a state-action pair has two outcomes and the Dyna model's
``random.choices`` matters.  Every case seeds python's ``random``, numpy's legacy global generator, the agent, both environments and the
training environment's action sampler."""

from __future__ import annotations

import random

import numpy as np

from tests.linear_support_oracle import corners_oracle, max_value_lp_oracle
from tests.pql_standin import TreasureGrid

BASE = dict(learning_rate=0.3, gamma=0.9, initial_epsilon=0.3, final_epsilon=0.3)
CASES = {
    "rand_d2": dict(d=2, slip=0.0, iters=3, steps=800, seed=1, kw=dict(use_gpi_policy=False, transfer_q_table=True)),
    "rand_d2_notransfer": dict(d=2, slip=0.0, iters=3, steps=800, seed=11, kw=dict(use_gpi_policy=False, transfer_q_table=False)),
    "rand_gpi_d2": dict(d=2, slip=0.0, iters=3, steps=800, seed=21, kw=dict(use_gpi_policy=True, transfer_q_table=True)),
    "rand_gpi_d3_notransfer": dict(d=3, slip=0.2, iters=3, steps=800, seed=31, kw=dict(use_gpi_policy=True, transfer_q_table=False)),
    "dyna_d3": dict(d=3, slip=0.2, iters=3, steps=600, seed=41, kw=dict(dyna=True, dyna_updates=5)),
    "dyna_pd_gpi_d3": dict(d=3, slip=0.2, iters=3, steps=600, seed=51, kw=dict(dyna=True, dyna_updates=5, gpi_pd=True, use_gpi_policy=True)),
    "ols_d2": dict(d=2, slip=0.0, iters=5, steps=600, seed=61, kw=dict(weight_selection_algo="ols", epsilon_ols=0.0)),
    "gpils_d2": dict(d=2, slip=0.0, iters=4, steps=600, seed=71, kw=dict(weight_selection_algo="gpi-ls", use_gpi_policy=True)),
}
ENV_SEED, EVAL_SEED, SAMPLER_SEED = 5, 6, 7
REF_POINT = np.array([0.0, -25.0, -25.0])


def _sorted_table(q_table: dict):
    keys = sorted(tuple(int(x) for x in k) for k in q_table)
    lookup = {tuple(int(x) for x in k): v for k, v in q_table.items()}
    return np.array(keys, dtype=np.int64).reshape(len(keys), 2), np.array([lookup[k] for k in keys], dtype=np.float64)


def model_record(pairs, outcomes, leaves, d):
    """pairs [(state tuple, action)] in model order; outcomes [[((next state tuple), reward tuple, terminal), count]] per pair in dict
    order; leaves: the tree's first len(pairs) leaves (or None)."""
    rec = dict(pair_state=np.array([p[0] for p in pairs], dtype=np.int64).reshape(len(pairs), 2),
               pair_action=np.array([p[1] for p in pairs], dtype=np.int64))
    flat = [(i, k, c) for i, outs in enumerate(outcomes) for k, c in outs]
    rec["out_pair"] = np.array([f[0] for f in flat], dtype=np.int64)
    rec["out_next"] = np.array([f[1][0] for f in flat], dtype=np.int64).reshape(len(flat), 2)
    rec["out_reward"] = np.array([f[1][1] for f in flat], dtype=np.float64).reshape(len(flat), d)
    rec["out_term"] = np.array([bool(f[1][2]) for f in flat], dtype=np.int64)
    rec["out_count"] = np.array([f[2] for f in flat], dtype=np.int64)
    if leaves is not None:
        rec["leaves"] = np.asarray(leaves, dtype=np.float64)
    return rec


def run_case(name: str, cls, seed: int, model_view, hook=None):
    """Train ``cls`` (the reference's MPMOQLearning or this package's) on case ``name``, one ``train`` call per iteration, and return the
    record: per iteration the weight, the training environment's actions, every policy's sorted q_table, ε, the policy count, the CCS and
    the model (``model_view(agent)`` -> (pairs, outcomes, leaves)).  Both sides take OLS's corner weights and optimistic bound from
    tests/linear_support_oracle.py.  ``hook(agent)``, if given, runs after construction."""
    c = CASES[name]
    d = c["d"]
    random.seed(seed)
    np.random.seed(seed)
    env = TreasureGrid(d=d, slip=c["slip"], seed=ENV_SEED)
    env.action_space.seed(SAMPLER_SEED)
    eval_env = TreasureGrid(d=d, slip=c["slip"], seed=EVAL_SEED)
    agent = cls(env, seed=seed, log=False, **BASE, **c["kw"])
    ls = agent.linear_support
    ls.verbose = False
    ls.compute_corner_weights = lambda: list(corners_oracle(np.vstack(ls.ccs)))
    ls.max_value_lp = lambda w_new: max_value_lp_oracle(ls.ccs, ls.visited_weights, w_new)
    if hook is not None:
        hook(agent)
    actions = []
    step = env.step

    def rec_step(a):
        actions.append(int(a))
        return step(a)

    env.step = rec_step
    weights = []
    orig_add = agent.linear_support.add_solution

    def add_solution(value, w):
        weights.append(np.array(w, dtype=np.float64))
        return orig_add(value, w)

    agent.linear_support.add_solution = add_solution
    rec = {}
    for it in range(c["iters"]):
        n0 = len(actions)
        agent.train(total_timesteps=c["steps"], eval_env=eval_env, ref_point=REF_POINT[:d], timesteps_per_iteration=c["steps"],
                    num_eval_episodes_for_front=1)
        r = {"weight": weights[-1], "actions": np.array(actions[n0:], dtype=np.int64),
             "epsilon": np.array([p.epsilon for p in agent.policies], dtype=np.float64),
             "n_policies": np.array([len(agent.policies)], dtype=np.int64),
             "ccs": np.array(agent.linear_support.ccs, dtype=np.float64).reshape(-1, d)}
        for j, p in enumerate(agent.policies):
            r[f"q{j}_keys"], r[f"q{j}_values"] = _sorted_table(p.q_table)
        if c["kw"].get("dyna"):
            r.update(model_record(*model_view(agent), d))
        rec.update({f"{it}/{k}": v for k, v in r.items()})
    env.step = step
    rec["seed"] = np.array([seed], dtype=np.int64)
    return agent, rec


def device_model_view(agent):
    """(pairs, outcomes, leaves) of this package's agent, from the host index and one copy of the device model."""
    st = agent._store
    idx, t = st.index, st.table
    pairs = [(idx.states[s], a) for s, a in idx.pairs]
    counts = t.counts.cpu().numpy()
    outcomes = [[((idx.states[k[0]], k[1], k[2]), int(counts[m, o])) for k, o in outs.items()] for m, outs in enumerate(idx.outcomes)]
    leaves = None
    if agent.gpi_pd:
        leaves = t.tree.cpu().numpy()[(1 << 17) - 1:][: len(pairs)]
    return pairs, outcomes, leaves
