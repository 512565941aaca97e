"""A small treasure grid world for Pareto Q-learning, and the golden cases run on it by both the reference's PQL and this package's.

mo-gymnasium is not installed here, so this stands in for deep-sea-treasure: integer-Box ``(row, col)`` observations (the
``ravel_multi_index`` path of ``_get_state_index``), four moves, walls and borders that leave the agent where it is (self-loops), terminal
treasures and a time limit.  Its map and values are this file's own.

- d = 2: reward (treasure, -1 per step), deterministic.
- d = 3: reward (treasure, -1 per step, -fuel), where a move slips with probability ``slip`` (the environment's own seeded generator) and
  then burns extra fuel; the agent still lands where it meant to, so the transitions stay deterministic, but the averages of
  ``avg_reward`` really average.
"""

from __future__ import annotations

import copy

import numpy as np

from morl_baselines_b200.testing import Box, Discrete, _Spec

MAP = [
    "S......",
    "a......",
    "#b.....",
    "##c....",
    "###d...",
    "####e.f",
]
TREASURE = {"a": 1.7, "b": 3.9, "c": 6.1, "d": 9.4, "e": 12.3, "f": 15.8}
MOVES = [(-1, 0), (1, 0), (0, -1), (0, 1)]  # up, down, left, right
FUEL = [0.21, 0.43, 0.17, 0.29]  # per intended move (d = 3)
SLIP_FUEL = 0.35


class TreasureGrid:
    def __init__(self, d: int = 2, slip: float = 0.0, seed: int = 0, horizon: int = 20):
        assert d in (2, 3)
        self.rows, self.cols = len(MAP), len(MAP[0])
        self.observation_space = Box(low=np.zeros(2), high=np.array([self.rows - 1, self.cols - 1]), dtype=np.dtype(np.int32))
        self.action_space = Discrete(4)
        self.reward_space = Box(-np.inf, np.inf, shape=(d,))
        self.reward_dim = d
        self.d, self.slip, self.horizon = d, slip, horizon
        self.unwrapped = self
        self.spec = _Spec(f"treasure-grid-d{d}-v0")
        self.metadata = {"render_modes": []}
        self._rng = np.random.default_rng(seed)
        self._pos = (0, 0)
        self._t = 0

    def reset(self, seed=None, options=None):
        if seed is not None:
            self._rng = np.random.default_rng(seed)
        self._pos, self._t = (0, 0), 0
        return np.array(self._pos, dtype=np.int32), {}

    def step(self, action):
        action = int(action)
        slipped = self.slip > 0.0 and self._rng.uniform() < self.slip
        r, c = self._pos[0] + MOVES[action][0], self._pos[1] + MOVES[action][1]
        if 0 <= r < self.rows and 0 <= c < self.cols and MAP[r][c] != "#":
            self._pos = (r, c)
        self._t += 1
        cell = MAP[self._pos[0]][self._pos[1]]
        treasure = TREASURE.get(cell, 0.0)
        rew = [treasure, -1.0] + ([-(FUEL[action] + (SLIP_FUEL if slipped else 0.0))] if self.d == 3 else [])
        terminated = cell in TREASURE
        truncated = self._t >= self.horizon
        return np.array(self._pos, dtype=np.int32), np.array(rew, dtype=np.float32), terminated, truncated, {}


# golden cases: environment, agent and training settings.  `seed` is the first agent seed tried by tests/golden/make_golden_pql.py, which
# records the seed it accepted.
CASES = {
    "hv_d2_g1": dict(d=2, slip=0.0, gamma=1.0, ref=(0.0, -25.0), action_eval="hypervolume", steps=3000, seed=1),
    "hv_d2_g099": dict(d=2, slip=0.0, gamma=0.99, ref=(0.0, -25.0), action_eval="hypervolume", steps=3000, seed=11),
    "hv_d3_slip": dict(d=3, slip=0.15, gamma=0.95, ref=(0.0, -25.0, -25.0), action_eval="hypervolume", steps=3000, seed=21),
    "card_d2": dict(d=2, slip=0.0, gamma=1.0, ref=(0.0, -25.0), action_eval="pareto_cardinality", steps=3000, seed=31),
}
EPS = dict(initial_epsilon=1.0, epsilon_decay_steps=2000, final_epsilon=0.1)
ENV_SEED, EVAL_SEED = 5, 6


def canonical(points) -> np.ndarray:
    """Points in the device table's canonical order: descending coordinate sum (added left to right), ties lexicographically descending."""
    pts = [tuple(float(x) for x in p) for p in points]

    def key(p):
        acc = p[0]
        for x in p[1:]:
            acc = acc + x
        return (acc,) + p

    return np.array(sorted(pts, key=key, reverse=True), dtype=np.float64).reshape(len(pts), -1)


def run_case(name: str, pql_cls, seed: int, check=None, **kw):
    """Train ``pql_cls`` (the reference's PQL or this package's) on case ``name`` with agent seed ``seed``.  Returns the agent and the
    record: every action, every greedy step's (step, state, scores), the final epsilon, counts, avg_reward and sets, the local PCS and the
    return ``track_policy`` reaches for each of its points (canonical order).  ``check``, if given, sees every greedy step's scores
    (``check.score(agent, state, scores)``) and a copy of the evaluation environment before each tracked point
    (``check.track(agent, point, env_copy)``)."""
    c = CASES[name]
    env = TreasureGrid(d=c["d"], slip=c["slip"], seed=ENV_SEED)
    eval_env = TreasureGrid(d=c["d"], slip=c["slip"], seed=EVAL_SEED)
    ref = np.array(c["ref"], dtype=np.float64)
    agent = pql_cls(env, ref, gamma=c["gamma"], seed=seed, log=False, **EPS, **kw)
    actions, greedy = [], []
    step = env.step

    def rec_step(a):
        actions.append(int(a))
        return step(a)

    env.step = rec_step
    attr = "score_hypervolume" if c["action_eval"] == "hypervolume" else "score_pareto_cardinality"
    score = getattr(agent, attr)

    def rec_score(state):
        out = score(state)
        if check is not None:
            check.score(agent, int(state), np.array(out, dtype=np.float64))
        greedy.append((agent.global_step, int(state), np.array(out, dtype=np.float64)))
        return out

    setattr(agent, attr, rec_score)
    pcs = agent.train(total_timesteps=c["steps"], eval_env=eval_env, ref_point=ref, action_eval=c["action_eval"], log_every=10**9)
    setattr(agent, attr, score)
    env.step = step
    pcs = canonical(pcs)
    tracked = []
    for p in pcs:
        if check is not None:
            check.track(agent, p, copy.deepcopy(eval_env))
        tracked.append(agent.track_policy(p, eval_env))
    tracked = np.array(tracked, dtype=np.float64).reshape(len(pcs), -1)
    nd = agent.non_dominated
    S, A = len(nd), len(nd[0])
    K = max(len(x) for row in nd for x in row)
    nd_arr = np.zeros((S, A, K, c["d"]))
    nd_count = np.zeros((S, A), dtype=np.int32)
    for s in range(S):
        for a in range(A):
            pts = canonical(nd[s][a])
            nd_arr[s, a, : len(pts)] = pts
            nd_count[s, a] = len(pts)
    record = dict(
        actions=np.array(actions, dtype=np.int64),
        greedy_step=np.array([g[0] for g in greedy], dtype=np.int64),
        greedy_state=np.array([g[1] for g in greedy], dtype=np.int64),
        greedy_scores=np.array([g[2] for g in greedy], dtype=np.float64).reshape(len(greedy), A),
        epsilon=np.array([agent.epsilon], dtype=np.float64),
        counts=np.asarray(agent.counts, dtype=np.float64),
        avg_reward=np.asarray(agent.avg_reward, dtype=np.float64),
        nd=nd_arr,
        nd_count=nd_count,
        pcs=pcs,
        tracked=tracked,
        seed=np.array([seed], dtype=np.int64),
    )
    return agent, record
