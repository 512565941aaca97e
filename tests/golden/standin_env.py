"""Stand-in vector-reward MDP for the hypervolume-parity protocol (SURVEY.md section 8(d): "If mo-gymnasium is unavailable on the
build box, use an in-repo stand-in vector-reward MDP for *both* engines and say so").  mo-gymnasium is not installed here, so the
reference (CPU, golden generation) and the CUDA engine (GPU test) are both trained on this environment.

TreasureChain: a 3-objective chain in the spirit of deep-sea-treasure.  Positions x = 0..2; every step costs TIME_COST units of
time (objective 2).  Actions: 0 = move right (walking off the end of the chain terminates the episode empty-handed), 1 = collect
treasure A (terminal), 2 = collect treasure B (terminal) -- every episode terminates within N_POS steps, no time-limit truncation.
Both treasures grow with x (concave), so the 6 "go to x, collect A|B" policies are mutually non-dominated and each is optimal for
some linear weight.  The constants were chosen (random search) so that every policy has an evaluation weight for which it beats the
runner-up by more than 1.0 in scalarised discounted return (about 6 % of the value scale): the hypervolume of a correctly trained
agent does not hinge on near-ties.  Deterministic; observations are one-hot position + elapsed-time fraction.
Spaces come from oracle.ref_harness (the gymnasium stand-ins both engines accept); action sampling is seeded per environment.
"""

from __future__ import annotations

import numpy as np

from oracle.ref_harness import Box, Discrete, _Spec

TA = np.array([10.0, 18.0, 21.0])
TB = np.array([12.0, 22.0, 25.5])
TIME_COST = 4.0
N_POS = 3
HORIZON = 3


class TreasureChain:
    def __init__(self, seed: int = 0):
        self.observation_space = Box(0.0, 1.0, shape=(N_POS + 1,))
        self.action_space = Discrete(3)
        self.action_space.seed(seed)
        self.reward_space = Box(-np.inf, np.inf, shape=(3,))
        self.reward_dim = 3
        self.unwrapped = self
        self.spec = _Spec("treasure-chain-v0")
        self.metadata = {"render_modes": []}
        self._x = 0
        self._t = 0

    def _obs(self):
        o = np.zeros(N_POS + 1, dtype=np.float32)
        o[self._x] = 1.0
        o[N_POS] = self._t / HORIZON
        return o

    def reset(self, seed=None, options=None):
        self._x, self._t = 0, 0
        return self._obs(), {}

    def step(self, action):
        a = int(action)
        r = np.array([0.0, 0.0, -TIME_COST], dtype=np.float32)
        terminated = False
        if a == 0:
            if self._x == N_POS - 1:
                terminated = True
            else:
                self._x += 1
        elif a == 1:
            r[0] = TA[self._x]
            terminated = True
        elif a == 2:
            r[1] = TB[self._x]
            terminated = True
        self._t += 1
        truncated = (not terminated) and self._t >= HORIZON
        return self._obs(), r, terminated, truncated, {}

    def pareto_front(self, gamma: float):
        """Discounted returns of the 2 * N_POS 'move right x times, then collect' policies."""
        pts = []
        for x in range(N_POS):
            time = -TIME_COST * sum(gamma**k for k in range(x + 1))
            pts.append(np.array([gamma**x * TA[x], 0.0, time]))
            pts.append(np.array([0.0, gamma**x * TB[x], time]))
        return pts


def robust_eval_weights(gamma: float, per_policy: int = 2, steps: int = 20, min_time_steps: int = 2):
    """Deterministic evaluation-weight list shared by both engines: for every policy of the true front, the ``per_policy`` interior
    grid weights (components k / steps, all > 0) for which it wins with the largest margin over the runner-up."""
    pts = np.array(TreasureChain().pareto_front(gamma))
    grid = []
    for a in range(1, steps):
        for b in range(1, steps - a):
            c = steps - a - b
            if c >= min_time_steps:
                grid.append(np.array([a, b, c], dtype=np.float64) / steps)
    grid = np.array(grid)
    scores = grid @ pts.T
    order = np.argsort(-scores, axis=1, kind="stable")
    rows = np.arange(len(grid))
    win, gap = order[:, 0], scores[rows, order[:, 0]] - scores[rows, order[:, 1]]
    out = []
    for p in range(len(pts)):
        idx = np.nonzero(win == p)[0]
        idx = idx[np.argsort(-gap[idx], kind="stable")][:per_policy]
        out.extend((grid[i].astype(np.float32), float(gap[i]), p) for i in idx)
    return out


HV_REF_POINT = np.array([-1.0, -1.0, -(TIME_COST * HORIZON + 1.0)])
