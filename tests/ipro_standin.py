"""Scripted runs of IPRO's and IPRO-2D's outer loop, shared by tests/golden/make_golden_ipro.py (which runs the reference's classes) and
the golden replay test (which runs this package's).

The learner is replaced after construction by :class:`ScriptedOracle`: ``train`` evaluates the utility it is given on a fixed finite point
set and returns a float64 copy of the best row, or, on chosen calls, that row lowered by 4 in every objective (a dominated answer, so
that a later call finds a point that beats it and ``replay`` runs).  All coordinates are multiples of 1/8 with |x| <= 64, so every box
volume and every partial hypervolume sum of a few hundred such points in d <= 4 is exact in float64: any exact hypervolume algorithm gives
the same bits, and the outer loop's discrete decisions can be compared exactly.
"""

from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from tests.nl_ppo_standin import RingVecEnv

MARGIN = 1e-5  # relative gap between the best and the second utility value: over 100 float32 rounding steps


class IproEnv(RingVecEnv):
    """The ring vector environment with the attributes an MOAgent reads at construction."""

    def __init__(self, num_envs=2, **kw):
        super().__init__(num_envs=num_envs, **kw)
        from morl_baselines_b200.testing import Discrete

        self.observation_space, self.action_space = self.single_observation_space, Discrete(self.single_action_space.n)
        self.unwrapped = self
        self.spec = SimpleNamespace(id="ring-v0")


def point_set(d: int, n: int, seed: int) -> np.ndarray:
    """n points in d objectives, multiples of 1/8: most near a sphere of radius 40 around (-8, ..., -8) (mutually non-dominated), a
    few inside it; every column has a unique maximum and minimum."""
    rng = np.random.default_rng(seed)
    while True:
        w = np.abs(rng.standard_normal((n, d))) + 0.05
        r = np.where(rng.random(n) < 0.8, 40.0, 40.0 * rng.random(n))
        pts = np.round(8 * (r[:, None] * w / np.linalg.norm(w, axis=1, keepdims=True) - 8.0)) / 8
        if all(np.sum(c == c.max()) == 1 and np.sum(c == c.min()) == 1 for c in pts.T):
            return pts


class ScriptedOracle:
    """Stands in for NLMOPPO: ``train(eval_env, u_func, pref, deterministic)`` returns the row of ``points`` with the largest utility
    (a fresh float64 array), lowered by 4 on the calls listed in ``dominated_calls`` (0-based)."""

    def __init__(self, points: np.ndarray, dominated_calls=(), check_margin: bool = True):
        self.points, self.dominated_calls, self.check_margin = np.asarray(points, dtype=np.float64), set(dominated_calls), check_margin
        self.calls, self.resets = 0, 0
        self.agent = "scripted-agent"

    def reset_agent(self, pref_dim):
        self.resets += 1

    def train(self, eval_env, u_func, pref=None, deterministic=False):
        import torch as th

        dev = pref.device if isinstance(pref, th.Tensor) else "cpu"
        vals = u_func(th.as_tensor(self.points, dtype=th.float32, device=dev)).double().cpu().numpy()
        order = np.argsort(-vals, kind="stable")
        if self.check_margin and len(vals) > 1:
            best, second = vals[order[0]], vals[order[1]]
            assert best - second > MARGIN * max(1.0, abs(best)), f"call {self.calls}: utility margin {best - second} too small"
        vec = self.points[order[0]].astype(np.float64).copy()
        if self.calls in self.dominated_calls:
            vec = vec - 4.0
        self.calls += 1
        return vec


# name -> class ("IPRO" / "IPRO2D"), d, number of points, point seed, constructor keywords, dominated calls (0-based), extrema given.
# A minimising run starts from given extrema: its linear phase maximises each objective, so it would bound the box from the wrong side.
CASES = {
    "ipro_d2_max": dict(cls="IPRO", d=2, n=24, pseed=1, ctor=dict(direction="maximize", max_iterations=10, update_freq=1), dominated=(),
                        extrema=False),
    "ipro_d2_min": dict(cls="IPRO", d=2, n=24, pseed=2, ctor=dict(direction="minimize", max_iterations=8, update_freq=2), dominated=(),
                        extrema=True),
    "ipro_d3_max_replay": dict(cls="IPRO", d=3, n=40, pseed=3, ctor=dict(direction="maximize", max_iterations=12, update_freq=1),
                               dominated=(6, 8, 10), extrema=False),
    "ipro_d3_min_extrema": dict(cls="IPRO", d=3, n=40, pseed=4, ctor=dict(direction="minimize", max_iterations=10, update_freq=2), dominated=(),
                                extrema=True),
    "ipro_d4_max_extrema": dict(cls="IPRO", d=4, n=48, pseed=5, ctor=dict(direction="maximize", max_iterations=10, update_freq=1), dominated=(),
                                extrema=True),
    "ipro_d4_max_replay": dict(cls="IPRO", d=4, n=48, pseed=6, ctor=dict(direction="maximize", max_iterations=10, update_freq=2),
                               dominated=(9, 11, 13), extrema=False),
    "ipro_d4_min_extrema": dict(cls="IPRO", d=4, n=48, pseed=9, ctor=dict(direction="minimize", max_iterations=8, update_freq=1), dominated=(),
                                extrema=True),
    "ipro2d_empty_queue": dict(cls="IPRO2D", d=2, n=12, pseed=7, ctor=dict(direction="maximize", max_iterations=40), dominated=(),
                               extrema=False),
    "ipro2d_replay": dict(cls="IPRO2D", d=2, n=24, pseed=8, ctor=dict(direction="maximize", max_iterations=12), dominated=(3, 5),
                          extrema=False),
}


def extrema_of(points: np.ndarray, sign: int):
    """(nadir, ideal) in the maximisation sign, widened by 1 (what the linear phase finds with offset 1)."""
    p = sign * points
    return p.min(axis=0) - 1, p.max(axis=0) + 1


def run_case(name: str, classes: dict, device: str = "auto"):
    """Run golden case ``name`` with the outer-loop classes {"IPRO": ..., "IPRO2D": ...}; returns a dict of arrays: every iteration's
    referent, pf, lower / upper points (IPRO), completed, robust points, open boxes (IPRO-2D: [k, 2, 2] nadir and ideal), hv,
    dominated_hv, discarded_hv, coverage, error and callback arguments, and the final front, Pareto set and counters."""
    c = CASES[name]
    # a minimising run gets the mirrored set, so that its front (in the maximisation sign) is as rich as a maximising run's
    points = point_set(c["d"], c["n"], c["pseed"]) * (-1 if c["ctor"]["direction"] == "minimize" else 1)
    env = IproEnv(num_envs=2, obs_dim=2, n_actions=3, d=c["d"])
    cls = classes[c["cls"]]
    kw = dict(tolerance=0.0, **c["ctor"])
    agent = cls(env, iter_total_timesteps=16, num_steps=8, anneal_lr=False, device=device, seed=11, log=False, **kw)
    oracle = ScriptedOracle(points, dominated_calls=c["dominated"])
    agent.agent = oracle
    out, rec = {}, {"iter": 0}

    decompose = agent.decompose_problem

    def recording_decompose(iteration, method="first"):
        sp = decompose(iteration, method)
        rec["referent"] = np.array(sp.referent, dtype=np.float64)
        return sp

    agent.decompose_problem = recording_decompose

    def snapshot(prefix):
        out[f"{prefix}/pf"] = np.array(agent.pf, dtype=np.float64).reshape(-1, c["d"])
        out[f"{prefix}/completed"] = np.array(agent.completed, dtype=np.float64).reshape(-1, c["d"])
        out[f"{prefix}/robust_points"] = np.array(agent.robust_points, dtype=np.float64).reshape(-1, c["d"])
        if c["cls"] == "IPRO":
            out[f"{prefix}/lower_points"] = np.array(agent.lower_points, dtype=np.float64).reshape(-1, c["d"])
            out[f"{prefix}/upper_points"] = np.array(agent.upper_points, dtype=np.float64).reshape(-1, c["d"])
        else:
            out[f"{prefix}/boxes"] = np.array([[b.nadir, b.ideal] for b in agent.box_queue], dtype=np.float64).reshape(-1, 2, 2)
        out[f"{prefix}/scalars"] = np.array([agent.hv, agent.dominated_hv, agent.discarded_hv, agent.coverage, agent.error], dtype=np.float64)

    def callback(iteration, hv, dominated_hv, discarded_hv, coverage, error):
        k = rec["iter"]
        out[f"it{k}/callback"] = np.array([iteration, hv, dominated_hv, discarded_hv, coverage, error], dtype=np.float64)
        out[f"it{k}/referent"] = rec["referent"]
        snapshot(f"it{k}")
        rec["iter"] = k + 1

    extrema = extrema_of(points, agent.sign) if c["extrema"] else None
    ps = agent.train(eval_env=None, ref_point=None, deterministic=True, extrema=extrema, callback=callback)
    snapshot("final")
    out["final/pareto_set"] = np.array([v for v, _ in ps], dtype=np.float64).reshape(-1, c["d"])
    out["final/counters"] = np.array([rec["iter"], agent.replay_triggered, oracle.calls, agent.total_hv], dtype=np.float64)
    out["points"] = points
    return out
