"""Golden vectors for Pareto Q-learning, produced by the unmodified reference's ``PQL`` on CPU (needs the reference's source tree, so it is
run by hand, not by the tests):
    python tests/golden/make_golden_pql.py   ->  tests/golden/pql.npz

Each case of ``tests/pql_standin.CASES`` trains the reference's agent on the treasure grid stand-in and records every action, every greedy
step's scores, the final epsilon, counts, averages and sets (canonical order), the local PCS and the return ``track_policy`` reaches for
each of its points, under ``<case>/...``.  pymoo's ``HV`` is replaced by the exact sweep of oracle/hv_oracle.py, ``gymnasium.spaces`` gets
the ``MultiDiscrete`` stand-in of morl_baselines_b200/testing.py.

Tie safety.  The device adds the volume's slabs in another order than the host sweep, so its scores may differ from the reference's in the
last bits; a case is reproducible bit for bit only if no greedy step hinges on that.  A seed is rejected when, at some greedy step of a
hypervolume case, (1) the maximum is an exact tie between actions whose Q-sets differ in their points above ``ref_point`` (the points that
span volume; equal spanning sets give equal volumes on both sides) and the maximum is not zero, or (2) the best score and the next distinct
one differ by less than 1e-9 relative.  It is also rejected when ``track_policy`` meets two vectors of one action that are equally close to
the target, or both within ``tol`` of it (the device scans them in canonical order, the reference in set order).  Seeds are tried from the
case's ``seed`` upwards; the accepted one is recorded.  A rerun writes the same bytes.
"""

from __future__ import annotations

import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from morl_baselines_b200.testing import MultiDiscrete  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
from tests.pql_standin import CASES, run_case  # noqa: E402

TRIES = 50


class Rejected(Exception):
    pass


class TieCheck:
    def __init__(self, case):
        self.hv = case["action_eval"] == "hypervolume"
        self.ref = np.array(case["ref"], dtype=np.float64)

    def score(self, agent, state, scores):
        if not self.hv:
            return
        best = scores.max()
        tied = np.flatnonzero(scores == best)
        if len(tied) > 1 and best != 0.0:
            spans = [{q for q in agent.get_q_set(state, a) if np.all(np.array(q) > self.ref)} for a in tied]
            if any(s != spans[0] for s in spans[1:]):
                raise Rejected(f"exact tie at {best} between differing Q-sets, state {state}")
        rest = scores[scores < best]
        if rest.size and best - rest.max() < 1e-9 * abs(best):
            raise Rejected(f"near tie {best} vs {rest.max()}, state {state}")

    def track(self, agent, point, env, tol=1e-3):
        """The reference's track_policy loop, raising where the scan order within one action could change its outcome."""
        target = np.array(point)
        state, _ = env.reset()
        terminated = truncated = False
        while not (terminated or truncated):
            state = agent._get_state_index(state)
            closest_dist, closest_action, found, new_target = np.inf, 0, False, target
            for action in range(agent.num_actions):
                im_rew = agent.avg_reward[state, action]
                qs = [np.array(q) for q in agent.non_dominated[state][action]]
                dists = [np.sum(np.abs(agent.gamma * q + im_rew - target)) for q in qs]
                if sum(d < tol for d in dists) > 1:
                    raise Rejected(f"two vectors within tol in state {state}, action {action}")
                best = min(dists)
                if best < closest_dist and sum(d == best for d in dists) > 1:
                    raise Rejected(f"equally close vectors in state {state}, action {action}")
                for q, dist in zip(qs, dists):
                    if dist < closest_dist:
                        closest_dist, closest_action, new_target = dist, action, q
                        if dist < tol:
                            found = True
                            break
                if found:
                    break
            state, _, terminated, truncated, _ = env.step(closest_action)
            target = new_target


def main():
    rh.install_stubs()
    sys.modules["gymnasium.spaces"].MultiDiscrete = MultiDiscrete
    pql = rh.import_reference("morl_baselines.multi_policy.pareto_q_learning.pql")
    out = {}
    for name, case in CASES.items():
        for seed in range(case["seed"], case["seed"] + TRIES):
            try:
                _, rec = run_case(name, pql.PQL, seed, check=TieCheck(case))
                break
            except Rejected as e:
                print(f"{name}: seed {seed} rejected: {e}")
        else:
            raise RuntimeError(f"{name}: no tie-safe seed in {TRIES} tries")
        print(f"{name}: seed {seed}, {len(rec['greedy_step'])} greedy steps, |pcs| = {len(rec['pcs'])}, max set {rec['nd'].shape[2]}")
        out.update({f"{name}/{k}": v for k, v in rec.items()})
    # fixed member order and timestamps, so a rerun gives the same bytes
    path = os.path.join(HERE, "pql.npz")
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(out[k]), allow_pickle=False)
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(zi, buf.getvalue())
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
