"""Golden vectors for multi-policy MO Q-learning, produced by the unmodified reference's ``MPMOQLearning`` on CPU (needs the reference's
source tree, so it is run by hand, not by the tests):
    python tests/golden/make_golden_mp_moq.py   ->  tests/golden/mp_moq.npz

Each case of ``tests/mp_moq_cases.CASES`` trains the reference's agent on the treasure grid stand-in and records, per iteration, the weight,
every action, every policy's sorted q_table, ε, the policy count, the CCS and the Dyna model (pair order, outcomes, counts, tree leaves),
under ``<case>/<iteration>/...``.  ``equally_spaced_weights`` (pymoo) is replaced by a stub that is never reached with ``log=False``.

Tie safety.  The device adds w . q left to right; numpy's dot may round differently in the last bit.  A greedy decision (own policy or
GPI) whose values all equal the left-to-right sums is reproduced exactly, ties included.  Otherwise a seed is rejected when the decision's
best and runner-up distinct values lie within 1e-9 relative, or it is an exact tie between entries whose Q vectors differ; it is also
rejected when a prioritised walk's query lies within 1e-9 relative of a left sum it is compared with.  Seeds are tried from the
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

from oracle import ref_harness as rh  # noqa: E402
from tests.mp_moq_cases import CASES, run_case  # noqa: E402

TRIES = 40
REL = 1e-9


class Rejected(Exception):
    pass


def seq_dot(v, w) -> float:
    """w . v as the device adds it: products left to right, one rounding each."""
    acc = float(v[0]) * float(w[0])
    for c in range(1, len(v)):
        acc = acc + float(v[c]) * float(w[c])
    return acc


def check_values(vals: np.ndarray, vecs: np.ndarray, w, what: str):
    """vals [n] scalarised values (numpy's dot), vecs [n, d] the Q vectors behind them.  A decision whose values all equal the device's
    left-to-right sums is reproduced exactly, ties included; any other must not hinge on the last bits."""
    if all(float(x) == seq_dot(v, w) for x, v in zip(vals, vecs)):
        return
    best = vals.max()
    tied = np.flatnonzero(vals == best)
    if len(tied) > 1 and any(not np.array_equal(vecs[i], vecs[tied[0]]) for i in tied[1:]):
        raise Rejected(f"{what}: exact tie at {best} between differing Q vectors")
    rest = vals[vals < best]
    if rest.size and best - rest.max() <= REL * max(abs(best), abs(rest.max())):
        raise Rejected(f"{what}: near tie {best} vs {rest.max()}")


def install_checks(mq, mp, pb):
    orig_eval = mq.MOQLearning.eval

    def q_rows(policy, obs):
        t = policy._state_to_tuple(obs)
        if t not in policy.q_table:
            return np.zeros((policy.action_dim, policy.reward_dim))
        return np.asarray(policy.q_table[t])

    def eval_(self, obs, w=None):
        if not self.use_gpi_policy and self._state_to_tuple(obs) in self.q_table:
            q = q_rows(self, obs)
            check_values(np.array([np.dot(v, self.weights) for v in q]), q, self.weights, "own greedy")
        return orig_eval(self, obs, w)

    mq.MOQLearning.eval = eval_
    orig_gpi = mp.MPMOQLearning._gpi_action

    def gpi(self, state, w):
        q = np.concatenate([q_rows(p, state) for p in self.policies])
        check_values(np.concatenate([p.scalarized_q_values(state, w) for p in self.policies]), q, w, "gpi")
        return orig_gpi(self, state, w)

    mp.MPMOQLearning._gpi_action = gpi

    def sample(self, batch_size):
        state = np.random.get_state()
        q = np.random.uniform(0, self.nodes[0][0], size=batch_size)
        np.random.set_state(state)
        node = 0
        qv = float(q[0])
        for nodes in self.nodes[1:]:
            node *= 2
            left = nodes[node]
            if abs(qv - left) <= REL * max(abs(qv), abs(left)):
                raise Rejected(f"walk query {qv} near left sum {left}")
            if qv > left:
                node += 1
                qv -= left
        return orig_sample(self, batch_size)

    orig_sample = pb.SumTree.sample
    pb.SumTree.sample = sample


def ref_model_view(agent):
    model = agent.policies[-1].model
    pairs = list(model.state_actions_pairs)
    outcomes = [list(model.model[sa].items()) for sa in pairs]
    leaves = model.priorities.nodes[-1][: len(pairs)].copy() if model.prioritize else None
    return pairs, outcomes, leaves


def main():
    rh.install_stubs()
    sys.modules["pymoo.util.ref_dirs"].get_reference_directions = lambda *a, **k: np.eye(2)
    mp = rh.import_reference("morl_baselines.multi_policy.multi_policy_moqlearning.mp_mo_q_learning")
    mq = rh.import_reference("morl_baselines.single_policy.ser.mo_q_learning")
    pb = rh.import_reference("morl_baselines.common.prioritized_buffer")
    install_checks(mq, mp, pb)
    out = {}
    for name, case in CASES.items():
        for seed in range(case["seed"], case["seed"] + TRIES):
            try:
                _, rec = run_case(name, mp.MPMOQLearning, seed, ref_model_view)
                break
            except Rejected as e:
                print(f"{name}: seed {seed} rejected: {e}")
        else:
            raise RuntimeError(f"{name}: no tie-safe seed in {TRIES} tries")
        print(f"{name}: seed {seed}, policies {[int(rec[f'{i}/n_policies'][0]) for i in range(case['iters'])]}")
        out.update({f"{name}/{k}": v for k, v in rec.items()})
    path = os.path.join(HERE, "mp_moq.npz")
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
