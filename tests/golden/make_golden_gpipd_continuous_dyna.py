"""Golden vectors for the Dyna half of GPIPDContinuousAction (reference multi_policy/gpi_pd/gpi_pd_continuous_action.py:216-235, :311-371,
:373-452, :548-555), produced by the unmodified reference on CPU (run in the build container only):

    python tests/golden/make_golden_gpipd_continuous_dyna.py   ->  tests/golden/gpipd_continuous_dyna.npz

The environment id contains "hopper", so the model rollout terminates rows with the hopper rule.  Dropout is disabled on the critics (p = 0:
CPU and CUDA generators differ), the policy's target noise (th.randn_like, :55) and the ensemble's sampling noise (th.randn,
probabilistic_ensemble.py:128) come from two seeded numpy streams.  Stored:
  * rollout: the initial networks and replay contents, an uncertainty threshold placed in the widest central gap of the uncertainties of a
    dry run (so CPU / GPU rounding cannot move a row across it), the model buffer after ``_rollout_dynamics`` (3 steps from 300 start rows
    into a ring of 200 slots, which wraps), its ptr / size and the last step's uncertainties;
  * update: the parameters and PER leaves after three whole updates on mixed real / imagined minibatches with a support of five weights;
  * fit: the ensemble after ``fit`` (normalize_inputs=True, the agent's default) for three epochs on X = [s | a], Y = [r | s' - s].
"""

from __future__ import annotations

import os
import random
import sys

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402

CFG = dict(OBS=11, ACT=3, D=3, B=16, N=256, ENV_ID="mo-hopper-standin-v4", ROLLOUT_B=300, ROLLOUT_LEN=3, DYN_BUF=200, REAL_RATIO=0.25,
           ARCH=[32, 32], DYN_ARCH=[32, 32], SEED_ROLLOUT=7, POLICY_NOISE_SEED=51, MODEL_NOISE_SEED=52, N_SUPPORT=5)


def sd_to_npz(out, prefix, sd):
    for k, v in sd.items():
        out[f"{prefix}/{k}"] = v.detach().cpu().numpy().copy()


class NoiseStream:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)

    def __call__(self, shape):
        return th.from_numpy(self.rng.standard_normal(tuple(shape)).astype(np.float32))


class TorchProxy:
    """Stands in for the name ``th`` inside the ensemble module: torch, except that randn comes from a seeded numpy stream."""

    def __init__(self, seed):
        self._stream = NoiseStream(seed)

    def randn(self, shape, device=None, **kw):
        return self._stream(shape)

    def __getattr__(self, name):
        return getattr(th, name)


def replay_contents(seed):
    """Seeded real transitions: hopper-like heights around 1.1 and angles around 0, so that some imagined rows stay alive for 3 steps."""
    c = CFG
    rng = np.random.default_rng(seed)
    obs = (rng.standard_normal((c["N"], c["OBS"])) * 0.5).astype(np.float32)
    obs[:, 0] = rng.uniform(0.6, 1.6, c["N"]).astype(np.float32)
    obs[:, 1] = rng.uniform(-0.3, 0.3, c["N"]).astype(np.float32)
    nobs = (obs + 0.05 * rng.standard_normal((c["N"], c["OBS"]))).astype(np.float32)
    act = rng.uniform(-1, 1, (c["N"], c["ACT"])).astype(np.float32)
    rew = rng.standard_normal((c["N"], c["D"])).astype(np.float32)
    done = (rng.random((c["N"], 1)) < 0.1).astype(np.float32)
    return obs, nobs, act, rew, done, (rng.random(c["N"]) + 0.1), rng.dirichlet(np.ones(c["D"]), c["N_SUPPORT"]).astype(np.float32)


def build_ref_agent(gm, threshold):
    c = CFG
    env = rh.FakeEnv(obs_dim=c["OBS"], continuous_action_dim=c["ACT"], reward_dim=c["D"])
    env.spec = rh._Spec(c["ENV_ID"])
    th.manual_seed(0)
    agent = gm.GPIPDContinuousAction(env, batch_size=c["B"], net_arch=c["ARCH"], num_q_nets=2, gradient_updates=3, per=True, buffer_size=c["N"], dyna=True,
                                     dynamics_net_arch=c["DYN_ARCH"], dynamics_rollout_len=c["ROLLOUT_LEN"], dynamics_rollout_starts=0,
                                     dynamics_rollout_batch_size=c["ROLLOUT_B"], dynamics_buffer_size=c["DYN_BUF"], dynamics_min_uncertainty=threshold,
                                     dynamics_real_ratio=c["REAL_RATIO"], log=False, seed=3, device="cpu")
    for net in agent.q_nets + agent.target_q_nets:
        for m in net.modules():
            if isinstance(m, th.nn.Dropout):
                m.p = 0.0
    obs, nobs, act, rew, done, prio, support = replay_contents(41)
    rb = agent.replay_buffer
    rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = obs, nobs, act, rew, done
    rb.size, rb.ptr = c["N"], 0
    rb.tree.batch_set(np.arange(c["N"]), prio)
    agent.set_weight_support(list(support))
    # a model with small, input-dependent disagreement: small state deltas keep rows alive over several steps, a narrow aleatoric part lets
    # the member disagreement rank the rows
    dyn = agent.dynamics
    with th.no_grad():
        dyn._fit_input_stats(np.hstack((obs, act)))
        dyn.layers[-1].W.mul_(0.15)
        dyn.max_logvar.fill_(-14.0)
        dyn.min_logvar.fill_(-18.0)
    dyn.elites = [4, 2]
    return agent, support


def rollout(agent, pm, w):
    c = CFG
    pm.th = TorchProxy(c["MODEL_NOISE_SEED"])
    stream = NoiseStream(c["POLICY_NOISE_SEED"])
    orig = th.randn_like
    th.randn_like = lambda t, **kw: stream(t.shape)
    try:
        np.random.seed(c["SEED_ROLLOUT"])
        agent._rollout_dynamics(w)
    finally:
        pm.th = th
        th.randn_like = orig


def main():
    assert rh.reference_available()
    th.set_num_threads(os.cpu_count() or 1)
    gm = rh.import_reference("morl_baselines.multi_policy.gpi_pd.gpi_pd_continuous_action")
    um = rh.import_reference("morl_baselines.common.model_based.utils")
    pm = rh.import_reference("morl_baselines.common.model_based.probabilistic_ensemble")
    out = {}

    # dry run with an infinite threshold: every step's uncertainties; the threshold goes in their widest central gap
    seen = []
    orig_step = um.ModelEnv.step

    def recording_step(self, obs, act, deterministic=False):
        r = orig_step(self, obs, act, deterministic)
        seen.append(np.asarray(r[3]["uncertainty"]).copy())
        return r

    agent, support = build_ref_agent(gm, 1e30)
    w = th.tensor(support[2])
    gm.ModelEnv.step = recording_step
    try:
        rollout(agent, pm, w)
    finally:
        gm.ModelEnv.step = orig_step
    allu = np.sort(np.concatenate(seen))
    lo, hi = int(0.3 * len(allu)), int(0.7 * len(allu))
    gaps = allu[lo + 1:hi] - allu[lo:hi - 1]
    k = lo + int(np.argmax(gaps))
    threshold = float(0.5 * (allu[k] + allu[k + 1]))
    print(f"{len(seen)} steps, rows per step {[len(s) for s in seen]}; uncertainties {allu[0]:.5f} .. {allu[-1]:.5f}; threshold {threshold:.6f} "
          f"in a gap of {gaps.max():.2e}")
    assert len(seen) == CFG["ROLLOUT_LEN"] and gaps.max() > 1e-4 * threshold

    agent, support = build_ref_agent(gm, threshold)
    out["threshold"] = np.float64(threshold)
    out["support"] = support
    sd_to_npz(out, "init_policy", agent.policy.state_dict())
    for i, q in enumerate(agent.q_nets):
        sd_to_npz(out, f"init_q{i}", q.state_dict())
    sd_to_npz(out, "init_dynamics", agent.dynamics.state_dict())
    rb = agent.replay_buffer
    for k_ in ("obs", "next_obs", "actions", "rewards", "dones"):
        out[f"rb_{k_}"] = getattr(rb, k_).copy()
    out["tree_leaves0"] = rb.tree.nodes[-1].copy()

    seen.clear()
    gm.ModelEnv.step = recording_step
    try:
        rollout(agent, pm, w)
    finally:
        gm.ModelEnv.step = orig_step
    db = agent.dynamics_buffer
    for k_ in ("obs", "next_obs", "actions", "rewards", "dones"):
        out[f"db_{k_}"] = getattr(db, k_).copy()
    out["db_ptr_size"] = np.array([db.ptr, db.size], np.int64)
    out["rows_per_step"] = np.array([len(s) for s in seen], np.int64)
    out["last_uncertainty"] = seen[-1]
    print("model buffer after the rollout: ptr", db.ptr, "size", db.size, "rows per step", out["rows_per_step"])
    assert int(out["rows_per_step"].sum()) > 0 and 0 < db.ptr and db.size == CFG["DYN_BUF"]

    # three whole updates on mixed minibatches (PER real rows + model rows, doubled batch over the support)
    stream = NoiseStream(99)
    orig = th.randn_like
    th.randn_like = lambda t, **kw: stream(t.shape)
    try:
        random.seed(15)
        np.random.seed(16)
        agent.global_step = 5
        agent.update(w)
    finally:
        th.randn_like = orig
    sd_to_npz(out, "final_policy", agent.policy.state_dict())
    for i, (q, tq) in enumerate(zip(agent.q_nets, agent.target_q_nets)):
        sd_to_npz(out, f"final_q{i}", q.state_dict())
        sd_to_npz(out, f"final_tq{i}", tq.state_dict())
    out["tree_leaves1"] = rb.tree.nodes[-1].copy()
    out["min_priority1"] = np.float64(rb.min_priority)

    # fit of the agent's ensemble on the real transitions, three epochs
    m_obs, m_actions, m_rewards, m_next_obs, _ = rb.get_all_data()
    X = np.hstack((m_obs, m_actions))
    Y = np.hstack((m_rewards, m_next_obs - m_obs))
    sd_to_npz(out, "fit_init", agent.dynamics.state_dict())
    np.random.seed(5)
    out["fit_mean_holdout"] = np.float64(agent.dynamics.fit(X, Y, batch_size=64, max_epochs=3))
    out["fit_elites"] = np.asarray(agent.dynamics.elites, np.int64)
    sd_to_npz(out, "fit_final", agent.dynamics.state_dict())

    path = os.path.join(HERE, "gpipd_continuous_dyna.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
