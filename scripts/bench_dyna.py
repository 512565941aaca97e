"""GPI-PD Dyna path (SURVEY 8(f)3) at the reference's default sizes: time of one `_rollout_dynamics` call (25,000 imagined transitions from a
64-policy support set, every row accepted: the worst case of the insert) and of one `ProbabilisticEnsemble.fit` epoch on 16,384 transitions.
    python scripts/bench_dyna.py                   CUDA engine (needs a GPU)
    python scripts/bench_dyna.py --impl reference  the unmodified reference on CPU through oracle/ref_harness (build container only)
One JSON object on stdout."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch as th

REF = "--impl" in sys.argv and sys.argv[sys.argv.index("--impl") + 1] == "reference"
OBS, A, D, N, P = 32, 8, 3, 16384, 64

if REF:
    from oracle import ref_harness as rh

    GPIPD = rh.import_reference("morl_baselines.multi_policy.gpi_pd.gpi_pd").GPIPD
    FakeEnv, Spec, dev = rh.FakeEnv, rh._Spec, "cpu"
    sync = lambda: None  # noqa: E731
else:
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPIPD
    from morl_baselines_b200.testing import FakeEnv, _Spec as Spec

    dev = th.device("cuda:0")
    sync = th.cuda.synchronize

rng = np.random.default_rng(0)
np.random.seed(0)
th.manual_seed(0)
env = FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D)
env.spec = Spec("mo-mountaincar-standin-v0")
ag = GPIPD(env, batch_size=128, per=True, buffer_size=N, log=False, seed=0, device=dev, dynamics_rollout_batch_size=25000, dynamics_buffer_size=100000,
           dynamics_uncertainty_threshold=1e9, dynamics_rollout_starts=0)
rb = ag.replay_buffer
rb.obs[:N] = rng.standard_normal((N, OBS)).astype(np.float32)
rb.next_obs[:N] = rb.obs[:N] + 0.1 * rng.standard_normal((N, OBS)).astype(np.float32)
rb.actions[:N] = rng.integers(0, A, size=(N, 1)).astype(np.uint8)
rb.rewards[:N] = rng.standard_normal((N, D)).astype(np.float32)
rb.dones[:N] = 0.0
rb.size, rb.ptr = N, 0
if hasattr(rb, "mark_all_dirty"):
    rb.mark_all_dirty()
rb.tree.batch_set(np.arange(N), np.full(N, 0.1))
ag.set_weight_support(list(rng.dirichlet(np.ones(D), P).astype(np.float32)))
w = th.tensor(ag.weight_support[0].cpu().numpy()).to(dev)
out = {"impl": "reference (CPU, %d threads)" % th.get_num_threads() if REF else "b200", "obs": OBS, "actions": A, "d": D, "support": P, "rollout_rows": 25000}


def timed(fn, n, warm):
    for _ in range(warm):
        fn()
    sync()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        sync()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


t = timed(lambda: ag._rollout_dynamics(w), n=2 if REF else 10, warm=0 if REF else 2)
out["rollout_dynamics_s"] = t
out["imagined_transitions_per_s"] = 25000 / t
# one training epoch of the ensemble on the whole buffer (the reference refits every 250 environment steps)
m_obs, m_act, m_rew, m_nobs, _ = rb.get_all_data()
one_hot = np.zeros((len(m_obs), A))
one_hot[np.arange(len(m_obs)), m_act.astype(int).reshape(-1)] = 1
X, Y = np.hstack((m_obs, one_hot)).astype(np.float32), np.hstack((m_rew, m_nobs - m_obs)).astype(np.float32)
ag.dynamics.fit(X, Y, max_epochs=1)  # warm-up (allocations, cuBLAS handles)
sync()
t0 = time.perf_counter()
ag.dynamics.fit(X, Y, max_epochs=3)
sync()
out["fit_s_per_epoch"] = (time.perf_counter() - t0) / 3
print(json.dumps(out))
