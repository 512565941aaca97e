"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

numpy restatement of one imagined Dyna step of the continuous-action GPI-PD rollout (reference gpi_pd_continuous_action.py:346-366): the
ensemble sample (``oracle.dyna_oracle.ensemble_sample``), the termination rule of the environment, the strict uncertainty gate and the
reference's row-by-row ``ReplayBuffer.add`` loop.  Pinned against the unmodified reference's rollout (tests/golden/gpipd_continuous_dyna.npz,
tests/test_dyna_commit_cpu.py); checker of ``morl_dyna_commit_f32`` (csrc/dyna.cu) in tests/test_dyna_commit_gpu.py."""

import numpy as np

from oracle.dyna_oracle import ensemble_sample


# termination rules of the continuous-action environments (reference common/model_based/utils.py:13-102), by the ids of
# morl_dyna_commit_f32 (MORL_TERM_*): float32 comparisons with IEEE NaN semantics, as the reference's numpy functions
def _done_hopper(nobs, rew):
    not_done = np.isfinite(nobs).all(-1) & (nobs[:, 1:] < 100).all(-1) & (nobs[:, 0] > np.float32(0.7)) & (np.abs(nobs[:, 1]) < np.float32(0.2))
    return ~not_done


def _done_humanoid(nobs, rew):
    return ~((np.float32(1.0) < nobs[:, 0]) & (nobs[:, 0] < np.float32(2.0)))


def _done_mountaincar(nobs, rew):
    return (nobs[:, 0] >= np.float32(0.45)) & (nobs[:, 1] >= np.float32(0.0))


def _done_lunarlander(nobs, rew):
    return (np.abs(nobs[:, 0]) >= np.float32(1.0)) | ((rew[:, 0] != 0) & (nobs[:, 6] >= np.float32(0.95)) & (nobs[:, 7] >= np.float32(0.95)))


TERM_RULES = {0: lambda nobs, rew: np.zeros(nobs.shape[0], bool), 1: _done_hopper, 2: _done_humanoid, 3: _done_mountaincar, 4: _done_lunarlander}


def commit(means, logvar, model_inds, noise, obs, act, rew_dim, rule, max_uncertainty, stores, ptr, size):
    """numpy restatement of one imagined step of morl_dyna_commit_f32 (reference gpi_pd_continuous_action.py:346-366): ``ensemble_sample``
    (obs added), then ``commit_rows``.  Returns (ptr, size, next_alive [alive, S], uncertainty [N], done [N] bool, keep [N] bool)."""
    sample, _, unc = ensemble_sample(means, logvar, model_inds, noise, obs, rew_dim)
    return commit_rows(sample, unc, obs, act, rew_dim, rule, max_uncertainty, stores, ptr, size)


def commit_rows(sample, unc, obs, act, rew_dim, rule, max_uncertainty, stores, ptr, size):
    """The termination rule, the strict uncertainty gate and a row-by-row ring append -- the reference's ``ReplayBuffer.add`` loop -- on a
    given sample [N, O] and uncertainty [N].  stores = (obs, next_obs, actions, rewards, dones) numpy arrays of the ring, modified in place."""
    rew, nobs = sample[:, :rew_dim], sample[:, rew_dim:]
    with np.errstate(invalid="ignore"):
        done = TERM_RULES[rule](nobs, rew)
        keep = unc < np.float32(max_uncertainty)
    st_obs, st_nobs, st_act, st_rew, st_done = stores
    cap = st_obs.shape[0]
    for i in np.flatnonzero(keep):
        st_obs[ptr], st_nobs[ptr], st_act[ptr], st_rew[ptr], st_done[ptr] = obs[i], nobs[i], act[i], rew[i], float(done[i])
        ptr = (ptr + 1) % cap
        size = min(size + 1, cap)
    return ptr, size, nobs[~done].copy(), unc, done, keep
