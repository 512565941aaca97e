"""The numpy restatement of one fused Dyna step (tests/dyna_commit_oracle.py ``commit``, the checker of morl_dyna_commit_f32) against the unmodified
reference's continuous-action rollout (tests/golden/gpipd_continuous_dyna.npz, frozen by tests/golden/make_golden_gpipd_continuous_dyna.py from
gpi_pd_continuous_action.py:336-371, whose row-by-row ``ReplayBuffer.add`` loop fills the model buffer), and the env-id -> device rule table.

The policy and ensemble forwards run in torch on the CPU, as in the reference; the rule outcomes, kept rows and buffer positions must be
identical, continuous values agree to 1e-5 relative."""

import os

import numpy as np
import pytest
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(OBS=11, ACT=3, D=3, N=256, ROLLOUT_B=300, ROLLOUT_LEN=3, DYN_BUF=200, DYN_ARCH=[32, 32], SEED_ROLLOUT=7, POLICY_NOISE_SEED=51,
           MODEL_NOISE_SEED=52, ELITES=[4, 2])


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "gpipd_continuous_dyna.npz"))


class _Noise:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)

    def __call__(self, shape):
        return th.from_numpy(self.rng.standard_normal(tuple(shape)).astype(np.float32))


def _sd(gold, prefix):
    return {k[len(prefix) + 1:]: th.from_numpy(gold[k]) for k in gold.files if k.startswith(prefix + "/")}


def _ensemble_raw(sd, x, n_layers):
    """Raw last-layer output [E, N, 2 O] of the reference's ensemble (normalised inputs, ReLU between EnsembleLayers)."""
    h = ((x - sd["inputs_mu"]) / sd["inputs_sigma"]).unsqueeze(0).repeat(sd["layers.0.W"].shape[0], 1, 1)
    for i in range(n_layers):
        h = th.baddbmm(sd[f"layers.{i}.b"], h, sd[f"layers.{i}.W"])
        if i < n_layers - 1:
            h = th.relu(h)
    return h


def test_oracle_commit_reproduces_reference_rollout(gold):
    from morl_baselines_b200.common.prioritized_buffer import PrioritizedReplayBuffer
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import Policy
    from morl_baselines_b200.testing import Box
    from oracle.dyna_oracle import clamp_logvar
    from tests import dyna_commit_oracle as do

    c = CFG
    OBS, ACT, D = c["OBS"], c["ACT"], c["D"]
    policy = Policy(OBS, D, ACT, Box(-1.0, 1.0, shape=(ACT,)), net_arch=[32, 32])
    policy.load_state_dict(_sd(gold, "init_policy"))
    dyn = _sd(gold, "init_dynamics")
    n_layers = len(c["DYN_ARCH"]) + 1
    rb = PrioritizedReplayBuffer((OBS,), ACT, rew_dim=D, max_size=c["N"])
    for k in ("obs", "next_obs", "actions", "rewards", "dones"):
        getattr(rb, k)[:] = gold[f"rb_{k}"]
    rb.size, rb.ptr = c["N"], 0
    rb.tree.batch_set(np.arange(c["N"]), gold["tree_leaves0"][:c["N"]])
    C = c["DYN_BUF"]
    stores = (np.zeros((C, OBS), np.float32), np.zeros((C, OBS), np.float32), np.zeros((C, ACT), np.float32), np.zeros((C, D), np.float32),
              np.zeros((C, 1), np.float32))
    weight = th.from_numpy(gold["support"][2])
    pol_noise, model_noise = _Noise(c["POLICY_NOISE_SEED"]), _Noise(c["MODEL_NOISE_SEED"])
    np.random.seed(c["SEED_ROLLOUT"])
    obs = th.from_numpy(rb.sample_obs(c["ROLLOUT_B"]))
    ptr, size, rows = 0, 0, []
    with th.no_grad():
        for _ in range(c["ROLLOUT_LEN"]):
            n = obs.shape[0]
            rows.append(n)
            act = policy(obs, weight.repeat(n, 1), noise=0.2, noise_clip=0.5, eps=pol_noise((n, ACT)))
            out = _ensemble_raw(dyn, th.cat((obs, act), dim=-1), n_layers).numpy()
            O = OBS + D
            noise = model_noise((out.shape[0], n, O)).numpy()
            inds = np.random.choice(c["ELITES"], size=n)
            lv = clamp_logvar(out[..., O:], dyn["max_logvar"].numpy().reshape(-1), dyn["min_logvar"].numpy().reshape(-1))
            ptr, size, alive, unc, done, keep = do.commit(out[..., :O], lv, inds, noise, obs.numpy(), act.numpy(), D, 1, float(gold["threshold"]), stores,
                                                          ptr, size)
            if len(alive) == 0:
                break
            obs = th.from_numpy(alive)
    assert rows == gold["rows_per_step"].tolist()
    assert [ptr, size] == gold["db_ptr_size"].tolist()
    np.testing.assert_allclose(unc, gold["last_uncertainty"], rtol=1e-5, atol=1e-7)
    for st, k in zip(stores, ("obs", "next_obs", "actions", "rewards", "dones")):
        want = gold[f"db_{k}"]
        if k == "dones":
            assert np.array_equal(st, want)
        else:
            np.testing.assert_allclose(st, want, rtol=1e-5, atol=1e-6, err_msg=k)


def test_oracle_rules_match_reference_outcomes():
    """The oracle's rule restatements (by device rule id) against the reference's outcomes frozen in termination_rules.npz."""
    from tests import dyna_commit_oracle as do
    from tests.golden.make_golden_reference_pins import termination_batch

    ref = np.load(os.path.join(ROOT, "tests", "golden", "termination_rules.npz"), allow_pickle=False)
    obs, act, nobs, rew = termination_batch()
    for rule, name in ((0, "false"), (1, "hopper"), (2, "humanoid"), (3, "mountaincar"), (4, "lunarlander")):
        with np.errstate(invalid="ignore"):
            got = do.TERM_RULES[rule](nobs, rew)
        assert np.array_equal(got, ref[name][:, 0].astype(bool)), name


def test_termination_rule_id_agrees_with_termination_fn_for():
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.model_based import utils

    ref = np.load(os.path.join(ROOT, "tests", "golden", "termination_rules.npz"), allow_pickle=False)
    by_fn = {utils.termination_fn_false: ops.TERM_NONE, utils.termination_fn_hopper: ops.TERM_HOPPER, utils.termination_fn_humanoid: ops.TERM_HUMANOID,
             utils.termination_fn_mountaincar: ops.TERM_MOUNTAINCAR, utils.termination_fn_lunarlander: ops.TERM_LUNARLANDER}
    for env_id in ref["env_ids"].tolist():
        fn = utils.termination_fn_for(env_id)
        if fn in by_fn:
            assert utils.termination_rule_id(env_id) == by_fn[fn], env_id
        else:  # minecart: discrete-action only, no device rule
            with pytest.raises(NotImplementedError):
                utils.termination_rule_id(env_id)
    for env_id in ("deep-sea-treasure-v0", "fake-momdp-v0"):
        with pytest.raises(NotImplementedError, match=env_id):
            utils.termination_rule_id(env_id)


def test_commit_argument_errors_need_no_device():
    """Bad rule ids and rules whose columns are missing are refused before anything touches a device."""
    import ctypes as C

    from morl_baselines_b200 import _lib

    lib = _lib.load()
    p = C.c_void_p(16)  # never dereferenced: the argument checks run first

    def call(rew_dim=3, O=14, rule=1, ptr=0, cap=8, N=4):
        return lib.morl_dyna_commit_f32(p, p, p, p, None, p, p, rew_dim, 5, N, O, 3, rule, 1.0, p, p, p, p, p, cap, ptr, p, p, p, p, None)

    assert call(rule=5) == -4 and call(rule=-1) == -4
    assert call(O=4, rew_dim=3, rule=1) == -2          # HOPPER needs s'[0], s'[1]
    assert call(O=10, rew_dim=3, rule=4) == -2         # LUNARLANDER needs s'[7]
    assert call(O=8, rew_dim=0, rule=4) == -2          # ... and r[0]
    assert call(O=3, rew_dim=3, rule=0) == -2          # no state columns
    assert call(ptr=8, cap=8) == -2 and call(N=0) == -2
    assert lib.morl_dyna_commit_workspace_bytes(0) == 0 and lib.morl_dyna_commit_workspace_bytes(10007) >= 10007
