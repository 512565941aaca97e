"""NLMOPPO against tests/golden/nl_mo_ppo.npz, which the unmodified reference produced on CPU (tests/golden/make_golden_nl_mo_ppo.py):
every update case (the kernels, and the autograd fallback for a shape outside their range) and both replayable train() runs."""

import os

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import nl_ppo_ops
from morl_baselines_b200.single_policy.ser.nl_mo_ppo import NLMOPPO
from tests.nl_ppo_standin import TRAIN_CASES, UPDATE_CASES, UTILITIES, FixedSampling, RingEnv, RingVecEnv, action_table, single_thread

pytestmark = pytest.mark.gpu
DEV = th.device("cuda")
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nl_mo_ppo.npz"))

# Errors are max |ours - reference| / max(1, max |reference|) per array; the reference ran in float32 on CPU with its own summation order.
# Measured worst over the cases on one H100 80GB HBM3 (700 W power limit) beside each bound.
W_TOL = 2e-6        # loss weights: 1.9e-7
STEP_TOL = 1e-6     # parameters after the first minibatch step: 3.5e-8
UPDATE_TOL = 1e-6   # parameters after a whole update: 3.5e-8 (the fallback's GAE from its own bootstrap value is held to it too)
STATS_TOL = 2e-6    # the statistics update() returns: 1.3e-7
TRAIN_TOL = 1e-5    # storage, final parameters and evaluation after three train() iterations: 4.6e-7 (values); accrued rewards and
                    # the evaluation result came out exact


def err(ours, ref) -> float:
    ours = ours.detach().double().cpu().numpy() if isinstance(ours, th.Tensor) else np.asarray(ours, np.float64)
    ref = np.asarray(ref, np.float64)
    return float(np.abs(ours - ref).max() / max(1.0, np.abs(ref).max()))


def golden_params(pre):
    return {k[len(pre) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(pre + "/")}


def params_err(agent, pre) -> float:
    ref = golden_params(pre)
    sd = agent.agent.state_dict()
    assert set(sd) == set(ref)
    return max(err(sd[k], ref[k]) for k in sd)


def build(c):
    th.manual_seed(c["seed"])
    with single_thread():
        return NLMOPPO(0, RingVecEnv(c["E"], **c["env"]), num_steps=c["T"], device=DEV, seed=c["seed"], **c["ctor"])


def load_case(name):
    """A learner of update case ``name`` with the golden synthetic batch in its storage and the reference's GAE outputs loaded."""
    c, pre = UPDATE_CASES[name], f"update_{name}"
    ag = build(c)
    assert params_err(ag, f"{pre}/init") == 0.0  # the same seeded construction
    g = lambda k: th.from_numpy(GOLDEN[f"{pre}/in/{k}"]).to(DEV)  # noqa: E731
    for k in ("obs", "acc_rewards", "actions", "rewards", "values", "dones", "logprobs"):
        getattr(ag, k).copy_(g(k))
    ag._next_obs.copy_(g("next_obs"))
    ag._next_acc.copy_(g("next_acc"))
    ag._next_done.copy_(g("next_done"))
    ag.u_func = UTILITIES[c["u"]]
    ag._set_pref(c["pref"])
    return ag, c, pre, g


def check_update_case(name):
    """Returns the measured errors (loss weights, first step, update, stats)."""
    ag, c, pre, g = load_case(name)
    assert ag.fused == (name != "a40_fallback")
    if ag.fused:  # the objective GAE from the reference's bootstrap value, bit for bit
        ret, adv = nl_ppo_ops.vector_gae_objectives(g("rewards"), g("values"), g("dones"), g("next_value"), g("next_done"), ag.gamma, ag.gae_lambda)
        assert th.equal(adv, g("advantages")) and th.equal(ret, g("returns"))
    else:  # the fallback's GAE, from its own bootstrap value
        ag._compute_advantages_and_returns()
        assert err(ag.advantages, GOLDEN[f"{pre}/in/advantages"]) < UPDATE_TOL and err(ag.returns, GOLDEN[f"{pre}/in/returns"]) < UPDATE_TOL
    ag.advantages.copy_(g("advantages"))
    ag.returns.copy_(g("returns"))
    errs = {"w": err(ag._compute_loss_weights(), GOLDEN[f"{pre}/loss_weights"])}
    if ag.fused:  # the first minibatch step alone, on a twin learner: the reference's first shuffle, the kernel pair, clip + Adam
        tw = load_case(name)[0]
        tw.advantages.copy_(g("advantages"))
        tw.returns.copy_(g("returns"))
        tw._compute_loss_weights()
        inds = np.arange(tw.batch_size)
        np.random.default_rng(c["seed"]).shuffle(inds)
        perm = th.as_tensor(inds[:tw.minibatch_size], device=DEV)
        nl_ppo_ops.nl_ppo_update(tw._net, *tw._batch(), perm, tw._w, tw.clip_coef, tw.ent_coef, tw.vf_coef, tw.norm_adv, tw.clip_vloss, tw._stats,
                                 tw._ws)
        tw.optimizer.step_fused(tw.max_grad_norm)
        errs["first"] = params_err(tw, f"{pre}/first")
    stats = ag.update()
    errs["after"] = params_err(ag, f"{pre}/after")
    errs["stats"] = err(np.array([float(s) for s in stats]), GOLDEN[f"{pre}/stats"])
    # the reference's number of shuffles, drawn from the learner's generator
    rng, inds = np.random.default_rng(c["seed"]), np.arange(ag.batch_size)
    for _ in range(int(GOLDEN[f"{pre}/shuffles"])):
        rng.shuffle(inds)
    assert rng.bit_generator.state == ag.rng.bit_generator.state
    return errs


@pytest.mark.parametrize("name", list(UPDATE_CASES))
def test_update_case_matches_reference(name):
    e = check_update_case(name)
    assert e["w"] < W_TOL, e
    assert e.get("first", 0.0) < STEP_TOL, e
    assert e["after"] < UPDATE_TOL, e
    assert e["stats"] < STATS_TOL, e


def check_train_case(name):
    """Returns the measured error of each recorded array of the run."""
    c, pre = TRAIN_CASES[name], f"train_{name}"
    ag = build(c)
    assert ag.fused and params_err(ag, f"{pre}/init") == 0.0
    table = action_table(c["seed"], ag.num_iterations * c["T"], c["E"], c["env"]["n_actions"])
    with FixedSampling(table) as fs:
        res = ag.train(RingEnv(**c["env"]), UTILITIES[c["u"]], c["pref"], deterministic=True)
    assert fs.k == len(table)
    # what depends on the actions and the environment alone is exact
    for k in ("obs", "actions", "rewards", "dones"):
        assert np.array_equal(getattr(ag, k).cpu().numpy(), GOLDEN[f"{pre}/last/{k}"]), k
    errs = {k: err(getattr(ag, k), GOLDEN[f"{pre}/last/{k}"]) for k in ("acc_rewards", "logprobs", "values", "advantages", "returns")}
    errs["final"] = params_err(ag, f"{pre}/final")
    errs["eval"] = err(res, GOLDEN[f"{pre}/eval"])
    return errs


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_train_run_matches_reference(name):
    e = check_train_case(name)
    assert all(v < TRAIN_TOL for v in e.values()), e
