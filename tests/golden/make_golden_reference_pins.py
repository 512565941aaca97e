"""Golden data of the two differential CPU tests that used to import the unmodified reference at test time:
    python tests/golden/make_golden_reference_pins.py  ->  tests/golden/port_vs_reference.npz, tests/golden/termination_rules.npz
Needs the reference checkout (MORL_REFERENCE_ROOT); the tests themselves only read the .npz files.

  port_vs_reference.npz : for per in (0, 1): the reference Envelope's initial q_net parameters, the replay indices and weight sets of three
                          ``update()`` calls, and its q_net parameters afterwards (tests/test_port_vs_reference.py)
  termination_rules.npz : the seeded batch of tests/test_dyna_cpu.py::test_termination_rules_match_reference and the outcome of each of
                          the reference's termination functions on it, plus the env-id -> rule table of the reference's ModelEnv
"""

import os
import sys

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_harness as rh  # noqa: E402
from oracle.envelope_update_port import synthetic_store  # noqa: E402

PORT_CASE = dict(OBS=12, A=5, D=3, W=6, B=16, N=512, net=[32, 32], steps=3)
RULES = ("false", "mountaincar", "minecart", "hopper", "lunarlander", "humanoid")
ENV_IDS = ("mo-hopper-v4", "mo-halfcheetah-v4", "mo-humanoid-v4", "mo-lunar-lander-v2", "mo-reacher-v4", "mo-mountaincar-v0", "minecart-v0",
           "mo-highway-v0", "mo-highway-fast-v0")


def termination_batch():
    rng = np.random.default_rng(0)
    n = 4000
    obs = (rng.standard_normal((n, 9)) * np.array([0.3, 0.3, 1, 1, 1, 1, 1, 1, 1])).astype(np.float32)
    nobs = (rng.standard_normal((n, 9)) * np.array([0.6, 0.15, 1, 1, 1, 1, 0.6, 0.6, 40])).astype(np.float32)
    nobs[:, 0] += 0.9  # heights / positions around the hopper, humanoid and mountain-car thresholds
    nobs[:, 6:8] += 0.8
    nobs[5, 3], nobs[6, 4], nobs[7, 8] = np.nan, np.inf, 250.0
    act = rng.integers(0, 2, (n, 4)).astype(np.float32)
    rew = (rng.standard_normal((n, 3)) * (rng.random((n, 1)) < 0.5)).astype(np.float32)
    return obs, act, nobs, rew


def gen_port():
    envm = rh.import_reference("morl_baselines.multi_policy.envelope.envelope")
    wm = rh.import_reference("morl_baselines.common.weights")
    c = PORT_CASE
    out = {}
    for per in (False, True):
        th.manual_seed(0)
        agent = envm.Envelope(rh.FakeEnv(obs_dim=c["OBS"], n_actions=c["A"], reward_dim=c["D"]), batch_size=c["B"], num_sample_w=c["W"], per=per,
                              buffer_size=c["N"], net_arch=c["net"], log=False, seed=3, device="cpu")
        store = synthetic_store(c["N"], c["OBS"], c["A"], c["D"], seed=1)
        rb = agent.replay_buffer
        rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
        rb.size, rb.ptr = c["N"], 0
        if per:
            rb.tree.batch_set(np.arange(c["N"]), np.full(c["N"], rb.min_priority))
        for k, v in agent.q_net.state_dict().items():
            out[f"per{int(per)}/init/{k}"] = v.numpy().copy()
        rng = np.random.default_rng(3)  # mirrors agent.np_random
        agent.global_step = 1
        for step in range(c["steps"]):
            np.random.seed(50 + step)
            # the reference's draws: replay indices from the global RNG first, then the weights from the agent's generator
            state = np.random.get_state()
            idx = rb.tree.sample(c["B"]) if per else np.random.choice(c["N"], c["B"], replace=True)
            np.random.set_state(state)
            out[f"per{int(per)}/idx{step}"] = np.asarray(idx, dtype=np.int64)
            out[f"per{int(per)}/wset{step}"] = np.asarray(wm.random_weights(c["D"], c["W"], dist="gaussian", rng=rng), dtype=np.float32)
            agent.update()
        for k, v in agent.q_net.state_dict().items():
            out[f"per{int(per)}/final/{k}"] = v.numpy().copy()
    np.savez_compressed(os.path.join(HERE, "port_vs_reference.npz"), **out)


def gen_termination():
    ref = rh.import_reference("morl_baselines.common.model_based.utils")
    obs, act, nobs, rew = termination_batch()
    out = {name: np.asarray(getattr(ref, f"termination_fn_{name}")(obs, act, nobs, rew), dtype=bool) for name in RULES}
    by_fn = {getattr(ref, f"termination_fn_{name}"): name for name in RULES}
    out["env_ids"] = np.array(ENV_IDS)
    out["env_rules"] = np.array([by_fn[ref.ModelEnv(None, e).termination_func] for e in ENV_IDS])
    np.savez_compressed(os.path.join(HERE, "termination_rules.npz"), **out)


if __name__ == "__main__":
    assert rh.reference_available()
    gen_port()
    gen_termination()
