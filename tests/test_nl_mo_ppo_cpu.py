"""NLMOPPO without a device: the kernels' supported range at and just outside each bound, the library's workspace size, and the stand-in
environment's replayability."""

import numpy as np
import pytest

from morl_baselines_b200 import nl_ppo_ops
from morl_baselines_b200.nl_ppo_ops import nl_ppo_supported
from tests.nl_ppo_standin import RingVecEnv


@pytest.mark.parametrize("args,ok", [
    ((2, 2, 2, 4, 64), True),
    ((1, 1, 0, 1, 1), True),
    ((0, 2, 2, 4, 64), False),                 # obs_dim >= 1
    ((2, 0, 0, 4, 64), False),                 # d >= 1
    ((2, 8, 8, 4, 64), True), ((2, 9, 9, 4, 64), False),   # d <= 8
    ((2, 3, 2, 4, 64), False),                 # pref_dim in {0, d}
    ((240, 8, 8, 4, 64), True), ((241, 8, 8, 4, 64), False),  # S + d + Dp <= 256
    ((248, 8, 0, 4, 64), True), ((249, 8, 0, 4, 64), False),
    ((2, 2, 2, 32, 64), True), ((2, 2, 2, 33, 64), False), ((2, 2, 2, 0, 64), False),  # 1 <= A <= 32
    ((2, 2, 2, 4, 4096), True), ((2, 2, 2, 4, 4097), False), ((2, 2, 2, 4, 0), False),  # 1 <= batch <= 4096
])
def test_supported_range(args, ok):
    assert nl_ppo_supported(*args) is ok


def test_workspace_independent_of_batch_and_zero_outside_range():
    from morl_baselines_b200 import _lib

    lib = _lib.load()
    K, d, A = 2 + 2 + 2, 2, 4
    params = 2 * (64 * K + 64 + 64 * 64 + 64) + 64 * d + d + 64 * A + A
    assert lib.morl_nl_ppo_workspace_bytes(2, d, 2, A) == 128 * (13 * 8 + 4 * params)
    assert lib.morl_nl_ppo_workspace_bytes(2, 9, 9, A) == 0
    assert nl_ppo_ops.N_STATS == 6


def test_standin_replays_from_seed():
    runs = []
    for _ in range(2):
        env = RingVecEnv(num_envs=3)
        obs, _ = env.reset(seed=5)
        seq = [obs]
        for t in range(30):
            o, r, te, tr, _ = env.step((np.arange(3) + t) % 4)
            seq += [o, r, te, tr]
        runs.append(seq)
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


# ---- tests/golden/nl_mo_ppo.npz, without a device ------------------------------------------------------------------------------------
import os  # noqa: E402

import torch as th  # noqa: E402

from morl_baselines_b200.single_policy.ser.nl_mo_ppo import Agent  # noqa: E402
from tests.nl_ppo_standin import TRAIN_CASES, UPDATE_CASES, single_thread  # noqa: E402

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nl_mo_ppo.npz"))
NAMES = [f"{net}.{i}.{k}" for net in ("critic", "actor") for i in (0, 2, 4) for k in ("weight", "bias")]


@pytest.mark.parametrize("pre,c", [(f"update_{n}", c) for n, c in UPDATE_CASES.items()] + [(f"train_{n}", c) for n, c in TRAIN_CASES.items()])
def test_golden_initial_parameters_are_the_seeded_agent(pre, c):
    """The Agent built after th.manual_seed(seed) has the reference's names, shapes and initial values."""
    th.manual_seed(c["seed"])
    with single_thread():
        sd = Agent(RingVecEnv(c["E"], **c["env"]), c["env"]["d"], c["env"]["d"]).state_dict()
    assert list(sd) == NAMES
    for k in NAMES:
        assert np.array_equal(sd[k].numpy(), GOLDEN[f"{pre}/init/{k}"]), k
        for stage in ("first", "after", "final"):
            if f"{pre}/{stage}/{k}" in GOLDEN.files:
                assert GOLDEN[f"{pre}/{stage}/{k}"].shape == sd[k].shape


@pytest.mark.parametrize("name", list(UPDATE_CASES))
def test_golden_update_case_is_consistent(name):
    c, pre = UPDATE_CASES[name], f"update_{name}"
    g = {k[len(pre) + 4:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(pre + "/in/")}
    T, E, d = c["T"], c["E"], c["env"]["d"]
    # the reference's GAE loop in float32, each operation rounded once (gamma and gamma * lambda rounded to float32 by the tensor ops)
    gm, gl = np.float32(0.99), np.float32(0.99 * 0.95)
    adv, last = np.zeros((T, E, d), np.float32), np.zeros((E, d), np.float32)
    for t in reversed(range(T)):
        nnt = (np.float32(1) - (g["next_done"] if t == T - 1 else g["dones"][t + 1]))[:, None]
        nv = g["next_value"] if t == T - 1 else g["values"][t + 1]
        last = ((g["rewards"][t] + (gm * nv) * nnt) - g["values"][t]) + (gl * nnt) * last
        adv[t] = last
    assert np.array_equal(adv, g["advantages"]) and np.array_equal(adv + g["values"], g["returns"])
    assert g["actions"].min() >= 0 and g["actions"].max() < c["env"]["n_actions"]
    if c["u"] == "linear":
        np.testing.assert_allclose(GOLDEN[f"{pre}/loss_weights"], np.arange(1, d + 1) / (d * (d + 1) / 2), rtol=1e-6)
    shuffles = int(GOLDEN[f"{pre}/shuffles"])
    if c["ctor"]["target_kl"] is None:
        assert shuffles == c["ctor"]["update_epochs"]
    else:
        assert 1 <= shuffles < c["ctor"]["update_epochs"]  # the case stops early
    assert 0.0 <= GOLDEN[f"{pre}/stats"][5] <= 1.0


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_golden_train_run_is_consistent(name):
    c, pre = TRAIN_CASES[name], f"train_{name}"
    last = {k: GOLDEN[f"{pre}/last/{k}"] for k in ("obs", "actions", "rewards", "dones", "values", "advantages", "returns")}
    assert np.array_equal(last["advantages"] + last["values"], last["returns"])
    assert last["actions"].min() >= 0 and last["actions"].max() < c["env"]["n_actions"]
    assert set(np.unique(last["dones"])) <= {0.0, 1.0}
    assert GOLDEN[f"{pre}/eval"].shape == (c["env"]["d"],) and np.all(np.isfinite(GOLDEN[f"{pre}/eval"]))
