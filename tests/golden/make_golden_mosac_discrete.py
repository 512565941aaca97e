"""Golden vectors for whole MOSACDiscrete updates, produced by the unmodified reference on CPU (run in the build container only):
    python tests/golden/make_golden_mosac_discrete.py   ->  tests/golden/mosac_discrete.npz

MOSACDiscrete.update (single_policy/ser/mosac_discrete_action.py:445-530): obs 8, 4 actions, 4 objectives, net_arch [32, 32], batch 16,
tau 0.5, three updates at global steps 100, 200, 300 with target_net_freq 200 (one target sync, at 200), autotune on and off.  The
update's own Categorical.sample() draws consume only torch's generator; the replay indices come from numpy's global stream.
Stored per case: the initial state dicts, the replay contents, the state dicts, log_alpha and alpha after the updates, and the losses
the reference logs at every update (global_step % 100 == 0)."""

from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402

OBS, A, D, B, N = 8, 4, 4, 16, 128
STEPS = (100, 200, 300)
LOSSES = ("qf1_loss", "qf2_loss", "actor_loss", "alpha_loss")


def sd_to_npz(out, prefix, sd):
    for k, v in sd.items():
        out[f"{prefix}/{k}"] = v.detach().cpu().numpy().copy()


def gen(out, autotune: bool):
    mm = rh.import_reference("morl_baselines.single_policy.ser.mosac_discrete_action")
    tag = f"autotune{int(autotune)}"
    logged = []
    mm.wandb = types.SimpleNamespace(log=lambda d: logged.append(dict(d)))
    th.manual_seed(0)
    env = rh.FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D)
    w = np.array([0.1, 0.4, 0.3, 0.2], dtype=np.float32)
    agent = mm.MOSACDiscrete(env, weights=w, batch_size=B, net_arch=[32, 32], log=True, seed=4, device="cpu", buffer_size=N, tau=0.5,
                             update_frequency=1, target_net_freq=200, autotune=autotune, alpha=0.3)
    rng = np.random.default_rng(41)
    buf = agent.buffer
    buf.obs[:] = rng.standard_normal((N, OBS)).astype(np.float32)
    buf.next_obs[:] = rng.standard_normal((N, OBS)).astype(np.float32)
    buf.actions[:] = rng.integers(0, A, (N, 1)).astype(np.float32)
    buf.rewards[:] = rng.standard_normal((N, D)).astype(np.float32)
    buf.dones[:] = (rng.random((N, 1)) < 0.2).astype(np.float32)
    buf.size, buf.ptr = N, 0
    for k in ("obs", "next_obs", "actions", "rewards", "dones"):
        out[f"{tag}/rb_{k}"] = getattr(buf, k).copy()
    for name in ("actor", "qf1", "qf2"):
        sd_to_npz(out, f"{tag}/init_{name}", getattr(agent, name).state_dict())
    np.random.seed(12)
    for step in STEPS:
        agent.global_step = step
        agent.update()
    assert len(logged) == len(STEPS)
    for name in ("actor", "qf1", "qf2", "qf1_target", "qf2_target"):
        sd_to_npz(out, f"{tag}/final_{name}", getattr(agent, name).state_dict())
    for k in LOSSES:
        if autotune or k != "alpha_loss":
            out[f"{tag}/{k}"] = np.array([d[f"losses_{agent.id}/{k}" if agent.id is not None else f"losses/{k}"] for d in logged], np.float64)
    if autotune:
        out[f"{tag}/final_log_alpha"] = agent.log_alpha.detach().numpy().copy()
    out[f"{tag}/final_alpha"] = np.float64(agent.alpha)
    print(tag, "done")


def main():
    assert rh.reference_available()
    th.set_num_threads(os.cpu_count() or 1)
    out = {}
    gen(out, True)
    gen(out, False)
    path = os.path.join(HERE, "mosac_discrete.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
