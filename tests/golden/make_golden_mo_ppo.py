"""Golden vectors for MO-PPO's advantage computation and update, produced by the unmodified reference on CPU (needs the reference's
source tree, so it is run by hand, not by the tests):
    python tests/golden/make_golden_mo_ppo.py   ->  tests/golden/mo_ppo.npz

MOPPO (single_policy/ser/mo_ppo.py): obs 11, act 3, d in {2, 3}, [8, 8] networks, 2 envs x 64 steps, 2 epochs x 4 minibatches, over
gae, clip_vloss, norm_adv on/off and ent_coef in {0, 0.01}, plus one target_kl case that stops after the first epoch.

The batch of case k comes from ``synthetic_batch(k, d)`` (numpy PCG64, reproduced by the tests), so only what the reference computed is
stored: the initial state dict per d, and per case the old log-probs (the reference network's log-probs plus the synthetic perturbation),
the critic's next_value, the outputs of ``_MOPPO__compute_advantages``, the parameters after the first minibatch step and after the
whole ``update()``, and how many shuffles the update drew."""

from __future__ import annotations

import itertools
import os
import sys
import types

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402

OBS, ACT, E, T = 11, 3, 2, 64
EPOCHS, MINIBATCHES = 2, 4
WEIGHTS = {2: np.array([0.3, 0.7], np.float32), 3: np.array([0.2, 0.5, 0.3], np.float32)}
ARCH = [8, 8]
NEXT_DONE = np.array([1.0, 0.0], np.float32)


def synthetic_batch(k: int, d: int) -> dict:
    """Case k's rollout contents.  ``pert`` is added to the reference network's log-probs to form the old log-probs: near the current
    policy (the first ratios are 1 up to it), with a tenth of the rows far outside the clip band."""
    g = np.random.default_rng(1000 + k)
    out = dict(obs=g.standard_normal((T, E, OBS)).astype(np.float32), actions=g.standard_normal((T, E, ACT)).astype(np.float32))
    pert = g.standard_normal(T * E).astype(np.float32) * 0.05
    pert[g.random(T * E) < 0.1] *= 20.0
    out["pert"] = pert
    out["rewards"] = g.standard_normal((T, E, d)).astype(np.float32)
    out["dones"] = (g.random((T, E)) < 0.08).astype(np.float32)
    out["values"] = g.standard_normal((T, E, d)).astype(np.float32)
    out["next_obs"] = g.standard_normal((E, OBS)).astype(np.float32)
    return out


def flat(sd) -> np.ndarray:
    """A state dict as one float32 vector, tensors in state-dict order (MOPPONet's order is the same here and in the reference)."""
    return np.concatenate([np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, np.float32).reshape(-1) for v in sd.values()])


def unflat(vec: np.ndarray, like) -> dict:
    """Inverse of ``flat`` for a state dict shaped like ``like``."""
    out, o = {}, 0
    for key, v in like.items():
        n = v.numel()
        out[key] = vec[o:o + n].reshape(tuple(v.shape))
        o += n
    assert o == len(vec)
    return out


def split_gae(vec: np.ndarray, d: int) -> dict:
    """The per-case vector of reference outputs: old log-probs [T, E], next_value [E, d], returns [T, E, d], advantages [T, E]."""
    sizes = (("logprobs", (T, E)), ("next_value", (E, d)), ("returns", (T, E, d)), ("advantages", (T, E)))
    out, o = {}, 0
    for name, shape in sizes:
        n = int(np.prod(shape))
        out[name] = vec[o:o + n].reshape(shape)
        o += n
    assert o == len(vec)
    return out


def cases():
    out = []
    for d, gae, clip_vloss, norm_adv, ent in itertools.product((2, 3), (1, 0), (1, 0), (1, 0), (0.0, 0.01)):
        out.append(dict(d=d, gae=gae, clip_vloss=clip_vloss, norm_adv=norm_adv, ent_coef=ent, target_kl=None))
    out.append(dict(d=2, gae=1, clip_vloss=1, norm_adv=1, ent_coef=0.0, target_kl=1e-6))  # breaks after the first epoch
    return out


def tag(c):
    kl = "none" if c["target_kl"] is None else "1e-6"
    return f"d{c['d']}_gae{c['gae']}_cv{c['clip_vloss']}_na{c['norm_adv']}_ent{c['ent_coef']}_kl{kl}"


class CountingRng:
    """np.random.Generator whose shuffle calls are counted."""

    def __init__(self, seed):
        self.g = np.random.default_rng(seed)
        self.shuffles = 0

    def shuffle(self, x):
        self.shuffles += 1
        self.g.shuffle(x)


def import_mo_ppo():
    rh.install_stubs()
    gym = sys.modules["gymnasium"]
    if getattr(gym, "__graft_stub__", False) and not hasattr(gym, "vector"):
        gym.vector = types.SimpleNamespace(SyncVectorEnv=object)  # named in a type annotation only
    return rh.import_reference("morl_baselines.single_policy.ser.mo_ppo")


def gen(out, c, k):
    mm = import_mo_ppo()
    mm.wandb = types.SimpleNamespace(log=lambda d: None)
    t = tag(c)
    d = c["d"]
    th.manual_seed(100 + d)
    net = mm.MOPPONet((OBS,), (ACT,), d, ARCH)
    init = flat(net.state_dict())
    if f"init_d{d}" in out:
        assert np.array_equal(out[f"init_d{d}"], init)
    out[f"init_d{d}"] = init
    rng = CountingRng(7 + k)
    envs = types.SimpleNamespace(num_envs=E)
    agent = mm.MOPPO(0, net, WEIGHTS[d], envs, steps_per_iteration=T, num_minibatches=MINIBATCHES, update_epochs=EPOCHS, gae=bool(c["gae"]),
                     clip_vloss=bool(c["clip_vloss"]), norm_adv=bool(c["norm_adv"]), ent_coef=c["ent_coef"], target_kl=c["target_kl"],
                     device="cpu", rng=rng)
    sb = synthetic_batch(k, d)
    b = agent.batch
    for f in ("obs", "actions", "rewards", "dones", "values"):
        getattr(b, f)[:] = th.from_numpy(sb[f])
    with th.no_grad():
        _, lp, _, _ = net.get_action_and_value(b.obs.reshape(-1, OBS), b.actions.reshape(-1, ACT))
    b.logprobs[:] = (lp + th.from_numpy(sb["pert"])).reshape(T, E)
    next_obs, next_done = th.from_numpy(sb["next_obs"]), th.from_numpy(NEXT_DONE)
    with th.no_grad():
        next_value = net.get_value(next_obs)
    returns, advantages = agent._MOPPO__compute_advantages(next_obs, next_done)
    agent.returns, agent.advantages = returns, advantages
    out[f"{t}/gae"] = np.concatenate([x.numpy().reshape(-1) for x in (b.logprobs, next_value, returns, advantages)])
    first = []
    step0 = agent.optimizer.step

    def step(*a, **kw):
        r = step0(*a, **kw)
        if not first:
            first.append(flat(net.state_dict()))
        return r

    agent.optimizer.step = step
    agent.update()
    out[f"{t}/params"] = np.stack([first[0], flat(net.state_dict())])  # after the first minibatch step, after the update
    out[f"{t}/shuffles"] = np.int64(rng.shuffles)
    print(t, "shuffles", rng.shuffles)


def main():
    assert rh.reference_available()
    th.set_num_threads(1)
    out = {}
    for k, c in enumerate(cases()):
        gen(out, c, k)
    path = os.path.join(HERE, "mo_ppo.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
