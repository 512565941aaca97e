"""Golden vectors for PCN and LCN, produced by the unmodified reference on CPU (needs the reference's source tree, so it is run by hand,
not by the tests):
    python tests/golden/make_golden_pcn.py   ->  tests/golden/pcn.npz

Every case runs on ``tests/pcn_standin.VarLengthEnv`` (episodes of 2 to 12 steps) and fills the heap with the episodes of
``episode_plan(case)`` (``pcn_standin.random_episode`` from a numpy seed, so the tests rebuild the same episodes), with one ranking pass
in the middle so that later positions follow rewritten scores and some episodes are evicted.

  update_<case>  : discrete (obs 4, 3 actions, d 2, H 64, B 37) and continuous (obs 5, act 2, d 3, H 32, B 40) PCN: the initial state
                   dict, the parameters after one ``update()`` and its prediction, and the parameters, losses and (discrete) entropies of
                   U = 6 consecutive updates;
  rank_<mode>    : LCN ``_choose_commands`` for distance_ref "nondominated" and "lambda_lorenz" (d 3, duplicated episodes included): the
                   heap (score, step) after each of two calls, and the commands;
  train_<algo>   : a short ``train()`` of PCN (discrete) and LCN: initial and final parameters, the heap (step, return, length) at the
                   end and each iteration's command.
"""

from __future__ import annotations

import os
import sys
import tempfile

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402
from tests.pcn_standin import VarLengthEnv, random_episode  # noqa: E402

UPDATE_CASES = {
    "disc": dict(env=dict(obs_dim=4, n_actions=3, reward_dim=2), scaling=[1.0, 1.0, 0.1], hidden=64, batch=37, lr=1e-3, seed=3),
    "cont": dict(env=dict(obs_dim=5, reward_dim=3, continuous_action_dim=2), scaling=[1.0, 0.5, 0.5, 0.1], hidden=32, batch=40, lr=1e-3,
                 seed=5),
}
N_UPDATES = 6
N_EPISODES, MAX_SIZE, RANK_AT, RANK_N = 30, 24, 18, 6


def episode_plan(seed: int):
    """(episode seed, step) of each heap insertion; the ranking pass (``_nlargest(RANK_N)``) runs before insertion RANK_AT."""
    return [(seed * 1000 + k, 3 * k + 1) for k in range(N_EPISODES)]


def fill(agent, env, seed: int, transition_cls, duplicate_every: int = 0):
    """Insert the plan's episodes; with ``duplicate_every`` every such episode is inserted twice (equal returns)."""
    prev = None
    for k, (ep_seed, step) in enumerate(episode_plan(seed)):
        if k == RANK_AT:
            agent._nlargest(RANK_N, *([agent.cd_threshold] if hasattr(agent, "cd_threshold") else []))
        if duplicate_every and prev is not None and k % duplicate_every == 0:
            o, a, r = prev
        else:
            o, a, r = random_episode(env, np.random.default_rng(ep_seed))
        prev = (o, a, r)
        agent._add_episode([transition_cls(oi, ai, ri.copy(), None, False) for oi, ai, ri in zip(o, a, r)], max_size=MAX_SIZE, step=step)


def params(model) -> dict:
    return {k: v.detach().cpu().numpy().copy() for k, v in model.state_dict().items()}


def put(out: dict, prefix: str, d: dict):
    for k, v in d.items():
        out[f"{prefix}/{k}"] = np.asarray(v)


def update_cases(out: dict):
    pcn = rh.import_reference("morl_baselines.multi_policy.pcn.pcn")
    for name, c in UPDATE_CASES.items():
        env = VarLengthEnv(**c["env"], seed=c["seed"])
        th.manual_seed(c["seed"])
        agent = pcn.PCN(env, np.array(c["scaling"], np.float32), learning_rate=c["lr"], batch_size=c["batch"], hidden_dim=c["hidden"], log=False,
                        seed=c["seed"], device="cpu")
        fill(agent, env, c["seed"], pcn.Transition)
        init = params(agent.model)
        rng_state = agent.np_random.bit_generator.state
        put(out, f"update_{name}/init", init)
        losses, ents = [], []
        for u in range(N_UPDATES):
            l, lp = agent.update()
            losses.append(l.detach().cpu().numpy())
            if name == "disc":
                lpn = lp.detach().cpu().numpy()
                ents.append(np.sum(-np.exp(lpn) * lpn))
            if u == 0:
                put(out, f"update_{name}/after1", params(agent.model))
                out[f"update_{name}/pred1"] = lp.detach().cpu().numpy()
        put(out, f"update_{name}/afterU", params(agent.model))
        out[f"update_{name}/loss"] = np.array(losses, np.float32)
        out[f"update_{name}/entropy"] = np.array(ents, np.float32)
        out[f"update_{name}/heap_steps"] = np.array([e[1] for e in agent.experience_replay])
        agent.np_random.bit_generator.state = rng_state


def rank_cases(out: dict):
    lcn = rh.import_reference("morl_baselines.multi_policy.lcn.lcn")
    for mode, lam in (("nondominated", None), ("lambda_lorenz", 0.4)):
        env = VarLengthEnv(obs_dim=3, n_actions=2, reward_dim=3, seed=11)
        agent = lcn.LCN(env, np.ones(4, np.float32), log=False, seed=11, device="cpu", distance_ref=mode, lcn_lambda=lam)
        agent.cd_threshold = 0.3
        fill(agent, env, 11, lcn.Transition, duplicate_every=7)
        cmds, heaps = [], []
        for n in (8, 5):
            cmds.append(np.concatenate(agent._choose_commands(n), axis=None))
            heaps.append(np.array([(float(e[0]), e[1]) for e in agent.experience_replay]))
            o, a, r = random_episode(env, np.random.default_rng(77))
            agent._add_episode([lcn.Transition(oi, ai, ri.copy(), None, False) for oi, ai, ri in zip(o, a, r)], max_size=MAX_SIZE, step=1000)
        out[f"rank_{mode}/commands"] = np.array(cmds, np.float32)
        out[f"rank_{mode}/heap0"] = heaps[0]
        out[f"rank_{mode}/heap1"] = heaps[1]


TRAIN = {
    "pcn": dict(env=dict(obs_dim=4, n_actions=3, reward_dim=2), scaling=[1.0, 1.0, 0.1], ctor=dict(learning_rate=1e-3, batch_size=32, seed=21),
                train=dict(total_timesteps=160, ref_point=np.array([-5.0, -5.0]), num_er_episodes=8, num_step_episodes=3, num_model_updates=5,
                           max_return=np.array([15.0, 15.0], np.float32), max_buffer_size=12, num_points_pf=3)),
    "lcn": dict(env=dict(obs_dim=3, n_actions=2, reward_dim=3), scaling=[1.0, 1.0, 1.0, 0.1], ctor=dict(learning_rate=1e-2, batch_size=16, seed=22),
                train=dict(total_timesteps=120, ref_point=np.zeros(3), num_er_episodes=10, num_step_episodes=2, num_model_updates=4,
                           max_return=np.full(3, 10.0, dtype=np.float32), max_buffer_size=12, num_points_pf=3, cd_threshold=0.2)),
}


def train_cases(out: dict):
    for algo, c in TRAIN.items():
        mod = rh.import_reference(f"morl_baselines.multi_policy.{algo}.{algo}")
        cls = mod.PCN if algo == "pcn" else mod.LCN
        env, eval_env = VarLengthEnv(**c["env"], seed=31), VarLengthEnv(**c["env"], seed=32)
        th.manual_seed(c["ctor"]["seed"])
        agent = cls(env, np.array(c["scaling"], np.float32), log=False, device="cpu", **c["ctor"])
        put(out, f"train_{algo}/init", params(agent.model))
        cmds = []
        choose = agent._choose_commands

        def recording(n, choose=choose, cmds=cmds):
            r, h = choose(n)
            cmds.append(np.concatenate([r, [h]]).astype(np.float32))
            return r, h

        agent._choose_commands = recording
        cwd = os.getcwd()
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            try:
                agent.train(eval_env=eval_env, **c["train"])
            finally:
                os.chdir(cwd)
        put(out, f"train_{algo}/final", params(agent.model))
        out[f"train_{algo}/commands"] = np.array(cmds)
        out[f"train_{algo}/heap_steps"] = np.array([e[1] for e in agent.experience_replay])
        out[f"train_{algo}/heap_returns"] = np.array([e[2][0].reward for e in agent.experience_replay])
        out[f"train_{algo}/heap_lengths"] = np.array([len(e[2]) for e in agent.experience_replay])
        out[f"train_{algo}/global_step"] = np.array(agent.global_step)


def main():
    th.set_num_threads(1)
    out: dict = {}
    update_cases(out)
    rank_cases(out)
    train_cases(out)
    path = os.path.join(HERE, "pcn.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
