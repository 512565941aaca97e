"""Host halves of PCN / LCN without a GPU: the heap mirror, the index draws, return-to-go and the ranking against the reference
(tests/golden/pcn.npz, and the reference itself where its source tree is available), and the model's state-dict keys."""

import os

import numpy as np
import pytest
import torch as th

from morl_baselines_b200.multi_policy.lcn.lcn import LCN
from morl_baselines_b200.multi_policy.pcn.pcn import (
    PCN,
    ContinuousActionsDefaultModel,
    DiscreteActionsDefaultModel,
    EpisodeHeap,
    draw_update_indices,
    return_to_go,
)
from oracle import ref_harness as rh
from tests.golden import make_golden_pcn as mg
from tests.pcn_standin import VarLengthEnv, random_episode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "pcn.npz"))
needs_reference = pytest.mark.skipif(not rh.reference_available(), reason="reference source tree not available")


def _host_non_dominated(solutions):
    """The repository's get_non_dominated_inds with the dominance test of the C oracle instead of the device kernel (same exact compares)."""
    from oracle import oracle as orc

    sol = np.asarray(solutions)
    return np.ones(len(sol), dtype=bool) if len(sol) < 2 else orc.pareto_mask(sol.reshape(len(sol), -1), False)


@pytest.fixture(autouse=True)
def host_pareto(monkeypatch):
    import morl_baselines_b200.multi_policy.lcn.lcn as lcn_mod
    import morl_baselines_b200.multi_policy.pcn.pcn as pcn_mod

    monkeypatch.setattr(pcn_mod, "get_non_dominated_inds", _host_non_dominated)
    monkeypatch.setattr(lcn_mod, "get_non_dominated_inds", _host_non_dominated)


class HostAgent:
    """The host half of a PCN / LCN agent: its heap, generator and ranking, with episodes kept as (return-to-go rows, length)."""

    def __init__(self, cls, seed, **attrs):
        self.agent = cls.__new__(cls)
        self.agent._heap = EpisodeHeap()
        self.agent.np_random = np.random.default_rng(seed)
        self.agent.__dict__.update(attrs)
        self.next_slot = 0

    def add(self, rewards, step):
        rtg = return_to_go(np.array(rewards, dtype=np.float32), self.agent.gamma)
        self.agent._heap.add(self.next_slot, rtg[0].copy(), len(rtg), step, mg.MAX_SIZE)
        self.next_slot += 1

    def fill(self, env, seed, duplicate_every=0):
        prev = None
        for k, (ep_seed, step) in enumerate(mg.episode_plan(seed)):
            if k == mg.RANK_AT:
                self.agent._nlargest(mg.RANK_N, self.agent._threshold())
            if duplicate_every and prev is not None and k % duplicate_every == 0:
                r = prev
            else:
                _, _, r = random_episode(env, np.random.default_rng(ep_seed))
            prev = r
            self.add(r, step)


@pytest.mark.parametrize("name", list(mg.UPDATE_CASES))
def test_heap_positions_follow_the_reference(name):
    c = mg.UPDATE_CASES[name]
    h = HostAgent(PCN, c["seed"], gamma=1.0)
    h.fill(VarLengthEnv(**c["env"], seed=c["seed"]), c["seed"])
    assert [e[1] for e in h.agent.experience_replay] == list(GOLDEN[f"update_{name}/heap_steps"])


@pytest.mark.parametrize("mode,lam", [("nondominated", None), ("lambda_lorenz", 0.4)])
def test_lcn_ranking_and_commands_bit_equal(mode, lam):
    h = HostAgent(LCN, 11, gamma=1.0, distance_ref=mode, lcn_lambda=lam, cd_threshold=0.3)
    env = VarLengthEnv(obs_dim=3, n_actions=2, reward_dim=3, seed=11)
    h.fill(env, 11, duplicate_every=7)
    for i, n in enumerate((8, 5)):
        r, hor = h.agent._choose_commands(n)
        assert r.dtype == np.float32 and np.array_equal(np.concatenate([r, [hor]]).astype(np.float32), GOLDEN[f"rank_{mode}/commands"][i])
        heap = np.array([(float(e[0]), e[1]) for e in h.agent.experience_replay])
        assert np.array_equal(heap, GOLDEN[f"rank_{mode}/heap{i}"])
        _, _, rew = random_episode(env, np.random.default_rng(77))
        h.add(rew, 1000)


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4])
def test_vector_timestep_draw_equals_sequential_draws(seed):
    lengths = np.random.default_rng(100 + seed).integers(1, 1000, size=57)
    a, b = np.random.default_rng(seed), np.random.default_rng(seed)
    pos, t = draw_update_indices(a, lengths, 64, 3)
    for u in range(3):
        p = b.choice(np.arange(len(lengths)), size=64, replace=True)
        assert np.array_equal(p, pos[u])
        assert np.array_equal([b.integers(0, lengths[i]) for i in p], t[u])
    assert a.random() == b.random()


@needs_reference
def test_return_to_go_bit_equal_to_reference():
    pcn = rh.import_reference("morl_baselines.multi_policy.pcn.pcn")
    rng = np.random.default_rng(0)
    for gamma in (1.0, 0.99, 0.9):
        rewards = rng.standard_normal((40, 3)).astype(np.float32) * 10
        ref = type("R", (), {"gamma": gamma, "experience_replay": []})()
        ts = [pcn.Transition(None, 0, r.copy(), None, False) for r in rewards]
        pcn.PCN._add_episode(ref, ts, max_size=5, step=1)
        assert np.array_equal(np.array([t.reward for t in ts]), return_to_go(rewards.copy(), gamma))


@needs_reference
@pytest.mark.parametrize("mode,lam", [("nondominated", None), ("lambda_lorenz", 0.7)])
def test_heap_mirror_tracks_reference_through_adds_and_rankings(mode, lam):
    lcn = rh.import_reference("morl_baselines.multi_policy.lcn.lcn")
    env_a, env_b = (VarLengthEnv(obs_dim=2, n_actions=2, reward_dim=4, seed=5) for _ in range(2))
    ref = lcn.LCN(env_a, np.ones(5, np.float32), log=False, seed=5, device="cpu", distance_ref=mode, lcn_lambda=lam)
    ref.cd_threshold = 0.25
    h = HostAgent(LCN, 5, gamma=1.0, distance_ref=mode, lcn_lambda=lam, cd_threshold=0.25)
    for k in range(60):
        o, a, r = random_episode(env_a, np.random.default_rng(k))
        _, _, r2 = random_episode(env_b, np.random.default_rng(k))
        ref._add_episode([lcn.Transition(oi, ai, ri.copy(), None, False) for oi, ai, ri in zip(o, a, r)], max_size=mg.MAX_SIZE, step=k + 1)
        h.add(r2, k + 1)
        if k % 9 == 8:
            assert np.array_equal(np.concatenate(ref._choose_commands(6), axis=None), np.concatenate(h.agent._choose_commands(6), axis=None))
        ref_heap = [(e[0], e[1], e[2][0].reward, len(e[2])) for e in ref.experience_replay]
        ours = [(e[0], e[1], h.agent._heap.returns[e[2]], h.agent._heap.lengths[e[2]]) for e in h.agent.experience_replay]
        assert len(ref_heap) == len(ours)
        for x, y in zip(ref_heap, ours):
            assert x[0] == y[0] and x[1] == y[1] and np.array_equal(x[2], y[2]) and x[3] == y[3]


def test_state_dict_keys():
    keys = ["scaling_factor", "s_emb.0.weight", "s_emb.0.bias", "c_emb.0.weight", "c_emb.0.bias", "fc.0.weight", "fc.0.bias", "fc.2.weight",
            "fc.2.bias"]
    for cls in (DiscreteActionsDefaultModel, ContinuousActionsDefaultModel):
        m = cls(4, 3, 2, np.ones(3, np.float32), 64)
        assert list(m.state_dict()) == keys
        assert not m.scaling_factor.requires_grad
    for name, c in mg.UPDATE_CASES.items():
        init = {k.split("/", 2)[2]: v for k, v in GOLDEN.items() if k.startswith(f"update_{name}/init/")}
        assert sorted(init) == sorted(keys)
        env = VarLengthEnv(**c["env"])
        cls = ContinuousActionsDefaultModel if "continuous_action_dim" in c["env"] else DiscreteActionsDefaultModel
        n_out = env.action_space.shape[0] if "continuous_action_dim" in c["env"] else env.action_space.n
        m = cls(env.observation_space.shape[0], n_out, env.reward_dim, np.array(c["scaling"], np.float32), c["hidden"])
        m.load_state_dict({k: th.from_numpy(v) for k, v in init.items()})
