"""MOPPO (single_policy/ser/mo_ppo.py) against the unmodified reference (tests/golden/mo_ppo.npz, tests/golden/make_golden_mo_ppo.py),
and the engine's own guarantees: the CUDA-graph update is bit-identical to the eager one, target_kl stops after the reference's number
of shuffles, anneal_lr follows the reference's schedule without a re-capture, and a deep copy is independent with a fresh Adam."""

import os
from copy import deepcopy

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import ops
from morl_baselines_b200.single_policy.ser.mo_ppo import MOPPO, MOPPONet, PPOReplayBuffer
from tests.golden.make_golden_mo_ppo import (ACT, ARCH, EPOCHS, MINIBATCHES, NEXT_DONE, OBS, WEIGHTS, CountingRng, E, T, cases, split_gae,
                                             synthetic_batch, tag, unflat)
from tests.ppo_standin import fake_vec_env

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mo_ppo.npz"))
CASES = list(enumerate(cases()))
# Deviation of the parameters after a whole update (2 epochs x 4 minibatches) from the reference's CPU run, as ``_rel_dev`` measures it:
# at most 8.7e-7 over the 33 cases (8.4e-7 after the first minibatch step), measured on an H100 80GB HBM3.  The device's float32
# forward and backward round differently from the CPU's, and Adam's first steps (which divide by sqrt(v) ~ |g|) carry those differences
# into every step.
FULL_UPDATE_TOL = 5e-6


class _StandIn:
    num_envs = E


def _agent(cuda, k, c, use_cuda_graph=True, rng=None):
    t = tag(c)
    d = c["d"]
    net = MOPPONet((OBS,), (ACT,), d, ARCH).to(cuda)
    net.load_state_dict({key: th.from_numpy(v) for key, v in unflat(G[f"init_d{d}"], net.state_dict()).items()})
    agent = MOPPO(0, net, WEIGHTS[d], _StandIn(), steps_per_iteration=T, num_minibatches=MINIBATCHES, update_epochs=EPOCHS, gae=bool(c["gae"]),
                  clip_vloss=bool(c["clip_vloss"]), norm_adv=bool(c["norm_adv"]), ent_coef=c["ent_coef"], target_kl=c["target_kl"], device=cuda,
                  rng=rng if rng is not None else CountingRng(7 + k), use_cuda_graph=use_cuda_graph)
    sb, ref = synthetic_batch(k, d), split_gae(G[f"{t}/gae"], d)
    for f in ("obs", "actions", "rewards", "dones", "values"):
        getattr(agent.batch, f).copy_(th.from_numpy(sb[f]))
    agent.batch.logprobs.copy_(th.from_numpy(ref["logprobs"]))
    # the reference's next_value (the critic's output on its CPU), so the returns can be compared bit for bit
    ops.vector_gae(agent.batch.rewards, agent.batch.values, agent.batch.dones, th.from_numpy(ref["next_value"]).to(cuda),
                   th.from_numpy(NEXT_DONE).to(cuda), agent._w32, agent.gamma, agent.gae_lambda, agent.gae, returns_out=agent.returns,
                   adv_out=agent.advantages)
    return agent


def _rel_dev(sd, ref_flat):
    """Largest parameter deviation from the reference, relative to each tensor's largest magnitude, floored at 0.01: after Adam's first
    steps ``actor_logstd`` is about the learning rate (3e-4) in size, and a step that divides a gradient by sqrt(v) + eps turns the
    float32 rounding of a small gradient into ~3e-8 absolute, which is 1e-4 of that tensor but far below any other parameter's scale."""
    worst = 0.0
    for key, ref in unflat(ref_flat, sd).items():
        v = sd[key]
        worst = max(worst, float(np.abs(v.detach().cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1e-2)))
    return worst


@pytest.mark.parametrize("k,c", CASES, ids=[tag(c) for _, c in CASES])
def test_update_matches_reference(cuda, k, c):
    agent = _agent(cuda, k, c, use_cuda_graph=False)
    # the engine's GAE outputs against the reference's (returns bit-exact)
    assert np.array_equal(agent.returns.cpu().numpy(), split_gae(G[f"{tag(c)}/gae"], c["d"])["returns"])
    step, first = agent.optimizer.step_fused, {}

    def record(*a, **kw):
        step(*a, **kw)
        if not first:
            first.update({key: v.detach().clone() for key, v in agent.networks.state_dict().items()})

    agent.optimizer.step_fused = record
    agent.update()
    dev_first = _rel_dev(first, G[f"{tag(c)}/params"][0])
    assert dev_first <= 1e-5, dev_first
    dev_full = _rel_dev(agent.networks.state_dict(), G[f"{tag(c)}/params"][1])
    assert dev_full <= FULL_UPDATE_TOL, f"full-update deviation {dev_full:.3g}"
    assert agent.np_random.shuffles == int(G[f"{tag(c)}/shuffles"])


@pytest.mark.parametrize("k,c", [CASES[0], CASES[-1], CASES[13]], ids=["plain", "target_kl", "other"])
def test_graph_and_eager_updates_are_bit_identical(cuda, k, c):
    a, b = _agent(cuda, k, c, use_cuda_graph=True), _agent(cuda, k, c, use_cuda_graph=False)
    for _ in range(2):
        a.update()
        b.update()
        for p, q in zip(a.networks.parameters(), b.networks.parameters()):
            assert th.equal(p, q)
        assert th.equal(a._stats, b._stats)
    assert a.np_random.shuffles == b.np_random.shuffles


def test_target_kl_stops_like_the_reference(cuda):
    k, c = CASES[-1]
    agent = _agent(cuda, k, c)
    agent.update()
    assert int(G[f"{tag(c)}/shuffles"]) == 1 and agent.np_random.shuffles == 1


def test_anneal_lr_follows_the_schedule_without_recapture(cuda):
    th.manual_seed(0)
    envs = fake_vec_env(2, obs_dim=OBS, act_dim=ACT, reward_dim=2)
    net = MOPPONet((OBS,), (ACT,), 2, [32, 32]).to(cuda)
    agent = MOPPO(0, net, WEIGHTS[2], envs, steps_per_iteration=16, num_minibatches=4, update_epochs=2, anneal_lr=True, learning_rate=3e-4,
                  device=cuda)
    graphs = None
    for it in range(1, 4):
        agent.train(0.0, it, 3)
        lr = (1.0 - (it - 1.0) / 3) * 3e-4
        assert agent._lr.item() == lr and agent.optimizer.param_groups[0]["lr"] == lr
        st = agent._graphs["all"]
        if graphs is None:
            graphs = st["graph"].graph
        assert st["graph"].graph is graphs and len(agent._graphs) == 1


def test_learning_rate_scalar_is_read_at_replay(cuda):
    """A graph captured at one learning rate, replayed after ``set_learning_rate``, equals an eager update at the new rate; the
    in-place ``become_copy_of`` (PGMORL's task-selection swap) resets the learner under the kept graph."""
    k, c = CASES[0]
    a = _agent(cuda, k, c)
    a.update()
    graph = a._graphs["all"]["graph"].graph
    a.become_copy_of(_agent(cuda, k, c, use_cuda_graph=False))
    a.np_random = CountingRng(7 + k)
    a.set_learning_rate(1e-4)
    a.update()
    assert a._graphs["all"]["graph"].graph is graph
    ref = _agent(cuda, k, c, use_cuda_graph=False)
    ref.set_learning_rate(1e-4)
    ref.update()
    for p, q in zip(a.networks.parameters(), ref.networks.parameters()):
        assert th.equal(p, q)


def test_deepcopy_is_independent_with_a_fresh_adam(cuda):
    k, c = CASES[0]
    agent = _agent(cuda, k, c)
    agent.update()
    agent.global_step = 123
    cp = deepcopy(agent)
    assert cp.global_step == 123 and cp.seed == 42 and cp.np_random is not agent.np_random
    assert len(cp.optimizer.state) == 0 and len(agent.optimizer.state) > 0
    for p, q in zip(agent.networks.parameters(), cp.networks.parameters()):
        assert th.equal(p, q) and p.data_ptr() != q.data_ptr()
    for f in PPOReplayBuffer.FIELDS:
        x, y = getattr(agent.batch, f), getattr(cp.batch, f)
        assert th.equal(x, y) and x.data_ptr() != y.data_ptr()
    before = [p.detach().clone() for p in agent.networks.parameters()]
    cp.update()
    for p, q in zip(agent.networks.parameters(), before):
        assert th.equal(p, q)
