"""The graph inputs of every graphed learner update are staged through pinned memory (common/graphed.Staging; Envelope: its one
pinned per-step pack).  When the host runs ahead of the device, a pinned input must not be rewritten while the asynchronous copy that
reads it is still queued; otherwise an update trains on a later update's minibatch.

Each case runs the same updates on two identically seeded agents with no injected noise.  Agent A captures its graphs, then holds the
stream with one bounded device spin and queues all updates without a synchronise, so the host is certainly ahead of the device.  Agent
B synchronises after every update.  Every parameter, optimiser moment and step counter, and every other tensor the learner keeps
(``log_alpha``, the temperature, the last losses, Envelope's sum tree) must be equal bit for bit."""

import random

import numpy as np
import pytest
import torch as th

from oracle.ref_harness import FakeEnv

pytestmark = pytest.mark.gpu

K = 4  # updates queued behind the held stream
HOLD_CYCLES = 100_000_000  # one spin of about 50 ms at the H100's clocks: longer than the host needs to queue K updates


def _fill(buf, rng, n, obs, act, d, act_dtype=np.float32, discrete=0):
    buf.obs[:n] = rng.standard_normal((n, obs)).astype(np.float32)
    buf.next_obs[:n] = rng.standard_normal((n, obs)).astype(np.float32)
    if discrete:
        buf.actions[:n] = rng.integers(0, discrete, (n, 1)).astype(act_dtype)
    else:
        buf.actions[:n] = rng.uniform(-1, 1, (n, act)).astype(act_dtype)
    buf.rewards[:n] = rng.standard_normal((n, d)).astype(np.float32)
    buf.dones[:n] = (rng.random((n, 1)) < 0.1).astype(np.float32)
    buf.size, buf.ptr = n, n % buf.max_size
    buf.mark_all_dirty()


def _tensors(obj, prefix=""):
    """(name, tensor) of every parameter, module buffer, optimiser state and plain tensor attribute of a learner."""
    out = []
    for name, v in vars(obj).items():
        mods = v if isinstance(v, (list, tuple)) and v and all(isinstance(m, th.nn.Module) for m in v) else [v]
        for i, m in enumerate(mods):
            if isinstance(m, th.nn.Module):
                out += [(f"{prefix}{name}[{i}].{k}", t) for k, t in m.state_dict().items()]
        if isinstance(v, th.optim.Optimizer):
            for j, st in enumerate(v.state.values()):
                out += [(f"{prefix}{name}.state[{j}].{k}", t) for k, t in st.items() if th.is_tensor(t)]
        elif th.is_tensor(v):
            out.append((f"{prefix}{name}", v))
    return out


def _mosac(cuda):
    from morl_baselines_b200.single_policy.ser.mosac_continuous_action import MOSAC

    agent = MOSAC(FakeEnv(obs_dim=11, continuous_action_dim=3, reward_dim=3), weights=np.array([0.2, 0.5, 0.3], np.float32), batch_size=32,
                  net_arch=[64, 64], log=False, seed=4, device=cuda, buffer_size=256)
    _fill(agent.buffer, np.random.default_rng(5), 256, 11, 3, 3)

    def update(step):
        agent.global_step = step  # policy_freq 2: two variants, with and without the actor / temperature steps
        agent.update()

    return agent, [lambda s=s: update(s) for s in range(2)], [lambda s=s: update(s) for s in range(2, 2 + K)], lambda: _tensors(agent)


def _mosac_discrete(cuda):
    from morl_baselines_b200.single_policy.ser.mosac_discrete_action import MOSACDiscrete

    agent = MOSACDiscrete(FakeEnv(obs_dim=8, n_actions=4, reward_dim=4), weights=np.array([0.1, 0.4, 0.3, 0.2], np.float32), batch_size=32,
                          net_arch=[64, 64], log=False, seed=4, device=cuda, buffer_size=256, tau=0.5, update_frequency=1,
                          target_net_freq=2)
    _fill(agent.buffer, np.random.default_rng(5), 256, 8, 1, 4, discrete=4)

    def update(step):
        agent.global_step = step  # target_net_freq 2: two variants, with and without the target sync
        agent.update()

    return agent, [lambda s=s: update(s) for s in range(2)], [lambda s=s: update(s) for s in range(2, 2 + K)], lambda: _tensors(agent)


def _capql(cuda):
    from morl_baselines_b200.multi_policy.capql.capql import CAPQL

    OBS, ACT, D = 9, 3, 2
    agent = CAPQL(FakeEnv(obs_dim=OBS, continuous_action_dim=ACT, reward_dim=D), batch_size=32, net_arch=[64, 64], log=False, seed=2,
                  device=cuda, buffer_size=1024, gradient_updates=3)
    rng = np.random.default_rng(5)
    for _ in range(256):
        w = rng.dirichlet(np.ones(D)).astype(np.float32)
        agent.replay_buffer.push(rng.standard_normal(OBS).astype(np.float32), rng.uniform(-1, 1, ACT).astype(np.float32), w,
                                 rng.standard_normal(D).astype(np.float32), rng.standard_normal(OBS).astype(np.float32), float(rng.random() < 0.1))
    return agent, [agent.update], [agent.update] * K, lambda: _tensors(agent)


def _gpils(cuda):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPILS

    OBS, A, D = 10, 4, 3
    agent = GPILS(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), batch_size=32, net_arch=[64, 64, 64], num_nets=2, gradient_updates=3, per=False,
                  drop_rate=0.0, buffer_size=256, log=False, seed=1, device=cuda, target_net_update_freq=3)
    _fill(agent.replay_buffer, np.random.default_rng(5), 256, OBS, 1, D, act_dtype=np.uint8, discrete=A)
    support = np.random.default_rng(6).dirichlet(np.ones(D), 8).astype(np.float32)  # > 5 weights: support picks and sampled weights
    agent.set_weight_support(list(support))
    w = th.tensor(support[2]).to(cuda)

    def update():
        agent.update(w)
        agent.global_step += 1

    return agent, [update], [update] * K, lambda: _tensors(agent)


def _gpils_continuous(cuda):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd_continuous_action import GPILSContinuousAction

    OBS, ACT, D = 11, 3, 3
    agent = GPILSContinuousAction(FakeEnv(obs_dim=OBS, continuous_action_dim=ACT, reward_dim=D), batch_size=32, net_arch=[64, 64], num_q_nets=2,
                                  gradient_updates=3, per=False, buffer_size=256, log=False, seed=3, device=cuda)
    _fill(agent.replay_buffer, np.random.default_rng(5), 256, OBS, ACT, D)
    agent.set_weight_support(list(np.random.default_rng(6).dirichlet(np.ones(D), 4).astype(np.float32)))
    w = agent.weight_support[1].clone()
    # delay_policy_update 2 over 3 steps per update: both variants, with and without the actor step
    return agent, [lambda: agent.update(w)], [lambda: agent.update(w)] * K, lambda: _tensors(agent)


def _mo_ppo(cuda):
    from morl_baselines_b200 import ops
    from morl_baselines_b200.single_policy.ser.mo_ppo import MOPPO, MOPPONet
    from tests.ppo_standin import fake_vec_env

    OBS, ACT, D = 6, 2, 2
    net = MOPPONet((OBS,), (ACT,), D, [32, 32]).to(cuda)
    agent = MOPPO(0, net, np.array([0.3, 0.7]), fake_vec_env(2, obs_dim=OBS, act_dim=ACT, reward_dim=D), steps_per_iteration=16,
                  num_minibatches=4, update_epochs=3, device=cuda, rng=np.random.default_rng(7))
    g = th.Generator(device=cuda).manual_seed(8)
    b = agent.batch
    for t in (b.obs, b.actions, b.rewards, b.values):
        t.copy_(th.randn(t.shape, device=cuda, generator=g))
    b.logprobs.copy_(-th.rand(b.logprobs.shape, device=cuda, generator=g))
    ops.vector_gae(b.rewards, b.values, b.dones, th.randn(2, D, device=cuda, generator=g), th.zeros(2, device=cuda), agent._w32, agent.gamma,
                   agent.gae_lambda, agent.gae, returns_out=agent.returns, adv_out=agent.advantages)

    def update():
        agent.prepare_update().graph()

    return agent, [update], [update] * K, lambda: _tensors(agent)


def _morld_mosac(cuda):
    from morl_baselines_b200.multi_policy.morld.morld import MORLD

    env = FakeEnv(obs_dim=6, continuous_action_dim=2, reward_dim=2, horizon=20)
    algo = MORLD(env, pop_size=5, exchange_every=60, update_passes=1, log=False, device=cuda, seed=0, weight_init_method="random",
                 policy_args={"learning_starts": 0, "batch_size": 16, "net_arch": [32, 32], "buffer_size": 256}, neighborhood_size=1)
    for p in algo.population:
        _fill(p.wrapped.get_buffer(), np.random.default_rng(10 + p.id), 64, 6, 2, 2)
        p.wrapped.global_step = 4

    def update():
        algo._update_others(algo.population[1])

    return algo, [update], [update] * K, lambda: [x for p in algo.population for x in _tensors(p.wrapped, f"population[{p.id}].")]


def _envelope(mode):
    """Envelope in one graph mode: sum tree in HBM ("device_per"), HBM replay mirror without PER ("device"), host-resident buffer ("host")."""

    def case(cuda):
        from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

        OBS, A, D = 12, 4, 3
        per = mode != "device"
        agent = Envelope(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), batch_size=32, num_sample_w=8, per=per, buffer_size=256,
                         net_arch=[64, 64, 64], gradient_updates=4, target_net_update_freq=2, log=False, seed=3, device=cuda,
                         replay_on_device=mode != "host")
        rb = agent.replay_buffer
        _fill(rb, np.random.default_rng(5), 256, OBS, 1, D, act_dtype=np.uint8, discrete=A)
        if per:
            rb.tree.batch_set(np.arange(256), np.random.default_rng(6).random(256) + 0.01)
        agent.global_step = 1

        def update():
            agent.update()
            agent.global_step += 1

        def state():
            out = _tensors(agent)
            if per:
                out += [("replay_buffer.tree", th.from_numpy(np.concatenate(rb.tree.nodes))),
                        ("replay_buffer.min_priority", th.tensor(rb.min_priority, dtype=th.float64))]
            return out

        def warmup():
            update()
            assert list(agent._graphs) == [mode]

        return agent, [warmup], [update] * K, state

    return case


CASES = {"mosac": _mosac, "mosac_discrete": _mosac_discrete, "capql": _capql, "gpils": _gpils, "gpils_continuous": _gpils_continuous,
         "mo_ppo": _mo_ppo, "morld_mosac": _morld_mosac, "envelope_device_per": _envelope("device_per"), "envelope_device": _envelope("device"),
         "envelope_host": _envelope("host")}


def _run(case, cuda, held: bool):
    random.seed(1)
    np.random.seed(2)
    th.manual_seed(3)
    agent, warmup, updates, state = case(cuda)
    for u in warmup:  # captures every graph variant the updates replay
        u()
    th.cuda.synchronize()
    if held:
        th.cuda._sleep(HOLD_CYCLES)
    for u in updates:
        u()
        if not held:
            th.cuda.synchronize()
    th.cuda.synchronize()
    return [(name, t.detach().clone()) for name, t in state()]


@pytest.mark.parametrize("name", list(CASES))
def test_updates_read_their_own_inputs_when_the_host_runs_ahead(cuda, name):
    ahead = _run(CASES[name], cuda, held=True)
    in_step = _run(CASES[name], cuda, held=False)
    assert [n for n, _ in ahead] == [n for n, _ in in_step] and len(ahead) > 0
    differ = [n for (n, a), (_, b) in zip(ahead, in_step) if not th.equal(a, b)]
    assert not differ, f"{len(differ)} of {len(ahead)} tensors differ, e.g. {differ[:5]}"
