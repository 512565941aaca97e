"""Whole-update parity of ``morl_baselines_b200.Envelope.update()`` against the UNMODIFIED reference at the BASELINE.json shapes.

tests/golden/envelope_update.npz holds what the reference's ``Envelope.update()`` (multi_policy/envelope/envelope.py:266-367) produced on
CPU for the north-star shape (obs 32, |A| 8, d 3, |W| 64, B 1024, 4x256), for BASELINE configs[1] (minecart dims, |W| 32, B 256) and
for a homotopy-schedule run (tests/golden/make_golden_envelope_update.py).  Here the CUDA engine -- device replay gather, tensor-core dense
layers on the B*|W| distinct rows (74-pair persistent schedule, tail split, snake order at the north-star shape), fused envelope-TD,
fused loss / priorities, hand-written backward, fused clip + Adam, CUDA-graph replay -- runs the same updates from the same initial
parameters, replay store, sum-tree and RNG streams.

Bounds (BASELINE.json north_star: "Q-values and losses within 1e-5 relative fp32"):
  * sampled indices, weight sets            : identical (host RNG mirror: global numpy RNG for the sum-tree walk, agent.np_random for the weights)
  * critic loss                             : 1e-5 relative (measured 0 .. 7e-7)
  * priorities (|w . td| + min_p)^alpha     : |p - p_ref| <= 1e-5 |p_ref| + 2e-6 on >= 99 % of the B rows (measured: 0 .. 7 of 1024 rows outside).
                                              td = Q - target with |Q|, |target| ~ 1; both engines carry ~1e-6 absolute fp32 GEMM noise on Q
                                              (different summation orders), a LARGE relative error on rows where w . td cancels to ~1e-4
                                              -- hence the absolute term -- and the envelope target is an ARGMAX over |W| x |A| = 512
                                              candidates: where the two best candidates are closer than that noise, a different GEMM
                                              (cuBLAS included) may select the other one and the row's target jumps -- hence the 1 %
                                              allowance.  (That the argmax itself is bit-exact on identical Q inputs is what
                                              tests/test_kernels_gpu.py pins against the reference's own outputs.)
  * parameters after the last update        : |p - p_ref| <= 1e-5 |p_ref| + 2e-6 on >= 98 % of the elements of every tensor (measured >= 99.2 %),
                                              never more than 2 lr per update, and the float64 sum of every tensor within 1e-6 of its abs-sum.
                                              Adam's first steps move every element by ~lr * g / |g| whatever |g| is: where a gradient
                                              element is at the level of its own rounding noise (~1e-8) the two engines legitimately step
                                              in different directions, so no per-element bound below lr can hold for ALL 212,760 elements.
"""

import os

import numpy as np
import pytest
import torch as th

from morl_baselines_b200.testing import FakeEnv
from tests.golden.envelope_update_cases import CASES, fill_agent, perturbed_target

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "envelope_update.npz")
LOSS_RTOL = 1e-5
PRIO_RTOL, PRIO_ATOL = 1e-5, 2e-6
PRIO_FRAC = 0.99
PARAM_RTOL, PARAM_ATOL, PARAM_FRAC = 1e-5, 2e-6, 0.98


def _run_case(name, cuda, tc, graph, **extra):
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope

    g = np.load(GOLD)
    c = CASES[name]
    agent = Envelope(FakeEnv(obs_dim=c["obs"], n_actions=c["A"], reward_dim=c["D"]), batch_size=c["B"], num_sample_w=c["W"], per=True,
                     buffer_size=c["N"], net_arch=c["net"], log=False, seed=c["seed"], device=cuda, use_cuda_graph=graph, use_tensor_cores=tc,
                     **c["kwargs"], **extra)
    assert agent.use_tensor_cores == tc
    fill_agent(agent, c)
    init = {k: th.from_numpy(g[f"{name}/init/{k}"]) for k in agent.q_net.state_dict()}
    agent.q_net.load_state_dict(init)
    agent.target_q_net.load_state_dict(perturbed_target(init))
    lr = agent.learning_rate
    for step in range(c["steps"]):
        agent.global_step = c["global_step0"] + step
        np.random.seed(c["np_seed"] + step)
        assert abs(float(agent.homotopy_lambda) - float(g[f"{name}/step{step}/lambda"])) < 1e-12
        agent.update()
        np.testing.assert_array_equal(agent._last_inds, g[f"{name}/step{step}/inds"], err_msg=f"{name} step {step}: replay indices")
        loss, ref = float(agent._last_loss), float(g[f"{name}/step{step}/loss"])
        assert abs(loss - ref) <= LOSS_RTOL * abs(ref), (name, step, loss, ref)
        pref = g[f"{name}/step{step}/priority"]
        perr = np.abs(agent._last_priority - pref)
        p_ok = perr <= PRIO_RTOL * np.abs(pref) + PRIO_ATOL
        assert p_ok.mean() >= PRIO_FRAC, (name, step, "priorities", float(p_ok.mean()), float(perr.max()))
        sums = np.array([float(v.double().sum()) for v in agent.q_net.state_dict().values()])
        np.testing.assert_allclose(sums, g[f"{name}/step{step}/param_sums"], rtol=0, atol=1e-6 * g[f"{name}/step{step}/param_abs_sums"].max())
    worst = 0.0
    for k, v in agent.q_net.state_dict().items():
        ref = g[f"{name}/final/{k}"]
        err = np.abs(v.cpu().numpy() - ref)
        ok = err <= PARAM_RTOL * np.abs(ref) + PARAM_ATOL
        assert (~ok).sum() <= max(3, (1 - PARAM_FRAC) * ok.size), (name, k, float(ok.mean()), float(err.max()))
        assert err.max() <= 2 * lr * c["steps"], (name, k, float(err.max()))
        worst = max(worst, float(err.max()))
    assert abs(agent.replay_buffer.min_priority - float(g[f"{name}/min_priority"])) <= 1e-5 * float(g[f"{name}/min_priority"])
    return worst


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("tc", [True, False])
def test_north_star_update_matches_unmodified_reference(cuda, tc, graph):
    """B = 1024, |W| = 64, 4 x 256: the exact configuration bench.py times."""
    _run_case("north_star", cuda, tc, graph)


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("tc", [True, False])
def test_config2_update_matches_unmodified_reference(cuda, tc, graph):
    _run_case("config2", cuda, tc, graph)


@pytest.mark.parametrize("graph", [True, False])
def test_homotopy_schedule_update_matches_unmodified_reference(cuda, graph):
    """lambda changes every update: the captured graph must read it from memory (it used to force the eager path)."""
    _run_case("homotopy", cuda, True, graph)


def test_north_star_update_bf16x3_operand_format(cuda):
    """The wide-range operand format (three bf16 planes, six MMAs per product) through the same goldens."""
    _run_case("north_star", cuda, True, True, tensor_core_format="bf16x3")


def test_north_star_update_split_accumulators(cuda):
    """The higher-accuracy accumulator mode of the forward GEMMs (leading / correction products in separate accumulators)."""
    _run_case("north_star", cuda, True, True, tensor_core_accumulators="split")
