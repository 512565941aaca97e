"""GPU tests of the tensor-core Q-network at the shapes this path gained: 512-wide hidden layers (per-layer launches, output columns in
two units, 16-word ReLU masks) and more than 64 scalarising weights per update (two-pass pair reduction, standalone envelope_td).

Each TCPairMlp.backward case runs the named-case check of tests/test_tc_mlp_grad_gpu.py (float64 restatement, magnitude bounds, mask
flips, the rejections of a 0.1 % scale error, swapped masks and doubled layers, layer 1 from the kernel's own dL/dh1) on a new shape.
The Envelope cases compare every .grad with the float64 gradient of the reference loss, the loss with float64 to 1e-6, and the eager
update with the CUDA-graph replay bit for bit.
"""

import numpy as np
import pytest
import torch as th

from tests.test_tc_mlp_grad_gpu import (
    C_PRODUCT,
    F16,
    F16X2_FLOOR,
    BF16,
    _loss64,
    _products,
    _ratio,
    _rejects,
    check_mask_flips,
    grad_bounds,
    kernel_masks,
    pair_rows,
    reference,
)
from tests.test_tc_mlp_grad_gpu import test_backward_matches_float64 as _backward_case
from tests.test_tc_mlp_grad_gpu import test_bf16x3_forward_only_widths as _bf16_forward_case

pytestmark = pytest.mark.gpu

# name -> (hidden widths, output columns, B, |W|, format, split accumulators, tc_mlp switches turned off, dL/dQ) as in CASES there
WIDE_CASES = {
    "2x512-o24-b1024w64": ((512,) * 2, 24, 1024, 64, F16, False, (), "dense"),
    "2x512-o72-b64w8-bf16": ((512,) * 2, 72, 64, 8, BF16, False, (), "dense"),
    "2x512-o24-b37w5-split": ((512,) * 2, 24, 37, 5, F16, True, (), "dense"),
    "4x512-o24-b1024w64": ((512,) * 4, 24, 1024, 64, F16, False, (), "dense"),
    "4x512-o24-b1024w64-sparse": ((512,) * 4, 24, 1024, 64, F16, False, (), "sparse"),
    "4x512-o24-b1024w64-bf16": ((512,) * 4, 24, 1024, 64, BF16, False, (), "dense"),
    "4x512-o24-b256w256": ((512,) * 4, 24, 256, 256, F16, False, (), "dense"),
    "3x320-o36-b300w70": ((320,) * 3, 36, 300, 70, F16, False, (), "dense"),
    "4x256-o24-b512w96": ((256,) * 4, 24, 512, 96, F16, False, (), "dense"),
    "4x256-o24-b512w128": ((256,) * 4, 24, 512, 128, F16, False, (), "dense"),
    "4x256-o24-b256w256": ((256,) * 4, 24, 256, 256, F16, False, (), "dense"),
    "4x256-o24-b256w256-bf16": ((256,) * 4, 24, 256, 256, BF16, False, (), "sparse"),
    "4x256-o24-b256w256-nochain": ((256,) * 4, 24, 256, 256, F16, False, ("_CHAIN", "_CHAIN_BWD"), "dense"),
}


@pytest.mark.parametrize("case", [pytest.param(v, id=k) for k, v in WIDE_CASES.items()])
def test_wide_backward_matches_float64(cuda, monkeypatch, case):
    _backward_case(cuda, monkeypatch, case)


@pytest.mark.parametrize("hidden,out,B,W", [((288, 288), 24, 37, 5), ((480, 480), 72, 64, 8)], ids=["2x288-o24", "2x480-o72"])
def test_wide_bf16x3_forward_only_widths(cuda, hidden, out, B, W):
    """bf16x3 hidden widths above 256 that are multiples of 32 but not of 64 (forward only: 288 = 256 + 32, 480 = 256 + 224 columns in
    the two column units): Q against float64, by the forward-only check of tests/test_tc_mlp_grad_gpu.py."""
    _bf16_forward_case(cuda, hidden, out, B, W)


def _agent(cuda, cfg, graph):
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope
    from morl_baselines_b200.testing import FakeEnv, synthetic_store

    OBS, A, D, B, W, N = cfg["obs"], cfg["A"], 3, cfg["B"], cfg["W"], 4096
    th.manual_seed(0)
    agent = Envelope(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), batch_size=B, num_sample_w=W, per=False, buffer_size=N, net_arch=list(cfg["net"]),
                     log=False, seed=3, device=cuda, use_cuda_graph=graph, use_tensor_cores=True)
    store = synthetic_store(N, OBS, A, D, seed=1)
    store["dones"][:] = 1.0  # target = reward: the comparison does not depend on the envelope argmax (tested elsewhere)
    rb = agent.replay_buffer
    rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
    rb.size, rb.ptr = N, 0
    rb.mark_all_dirty()
    return agent, store


UPDATE_CASES = {
    "4x512-w64": dict(net=(512,) * 4, obs=32, A=8, B=1024, W=64),
    "4x256-w256": dict(net=(256,) * 4, obs=32, A=8, B=256, W=256),
}


@pytest.mark.parametrize("cfg", [pytest.param(v, id=k) for k, v in UPDATE_CASES.items()])
def test_wide_envelope_update(cuda, cfg):
    """One Envelope.update() eager and one through the CUDA graph, from the same state: identical loss, .grad and parameters after the
    step; every .grad within the float64 bound of the reference loss's gradient; the loss within 1e-6 of float64."""
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.weights import random_weights

    runs = []
    for graph in (False, True):
        agent, store = _agent(cuda, cfg, graph)
        params0 = [p.detach().clone() for p in agent.q_net.parameters()]
        agent.global_step = 1
        np.random.seed(50)
        ops.plane_overflow_count(reset=True)
        agent.update()
        th.cuda.synchronize()
        assert ops.plane_overflow_count() == 0
        assert not agent.fused_head_active  # K = 512 or |W| > 64: output-layer GEMMs + standalone envelope_td
        runs.append((agent, store, params0))
    (eager, store, params0), (graphed, _, _) = runs
    assert float(eager._last_loss) == float(graphed._last_loss)
    for pe, pg in zip(eager.q_net.parameters(), graphed.q_net.parameters()):
        assert th.equal(pe.grad, pg.grad) and th.equal(pe, pg)
    assert np.array_equal(eager._last_inds, graphed._last_inds)

    net, A, D, B, W = list(cfg["net"]), cfg["A"], 3, cfg["B"], cfg["W"]
    rng = np.random.default_rng(3)  # the agent's weight stream (seed=3)
    wset = th.tensor(random_weights(D, W, dist="gaussian", rng=rng)).float().to(cuda)
    assert th.equal(wset, eager._static["wset"])
    inds = eager._last_inds
    feats = th.from_numpy(store["obs"][inds]).to(cuda)
    act = th.from_numpy(store["actions"][inds].astype(np.int64)).to(cuda).view(-1)
    rew = th.from_numpy(store["rewards"][inds]).to(cuda)
    n = len(net) + 1
    params = list(zip(params0[0::2], params0[1::2]))
    x = pair_rows(feats, wset)
    plan = eager._tc_train
    masks = kernel_masks(plan, net)
    ref = reference(params, x, masks, th.zeros(B * W, A * D, device=cuda))
    check_mask_flips(ref, masks)
    q_ratio, q_ok = _ratio(plan.q, ref["q"], C_PRODUCT * n * ref["qmag"])
    assert q_ok, q_ratio
    loss_ref, _ = _loss64(ref["q"], act, rew, wset, 0.0, A, D)
    loss = float(eager._last_loss)
    assert abs(loss - loss_ref) <= 1e-6 * abs(loss_ref), (loss, loss_ref)
    _, dq = _loss64(plan.q.double(), act, rew, wset, 0.0, A, D)
    ref = reference(params, x, masks, dq, floor=F16X2_FLOOR * float(dq.abs().max()))
    bounds = grad_bounds(ref, _products(n, B * W))
    ratios = []
    for i, (p, r, b) in enumerate(zip(eager.q_net.parameters(), ref["grads"], bounds)):
        ratio, ok = _ratio(p.grad, r, b)
        ratios.append(ratio)
        assert ok, f"parameter {i}: max err / bound = {ratio:.3g}"
    print(f"\n[wide-update] {net} B {B} W {W}: Q {q_ratio:.3g}, loss rel err {abs(loss - loss_ref) / abs(loss_ref):.3g}, "
          f"grads {' '.join(f'{r:.3g}' for r in ratios)}")
    assert _rejects([p.grad for p in eager.q_net.parameters()], [r * (1 + 1e-3) for r in ref["grads"]], bounds)
