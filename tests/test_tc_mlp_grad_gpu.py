"""GPU tests of the tensor-core Q-network's hand-written backward (morl_baselines_b200/tc_mlp.py: TCPairMlp.backward, per layer and
chained) against float64, at the network shapes the Envelope's tensor-core update accepts, and of the gradients one Envelope.update()
leaves in the parameters' .grad.

The whole-update tests cannot see a gradient tensor that is off by a positive constant: Adam's step m / (sqrt(v) + eps) and the common
clip coefficient of clip_grad_norm_ are both invariant to it.  These tests compare the gradient values themselves.

Reference.  The forward over the pair rows x[b*W + j] = [feats[b] | wset[j]] and the backward written out layer by layer,
    G_n = dL/dQ,   dW_l = G_l^T H_{l-1},   db_l = sum over rows of G_l,   G_{l-1} = (G_l W_l) * M_{l-1},
in float64, with the ReLU masks M the kernels recorded (plan.hbits).  A pre-activation that rounds to the other side of zero is then not
counted as an arithmetic error; every case checks that the kernel's masks differ from the float64 signs only where |pre-activation| is
within the forward bound.

Bound.  The same computation on magnitudes (|W|, |b|, |x|, |dL/dQ| through the same masks), times C_PRODUCT = 2e-6 (the per-product
constant of tests/test_gemm_gpu.py) for every product on the way to the tensor: the n Linear layers of the path (forward products into
H_{l-1}, dX products down to G_l, the dL/dQ split, the pair reduction of layer 1) plus the row reduction of the gradient itself, counted
as max(1, sqrt(rows / 4096)) products (the allowance of the split-K weight-gradient test).  For the f16x2 format, an element of a
gradient plane below 2^-14 / s_g keeps an absolute accuracy of only 2^-26 of the largest dL/dQ element (tc_mlp.py); that floor enters at
every split and is carried through the same masks and |W| without a constant.
"""

import math

import numpy as np
import pytest
import torch as th
from torch import nn

pytestmark = pytest.mark.gpu

C_PRODUCT = 2e-6   # per split-operand product (tests/test_gemm_gpu.py)
F16X2_FLOOR = 2.0**-26  # times max|dL/dQ|: absolute accuracy of an f16x2 gradient plane element (tc_mlp.py)
F16, BF16 = 1, 0   # ops.FMT_F16X2, ops.FMT_BF16X3
FEAT, WDIM = 12, 3


def _products(n_lin, rows):
    """Products on the path of a gradient tensor of an n_lin-layer network reduced over `rows` pair rows."""
    return n_lin + max(1.0, math.sqrt(rows / 4096))


def pair_rows(feats, wset):
    """x[b*W + j] = [feats[b] | wset[j]] in float64."""
    B, W = feats.shape[0], wset.shape[0]
    return th.cat([feats.double().repeat_interleave(W, 0), wset.double().repeat(B, 1)], dim=1)


def reference(params, x, masks, dq, floor=0.0):
    """float64 forward / backward of the Linear-ReLU stack ``params`` [(weight, bias), ...] on the pair rows x with the hidden masks
    ``masks`` (0 / 1 per hidden layer), seeded with dL/dQ = dq.  Alongside each value it returns the magnitude terms of its bound:
    ``qmag`` / ``premag`` / ``gmag`` (|.| propagated through the same masks) and ``gabs`` (an absolute error ``floor`` added at every
    gradient split, propagated through |W| and the masks; None without a floor)."""
    Ws = [w.detach().double() for w, _ in params]
    bs = [b.detach().double() for _, b in params]
    n = len(Ws)
    H, Hm, pre, premag = [x], [x.abs()], [], []
    for l in range(n - 1):
        z = H[-1] @ Ws[l].t() + bs[l]
        zm = Hm[-1] @ Ws[l].abs().t() + bs[l].abs()
        pre.append(z)
        premag.append(zm)
        H.append(z * masks[l])
        Hm.append(zm * masks[l])
    q = H[-1] @ Ws[-1].t() + bs[-1]
    qmag = Hm[-1] @ Ws[-1].abs().t() + bs[-1].abs()
    G, Gm = dq.double(), dq.double().abs()
    Ga = th.full_like(G, float(floor)) if floor else None
    grads, gmag, gabs = [None] * (2 * n), [None] * (2 * n), [None] * (2 * n)
    for l in range(n - 1, -1, -1):
        grads[2 * l], grads[2 * l + 1] = G.t() @ H[l], G.sum(0)
        gmag[2 * l], gmag[2 * l + 1] = Gm.t() @ Hm[l], Gm.sum(0)
        if Ga is not None:
            gabs[2 * l], gabs[2 * l + 1] = Ga.t() @ Hm[l], Ga.sum(0)
        if l:
            G = (G @ Ws[l]) * masks[l - 1]
            Gm = (Gm @ Ws[l].abs()) * masks[l - 1]
            if Ga is not None:
                Ga = (Ga @ Ws[l].abs() + floor) * masks[l - 1]
    return {"q": q, "qmag": qmag, "pre": pre, "premag": premag, "grads": grads, "gmag": gmag, "gabs": gabs if Ga is not None else None}


def grad_bounds(ref, k):
    """Elementwise bound of every gradient tensor: C_PRODUCT * k * magnitude (+ the absolute floor terms)."""
    out = []
    for i, m in enumerate(ref["gmag"]):
        b = C_PRODUCT * k * m
        if ref["gabs"] is not None:
            b = b + ref["gabs"][i]
        out.append(b)
    return out


def _ratio(got, want, bound):
    err = (got.double() - want).abs()
    return float((err / bound.clamp_min(1e-300)).max()), bool((err <= bound).all())


def _rejects(got, wants, bounds):
    """True if the comparison fails for at least one element of one tensor."""
    return any(not _ratio(g, w, b)[1] for g, w, b in zip(got, wants, bounds))


def kernel_masks(plan, widths):
    from morl_baselines_b200 import ops

    return [ops.unpack_relu_bits(bits, h).double() for bits, h in zip(plan.hbits, widths)]


def check_mask_flips(ref, masks):
    """The recorded masks differ from the float64 signs only where |pre-activation| is within the forward bound (layer l's
    pre-activation is the end of l + 1 products); returns the number of flips."""
    flips = 0
    for l, (z, zm, m) in enumerate(zip(ref["pre"], ref["premag"], masks)):
        flip = (m > 0) != (z > 0)
        bound = C_PRODUCT * (l + 1) * zm
        assert bool((z.abs()[flip] <= bound[flip]).all()), f"hidden layer {l}: a ReLU mask bit differs from the float64 sign beyond the bound"
        flips += int(flip.sum())
    return flips


def _net(cuda, hidden, out, seed):
    th.manual_seed(seed)
    layers, d = [], FEAT + WDIM
    for h in hidden:
        layers += [nn.Linear(d, h), nn.ReLU()]
        d = h
    layers.append(nn.Linear(d, out))
    return nn.Sequential(*layers).to(cuda)


def _dq(cuda, kind, M, out, seed):
    """dL/dQ with magnitudes spread over 2^-9 .. 2^9 (1e-3 times): the smallest elements are below 2^-16 of the largest, where the
    f16x2 planes keep absolute accuracy only.  "sparse": only the taken action's 3 columns of a row are non-zero (the loss's structure)."""
    g = th.Generator(device=cuda).manual_seed(seed)
    mag = 1e-3 * th.exp2(th.rand(M, out, device=cuda, generator=g) * 18 - 9)
    dq = th.where(th.rand(M, out, device=cuda, generator=g) < 0.5, -mag, mag)
    if kind == "sparse":
        act = th.randint(0, out // 3, (M,), device=cuda, generator=g)
        keep = (th.arange(out, device=cuda)[None, :] // 3) == act[:, None]
        dq = dq * keep
    return dq.contiguous()


# name -> (hidden widths, output columns, B, |W|, format, split accumulators, tc_mlp switches turned off, dL/dQ)
CASES = {
    "2x64-o4-b1w64": ((64,) * 2, 4, 1, 64, F16, False, (), "dense"),
    "3x64-o24-b37w5": ((64,) * 3, 24, 37, 5, F16, False, (), "dense"),
    "3x64-o24-b64w8-bf16": ((64,) * 3, 24, 64, 8, BF16, False, (), "sparse"),
    "3x64-o36-b300w1-split": ((64,) * 3, 36, 300, 1, F16, True, (), "dense"),
    "3x128-o32-b64w8": ((128,) * 3, 32, 64, 8, F16, False, (), "dense"),
    "3x128-o72-b37w5-bf16": ((128,) * 3, 72, 37, 5, BF16, False, (), "dense"),
    "3x128-o24-b3000w2": ((128,) * 3, 24, 3000, 2, F16, False, (), "dense"),
    "2x192-o36-b64w8": ((192,) * 2, 36, 64, 8, F16, False, (), "dense"),
    "2x192-o72-b300w1-split": ((192,) * 2, 72, 300, 1, F16, True, (), "dense"),
    "2x192-o24-b1w64-bf16": ((192,) * 2, 24, 1, 64, BF16, False, (), "dense"),
    "2x256-o24-b64w8": ((256,) * 2, 24, 64, 8, F16, False, (), "dense"),
    "2x256-o256-b37w5": ((256,) * 2, 256, 37, 5, F16, False, (), "dense"),
    "3x256-o24-b1024w64": ((256,) * 3, 24, 1024, 64, F16, False, (), "dense"),
    "3x256-o72-b64w8-bf16": ((256,) * 3, 72, 64, 8, BF16, False, (), "dense"),
    "4x256-o24-b1024w64": ((256,) * 4, 24, 1024, 64, F16, False, (), "dense"),
    "4x256-o24-b1024w64-sparse": ((256,) * 4, 24, 1024, 64, F16, False, (), "sparse"),
    "4x256-o24-b1024w64-bf16": ((256,) * 4, 24, 1024, 64, BF16, False, (), "dense"),
    "4x256-o24-b1024w64-split": ((256,) * 4, 24, 1024, 64, F16, True, (), "dense"),
    "4x256-o24-b1024w64-nochain": ((256,) * 4, 24, 1024, 64, F16, False, ("_CHAIN", "_CHAIN_BWD"), "dense"),
    "4x256-o36-b37w5": ((256,) * 4, 36, 37, 5, F16, False, (), "dense"),
    "4x256-o72-b300w1": ((256,) * 4, 72, 300, 1, F16, False, (), "dense"),
    "4x256-o256-b64w8-bf16": ((256,) * 4, 256, 64, 8, BF16, False, (), "dense"),
    "4x256-o32-b3000w2": ((256,) * 4, 32, 3000, 2, F16, False, (), "dense"),
    "4x256-o4-b1w64": ((256,) * 4, 4, 1, 64, F16, False, (), "dense"),
    "4x256-o24-b64w8-nonarrow": ((256,) * 4, 24, 64, 8, F16, False, ("_NARROW_HEAD",), "dense"),
    "4x256-o24-b64w8-nosnake": ((256,) * 4, 24, 64, 8, F16, False, ("_SNAKE",), "dense"),
}


@pytest.mark.parametrize("case", [pytest.param(v, id=k) for k, v in CASES.items()])
def test_backward_matches_float64(cuda, monkeypatch, case):
    from morl_baselines_b200 import ops, tc_mlp

    hidden, out, B, W, fmt, split, off, kind = case
    for name in off:
        monkeypatch.setattr(tc_mlp, name, False)
    M, n = B * W, len(hidden) + 1
    net = _net(cuda, hidden, out, seed=M + out + n)
    assert tc_mlp.TCPairMlp.trainable_supported(net, W, fmt)
    g = th.Generator(device=cuda).manual_seed(M + 7 * out)
    feats = th.randn(B, FEAT, device=cuda, generator=g)
    wset = th.rand(W, WDIM, device=cuda, generator=g)
    dq = _dq(cuda, kind, M, out, seed=M + out)
    ops.plane_overflow_count(reset=True)
    plan = tc_mlp.TCPairMlp(net, FEAT, B, W, trainable=True, fmt=fmt, split_acc=split)
    assert plan.ld_last == (out + 63) // 64 * 64
    chained = not split and "_CHAIN" not in off and hidden[0] == 256 and ops.gemm_chain_supported(fmt, M, 256)
    assert plan.chain_supported() == chained
    plan.refresh_weights()
    q = plan.forward_pairs(feats, wset).clone()
    grads = [t.clone() for t in plan.backward(feats, wset, dq)]
    th.cuda.synchronize()
    assert ops.plane_overflow_count() == 0

    params = [(l.weight, l.bias) for l in plan.lin]
    x = pair_rows(feats, wset)
    masks = kernel_masks(plan, hidden)
    floor = F16X2_FLOOR * float(dq.abs().max()) if fmt == F16 else 0.0
    ref = reference(params, x, masks, dq, floor=floor)
    flips = check_mask_flips(ref, masks)
    qbound = C_PRODUCT * n * ref["qmag"]
    q_ratio, q_ok = _ratio(q, ref["q"], qbound)
    k = _products(n, M)
    bounds = grad_bounds(ref, k)
    ratios = [_ratio(t, r, b) for t, r, b in zip(grads, ref["grads"], bounds)]
    print(f"\n[grad-check] {'-'.join(map(str, hidden))} out {out} B {B} W {W} fmt {fmt} split {split} off {off} {kind}: "
          f"Q {q_ratio:.3g}, grads {' '.join(f'{r:.3g}' for r, _ in ratios)}, mask flips {flips}")
    assert q_ok, f"Q: max err / bound = {q_ratio:.3g} (bound {C_PRODUCT} x {n} products x magnitude)"
    for i, (r, ok) in enumerate(ratios):
        what = f"{'bias' if i & 1 else 'weight'} gradient of Linear {i // 2 + 1}"
        assert ok, f"{what}: max err / bound = {r:.3g} (bound {C_PRODUCT} x {k:.3g} products x magnitude{' + f16x2 floor' if floor else ''})"

    # the comparison tells a wrong gradient from a right one: all gradients 0.1 % too large, one hidden layer's ReLU mask swapped with
    # the next one's (forward and backward), and any single tensor of layers 2.. twice too large are each rejected.  (The magnitude bound
    # grows ~10x per dX product relative to the value itself: `resolution` is the smallest relative scale error each tensor still
    # detects; layer 1 of a deep net over 65,536 rows resolves only ~100 %, hence the check from the kernel's own dL/dh1 below.)
    resolution = [float((b / r.abs())[r != 0].min()) for r, b in zip(ref["grads"], bounds)]
    print(f"[grad-check]   resolution {' '.join(f'{v:.2g}' for v in resolution)}")
    assert _rejects(grads, [r * (1 + 1e-3) for r in ref["grads"]], bounds)
    swapped = [masks[1], masks[0]] + masks[2:]
    ref_sw = reference(params, x, swapped, dq, floor=floor)
    assert _rejects(grads, ref_sw["grads"], grad_bounds(ref_sw, k))
    for i, (t, r, b) in enumerate(zip(grads[2:], ref["grads"][2:], bounds[2:]), start=2):
        assert _rejects([t], [2 * r], [b]), f"gradient tensor {i}: a factor 2 passes the bound"

    # layer 1 from the kernel's own dL/dh1 planes (what pairs_grad_reduce reads): dU = sum_j G1, dV = sum_b G1, dW1 = [dU^T feats |
    # dV^T wset], db1 = sum_j dV in float64, bound C_PRODUCT x 2 products (the pair reduction, the layer-1 kernel) x the row-count growth
    # x magnitude; here a 1 % error of either tensor is rejected
    g1 = plan._gbufs[-1] if plan._gbufs is not None else plan.g[1]  # chained backward: one buffer per layer; per layer: G_1 lands in g[1]
    G1 = g1.double().sum(0)[:, : hidden[0]] / (float(plan.s_g) if plan.s_g is not None else 1.0)
    G1, G1m = G1.view(B, W, -1), G1.abs().view(B, W, -1)
    f64, w64 = feats.double(), wset.double()
    ref1 = [th.cat([G1.sum(1).t() @ f64, G1.sum(0).t() @ w64], 1), G1.sum((0, 1))]
    mag1 = [th.cat([G1m.sum(1).t() @ f64.abs(), G1m.sum(0).t() @ w64.abs()], 1), G1m.sum((0, 1))]
    bounds1 = [C_PRODUCT * 2 * max(1.0, math.sqrt(M / 4096)) * m for m in mag1]
    for i in range(2):
        r, ok = _ratio(grads[i], ref1[i], bounds1[i])
        print(f"[grad-check]   layer 1 from the kernel's dL/dh1: tensor {i} {r:.3g}")
        assert ok, f"{'bias' if i else 'weight'} gradient of Linear 1 from the kernel's dL/dh1: max err / bound = {r:.3g}"
        assert _rejects([grads[i]], [ref1[i] * (1 + 1e-2)], [bounds1[i]])


@pytest.mark.parametrize("hidden,out,B,W", [((96, 96), 24, 37, 5), ((160,) * 3, 72, 64, 8)], ids=["2x96-o24", "3x160-o72"])
def test_bf16x3_forward_only_widths(cuda, hidden, out, B, W):
    """bf16x3 hidden widths that are multiples of 32 but not of 64: forward-only plans (no hand-written backward); Q against float64
    (ReLU is 1-Lipschitz, so the magnitudes without masks bound the error whichever side of zero a pre-activation lands on)."""
    from morl_baselines_b200 import ops, tc_mlp

    net = _net(cuda, hidden, out, seed=sum(hidden) + out)
    assert tc_mlp.TCPairMlp.supported(net, BF16) and not tc_mlp.TCPairMlp.trainable_supported(net, W, BF16)
    g = th.Generator(device=cuda).manual_seed(B + W)
    feats, wset = th.randn(B, FEAT, device=cuda, generator=g), th.rand(W, WDIM, device=cuda, generator=g)
    plan = tc_mlp.TCPairMlp(net, FEAT, B, W, fmt=BF16)
    plan.refresh_weights()
    q = plan.forward_pairs(feats, wset).clone()
    h = pair_rows(feats, wset)
    hm = h.abs()
    lin = plan.lin
    for l in lin[:-1]:
        w, b = l.weight.detach().double(), l.bias.detach().double()
        h = (h @ w.t() + b).clamp_min(0)
        hm = hm @ w.abs().t() + b.abs()
    w, b = lin[-1].weight.detach().double(), lin[-1].bias.detach().double()
    ref, bound = h @ w.t() + b, C_PRODUCT * len(lin) * (hm @ w.abs().t() + b.abs())
    r, ok = _ratio(q, ref, bound)
    print(f"\n[grad-check] bf16x3 forward {hidden} out {out}: Q {r:.3g}")
    assert ok, r
    assert _rejects([q], [ref * (1 + 5e-2)], [bound])  # (without masks the bound resolves 0.07 % at 2 x 96, 1.4 % at 3 x 160)
    assert ops.plane_overflow_count() == 0


def test_reference_equals_autograd(cuda):
    """Self-check of the restatement: with float64's own masks it is torch.autograd in float64."""
    for hidden, out, B, W in (((64,) * 3, 24, 37, 5), ((256,) * 4, 72, 16, 8)):
        net = _net(cuda, hidden, out, seed=3).double()
        g = th.Generator(device=cuda).manual_seed(1)
        feats, wset = th.randn(B, FEAT, device=cuda, generator=g), th.rand(W, WDIM, device=cuda, generator=g)
        x = pair_rows(feats, wset)
        dq = _dq(cuda, "dense", B * W, out, seed=2).double()
        masks, h = [], x
        for l in [m for m in net if isinstance(m, nn.Linear)][:-1]:
            h = l(h)
            masks.append((h > 0).double())
            h = h.clamp_min(0)
        ref = reference([(l.weight, l.bias) for l in net if isinstance(l, nn.Linear)], x, masks, dq)
        q = net(x)
        auto = th.autograd.grad((q * dq).sum(), list(net.parameters()))
        assert float((ref["q"] - q).abs().max()) <= 1e-12 * float(q.abs().max())
        for a, r in zip(auto, ref["grads"]):
            assert float((a - r).abs().max()) <= 1e-12 * float(a.abs().max())


# ---------------------------------------------------------------------------------------------------- one Envelope update
def _loss64(q, act, rew, wset, lam, A, D):
    """The reference's critic loss (envelope.py:301-313, oracle/envelope_update_port.py) on rows b*W + j with every done = 1, so the
    target is the reward; returns (loss, dL/dQ) in float64."""
    W = wset.shape[0]
    q = q.detach().requires_grad_(True)
    qv = q.view(-1, A, D).gather(1, act.repeat_interleave(W).view(-1, 1, 1).expand(-1, 1, D)).squeeze(1)
    tq = rew.double().repeat_interleave(W, 0)
    w = wset.double().repeat(act.shape[0], 1)
    loss = th.nn.functional.mse_loss(qv, tq)
    if lam > 0:
        aux = th.nn.functional.mse_loss((qv * w).sum(1), (tq * w).sum(1))
        loss = (1 - lam) * loss + lam * aux
    (dq,) = th.autograd.grad(loss, q)
    return float(loss), dq


UPDATE_CASES = {
    "3x64-b32w8-eager": dict(net=(64,) * 3, graph=False),
    "3x64-b32w8-graph": dict(net=(64,) * 3, graph=True),
    "3x128-b32w8": dict(net=(128,) * 3, graph=True),
    "north-star-eager": dict(net=(256,) * 4, obs=32, A=8, B=1024, W=64, graph=False),
    "north-star-graph": dict(net=(256,) * 4, obs=32, A=8, B=1024, W=64, graph=True),
    "4x256-ad36-general-head": dict(net=(256,) * 4, A=12, B=64, W=8, graph=True),
    "3x64-homotopy": dict(net=(64,) * 3, lam=0.3, graph=True),
    "4x256-bf16x3": dict(net=(256,) * 4, B=64, W=8, fmt="bf16x3", graph=True),
    "4x256-split-acc": dict(net=(256,) * 4, B=64, W=8, acc="split", graph=True),
}


@pytest.mark.parametrize("cfg", [pytest.param(v, id=k) for k, v in UPDATE_CASES.items()])
def test_envelope_update_gradients_match_float64(cuda, cfg):
    """After one update, every q_net parameter's .grad (FusedClipAdam only reads it; the clip coefficient is applied inside the Adam
    kernel) equals the float64 gradient of the reference loss at the parameters before the step, on the same minibatch and weights."""
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.weights import random_weights
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope
    from morl_baselines_b200.testing import FakeEnv, synthetic_store

    net, graph = list(cfg["net"]), cfg["graph"]
    OBS, A, D, B, W, N = cfg.get("obs", 12), cfg.get("A", 4), 3, cfg.get("B", 32), cfg.get("W", 8), 2048
    lam, fmt = cfg.get("lam", 0.0), cfg.get("fmt", "f16x2")
    th.manual_seed(0)
    agent = Envelope(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), batch_size=B, num_sample_w=W, per=False, buffer_size=N, net_arch=net,
                     log=False, seed=3, device=cuda, use_cuda_graph=graph, use_tensor_cores=True, initial_homotopy_lambda=lam,
                     tensor_core_format=fmt, tensor_core_accumulators=cfg.get("acc", "single"))
    store = synthetic_store(N, OBS, A, D, seed=1)
    store["dones"][:] = 1.0  # target = reward: the comparison does not depend on the envelope argmax (tested elsewhere)
    rb = agent.replay_buffer
    rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
    rb.size, rb.ptr = N, 0
    rb.mark_all_dirty()
    params0 = [p.detach().clone() for p in agent.q_net.parameters()]
    rng = np.random.default_rng(3)  # the agent's weight stream (seed=3)
    agent.global_step = 1
    np.random.seed(50)
    ops.plane_overflow_count(reset=True)
    agent.update()
    th.cuda.synchronize()
    assert ops.plane_overflow_count() == 0
    if A * D > 32:
        assert not agent.fused_head_active
    wset = th.tensor(random_weights(D, W, dist="gaussian", rng=rng)).float().to(cuda)
    assert th.equal(wset, agent._static["wset"])
    inds = agent._last_inds
    feats = th.from_numpy(store["obs"][inds]).to(cuda)
    act = th.from_numpy(store["actions"][inds].astype(np.int64)).to(cuda).view(-1)
    rew = th.from_numpy(store["rewards"][inds]).to(cuda)

    n = len(net) + 1
    params = list(zip(params0[0::2], params0[1::2]))
    x = pair_rows(feats, wset)
    plan = agent._tc_train
    masks = kernel_masks(plan, net)
    ref = reference(params, x, masks, th.zeros(B * W, A * D, device=cuda))  # forward half: Q and its bound
    check_mask_flips(ref, masks)
    q_ratio, q_ok = _ratio(plan.q, ref["q"], C_PRODUCT * n * ref["qmag"])  # the training pass's Q (fp32, rows b*W + j)
    assert q_ok, q_ratio
    loss_ref, _ = _loss64(ref["q"], act, rew, wset, lam, A, D)
    loss = float(agent._last_loss)
    assert abs(loss - loss_ref) <= 1e-6 * abs(loss_ref), (loss, loss_ref)
    # the backward is seeded with dL/dQ at the kernel's own Q (checked just above): a Q error within its bound would otherwise move
    # dL/dQ = 2 (q - r) / (N D) by far more than the backward's own rounding when |q - r| << |Q|'s magnitude sum
    _, dq = _loss64(plan.q.double(), act, rew, wset, lam, A, D)
    floor = F16X2_FLOOR * float(dq.abs().max()) if fmt == "f16x2" else 0.0
    ref = reference(params, x, masks, dq, floor=floor)
    rows = B * W
    bounds = grad_bounds(ref, _products(n, rows))
    ratios = []
    for i, (p, r, b) in enumerate(zip(agent.q_net.parameters(), ref["grads"], bounds)):
        ratio, ok = _ratio(p.grad, r, b)
        ratios.append(ratio)
        assert ok, f"parameter {i}: max err / bound = {ratio:.3g}"
    print(f"\n[grad-check] update {net} B {B} W {W} A {A} lam {lam} {fmt} graph {graph}: loss rel err {abs(loss - loss_ref) / abs(loss_ref):.3g}, "
          f"grads {' '.join(f'{r:.3g}' for r in ratios)}, resolution "
          f"{' '.join(f'{float((b / r.abs())[r != 0].min()):.2g}' for r, b in zip(ref['grads'], bounds))}")
    assert _rejects([p.grad for p in agent.q_net.parameters()], [r * (1 + 1e-3) for r in ref["grads"]], bounds)
