"""GPI-PD's Q-networks on the tensor cores (tc_mlp.TCProductMlp): the LayerNorm / dropout epilogue of the K-major GEMM
(morl_gemm_planes_ln_f32), its Philox dropout stream, the product-conditioned first layer, the whole plan against a float64 copy of QNet, and
GPIPD with use_tensor_cores=True against the library path.

Error bound of the epilogue: the GEMM's pre-activation z carries at most E = C_PRODUCT (|A| |B|^T + |b|) per element (C_PRODUCT = 2e-6 as in
tests/test_gemm_wide_gpu.py); dropout multiplies it by the keep scale s.  Through LayerNorm y_i = (x_i - mean) r gamma_i + beta_i,
r = (var + eps)^-1/2, a perturbation of at most e = s max_row(E) per element moves x_i - mean by <= 2 e and r by <= 2 e r^2 (r sigma <= 1), so
|dy_i| <= 2 e |gamma_i| r (1 + r |x_i - mean|); the fp32 sums of N <= 256 terms add 2^-16 (|gamma_i| r (|x_i - mean| + max_row |x|) + |beta_i|).
ReLU is 1-Lipschitz."""

import copy

import numpy as np
import pytest
import torch as th
from torch import nn

pytestmark = pytest.mark.gpu
C_PRODUCT = 2e-6
FMTS = [pytest.param(1, id="f16x2"), pytest.param(0, id="bf16x3")]


def _scale(fmt, value, dev):
    from morl_baselines_b200 import ops

    return ops.scale_tensor(value, dev) if fmt == ops.FMT_F16X2 else None


def _operands(cuda, fmt, M, N, K, seed):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(seed)
    x = th.randn(M, K, device=cuda, generator=g)
    w = th.randn(N, K, device=cuda, generator=g) / 16
    b = th.randn(N, device=cuda, generator=g) * 0.1
    gamma = 1 + 0.2 * th.randn(N, device=cuda, generator=g)
    beta = 0.1 * th.randn(N, device=cuda, generator=g)
    sx, sw = _scale(fmt, 8.0, cuda), _scale(fmt, 1024.0, cuda)
    return x, w, b, gamma, beta, sx, sw, ops.split_planes(x, fmt, scale=sx), ops.split_planes(w, fmt, scale=sw)


def _dropout_state(cuda, seed=1234, offset=7):
    return th.tensor([seed], dtype=th.int64, device=cuda), th.tensor([offset], dtype=th.int32, device=cuda)


def _ln_reference(z, keep, s, gamma, beta, eps, E):
    """float64 relu(LN(dropout(z))) and its error bound (module docstring)."""
    x = z * keep * s
    mean = x.mean(1, keepdim=True)
    d = x - mean
    r = 1.0 / th.sqrt((d * d).mean(1, keepdim=True) + eps)
    y = d * r * gamma.double() + beta.double()
    e = s * E.max(1, keepdim=True).values
    g = gamma.double().abs()
    bound = 2 * e * g * r * (1 + r * d.abs()) + 2.0 ** -16 * (g * r * (d.abs() + x.abs().max(1, keepdim=True).values) + beta.double().abs())
    return y.clamp_min(0), bound


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("K", [64, 256, 512])
@pytest.mark.parametrize("N", [64, 128, 192, 256])
@pytest.mark.parametrize("M", [128, 1000, 65536])
def test_ln_dropout_epilogue_against_float64(cuda, fmt, M, N, K):
    from morl_baselines_b200 import ops

    x, w, b, gamma, beta, sx, sw, xp, wp = _operands(cuda, fmt, M, N, K, M + N + K + fmt)
    ops.plane_overflow_count(reset=True)
    # LayerNorm and dropout off: bit for bit the plain ReLU GEMM (fp32 output and planes)
    c0, p0 = ops.gemm_planes(xp, wp, N, bias=b, relu=True, out_f32=True, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx)
    c1, p1 = ops.gemm_planes_ln(xp, wp, N, bias=b, out_f32=True, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx)
    assert th.equal(c0, c1) and th.equal(p0.view(th.int16), p1.view(th.int16))
    # LayerNorm + dropout p = 0.1 against float64 with the kernel's own keep bits
    p, eps = 0.1, 1e-5
    seed, off = _dropout_state(cuda, seed=M * 31 + N)
    bits = ops.empty_relu_bits(M, cuda, N).zero_()
    c, planes = ops.gemm_planes_ln(xp, wp, N, bias=b, ln_weight=gamma, ln_bias=beta, ln_eps=eps, drop_p=p, drop_seed=seed, drop_offset=off,
                                   drop_salt=3, out_f32=True, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits)
    keep = ops.unpack_relu_bits(bits, N).double()
    z = x.double() @ w.double().t() + b.double()
    E = C_PRODUCT * (x.abs().double() @ w.abs().double().t() + b.abs().double())
    ref, bound = _ln_reference(z, keep, float(np.float32(1 / (1 - p))), gamma, beta, eps, E)
    err = (c.double() - ref).abs()
    assert bool((err <= bound).all()), f"max err / bound = {float((err / bound).max()):.3g}"
    # the planes hold c_scale * output, applied after the ReLU
    rec = planes.double().sum(0) / (8.0 if fmt == ops.FMT_F16X2 else 1.0)
    assert float(((rec - c.double()).abs() - 2.0 ** -20 * c.double().abs()).max()) <= 2.0 ** -24
    assert ops.plane_overflow_count() == 0


def _philox(ctr, key):
    """Philox4x32-10 on numpy uint64 arrays holding 32-bit words (ctr: 4 arrays, key: 2 ints)."""
    m32 = np.uint64(0xFFFFFFFF)
    c = [np.asarray(v, dtype=np.uint64) & m32 for v in ctr]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & m32, p1 & m32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & m32, p0 & m32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m32, (k1 + np.uint64(0xBB67AE85)) & m32
    return c


def test_philox_restatement_known_answers():
    # Random123 known-answer vectors of philox4x32-10
    assert [int(v) for v in _philox([0, 0, 0, 0], (0, 0))] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert [int(v) for v in _philox([0xFFFFFFFF] * 4, (0xFFFFFFFF, 0xFFFFFFFF))] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


@pytest.mark.parametrize("fmt", FMTS)
def test_dropout_mask_is_documented_philox_stream(cuda, fmt):
    """keep(row, col) = Philox4x32-10(counter = (offset, salt, row, group), key = seed)[i] >= round(p 2^32), with group = 8 (col / 32) + 2 (col % 8 / 2)
    ... as documented in gemm_planes.cu (ln_dropout_unit)."""
    from morl_baselines_b200 import ops

    M, N, K, p = 300, 192, 64, 0.3
    *_, sx, sw, xp, wp = _operands(cuda, fmt, M, N, K, 5)
    seed_v, off_v, salt = 0x0123456789ABCDEF, 11, 5
    seed, off = _dropout_state(cuda, seed_v, off_v)
    bits = ops.empty_relu_bits(M, cuda, N).zero_()
    ops.gemm_planes_ln(xp, wp, N, drop_p=p, drop_seed=seed, drop_offset=off, drop_salt=salt, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits)
    got = ops.unpack_relu_bits(bits, N).cpu().numpy()
    col = np.arange(N)
    c, q, l4, e = col // 32, (col % 32) // 8, (col % 8) // 2, col % 2
    k, i = q // 2, 2 * (q % 2) + e
    grp = 8 * c + 2 * l4 + k
    rows = np.arange(M)[:, None]
    draws = _philox([np.full((M, N), off_v), np.full((M, N), salt), np.broadcast_to(rows, (M, N)), np.broadcast_to(grp, (M, N))],
                    (seed_v & 0xFFFFFFFF, seed_v >> 32))
    draw = np.choose(np.broadcast_to(i, (M, N)), draws)
    assert np.array_equal(got, draw >= np.uint64(round(p * 2 ** 32)))


@pytest.mark.parametrize("p", [0.01, 0.1, 0.5])
def test_dropout_keep_fraction(cuda, p):
    from morl_baselines_b200 import ops

    M, N, K = 8192, 256, 64
    *_, sx, sw, xp, wp = _operands(cuda, 1, M, N, K, 9)
    seed, off = _dropout_state(cuda)
    bits = ops.empty_relu_bits(M, cuda, N).zero_()
    ops.gemm_planes_ln(xp, wp, N, drop_p=p, drop_seed=seed, drop_offset=off, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits)
    n = M * N  # 2.1e6 elements
    kept = float(ops.unpack_relu_bits(bits, N).sum())
    sigma = (p * (1 - p) / n) ** 0.5
    assert abs(kept / n - (1 - p)) <= 5 * sigma, (kept / n, 1 - p, sigma)


def test_dropout_masks_fresh_per_pass_layer_and_graph_replay(cuda):
    from morl_baselines_b200 import ops

    M, N, K, p = 1024, 128, 64, 0.5
    *_, sx, sw, xp, wp = _operands(cuda, 1, M, N, K, 13)
    seed, off = _dropout_state(cuda)

    def mask(salt=0):
        bits = ops.empty_relu_bits(M, cuda, N).zero_()
        ops.gemm_planes_ln(xp, wp, N, drop_p=p, drop_seed=seed, drop_offset=off, drop_salt=salt, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits)
        return bits

    a, b = mask(), mask()
    assert th.equal(a, b), "same seed and offset: same mask"
    assert not th.equal(a, mask(salt=1)), "layers of one pass draw different masks"
    ops.philox_advance(off)
    assert not th.equal(a, mask()), "successive passes draw different masks"
    seed2, _ = _dropout_state(cuda, seed=99)
    bits2 = ops.empty_relu_bits(M, cuda, N).zero_()
    ops.gemm_planes_ln(xp, wp, N, drop_p=p, drop_seed=seed2, drop_offset=off, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits2)
    assert not th.equal(bits2, mask()), "different seeds draw different masks"
    # a captured pass (advance + GEMM) draws a fresh mask on every replay
    bits = ops.empty_relu_bits(M, cuda, N).zero_()
    cp = ops.empty_planes(1, M, N, cuda)
    s = th.cuda.Stream()
    s.wait_stream(th.cuda.current_stream())
    with th.cuda.stream(s):
        ops.philox_advance(off)
        ops.gemm_planes_ln(xp, wp, N, drop_p=p, drop_seed=seed, drop_offset=off, c_planes=cp, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits)
    th.cuda.current_stream().wait_stream(s)
    graph = th.cuda.CUDAGraph()
    with th.cuda.graph(graph):
        ops.philox_advance(off)
        ops.gemm_planes_ln(xp, wp, N, drop_p=p, drop_seed=seed, drop_offset=off, c_planes=cp, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits)
    seen = []
    for _ in range(3):
        graph.replay()
        seen.append(bits.clone())
    assert not th.equal(seen[0], seen[1]) and not th.equal(seen[1], seen[2])
    # p = 0 keeps everything
    bits0 = ops.empty_relu_bits(M, cuda, N).zero_()
    ops.gemm_planes_ln(xp, wp, N, drop_p=0.0, drop_seed=seed, drop_offset=off, a_scale=sx, b_scale=sw, c_scale=sx, drop_bits_out=bits0)
    assert bool(ops.unpack_relu_bits(bits0, N).all())


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("B,P,H", [(1024, 64, 256), (37, 5, 128), (9, 16, 32)])
def test_product_layer(cuda, fmt, B, P, H):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(B + P + H)
    u = th.randn(B, H, device=cuda, generator=g).clamp_min(0) * 3
    v = th.randn(P, H, device=cuda, generator=g).clamp_min(0)
    s = _scale(fmt, 2.0, cuda)
    planes = ops.pairs_product_split(u, v, fmt=fmt, scale=s)
    ref = (u[:, None] * v[None]).reshape(B * P, H)
    rec = planes.double().sum(0) / (2.0 if fmt == ops.FMT_F16X2 else 1.0)
    if fmt == ops.FMT_BF16X3:  # three bf16 planes carry all 24 bits: the product itself, bit for bit
        assert th.equal(rec.float(), ref)
    else:
        assert float(((rec - ref.double()).abs() - 2.0 ** -21 * ref.double().abs()).max()) <= 2.0 ** -25
    # the feature maps u = relu(s Ls^T + bs), v = relu(m Lw^T + bw)
    obs, m = th.randn(B, 7, device=cuda, generator=g), th.rand(P, 3, device=cuda, generator=g)
    ls, lw = nn.Linear(7, H).to(cuda), nn.Linear(3, H).to(cuda)
    uu, vv = ops.product_layer1_uv(obs, ls.weight, ls.bias, m, lw.weight, lw.bias)
    for got, x, l in ((uu, obs, ls), (vv, m, lw)):
        ref64 = (x.double() @ l.weight.double().t() + l.bias.double()).clamp_min(0)
        bnd = 4 * 2.0 ** -24 * (x.double().abs() @ l.weight.double().abs().t() + l.bias.double().abs()) * x.shape[1]
        assert bool(((got.double() - ref64).abs() <= bnd).all())


def _qnet(cuda, arch, A, D, drop=0.01, ln=True, obs=8, seed=0):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import QNet

    th.manual_seed(seed)
    q = QNet((obs,), A, D, arch, drop_rate=drop, layer_norm=ln).to(cuda)
    with th.no_grad():  # non-trivial LayerNorm affine parameters and biases
        for m in q.modules():
            if isinstance(m, nn.LayerNorm):
                m.weight.normal_(1.0, 0.2)
                m.bias.normal_(0.0, 0.1)
            if isinstance(m, nn.Linear):
                m.bias.normal_(0.0, 0.05)
    return q


def _float64_forward(q64, plan, obs, M, masks):
    """QNet forward in float64 with the plan's recorded keep masks (masks None: module as is, eval mode)."""
    from morl_baselines_b200 import ops

    sf = q64.state_features(obs.double())
    wf = q64.weights_features(M.double())
    h = (sf[:, None] * wf[None]).reshape(-1, sf.shape[1])
    if masks is None:
        return q64.net(h)
    rows = h.shape[0]
    mods = list(q64.net)
    i, k = 0, 0
    while i < len(mods) - 1:
        z = mods[i](h)
        i += 1
        if isinstance(mods[i], nn.Dropout):
            keep = ops.unpack_relu_bits(masks[k][:rows], z.shape[1]).double()
            z = z * keep * float(np.float32(1 / (1 - mods[i].p)))
            i += 1
        if isinstance(mods[i], nn.LayerNorm):
            z = mods[i](z)
            i += 1
        h = z.clamp_min(0)
        i += 1
        k += 1
    return mods[-1](h)


@pytest.mark.parametrize("AD", [(6, 3), (8, 3), (8, 5)], ids=["AD18", "AD24", "AD40"])
@pytest.mark.parametrize("fmt,arch", [pytest.param(1, (256,) * 4, id="f16x2-256x4"), pytest.param(0, (256,) * 4, id="bf16x3-256x4"),
                                      pytest.param(1, (128,) * 3, id="f16x2-128x3"), pytest.param(0, (128,) * 3, id="bf16x3-128x3"),
                                      pytest.param(0, (32,) * 3, id="bf16x3-32x3"), pytest.param(0, (96,) * 3, id="bf16x3-96x3")])
def test_plan_against_float64_qnet(cuda, fmt, arch, AD):
    from morl_baselines_b200.tc_mlp import TCProductMlp

    A, D = AD
    q = _qnet(cuda, arch, A, D)
    q64 = copy.deepcopy(q).double()
    plan = TCProductMlp(q, 4096, fmt)
    plan.record_masks()
    g = th.Generator(device=cuda).manual_seed(3)
    for B, P in ((64, 16), (37, 5)):  # 1024 rows (narrow head when A*D <= 32) and a ragged call on views
        obs = th.randn(B, 8, device=cuda, generator=g)
        M = th.rand(P, D, device=cuda, generator=g)
        M = M / M.sum(1, keepdim=True)
        for train in (False, True):
            q.train(train)
            q64.train(False)
            got = plan.forward_pairs(obs, M).double()
            with th.no_grad():
                ref = _float64_forward(q64, plan, obs, M, plan.drop_bits if train else None)
            tol = 1e-4 * float(ref.abs().max())
            err = float((got - ref).abs().max())
            assert err <= tol, f"B={B} P={P} train={train}: max err {err:.3g} > {tol:.3g}"
    q.train(True)


def _agents(cuda, arch=(256,) * 4, fmt="f16x2", drop=0.0, obs=8, A=6, D=3, **kw):
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPIPD
    from morl_baselines_b200.testing import FakeEnv

    out = []
    for tc in (False, True):
        env = FakeEnv(obs_dim=obs, n_actions=A, reward_dim=D)
        out.append(GPIPD(env, net_arch=list(arch), drop_rate=drop, layer_norm=True, dyna=False, per=True, buffer_size=70000, log=False, seed=1,
                         device=cuda, use_tensor_cores=tc, tensor_core_format=fmt, **kw))
    lib, tc = out
    for a, b in zip(lib.q_nets + lib.target_q_nets, tc.q_nets + tc.target_q_nets):
        b.load_state_dict(a.state_dict())
    return lib, tc


def _fill(agent, n, rng):
    D, A, OBS = agent.reward_dim, agent.action_dim, agent.observation_shape[0]
    for _ in range(n):
        agent.replay_buffer.add(rng.standard_normal(OBS), rng.integers(A), rng.standard_normal(D), rng.standard_normal(OBS), rng.random() < 0.05)


@pytest.mark.parametrize("fmt", ["f16x2", "bf16x3"])
def test_gpipd_envelope_target_and_gpi_indices(cuda, fmt):
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.weights import equally_spaced_weights

    lib, tc = _agents(cuda, fmt=fmt)
    support = equally_spaced_weights(3, 16)
    for a in (lib, tc):
        a.set_weight_support(support)
    g = th.Generator(device=cuda).manual_seed(0)
    obs = th.randn(1024, 8, device=cuda, generator=g)
    w = th.tensor(support[5], device=cuda, dtype=th.float32).reshape(1, 3)
    M = lib._support_matrix()
    t_lib, _ = lib._envelope_target(obs, w, M)
    t_tc, _ = tc._envelope_target(obs, w, M)
    with th.no_grad():
        q_lib = th.stack([n.forward_pairs(obs, M) for n in lib.target_q_nets])
    q_tc = th.empty_like(q_lib)
    for i, plan in enumerate(tc._tc(1024 * 16)[1]):
        plan.forward_pairs(obs, M, out=q_tc[i].view(1024 * 16, -1))
    tol = 1e-4 * float(q_lib.abs().max())
    assert float((q_tc - q_lib).abs().max()) <= tol
    assert float((t_tc - t_lib).abs().max()) <= tol
    # GPI argmax: identical except where the two choices' scalarised values lie within the error bound
    _, pol_l, act_l = ops.gpi_envelope(q_lib[:1], w)
    _, pol_t, act_t = ops.gpi_envelope(q_tc[:1], w)
    sc = (q_lib[0].double() * w.double().reshape(1, 1, 1, 3)).sum(-1)  # [B, P, A]
    r = th.arange(1024, device=cuda)
    diff = (pol_l != pol_t) | (act_l != act_t)
    gap = (sc[r, pol_l.long(), act_l.long()] - sc[r, pol_t.long(), act_t.long()]).abs()
    assert bool((gap[diff] <= 2 * tol).all())


def test_gpipd_reset_priorities_and_graphed_update(cuda):
    from morl_baselines_b200.common.weights import equally_spaced_weights

    lib, tc = _agents(cuda, arch=(128,) * 3)
    support = equally_spaced_weights(3, 16)
    rng = np.random.default_rng(0)
    _fill(lib, 65536 + 300, rng)  # four chunks, the last one ragged
    for k in ("obs", "next_obs", "actions", "rewards", "dones"):
        getattr(tc.replay_buffer, k)[:] = getattr(lib.replay_buffer, k)
    tc.replay_buffer.size, tc.replay_buffer.ptr = lib.replay_buffer.size, lib.replay_buffer.ptr
    tc.replay_buffer.mark_all_dirty()
    w = th.tensor(support[3], device=cuda, dtype=th.float32)
    for a in (lib, tc):
        a.set_weight_support(support)
        a._reset_priorities(w)
    n = lib.replay_buffer.size
    pl, pt = lib.replay_buffer.tree.nodes[-1][:n], tc.replay_buffer.tree.nodes[-1][:n]
    np.testing.assert_allclose(pt, pl, rtol=1e-3, atol=1e-6)
    # update() replays its CUDA graph with the tensor-core envelope target
    tc.global_step = 1
    before = [p.detach().clone() for p in tc.q_nets[0].parameters()]
    graphs = []
    for _ in range(3):
        tc.update(w)
        assert np.isfinite(float(tc._last_loss))
        assert len(tc._graphs) == 1, "the update ran eagerly instead of through its CUDA graph"
        graphs.append(next(iter(tc._graphs.values()))["graph"])
    assert graphs[0] is graphs[1] is graphs[2], "the update graph was captured more than once"
    assert any(not th.equal(a, b) for a, b in zip(before, tc.q_nets[0].parameters()))


def test_gpipd_plan_seeds_follow_torch_manual_seed(cuda):
    seeds = []
    for _ in range(2):
        th.manual_seed(123)
        _, tc = _agents(cuda, arch=(128,) * 3)
        q0, tg = tc._tc_plans
        seeds.append([int(p.seed) for p in [q0] + tg])
    assert seeds[0] == seeds[1] and len(set(seeds[0])) == 3


def test_gpipd_dyna_rollout_golden_bf16x3(cuda):
    """_rollout_dynamics on the frozen case of tests/golden/dyna.npz (widths 32: bf16x3) through the tensor-core plan, set up as
    tests/test_dyna_gpu.py sets up the library path: accepted rows, GPI actions and termination flags identical to the reference."""
    import os

    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPIPD
    from morl_baselines_b200.testing import FakeEnv, _Spec

    from tests.test_dyna_gpu import DYN as c
    from tests.test_dyna_gpu import _load_sd, _Noise

    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dyna.npz"))
    env = FakeEnv(obs_dim=c["OBS"], n_actions=c["A"], reward_dim=c["D"])
    env.spec = _Spec(c["ENV_ID"])
    agent = GPIPD(env, batch_size=c["B"], net_arch=[32, 32, 32], num_nets=2, gradient_updates=2, dyna=True, per=True, gpi_pd=True, drop_rate=0.0,
                  layer_norm=True, buffer_size=c["N"], log=False, seed=1, device=cuda, target_net_update_freq=3, dynamics_net_arch=[32, 32],
                  dynamics_rollout_batch_size=c["ROLLOUT_B"], dynamics_rollout_len=c["ROLLOUT_LEN"], dynamics_buffer_size=c["DYN_BUF"],
                  dynamics_uncertainty_threshold=float(gold["dyn/threshold"]), dynamics_rollout_starts=0, real_ratio=0.5,
                  use_tensor_cores=True, tensor_core_format="bf16x3")
    for i, (net, tnet) in enumerate(zip(agent.q_nets, agent.target_q_nets)):
        _load_sd(net, gold, f"dyn/init{i}", cuda)
        tnet.load_state_dict(net.state_dict())
    _load_sd(agent.dynamics, gold, "dyn/init_dynamics", cuda)
    agent.dynamics.elites = [4, 2]
    rb = agent.replay_buffer
    for k in ("obs", "next_obs", "actions", "rewards", "dones"):
        getattr(rb, k)[:] = gold[f"dyn/rb_{k}"]
    rb.size, rb.ptr = c["N"], 0
    rb.mark_all_dirty()
    rb.tree.batch_set(np.arange(c["N"]), gold["dyn/tree_leaves0"][: c["N"]])  # the rollout's start states are drawn from the PER tree
    agent.set_weight_support(list(gold["dyn/support"]))
    w = th.tensor(gold["dyn/support"][2]).to(cuda)
    agent.dynamics.noise_fn = _Noise(c["NOISE_SEED"])
    np.random.seed(c["SEED_ROLLOUT"])
    added = agent._rollout_dynamics(w)
    db = agent.dynamics_buffer
    assert [db.ptr, db.size] == list(gold["dyn/db_ptr_size"]) and added > db.size
    assert np.array_equal(db.actions, gold["dyn/db_actions"]), "GPI actions / accepted rows differ"
    assert np.array_equal(db.dones, gold["dyn/db_dones"]), "termination flags differ"
    np.testing.assert_allclose(db.obs, gold["dyn/db_obs"], rtol=1e-5, atol=2e-6)


def test_unsupported_shapes_raise(cuda):
    from morl_baselines_b200 import _lib, ops
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPIPD, QNet
    from morl_baselines_b200.tc_mlp import TCProductMlp
    from morl_baselines_b200.testing import FakeEnv

    with pytest.raises(_lib.MorlB200Error):
        TCProductMlp(QNet((1, 84, 84), 4, 3, [256, 256]).to(cuda), 1024, ops.FMT_F16X2)  # NatureCNN features
    with pytest.raises(_lib.MorlB200Error, match="use_tensor_cores=False"):
        GPIPD(FakeEnv(obs_dim=8, n_actions=4, reward_dim=3), net_arch=[96, 96, 96], dyna=False, log=False, device=cuda, use_tensor_cores=True,
              tensor_core_format="f16x2")
    with pytest.raises(_lib.MorlB200Error, match="use_tensor_cores=False"):
        GPIPD(FakeEnv(obs_dim=8, n_actions=4, reward_dim=3), net_arch=[512, 512], dyna=False, log=False, device=cuda, use_tensor_cores=True)
    *_, sx, sw, xp, wp = _operands(cuda, 1, 256, 288, 64, 1)
    with pytest.raises(_lib.MorlB200Error):
        ops.gemm_planes_ln(xp, wp, 288, a_scale=sx, b_scale=sw)  # wider than one column unit
    plan = TCProductMlp(_qnet(cuda, (128,) * 3, 4, 3), 100)
    with pytest.raises(_lib.MorlB200Error):
        plan.forward_pairs(th.randn(11, 8, device=cuda), th.rand(10, 3, device=cuda))  # more pair rows than the plan holds
