"""GPU tests of how the wgmma GEMM kernels (csrc/gemm_planes.cu) are fed and drained: 384-thread CTAs with re-allocated registers, two
TMA-store staging tiles per consumer warp, the weight-gradient kernel instantiated per width.  None of that may change a result: the
same product computed in a different tile order, with a different number of bulk stores per unit (narrow output), per layer or chained,
must give identical planes, ReLU bits and fp32 outputs, and the values must still agree with float64."""

import pytest
import torch as th

pytestmark = pytest.mark.gpu

FMTS = [pytest.param(1, id="f16x2"), pytest.param(0, id="bf16x3")]
# (M, N, K): the update's hidden layer; 257 row tiles, the last one ragged; a narrow output (one bulk store per unit and warp)
SHAPES = [(65536, 256, 256), (32800, 256, 256), (32800, 24, 256)]


def _scale(fmt, value, dev):
    from morl_baselines_b200 import ops

    return ops.scale_tensor(value, dev) if fmt == ops.FMT_F16X2 else None


def _bound(a, b):
    return 2e-6 * (a.abs().double() @ b.abs().double().t()) + 1e-30


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_forward_and_dx_forms_do_not_depend_on_tile_order(cuda, fmt, M, N, K):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(M + N)
    x = th.randn(M, K, device=cuda, generator=g)
    w = th.randn(N, K, device=cuda, generator=g) / 16
    b = th.randn(N, device=cuda, generator=g) * 0.1
    sx, sw, sg = _scale(fmt, 8.0, cuda), _scale(fmt, 1024.0, cuda), _scale(fmt, 64.0, cuda)
    n_pad = (N + 31) // 32 * 32
    xp, wp = ops.split_planes(x, fmt, scale=sx), ops.split_planes(w, fmt, rows_pad=n_pad, scale=sw)
    ops.plane_overflow_count(reset=True)
    # forward form: bias + ReLU, fp32 and planes and bits
    outs = []
    for rev in (False, True):
        bits = ops.empty_relu_bits(M, cuda).zero_()
        c, p = ops.gemm_planes(xp, wp, N, bias=b, relu=True, out_f32=True, out_planes=True, reverse_tiles=rev, a_scale=sx, b_scale=sw, c_scale=sx,
                               relu_bits_out=bits)
        outs.append((c, p, bits))
    for c, p, bits in outs[1:]:
        assert th.equal(c, outs[0][0]) and th.equal(p.view(th.int16), outs[0][1].view(th.int16)) and th.equal(bits, outs[0][2])
    c0, p0, bits0 = outs[0]
    assert th.equal(ops.unpack_relu_bits(bits0, n_pad)[:, :N], c0 > 0)
    ref = (x.double() @ w.double().t() + b.double()).clamp_min(0)
    assert bool(((c0.double() - ref).abs() <= _bound(x, w)).all())
    # planes-only call (what the update runs; output scale folded into the epilogue constants): same planes, same bits
    bits1 = ops.empty_relu_bits(M, cuda).zero_()
    _, p1 = ops.gemm_planes(xp, wp, N, bias=b, relu=True, out_f32=False, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx, relu_bits_out=bits1)
    assert th.equal(p1.view(th.int16), p0.view(th.int16)) and th.equal(bits1, bits0)
    # dX form: G . W masked by the recorded bits (G [M, N] against W^T [K, N]; N is the reduction length here, so only N = 256 has it)
    if N == 256:
        gr = th.randn(M, N, device=cuda, generator=g) * 1e-3
        gp = ops.split_planes(gr, fmt, scale=sg)
        wt = ops.split_planes(w, fmt, transpose=True, scale=sw)  # [K, N]
        hbits = ops.empty_relu_bits(M, cuda).zero_()
        h, _ = ops.gemm_planes(xp, ops.split_planes(th.randn(K, K, device=cuda, generator=g) / 16, fmt, scale=sw), K, relu=True, out_f32=True,
                               a_scale=sx, b_scale=sw, relu_bits_out=hbits)
        dx = [ops.gemm_planes(gp, wt, K, relu_bits_in=hbits, out_f32=True, out_planes=True, reverse_tiles=rev, a_scale=sg, b_scale=sw, c_scale=sg)
              for rev in (False, True)]
        assert th.equal(dx[0][0], dx[1][0]) and th.equal(dx[0][1].view(th.int16), dx[1][1].view(th.int16))
        ref = (gr.double() @ w.double()) * (h > 0)
        assert bool(((dx[0][0].double() - ref).abs() <= _bound(gr, w.t())).all())
    assert ops.plane_overflow_count() == 0


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("n_chains", [1, 2])
@pytest.mark.parametrize("M", [65536, 32800, 1280])  # 257 tiles (ragged last one); 1280: fewer tiles than CTAs
def test_dx_chain_equals_per_layer_launches(cuda, fmt, n_chains, M):
    """The backward form of the chained launch (no ReLU, outputs masked by recorded ReLU bits, first layer reading a 64-wide input) against
    one launch per layer: every plane tensor bit for bit."""
    from morl_baselines_b200 import ops

    H, K0, n_layers = 256, 64, 3
    g = th.Generator(device=cuda).manual_seed(M + n_chains)
    sa = _scale(fmt, 64.0, cuda)
    acts, weights, scales, masks, refs = [], [], [], [], []
    for c in range(n_chains):
        a0 = ops.split_planes(th.randn(M, K0, device=cuda, generator=g) * 1e-2, fmt, scale=sa)
        ws, sws, ms = [], [], []
        for l in range(n_layers):
            k = K0 if l == 0 else H
            sw = _scale(fmt, 1024.0 * (1 + l), cuda)
            ws.append(ops.split_planes(th.randn(H, k, device=cuda, generator=g) / 16, fmt, scale=sw))
            sws.append(sw)
            ms.append(th.randint(-2**31, 2**31 - 1, (M, 8), device=cuda, generator=g, dtype=th.int64).to(th.int32))
        a, ref = a0, []
        for l in range(n_layers):
            _, a = ops.gemm_planes(a, ws[l], H, out_f32=False, out_planes=True, a_scale=sa, b_scale=sws[l], c_scale=sa, relu_bits_in=ms[l])
            ref.append(a)
        acts.append([a0] + [ops.empty_planes(fmt, M, H, cuda).zero_() for _ in range(n_layers)])
        weights.append(ws); scales.append(sws); masks.append(ms); refs.append(ref)
    chain = ops.GemmChain(acts, weights, None, None if fmt != ops.FMT_F16X2 else scales, None, act_scale=sa, relu=False, bits_in=masks, k_first=K0)
    for _ in range(2):
        chain()
    th.cuda.synchronize()
    for c in range(n_chains):
        for l in range(n_layers):
            assert th.equal(acts[c][l + 1].view(th.int16), refs[c][l].view(th.int16)), f"planes differ: chain {c} layer {l}"
        assert float(refs[c][-1].float().abs().max()) > 0


def test_overflow_in_the_epilogue_is_still_flagged(cuda):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(5)
    x = th.randn(1000, 256, device=cuda, generator=g)
    w = th.randn(256, 256, device=cuda, generator=g) / 16
    sx, sw = ops.scale_tensor(8.0, cuda), ops.scale_tensor(1024.0, cuda)
    xp, wp = ops.split_planes(x, ops.FMT_F16X2, scale=sx), ops.split_planes(w, ops.FMT_F16X2, scale=sw)
    ops.plane_overflow_count(reset=True)
    ops.gemm_planes(xp, wp, 256, out_f32=False, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx)
    assert ops.plane_overflow_count() == 0
    _, p = ops.gemm_planes(xp, wp, 256, out_f32=False, out_planes=True, a_scale=sx, b_scale=sw, c_scale=ops.scale_tensor(2.0**20, cuda))
    assert ops.plane_overflow_count(reset=True) > 0 and not bool(th.isfinite(p.float()).all())


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("hc", [64, 128, 192, 256])
def test_weight_gradient_widths_with_and_without_bias_gradient(cuda, fmt, hc):
    """The weight-gradient kernel is instantiated per width of H and with / without the fused bias gradient: same dW from both, against float64."""
    from morl_baselines_b200 import ops

    M, gc = 20000, 256
    g = th.Generator(device=cuda).manual_seed(hc)
    G = th.randn(M, gc, device=cuda, generator=g) * 1e-4
    Hm = th.randn(M, hc, device=cuda, generator=g).clamp_min(0)
    sg, sh = _scale(fmt, 2.0**20, cuda), _scale(fmt, 8.0, cuda)
    Gp, Hp = ops.split_planes(G, fmt, scale=sg), ops.split_planes(Hm, fmt, scale=sh)
    dW = ops.gemm_planes_mn(Gp, gc, Hp, hc, g_scale=sg, h_scale=sh)
    cs = th.full((gc,), float("nan"), device=cuda)
    dW2 = ops.gemm_planes_mn(Gp, gc, Hp, hc, colsum=cs, g_scale=sg, h_scale=sh)
    assert th.equal(dW, dW2)
    ref = G.double().t() @ Hm.double()
    bound = 2e-6 * (G.abs().double().t() @ Hm.abs().double()) * (M / 4096) ** 0.5 + 1e-30
    assert bool(((dW.double() - ref).abs() <= bound).all())
    assert th.allclose(cs.double(), G.double().sum(0), rtol=1e-5, atol=1e-5 * float(G.abs().sum(0).max()))
