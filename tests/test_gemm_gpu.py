"""GPU tests of the wgmma split-operand GEMMs (csrc/gemm_planes.cu) against a float64 reference, for both operand formats:
f16x2 (two fp16 planes of a power-of-two-scaled operand, three MMAs) and bf16x3 (three bf16 planes, six MMAs).

Tolerance: the expansions are exact to ~2^-22 (f16x2) / 2^-24 (bf16x3) per product and accumulate in fp32, so the result must agree
with the float64 product to fp32-GEMM accuracy: |err| <= 2e-6 * (|A| . |B|^T) elementwise (2e-6 ~ 32 ulp of headroom for the
K = 256 accumulation; a plain FP16 / BF16 / TF32 GEMM misses this bound by two to three orders of magnitude)."""

import numpy as np
import pytest
import torch as th

pytestmark = pytest.mark.gpu

FMTS = [pytest.param(1, id="f16x2"), pytest.param(0, id="bf16x3")]


def _ref(a, b, bias):
    r = a.double() @ b.double().t()
    if bias is not None:
        r = r + bias.double()
    return r


def _bound(a, b):
    return 2e-6 * (a.abs().double() @ b.abs().double().t()) + 1e-30


def _scale(fmt, value, dev):
    from morl_baselines_b200 import ops

    return ops.scale_tensor(value, dev) if fmt == ops.FMT_F16X2 else None


def _sum(p):
    return sum(p[i].double() for i in range(p.shape[0]))


@pytest.mark.parametrize("fmt", FMTS)
def test_split_planes_reproduce_the_operand(cuda, fmt):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(0)
    if fmt == ops.FMT_F16X2:  # fp16 exponent range: moderate dynamic range, power-of-two scale
        x = th.randn(300, 70, device=cuda, generator=g) * th.exp(th.randn(300, 70, device=cuda, generator=g))
        sc, rel = ops.scale_tensor(64.0, cuda), 2.0**-21
    else:
        x = th.randn(300, 70, device=cuda, generator=g) * th.exp(3 * th.randn(300, 70, device=cuda, generator=g))
        sc, rel = None, 2.0**-23
    p = ops.split_planes(x, fmt, rows_pad=320, ldp=128, scale=sc)
    s = _sum(p) / (64.0 if sc is not None else 1.0)
    assert th.all(s[300:] == 0) and th.all(s[:, 70:] == 0)
    big = x.abs() > 1e-3  # (f16x2: elements below 2^-14 / scale keep absolute, not relative, accuracy)
    assert float(((s[:300, :70] - x.double()).abs() / x.abs().double())[big].max()) <= rel
    assert float((s[:300, :70] - x.double()).abs().max()) <= rel * float(x.abs().max())
    pt = ops.split_planes(x, fmt, transpose=True, scale=sc)
    assert th.equal(pt[0][:70, :300], p[0][:300, :70].t())


def test_f16x2_overflow_is_flagged(cuda):
    from morl_baselines_b200 import ops

    ops.plane_overflow_count(reset=True)
    x = th.ones(64, 64, device=cuda)
    ops.split_planes(x, ops.FMT_F16X2, scale=ops.scale_tensor(1024.0, cuda))
    assert ops.plane_overflow_count() == 0
    x[3, 5] = 100.0  # 100 * 1024 > 65504
    p = ops.split_planes(x, ops.FMT_F16X2, scale=ops.scale_tensor(1024.0, cuda))
    assert ops.plane_overflow_count(reset=True) > 0 and not bool(th.isfinite(p.float()).all())
    assert ops.plane_overflow_count() == 0


def test_amax_scale(cuda):
    from morl_baselines_b200 import ops

    ws = th.zeros(2, device=cuda, dtype=th.int32)
    out = th.zeros(1, device=cuda)
    g = th.Generator(device=cuda).manual_seed(4)
    for n, mag in ((65536 * 24, 3e-5), (1000, 7.0), (13, 1e-9), (5, 0.0)):
        x = th.randn(n, device=cuda, generator=g) * mag
        ops.amax_scale(x, 9, out, ws)
        amax, s = float(x.abs().max()), float(out)
        assert int(ws.abs().sum()) == 0  # workspace left zeroed
        if amax == 0:
            assert s == 1.0
        else:
            assert np.log2(s) == round(np.log2(s)) and 2.0**8 <= amax * s < 2.0**9, (amax, s)


@pytest.mark.parametrize("split", [False, True], ids=["single", "split"])
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M,N,K", [(128, 256, 256), (1000, 256, 256), (65536, 256, 256), (4096, 24, 256), (777, 256, 64), (513, 64, 64)])
@pytest.mark.parametrize("relu", [False, True])
def test_gemm_planes_matches_float64(cuda, fmt, M, N, K, relu, split):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(M + N + K)
    a = th.randn(M, K, device=cuda, generator=g)
    b = th.randn(N, K, device=cuda, generator=g) / np.sqrt(K)
    bias = th.randn(N, device=cuda, generator=g)
    sa, sb, sc = _scale(fmt, 8.0, cuda), _scale(fmt, 4096.0, cuda), _scale(fmt, 16.0, cuda)
    ap = ops.split_planes(a, fmt, scale=sa)
    bp = ops.split_planes(b, fmt, rows_pad=(N + 31) // 32 * 32, scale=sb)
    c, cp = ops.gemm_planes(ap, bp, N, bias=bias, relu=relu, out_f32=True, out_planes=(N % 32 == 0), a_scale=sa, b_scale=sb, c_scale=sc,
                            split_acc=split)
    ref = _ref(a, b, bias)
    if relu:
        ref = ref.clamp_min(0)
    err = (c.double() - ref).abs()
    bound = _bound(a, b) + 2e-6 * bias.abs().double()
    assert bool((err <= bound).all()), float((err / bound).max())
    # a plain fp32 cuBLAS product sits inside the same bound (sanity of the bound itself)
    c32 = th.addmm(bias, a, b.t())
    c32 = c32.clamp_min(0) if relu else c32
    assert bool(((c32.double() - ref).abs() <= bound).all())
    if cp is not None:
        s = _sum(cp) / (16.0 if sc is not None else 1.0)
        assert float((s - c.double()).abs().max()) <= 2.0**-21 * float(c.abs().max())
    assert ops.plane_overflow_count() == 0


@pytest.mark.parametrize("fmt", FMTS)
def test_gemm_relu_bits_and_chaining(cuda, fmt):
    """Two chained layers through the plane format (no fp32 round trip) and the ReLU-backward mask recorded by the forward call."""
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(5)
    M, H = 2048, 256
    x = th.randn(M, H, device=cuda, generator=g)
    w1 = th.randn(H, H, device=cuda, generator=g) / 16
    w2 = th.randn(H, H, device=cuda, generator=g) / 16
    b1 = th.randn(H, device=cuda, generator=g) * 0.1
    sx, sw, sg = _scale(fmt, 8.0, cuda), _scale(fmt, 1024.0, cuda), _scale(fmt, 64.0, cuda)
    xp = ops.split_planes(x, fmt, scale=sx)
    h1_bits = ops.empty_relu_bits(M, cuda)
    _, h1p = ops.gemm_planes(xp, ops.split_planes(w1, fmt, scale=sw), H, bias=b1, relu=True, out_f32=False, out_planes=True, a_scale=sx, b_scale=sw,
                             c_scale=sx, relu_bits_out=h1_bits)
    y, _ = ops.gemm_planes(h1p, ops.split_planes(w2, fmt, scale=sw), H, a_scale=sx, b_scale=sw)
    h1 = (x.double() @ w1.double().t() + b1.double()).clamp_min(0)
    ref = h1 @ w2.double().t()
    assert float((y.double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    # backward of layer 2 w.r.t. h1, masked by relu'(h1):  dH = (dY . W2) * [h1 > 0]
    dy = th.randn(M, H, device=cuda, generator=g)
    dh, _ = ops.gemm_planes(ops.split_planes(dy, fmt, scale=sg), ops.split_planes(w2, fmt, transpose=True, scale=sw), H, relu_bits_in=h1_bits,
                            a_scale=sg, b_scale=sw)
    ref_dh = (dy.double() @ w2.double()) * (h1 > 0)
    assert float((dh.double() - ref_dh).abs().max()) <= 1e-5 * float(ref_dh.abs().max())


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M,H", [(2048, 256), (65536, 256), (777, 128), (100, 64)])
def test_gemm_relu_bit_masks(cuda, fmt, M, H):
    """ReLU backward from the bit masks: the forward call records [h > 0] (32 B per row), the backward call masks with it.  The bits must
    equal the sign pattern of the fp32 output of the same call exactly, and the masked product must equal the unmasked one with the cleared
    outputs zeroed, bit for bit."""
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(17)
    x = th.randn(M, H, device=cuda, generator=g)
    w1 = th.randn(H, H, device=cuda, generator=g) / 8
    w2 = th.randn(H, H, device=cuda, generator=g) / 8
    b1 = th.randn(H, device=cuda, generator=g) * 0.1
    sx, sw, sg = _scale(fmt, 8.0, cuda), _scale(fmt, 1024.0, cuda), _scale(fmt, 64.0, cuda)
    xp, w1p = ops.split_planes(x, fmt, scale=sx), ops.split_planes(w1, fmt, scale=sw)
    bits = ops.empty_relu_bits(M, cuda).fill_(-1)
    h, _ = ops.gemm_planes(xp, w1p, H, bias=b1, relu=True, out_f32=True, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx, relu_bits_out=bits)
    got = ops.unpack_relu_bits(bits, H)
    assert th.equal(got, h > 0)
    assert 0.2 < float(got.float().mean()) < 0.8
    # planes-only call (the form the update uses: output scale folded into the epilogue constants) records the same bits
    bits2 = ops.empty_relu_bits(M, cuda).fill_(0)
    ops.gemm_planes(xp, w1p, H, bias=b1, relu=True, out_f32=False, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx, relu_bits_out=bits2)
    assert th.equal(ops.unpack_relu_bits(bits2, H), got)
    # backward: G . W2 masked by the bits == the unmasked product where h > 0, zero elsewhere == reference
    gr = th.randn(M, H, device=cuda, generator=g) * 1e-3
    gp = ops.split_planes(gr, fmt, scale=sg)
    w2p = ops.split_planes(w2, fmt, scale=sw)
    d_bits, _ = ops.gemm_planes(gp, w2p, H, relu_bits_in=bits, out_f32=True, a_scale=sg, b_scale=sw)
    d_unmasked, _ = ops.gemm_planes(gp, w2p, H, out_f32=True, a_scale=sg, b_scale=sw)
    assert th.equal(d_bits, th.where(h > 0, d_unmasked, 0))
    ref = _ref(gr, w2, None) * (h > 0)
    assert bool(((d_bits.double() - ref).abs() <= _bound(gr, w2)).all())
    # the planes-output form of the backward call (what the update runs) carries the same values
    _, dpl = ops.gemm_planes(gp, w2p, H, relu_bits_in=bits, out_f32=False, out_planes=True, a_scale=sg, b_scale=sw, c_scale=sg)
    s = _sum(dpl) / (64.0 if sg is not None else 1.0)
    assert float((s - d_bits.double()).abs().max()) <= 2.0**-21 * float(d_bits.abs().max())
    assert ops.plane_overflow_count() == 0


@pytest.mark.parametrize("fmt", FMTS)
def test_pairs_relu_split_bit_masks(cuda, fmt):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(19)
    for B, W, H in [(37, 5, 64), (1024, 64, 256), (3, 7, 96), (9, 5, 256), (33, 18, 256)]:  # H = 256: the warp-per-transition kernel
        u, v = th.randn(B, H, device=cuda, generator=g), th.randn(W, H, device=cuda, generator=g)
        bits = ops.empty_relu_bits(B * W, cuda).fill_(0)
        hp = ops.pairs_relu_split(u, v, fmt=fmt, scale=_scale(fmt, 2.0, cuda), relu_bits_out=bits)
        ref = (u[:, None, :] + v[None, :, :]).reshape(B * W, H)
        assert th.equal(ops.unpack_relu_bits(bits, H), ref > 0)
        back = _sum(hp) / (2.0 if fmt == ops.FMT_F16X2 else 1.0)
        assert float((back - ref.clamp_min(0).double()).abs().max()) <= 2.0**-21 * float(ref.abs().max())
        assert th.equal(hp, ops.pairs_relu_split(u, v, fmt=fmt, scale=_scale(fmt, 2.0, cuda)))  # planes unchanged by the extra output


@pytest.mark.parametrize("fmt", FMTS)
def test_pairs_relu_split(cuda, fmt):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(1)
    u, v = th.randn(37, 256, device=cuda, generator=g), th.randn(5, 256, device=cuda, generator=g)
    sc = _scale(fmt, 8.0, cuda)
    p = ops.pairs_relu_split(u, v, fmt=fmt, scale=sc)
    ref = (u.unsqueeze(1) + v.unsqueeze(0)).clamp_min(0).view(-1, 256)
    s = _sum(p) / (8.0 if sc is not None else 1.0)
    assert float((s - ref.double()).abs().max()) <= 2.0**-21 * float(ref.abs().max())


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("M,gc,hc", [(65536, 256, 256), (5000, 256, 256), (4096, 24, 256), (1000, 128, 64), (333, 256, 192),
                                     (5000, 4, 256), (4096, 36, 192), (1000, 72, 128)])  # (output layers: ldg 64, 64, 128)
def test_gemm_mn_weight_gradient(cuda, fmt, M, gc, hc):
    """dW[n, k] = sum_m G[m, n] H[m, k] (MN-major operands, split-K) against float64."""
    from morl_baselines_b200 import ops

    g_ = th.Generator(device=cuda).manual_seed(M + gc)
    G = th.randn(M, gc, device=cuda, generator=g_) * 1e-4
    H = th.randn(M, hc, device=cuda, generator=g_).clamp_min(0)
    sg, sh = _scale(fmt, 2.0**20, cuda), _scale(fmt, 8.0, cuda)
    Gp = ops.split_planes(G, fmt, ldp=(gc + 63) // 64 * 64, scale=sg)
    Hp = ops.split_planes(H, fmt, ldp=(hc + 63) // 64 * 64, scale=sh)
    dW = ops.gemm_planes_mn(Gp, gc, Hp, hc, g_scale=sg, h_scale=sh)
    ref = G.double().t() @ H.double()
    bound = 2e-6 * (G.abs().double().t() @ H.abs().double()) * max(1.0, np.sqrt(M / 4096)) + 1e-30
    err = (dW.double() - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    dWt = ops.gemm_planes_mn(Gp, gc, Hp, hc, transpose_out=True, g_scale=sg, h_scale=sh)
    assert th.equal(dWt, dW.t().contiguous())
    # bias gradient fused into the same pass (G^T . ones on the tensor cores); the weight gradient must be unchanged by it
    cs2 = th.full((gc,), float("nan"), device=cuda)
    dW2 = ops.gemm_planes_mn(Gp, gc, Hp, hc, colsum=cs2, g_scale=sg, h_scale=sh)
    assert th.equal(dW2, dW)
    np.testing.assert_allclose(cs2.cpu().numpy(), G.double().sum(0).cpu().numpy(), rtol=1e-5, atol=1e-5 * float(G.abs().sum(0).max()))


@pytest.mark.parametrize("B,W,F,D,H", [(1024, 64, 32, 3, 256), (37, 5, 11, 2, 64), (3, 70, 7, 4, 300), (8, 8, 59, 3, 32)])
def test_pair_layer1_kernels(cuda, B, W, F, D, H):
    """Separable first layer on the pair batch: u = feats W1_s^T, v = wset W1_w^T + b1 in one launch, against float64; fp32 FMA
    chains -> 1e-6 of the magnitude sums."""
    from morl_baselines_b200 import ops

    g_ = th.Generator(device=cuda).manual_seed(B + 3 * W + F)
    feats, wset = th.randn(B, F, device=cuda, generator=g_), th.rand(W, D, device=cuda, generator=g_)
    W1, b1 = th.randn(H, F + D, device=cuda, generator=g_) / 4, th.randn(H, device=cuda, generator=g_)
    u, v = ops.pair_layer1_uv(feats, wset, W1, b1)
    ru = feats.double() @ W1[:, :F].double().t()
    rv = wset.double() @ W1[:, F:].double().t() + b1.double()
    assert float((u.double() - ru).abs().max()) <= 1e-6 * float((feats.abs().double() @ W1[:, :F].abs().double().t()).max())
    assert float((v.double() - rv).abs().max()) <= 1e-6 * float((wset.abs().double() @ W1[:, F:].abs().double().t() + b1.abs().double()).max())


@pytest.mark.parametrize("B,W,F,D,H", [(1024, 64, 32, 3, 256), (256, 32, 7, 3, 256), (37, 5, 11, 2, 64), (3, 70, 7, 4, 300), (8, 8, 59, 3, 32)])
def test_pair_layer1_grad(cuda, B, W, F, D, H):
    """dW1 = [dU^T feats | dV^T wset], db1 = colsum(dV) in one launch (split reduction, fixed summation order), against float64;
    run twice on the same workspace: the arrival counters must reset themselves and the result must be bit-identical."""
    from morl_baselines_b200 import ops

    g_ = th.Generator(device=cuda).manual_seed(B + 3 * W + F)
    feats, wset = th.randn(B, F, device=cuda, generator=g_), th.rand(W, D, device=cuda, generator=g_)
    dU, dV = th.randn(B, H, device=cuda, generator=g_), th.randn(W, H, device=cuda, generator=g_)
    ws = ops.pair_layer1_grad_workspace(F, D, H, cuda)
    dW1, db1 = ops.pair_layer1_grad(dU, dV, feats, wset, workspace=ws)
    ref_w = th.cat([dU.double().t() @ feats.double(), dV.double().t() @ wset.double()], dim=1)
    mag_w = th.cat([dU.abs().double().t() @ feats.abs().double(), dV.abs().double().t() @ wset.abs().double()], dim=1)
    assert float((dW1.double() - ref_w).abs().max()) <= 2e-6 * float(mag_w.max())
    assert float((db1.double() - dV.double().sum(0)).abs().max()) <= 2e-6 * float(dV.abs().double().sum(0).max())
    dW1b, db1b = ops.pair_layer1_grad(dU, dV, feats, wset, workspace=ws)
    assert th.equal(dW1, dW1b) and th.equal(db1, db1b)


@pytest.mark.parametrize("fmt", FMTS)
def test_split_vectorised_path_matches_scalar_path(cuda, fmt):
    """ldp % 8 == 0 takes the 8-columns-per-thread kernel; an unaligned source (ld_src % 4 != 0) and ragged columns must give the same
    planes as the transposed-input scalar kernel."""
    from morl_baselines_b200 import ops

    g_ = th.Generator(device=cuda).manual_seed(9)
    sc = _scale(fmt, 32.0, cuda)
    for rows, cols in ((65536, 24), (1000, 250), (77, 13)):
        x = th.randn(rows, cols, device=cuda, generator=g_)
        ldp = (cols + 31) // 32 * 32
        a = ops.split_planes(x, fmt, ldp=ldp, scale=sc)  # vectorised
        b = ops.split_planes(x.t().contiguous(), fmt, ldp=ldp, transpose=True, scale=sc)  # scalar kernel on the transposed source
        assert th.equal(a, b)
        s = _sum(a) / (32.0 if sc is not None else 1.0)
        assert float(s[:, :cols].sub(x.double()).abs().max()) <= 2.0**-21 * float(x.abs().max())
        assert float(a[:, :, cols:].float().abs().max()) == 0.0


@pytest.mark.parametrize("fmt", FMTS)
def test_pairs_grad_reduce(cuda, fmt):
    """dU = sum_j G, dV = sum_b G from the planes of G [B*W, H] against the float64 sums of the planes' exact values: an fp32 sum of
    `count` terms in any order is within count * 2^-24 * sum |terms|.  Shapes: |W| > 64 (two-pass path), B > 2368 with |W| <= 64
    (more than 296 chunks: the row-block + column-sum fallback), a single transition, a single weight vector; every H the update uses."""
    from morl_baselines_b200 import ops

    g_ = th.Generator(device=cuda).manual_seed(2)
    sc = _scale(fmt, 16.0, cuda)
    for H in (64, 128, 192, 256):
        for B, W in ((37, 5), (64, 64), (300, 33), (5, 70), (3000, 2), (1, 64), (37, 1)):
            G = th.randn(B * W, H, device=cuda, generator=g_)
            Gp = ops.split_planes(G, fmt, scale=sc)
            dU, dV = ops.pairs_grad_reduce(Gp, B, W, scale=sc)
            terms = Gp.double().view(Gp.shape[0], B, W, H) / (16.0 if sc is not None else 1.0)  # the exact values the kernel adds
            for got, axis, count in ((dU, 2, W * Gp.shape[0]), (dV, 1, B * Gp.shape[0])):
                ref = terms.sum(axis).sum(0)
                bound = count * 2.0**-24 * terms.abs().sum(axis).sum(0)
                err = (got.double() - ref).abs()
                assert bool((err <= bound).all()), (H, B, W, axis, float((err / bound).max()))


@pytest.mark.parametrize("fmt", FMTS)
def test_gemm_alternative_kernels_still_correct(cuda, fmt):
    """split_acc=True: a 256-wide output runs as two 128-column units, a 160-wide one as 128 + 32 -- cross-checks against float64."""
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(3)
    a = th.randn(5000, 256, device=cuda, generator=g)
    b = th.randn(256, 256, device=cuda, generator=g) / 16
    ref = a.double() @ b.double().t()
    sa, sb = _scale(fmt, 8.0, cuda), _scale(fmt, 1024.0, cuda)
    ap = ops.split_planes(a, fmt, scale=sa)
    for n in (256, 160):
        c, _ = ops.gemm_planes(ap, ops.split_planes(b[:n].contiguous(), fmt, scale=sb), n, a_scale=sa, b_scale=sb, split_acc=True)
        err = float((c.double() - ref[:, :n]).abs().max())
        assert err < 2e-5, (n, err)


@pytest.mark.parametrize("fmt", FMTS)
def test_reverse_tile_order_and_multi_split_are_bit_identical(cuda, fmt):
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(11)
    a = th.randn(40000, 256, device=cuda, generator=g)
    ws = [th.randn(256, 256, device=cuda, generator=g) / 16, th.randn(24, 256, device=cuda, generator=g), th.randn(256, 64, device=cuda, generator=g)]
    sa, sw = _scale(fmt, 8.0, cuda), _scale(fmt, 512.0, cuda)
    ap = ops.split_planes(a, fmt, scale=sa)
    singles = [ops.split_planes(ws[0], fmt, scale=sw), ops.split_planes(ws[1], fmt, rows_pad=32, scale=sw),
               ops.split_planes(ws[2], fmt, rows_pad=64, ldp=256, transpose=True, scale=sw)]
    multi = [th.empty_like(s) for s in singles]
    ops.split_planes_multi([(ws[0], multi[0], False, sw), (ws[1], multi[1], False, sw), (ws[2], multi[2], True, sw)], fmt)
    for s, m in zip(singles, multi):
        assert th.equal(s, m)
    c0, p0 = ops.gemm_planes(ap, singles[0], 256, relu=True, out_f32=True, out_planes=True, a_scale=sa, b_scale=sw, c_scale=sa)
    c1, p1 = ops.gemm_planes(ap, singles[0], 256, relu=True, out_f32=True, out_planes=True, reverse_tiles=True, a_scale=sa, b_scale=sw, c_scale=sa)
    assert th.equal(c0, c1) and th.equal(p0, p1)


def test_multi_split_auto_scale(cuda):
    """auto_scale jobs derive a power-of-two scale from their own matrix (amax * s in [2^13, 2^14)), publish it, and the plain and the
    transposed job of the same matrix agree on it."""
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(12)
    w = th.randn(256, 256, device=cuda, generator=g) * 0.07
    w2 = th.randn(24, 256, device=cuda, generator=g) * 3.0
    s1, s2 = ops.scale_tensor(1.0, cuda), ops.scale_tensor(1.0, cuda)
    outs = [ops.empty_planes(ops.FMT_F16X2, 256, 256, cuda), ops.empty_planes(ops.FMT_F16X2, 256, 256, cuda), ops.empty_planes(ops.FMT_F16X2, 32, 256, cuda)]
    ops.split_planes_multi([(w, outs[0], False, s1, 14), (w, outs[1], True, s1, 14), (w2, outs[2], False, s2, 14)], ops.FMT_F16X2)
    for s, m in ((s1, w), (s2, w2)):
        v = float(s) * float(m.abs().max())
        assert 2.0**13 <= v < 2.0**14 and np.log2(float(s)) == round(np.log2(float(s)))
    assert th.equal(outs[1], outs[0].transpose(1, 2).contiguous())
    rec = _sum(outs[0]) / float(s1)
    assert float((rec - w.double()).abs().max()) <= 2.0**-21 * float(w.abs().max())
    rec2 = _sum(outs[2])[:24] / float(s2)
    assert float((rec2 - w2.double()).abs().max()) <= 2.0**-21 * float(w2.abs().max())
    assert ops.plane_overflow_count() == 0


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("n_chains,M,n_layers", [(2, 65536, 3), (1, 65536, 3), (2, 38400, 2), (1, 1280, 3), (2, 1000, 3), (1, 512, 1), (2, 19200, 4)])
def test_gemm_chain_equals_per_layer_launches(cuda, fmt, n_chains, M, n_layers):
    """morl_gemm_chain_f32 (hidden layers of one / two networks in ONE persistent launch; intermediate activations re-read from L2) must
    reproduce the per-layer morl_gemm_planes_f32 launches BIT FOR BIT: every intermediate and final activation plane and every ReLU bit
    mask.  Shapes: the north-star row count (256 tiles on 74 pairs: groups of 2 + 2 / 2 + 1 tiles), fewer tiles than pairs, a ragged last
    tile (M = 1000), a single layer, four layers (8 jobs)."""
    from morl_baselines_b200 import ops

    H = 256
    g = th.Generator(device=cuda).manual_seed(M + 7 * n_chains + n_layers)
    sa = _scale(fmt, 2.0, cuda)
    chains = []
    for c in range(n_chains):
        x = th.randn(M, H, device=cuda, generator=g).relu_()
        a0 = ops.split_planes(x, fmt, rows_pad=M, ldp=H, scale=sa)
        ws, bs, sws = [], [], []
        for l in range(n_layers):
            w = th.randn(H, H, device=cuda, generator=g) / 16.0
            sw = _scale(fmt, 2048.0 * (1 + l), cuda)
            ws.append(ops.split_planes(w, fmt, rows_pad=H, ldp=H, scale=sw))
            sws.append(sw)
            bs.append(th.randn(H, device=cuda, generator=g) * 0.1)
        chains.append((a0, ws, bs, sws))
    # reference: one launch per layer
    ref_acts, ref_bits = [], []
    for a0, ws, bs, sws in chains:
        a, acts, bits = a0, [], []
        for l in range(n_layers):
            bt = ops.empty_relu_bits(M, cuda).zero_()
            _, a = ops.gemm_planes(a, ws[l], H, bias=bs[l], relu=True, out_f32=False, out_planes=True, a_scale=sa, b_scale=sws[l], c_scale=sa, relu_bits_out=bt)
            acts.append(a)
            bits.append(bt)
        ref_acts.append(acts)
        ref_bits.append(bits)
    # chained launch into fresh buffers
    outs = [[ops.empty_planes(fmt, M, H, cuda).zero_() for _ in range(n_layers)] for _ in range(n_chains)]
    obits = [[ops.empty_relu_bits(M, cuda).zero_() for _ in range(n_layers)] for _ in range(n_chains)]
    chain = ops.GemmChain([[chains[c][0]] + outs[c] for c in range(n_chains)], [chains[c][1] for c in range(n_chains)], [chains[c][2] for c in range(n_chains)],
                          None if fmt != ops.FMT_F16X2 else [chains[c][3] for c in range(n_chains)], obits, act_scale=sa)
    for _ in range(2):  # (twice: the second launch overwrites identical values, a stale-read would not survive the comparison of layer 1 only)
        chain()
    th.cuda.synchronize()
    for c in range(n_chains):
        for l in range(n_layers):
            assert th.equal(outs[c][l].view(th.int16), ref_acts[c][l].view(th.int16)), f"planes differ: chain {c} layer {l}"
            assert th.equal(obits[c][l], ref_bits[c][l]), f"ReLU bits differ: chain {c} layer {l}"
