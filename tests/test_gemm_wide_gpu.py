"""GPU tests of the wgmma GEMM kernels (csrc/gemm_planes.cu) and the layer-1 kernels at widths above 256 columns.

K-major kernel: an output wider than 256 columns runs as two column units [0, 256) and [256, N_pad) of the same row tile, each with the
arithmetic of an ordinary <= 256-column launch.  So the wide launch must equal, bit for bit, the same product run as two launches over
the <= 256-column halves of the weight (fp32 output, re-split planes, ReLU bits), in the forward form (bias, ReLU, bits out) and in the dX
form (ReLU-bit mask in).  Values are checked against float64 with the magnitude bound of tests/test_tc_mlp_grad_gpu.py: C_PRODUCT = 2e-6
per split-operand product times the magnitude sum |A| |B|^T (+ |bias|).

ReLU bit masks above 256 columns: [rows][16] int32, word 8 * half + (c & 1) * 4 + ((c >> 1) & 3) for 32-column chunk c of the half, so each
half of the row is exactly the 8-word mask of the half's own launch.

Weight-gradient kernel: H operands up to 512 columns wide are two k units of <= 256; the result is within count * 2^-24 * sum |terms| of the
float64 sum of the exact plane values (count = number of rows reduced), with and without the fused bias gradient.
"""

import pytest
import torch as th

pytestmark = pytest.mark.gpu

C_PRODUCT = 2e-6
FMTS = [pytest.param(1, id="f16x2"), pytest.param(0, id="bf16x3")]
M_ROWS = 32800  # 257 row tiles, the last one ragged


def _scale(fmt, value, dev):
    from morl_baselines_b200 import ops

    return ops.scale_tensor(value, dev) if fmt == ops.FMT_F16X2 else None


def _i16(p):
    return p.view(th.int16)


def _within(got, ref, bound):
    err = (got.double() - ref).abs()
    return float((err / bound.clamp_min(1e-300)).max()), bool((err <= bound).all())


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("K", [320, 512])
@pytest.mark.parametrize("N", [288, 384, 512])
def test_wide_kmajor_equals_two_halves_and_float64(cuda, fmt, N, K):
    from morl_baselines_b200 import ops

    M = M_ROWS
    g = th.Generator(device=cuda).manual_seed(N + K + fmt)
    x = th.randn(M, K, device=cuda, generator=g)
    w = th.randn(N, K, device=cuda, generator=g) / 16
    b = th.randn(N, device=cuda, generator=g) * 0.1
    sx, sw, sg = _scale(fmt, 8.0, cuda), _scale(fmt, 1024.0, cuda), _scale(fmt, 64.0, cuda)
    xp, wp = ops.split_planes(x, fmt, scale=sx), ops.split_planes(w, fmt, scale=sw)
    halves = [(0, 256), (256, N)]
    ops.plane_overflow_count(reset=True)

    # ---- forward form: bias + ReLU, fp32 + planes + 16-word bits; both tile orders
    outs = []
    for rev in (False, True):
        bits = ops.empty_relu_bits(M, cuda, N).zero_()
        assert tuple(bits.shape) == (M, 16)
        c, p = ops.gemm_planes(xp, wp, N, bias=b, relu=True, out_f32=True, out_planes=True, reverse_tiles=rev, a_scale=sx, b_scale=sw, c_scale=sx,
                               relu_bits_out=bits)
        outs.append((c, p, bits))
    c, p, bits = outs[0]
    assert th.equal(outs[1][0], c) and th.equal(_i16(outs[1][1]), _i16(p)) and th.equal(outs[1][2], bits)
    for h, (lo, hi) in enumerate(halves):
        hb = ops.empty_relu_bits(M, cuda, hi - lo).zero_()
        ch, ph = ops.gemm_planes(xp, wp[:, lo:hi].contiguous(), hi - lo, bias=b[lo:hi].contiguous(), relu=True, out_f32=True, out_planes=True,
                                 a_scale=sx, b_scale=sw, c_scale=sx, relu_bits_out=hb)
        assert th.equal(c[:, lo:hi], ch), f"fp32 output, columns [{lo}, {hi})"
        assert th.equal(_i16(p[:, :, lo:hi]), _i16(ph)), f"planes, columns [{lo}, {hi})"
        assert th.equal(bits[:, 8 * h : 8 * h + 8], hb), f"bit words of half {h}"
    # planes-only call (the hidden layers of the update; output scale folded into the epilogue): same planes and bits
    bits1 = ops.empty_relu_bits(M, cuda, N).zero_()
    _, p1 = ops.gemm_planes(xp, wp, N, bias=b, relu=True, out_f32=False, out_planes=True, a_scale=sx, b_scale=sw, c_scale=sx, relu_bits_out=bits1)
    assert th.equal(_i16(p1), _i16(p)) and th.equal(bits1, bits)
    # float64: values within the bound; mask bits equal the float64 signs except inside the bound
    pre = x.double() @ w.double().t() + b.double()
    bound = C_PRODUCT * (x.abs().double() @ w.abs().double().t() + b.abs().double())
    r, ok = _within(c, pre.clamp_min(0), bound)
    assert ok, f"forward: max err / bound = {r:.3g}"
    mask = ops.unpack_relu_bits(bits, N)
    assert th.equal(mask, c > 0)
    flip = mask != (pre > 0)
    assert bool((pre.abs()[flip] <= bound[flip]).all()), "a ReLU bit differs from the float64 sign beyond the forward bound"
    print(f"\n[wide] N {N} K {K} fmt {fmt}: forward err/bound {r:.3g}, mask flips {int(flip.sum())}")

    # ---- split accumulators: 128-column units, the same as the halves in split mode
    cs, _ = ops.gemm_planes(xp, wp, N, bias=b, relu=True, a_scale=sx, b_scale=sw, split_acc=True)
    for lo, hi in halves:
        ch, _ = ops.gemm_planes(xp, wp[:, lo:hi].contiguous(), hi - lo, bias=b[lo:hi].contiguous(), relu=True, a_scale=sx, b_scale=sw, split_acc=True)
        assert th.equal(cs[:, lo:hi], ch)
    assert _within(cs, pre.clamp_min(0), bound)[1]

    # ---- dX form: out [M, N] = G [M, K] . W2 [K, N], masked by the recorded 16-word bits; fp32 + planes, both tile orders
    gr = th.randn(M, K, device=cuda, generator=g) * 1e-3
    w2 = th.randn(K, N, device=cuda, generator=g) / 16
    gp = ops.split_planes(gr, fmt, scale=sg)
    wt = ops.split_planes(w2, fmt, transpose=True, scale=sw)  # [P, N, K]
    dx = [ops.gemm_planes(gp, wt, N, relu_bits_in=bits, out_f32=True, out_planes=True, reverse_tiles=rev, a_scale=sg, b_scale=sw, c_scale=sg)
          for rev in (False, True)]
    assert th.equal(dx[0][0], dx[1][0]) and th.equal(_i16(dx[0][1]), _i16(dx[1][1]))
    for h, (lo, hi) in enumerate(halves):
        ch, ph = ops.gemm_planes(gp, wt[:, lo:hi].contiguous(), hi - lo, relu_bits_in=bits[:, 8 * h : 8 * h + 8].contiguous(), out_f32=True,
                                 out_planes=True, a_scale=sg, b_scale=sw, c_scale=sg)
        assert th.equal(dx[0][0][:, lo:hi], ch) and th.equal(_i16(dx[0][1][:, :, lo:hi]), _i16(ph)), f"dX, columns [{lo}, {hi})"
    m = mask.double()
    ref = (gr.double() @ w2.double()) * m
    bdx = C_PRODUCT * (gr.abs().double() @ w2.abs().double()) * m
    r, ok = _within(dx[0][0], ref, bdx)
    assert ok, f"dX: max err / bound = {r:.3g}"
    assert float(dx[0][0][~mask].abs().max()) == 0.0
    assert ops.plane_overflow_count() == 0


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("N,n_pad", [(256, 288), (200, 512), (24, 288)])
def test_bit_mask_pitch_follows_padded_width(cuda, fmt, N, n_pad):
    """Weight planes padded beyond 256 rows for an output of <= 256 columns (N <= 256 < N_pad): the kernel visits every chunk below
    N_pad, so the bit masks are [M][16] words (the width is N_pad).  Forward (bits out) and dX (bits in) equal the launch over the unpadded
    planes; the padding chunks' words hold zeros; an 8-word mask for this shape is refused."""
    from morl_baselines_b200 import _lib, ops

    M, K = 1000, 128
    g = th.Generator(device=cuda).manual_seed(N + n_pad + fmt)
    x = th.randn(M, K, device=cuda, generator=g)
    w = th.randn(N, K, device=cuda, generator=g) / 16
    b = th.randn(N, device=cuda, generator=g) * 0.1
    sx, sw = _scale(fmt, 8.0, cuda), _scale(fmt, 1024.0, cuda)
    xp = ops.split_planes(x, fmt, scale=sx)
    n32 = (N + 31) // 32 * 32
    wp = ops.split_planes(w, fmt, rows_pad=n32, scale=sw)
    wpad = ops.split_planes(w, fmt, rows_pad=n_pad, scale=sw)  # rows [N, n_pad) zero
    bits_ref = ops.empty_relu_bits(M, cuda, n32).zero_()
    c_ref, _ = ops.gemm_planes(xp, wp, N, bias=b, relu=True, a_scale=sx, b_scale=sw, relu_bits_out=bits_ref)
    guard = th.full((M + 64, 16), -1, device=cuda, dtype=th.int32)  # 64 rows beyond the mask: must stay untouched
    bits = guard[:M]
    bits.zero_()
    assert tuple(bits.shape) == (M, ops.relu_bits_words(n_pad)) and bits.is_contiguous()
    c, _ = ops.gemm_planes(xp, wpad, N, bias=b, relu=True, a_scale=sx, b_scale=sw, relu_bits_out=bits)
    th.cuda.synchronize()
    assert th.equal(c, c_ref)
    assert bool((guard[M:] == -1).all()), "a bit-mask write went past the last row"
    assert th.equal(ops.unpack_relu_bits(bits, N), c > 0)
    chunks = th.arange(n32 // 32, device=cuda)
    assert th.equal(bits[:, ops.relu_bits_word(chunks)], bits_ref[:, ops.relu_bits_word(chunks)])
    pad_words = sorted(set(range(16)) - set(ops.relu_bits_word(chunks).tolist()))
    assert int(bits[:, pad_words].abs().sum()) == 0, "padding chunks must record no positive column"
    with pytest.raises(_lib.MorlB200Error):
        ops.gemm_planes(xp, wpad, N, bias=b, relu=True, a_scale=sx, b_scale=sw, relu_bits_out=ops.empty_relu_bits(M, cuda, N))
    # dX form reading the same mask: out [M, N] = G [M, K2] . W2 [K2, N] masked by the bits, padded weight rows beyond N
    K2 = 64
    gr = th.randn(M, K2, device=cuda, generator=g) * 1e-3
    w2 = th.randn(K2, N, device=cuda, generator=g) / 16
    gp = ops.split_planes(gr, fmt, scale=sx)
    wt = ops.split_planes(w2, fmt, transpose=True, rows_pad=n32, scale=sw)
    wt_pad = ops.split_planes(w2, fmt, transpose=True, rows_pad=n_pad, scale=sw)
    d_ref, _ = ops.gemm_planes(gp, wt, N, relu_bits_in=bits_ref, a_scale=sx, b_scale=sw)
    d, _ = ops.gemm_planes(gp, wt_pad, N, relu_bits_in=bits, a_scale=sx, b_scale=sw)
    assert th.equal(d, d_ref)
    assert float(d[~(c > 0)].abs().max()) == 0.0


@pytest.mark.parametrize("fmt", FMTS)
def test_wide_output_rejects_beyond_512(cuda, fmt):
    from morl_baselines_b200 import _lib, ops

    xp = ops.split_planes(th.randn(256, 64, device=cuda), fmt)
    wp = ops.split_planes(th.randn(544, 64, device=cuda), fmt)
    with pytest.raises(_lib.MorlB200Error):
        ops.gemm_planes(xp, wp, 544)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("ldh", [320, 512])
@pytest.mark.parametrize("gc", [24, 512])
def test_wide_weight_gradient(cuda, fmt, ldh, gc):
    """dW [gc, ldh] = G^T H with H 320 / 512 wide (two k units) and G 24 / 512 wide (one / four 128-column tiles), with and without the
    fused bias gradient: within count * 2^-24 * sum |terms| of float64; deterministic; the bias gradient does not change dW."""
    from morl_baselines_b200 import ops

    M = 65536
    g_ = th.Generator(device=cuda).manual_seed(ldh + gc + fmt)
    G = th.randn(M, gc, device=cuda, generator=g_) * 1e-4
    H = th.randn(M, ldh, device=cuda, generator=g_).clamp_min(0)
    sg, sh = _scale(fmt, 2.0**20, cuda), _scale(fmt, 8.0, cuda)
    Gp = ops.split_planes(G, fmt, ldp=(gc + 63) // 64 * 64, scale=sg)
    Hp = ops.split_planes(H, fmt, ldp=ldh, scale=sh)
    dW = ops.gemm_planes_mn(Gp, gc, Hp, ldh, g_scale=sg, h_scale=sh)
    Ge = Gp.double().sum(0)[:, :gc] / (2.0**20 if sg is not None else 1.0)  # the exact values the kernel multiplies
    He = Hp.double().sum(0) / (8.0 if sh is not None else 1.0)
    ref = Ge.t() @ He
    bound = M * 2.0**-24 * (Ge.abs().t() @ He.abs())
    r, ok = _within(dW, ref, bound)
    assert ok, f"dW: max err / bound = {r:.3g}"
    assert th.equal(ops.gemm_planes_mn(Gp, gc, Hp, ldh, g_scale=sg, h_scale=sh), dW)
    cs = th.full((gc,), float("nan"), device=cuda)
    dW2 = ops.gemm_planes_mn(Gp, gc, Hp, ldh, colsum=cs, g_scale=sg, h_scale=sh)
    assert th.equal(dW2, dW)
    r, ok = _within(cs, Ge.sum(0), M * 2.0**-24 * Ge.abs().sum(0))
    assert ok, f"bias gradient: max err / bound = {r:.3g}"
    assert th.equal(ops.gemm_planes_mn(Gp, gc, Hp, ldh, transpose_out=True, g_scale=sg, h_scale=sh), dW.t().contiguous())
    print(f"\n[wide-mn] gc {gc} ldh {ldh} fmt {fmt}: dW err/bound {r:.3g}")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("B,W", [(256, 64), (64, 128), (17, 256)])
def test_pairs_relu_split_h512(cuda, fmt, B, W):
    """Layer 1 at H = 512: the planes of relu(u[b] + v[j]) sum to the fp32 value (to the format's 2^-21), and the 16-word bits hold its
    signs in the documented word order."""
    from morl_baselines_b200 import ops

    H = 512
    g_ = th.Generator(device=cuda).manual_seed(B + W)
    u, v = th.randn(B, H, device=cuda, generator=g_), th.randn(W, H, device=cuda, generator=g_)
    sc = _scale(fmt, 2.0, cuda)
    bits = ops.empty_relu_bits(B * W, cuda, H).fill_(0)
    hp = ops.pairs_relu_split(u, v, fmt=fmt, scale=sc, relu_bits_out=bits)
    ref = (u[:, None, :] + v[None, :, :]).reshape(B * W, H).clamp_min(0)
    back = hp.double().sum(0) / (2.0 if sc is not None else 1.0)
    assert float((back - ref.double()).abs().max()) <= 2.0**-21 * float(ref.abs().max())
    assert th.equal(ops.unpack_relu_bits(bits, H), ref > 0)
    # word order: chunk c of the row (32 columns) in word 8 (c >> 3) + (c & 1) 4 + ((c >> 1) & 3)
    pos = (ref > 0).view(B * W, 16, 32).to(th.int64) << th.arange(32, device=cuda)
    packed = pos.sum(2)  # [rows, chunk]
    words = th.empty_like(packed)
    c = th.arange(16, device=cuda)
    words[:, 8 * (c >> 3) + (c & 1) * 4 + ((c >> 1) & 3)] = packed
    assert th.equal(bits.to(th.int64) & 0xFFFFFFFF, words)


@pytest.mark.parametrize("fmt", FMTS)
def test_pairs_grad_reduce_h512(cuda, fmt):
    """dU = sum_j G, dV = sum_b G at H = 512, one-pass (|W| <= 64) and two-pass (|W| > 64) forms: within count * 2^-24 * sum |terms|
    of the float64 sums of the planes' exact values."""
    from morl_baselines_b200 import ops

    H = 512
    g_ = th.Generator(device=cuda).manual_seed(5)
    sc = _scale(fmt, 16.0, cuda)
    for B, W in ((1024, 64), (37, 5), (512, 128), (256, 256), (3, 70)):
        G = th.randn(B * W, H, device=cuda, generator=g_)
        Gp = ops.split_planes(G, fmt, scale=sc)
        dU, dV = ops.pairs_grad_reduce(Gp, B, W, scale=sc)
        terms = Gp.double().view(Gp.shape[0], B, W, H) / (16.0 if sc is not None else 1.0)
        for got, axis, count in ((dU, 2, W * Gp.shape[0]), (dV, 1, B * Gp.shape[0])):
            ref = terms.sum(axis).sum(0)
            bound = count * 2.0**-24 * terms.abs().sum(axis).sum(0)
            r, ok = _within(got, ref, bound)
            assert ok, (B, W, axis, r)


def test_pair_layer1_kernels_h512(cuda):
    """u / v and dW1 / db1 of the separable first layer at H = 512 (and |W| = 256) against float64 (bounds of tests/test_gemm_gpu.py)."""
    from morl_baselines_b200 import ops

    B, W, F, D, H = 1024, 256, 32, 3, 512
    g_ = th.Generator(device=cuda).manual_seed(7)
    feats, wset = th.randn(B, F, device=cuda, generator=g_), th.rand(W, D, device=cuda, generator=g_)
    W1, b1 = th.randn(H, F + D, device=cuda, generator=g_) / 4, th.randn(H, device=cuda, generator=g_)
    u, v = ops.pair_layer1_uv(feats, wset, W1, b1)
    ru = feats.double() @ W1[:, :F].double().t()
    rv = wset.double() @ W1[:, F:].double().t() + b1.double()
    assert float((u.double() - ru).abs().max()) <= 1e-6 * float((feats.abs().double() @ W1[:, :F].abs().double().t()).max())
    assert float((v.double() - rv).abs().max()) <= 1e-6 * float((wset.abs().double() @ W1[:, F:].abs().double().t() + b1.abs().double()).max())
    dU, dV = th.randn(B, H, device=cuda, generator=g_), th.randn(W, H, device=cuda, generator=g_)
    ws = ops.pair_layer1_grad_workspace(F, D, H, cuda)
    dW1, db1 = ops.pair_layer1_grad(dU, dV, feats, wset, workspace=ws)
    ref_w = th.cat([dU.double().t() @ feats.double(), dV.double().t() @ wset.double()], dim=1)
    mag_w = th.cat([dU.abs().double().t() @ feats.abs().double(), dV.abs().double().t() @ wset.abs().double()], dim=1)
    assert float((dW1.double() - ref_w).abs().max()) <= 2e-6 * float(mag_w.max())
    assert float((db1.double() - dV.double().sum(0)).abs().max()) <= 2e-6 * float(dV.abs().double().sum(0).max())
    dW1b, db1b = ops.pair_layer1_grad(dU, dV, feats, wset, workspace=ws)
    assert th.equal(dW1, dW1b) and th.equal(db1, db1b)
