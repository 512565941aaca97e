"""The f16x2 chained hidden layers with the activation tile resident in shared memory (csrc/gemm_planes.cu: gemm_chain_resident_kernel),
in both input modes, against per-layer morl_gemm_planes_f32 launches: every stored activation plane and every ReLU bit mask must be
BIT-identical (the MMAs run in the same order)."""

import pytest
import torch as th

pytestmark = pytest.mark.gpu

H = 256


@pytest.fixture(scope="module")
def cuda():
    if not th.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return th.device("cuda:0")


def _weights(ops, g, cuda, n_layers, k_first=H):
    ws, bs, sws = [], [], []
    for l in range(n_layers):
        k = k_first if l == 0 else H
        w = th.randn(H, k, device=cuda, generator=g) / 16.0
        sw = ops.scale_tensor(2048.0 * (1 + l), cuda)
        ws.append(ops.split_planes(w, ops.FMT_F16X2, rows_pad=H, ldp=k, scale=sw))
        sws.append(sw)
        bs.append(th.randn(H, device=cuda, generator=g) * 0.1)
    return ws, bs, sws


def _per_layer(ops, a, ws, bs, sws, sa, M):
    acts, bits = [], []
    for l in range(len(ws)):
        bt = ops.empty_relu_bits(M, a.device).zero_()
        _, a = ops.gemm_planes(a, ws[l], H, bias=bs[l], relu=True, out_f32=False, out_planes=True, a_scale=sa, b_scale=sws[l], c_scale=sa, relu_bits_out=bt)
        acts.append(a)
        bits.append(bt)
    return acts, bits


@pytest.mark.parametrize("n_chains,B,W,n_layers", [(2, 1024, 64, 3), (1, 1024, 64, 3), (2, 21, 48, 3), (1, 37, 48, 2), (2, 100, 48, 4), (1, 8, 32, 4)])
def test_pair_chain_equals_pairs_split_and_per_layer_launches(cuda, n_chains, B, W, n_layers):
    """Pair mode (morl_gemm_chain_pairs_f32) against pairs_relu_split + one launch per layer: the bench shape (B W = 65,536, one and two
    chains), ragged row counts with W not dividing 128, 2 and 4 layers.  Stored outputs: every layer, and the last one only (the no-grad
    pass), where the other output buffers must stay untouched."""
    from morl_baselines_b200 import ops

    M = B * W
    g = th.Generator(device=cuda).manual_seed(M + n_chains + n_layers)
    sa = ops.scale_tensor(2.0, cuda)
    chains = []
    for c in range(n_chains):
        u = th.randn(B, H, device=cuda, generator=g)
        v = th.randn(W, H, device=cuda, generator=g) * 0.5
        chains.append((u, v) + _weights(ops, g, cuda, n_layers))
    refs = []
    for u, v, ws, bs, sws in chains:
        h0 = ops.pairs_relu_split(u, v, scale=sa)
        refs.append(_per_layer(ops, h0, ws, bs, sws, sa, M))
    for last_only in (False, True):
        outs = [[ops.empty_planes(ops.FMT_F16X2, M, H, cuda).fill_(7) for _ in range(n_layers)] for _ in range(n_chains)]
        obits = [[ops.empty_relu_bits(M, cuda).zero_() for _ in range(n_layers)] for _ in range(n_chains)]
        stored = [[o if (l == n_layers - 1 or not last_only) else None for l, o in enumerate(oc)] for oc in outs]
        chain = ops.GemmChainPairs(stored, [ch[2] for ch in chains], B, W, [ch[3] for ch in chains], [ch[4] for ch in chains], obits, act_scale=sa)
        for _ in range(2):
            chain([ch[0] for ch in chains], [ch[1] for ch in chains])
        th.cuda.synchronize()
        for c in range(n_chains):
            for l in range(n_layers):
                if stored[c][l] is None:
                    assert bool((outs[c][l] == 7).all()), f"unstored output written: chain {c} layer {l}"
                else:
                    assert th.equal(outs[c][l].view(th.int16), refs[c][0][l].view(th.int16)), f"planes differ: chain {c} layer {l}"
                assert th.equal(obits[c][l], refs[c][1][l]), f"ReLU bits differ: chain {c} layer {l}"


@pytest.mark.parametrize("M,n_layers", [(1000, 3), (65536, 2)])
def test_dx_chain_with_k_first_32_and_bits_in(cuda, M, n_layers):
    """Planes mode with a 32-wide first reduction (one K block of the resident kernel) and ReLU-backward masks, no ReLU: against per-layer
    launches on the input zero-padded to 64 columns (the extra products are exact zeros)."""
    from morl_baselines_b200 import ops

    g = th.Generator(device=cuda).manual_seed(M + n_layers)
    sg = ops.scale_tensor(4.0, cuda)
    x = th.randn(M, 32, device=cuda, generator=g)
    a0 = ops.split_planes(x, ops.FMT_F16X2, rows_pad=M, ldp=32, scale=sg)
    a0_pad = ops.split_planes(th.nn.functional.pad(x, (0, 32)), ops.FMT_F16X2, rows_pad=M, ldp=64, scale=sg)
    ws, _, sws = _weights(ops, g, cuda, n_layers)
    w0 = th.randn(H, 32, device=cuda, generator=g) / 16.0
    ws[0] = ops.split_planes(w0, ops.FMT_F16X2, rows_pad=H, ldp=32, scale=sws[0])
    w0p = ops.split_planes(th.nn.functional.pad(w0, (0, 32)), ops.FMT_F16X2, rows_pad=H, ldp=64, scale=sws[0])
    bits_in = [th.randint(-2 ** 31, 2 ** 31 - 1, (M, 8), device=cuda, dtype=th.int32, generator=g) for _ in range(n_layers)]
    ref, a = [], a0_pad
    for l in range(n_layers):
        _, a = ops.gemm_planes(a, w0p if l == 0 else ws[l], H, relu_bits_in=bits_in[l], out_f32=False, out_planes=True, a_scale=sg, b_scale=sws[l],
                               c_scale=sg)
        ref.append(a)
    outs = [ops.empty_planes(ops.FMT_F16X2, M, H, cuda).zero_() for _ in range(n_layers)]
    chain = ops.GemmChain([[a0] + outs], [ws], None, [sws], None, act_scale=sg, relu=False, bits_in=[bits_in], k_first=32)
    chain()
    th.cuda.synchronize()
    for l in range(n_layers):
        assert th.equal(outs[l].view(th.int16), ref[l].view(th.int16)), f"planes differ: layer {l}"


def test_overflowing_pair_input_raises_the_flag(cuda):
    """A pair input beyond the fp16 range (|s x| > 65,504) is counted by morl_plane_overflow_count, as pairs_relu_split counts it."""
    from morl_baselines_b200 import ops

    B, W = 64, 8
    g = th.Generator(device=cuda).manual_seed(3)
    sa = ops.scale_tensor(2.0, cuda)
    u = th.randn(B, H, device=cuda, generator=g)
    u[5, 17] = 1e6
    v = th.randn(W, H, device=cuda, generator=g)
    ws, bs, sws = _weights(ops, g, cuda, 2)
    out = ops.empty_planes(ops.FMT_F16X2, B * W, H, cuda)
    ops.plane_overflow_count(reset=True)
    ops.GemmChainPairs([[None, out]], [ws], B, W, [bs], [sws], act_scale=sa)([u], [v])
    assert ops.plane_overflow_count(reset=True) > 0
