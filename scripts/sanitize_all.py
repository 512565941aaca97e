"""Small launches of EVERY kernel of libmorl_b200.so for compute-sanitizer (SURVEY.md section 5):

    compute-sanitizer --tool memcheck|racecheck|synccheck|initcheck python scripts/sanitize_all.py [group ...]

groups: envelope td gemm optim pareto replay layer1 qhead dyna chain corners ppo pcn eupg nl_ppo hv_batch pql moq (default: all; dyna includes the fused Dyna commit).  Shapes are small (sanitizer slows kernels 10-100x) but exercise
every code path: all envelope kernel families, both GEMM operand formats x CTA modes x accumulator modes, MN split-K GEMM with the fused
column sums, every split / reduction helper, the loss kernels (discrete SAC's included), Adam, polyak, Pareto + front records, replay gather,
the corner-weight enumeration, MO-PPO's vector GAE and loss (racecheck: the loss kernel's CTA reductions), PCN's update and forward,
EUPG's returns, update and probabilities."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch as th

from morl_baselines_b200 import ops

dev = th.device("cuda:0")
g = th.Generator(device=dev).manual_seed(0)
if os.environ.get("SAN_ZERO_PLANES") == "1":
    # initcheck does not see the writes of TMA bulk tensor STORES (cp.async.bulk.tensor ... global.shared::cta): plane tensors produced
    # by the GEMM epilogue then look uninitialised to later readers.  Pre-zeroing every plane allocation separates that tool artefact
    # from a genuine read of memory nobody wrote.
    _empty = ops.empty_planes
    ops.empty_planes = lambda *a, **k: _empty(*a, **k).zero_()
groups = set(sys.argv[1:]) or {"envelope", "td", "gemm", "optim", "pareto", "replay", "layer1", "qhead", "dyna", "chain", "corners", "ppo", "pcn", "eupg", "nl_ppo", "hv_batch", "pql", "moq"}


def rn(*s, scale=1.0):
    return th.randn(*s, device=dev, generator=g) * scale


if "envelope" in groups:
    for (B, W, A, D) in [(40, 64, 8, 3), (9, 48, 4, 2)]:
        q_on, q_tg, wset, rew, done = rn(B, W, A, D), rn(B, W, A, D), th.rand(W, D, device=dev, generator=g), rn(B, D), th.zeros(B, device=dev)
        ref = None
        for path in ("v1", "v3", "wp"):
            if path == "wp" and W <= 32:
                continue
            os.environ["MORL_ENVELOPE_PATH"] = path
            out = ops.envelope_td(q_on, q_tg, wset, rew, done, 0.99)
            th.cuda.synchronize()
            ref = ref or out
            assert all(th.equal(a, b) for a, b in zip(ref, out)), path
        os.environ.pop("MORL_ENVELOPE_PATH", None)
    print("envelope ok")

if "td" in groups:
    B, W, A, D = 24, 8, 4, 3
    q = rn(B * W, A, D)
    ops.greedy_td(q, rn(B * W, A, D), th.rand(W, D, device=dev, generator=g), rn(B, D), th.zeros(B, device=dev), 0.99, ops.DOT_UNFUSED, ops.MAP_TILE, ops.MAP_BLOCK)
    act = th.randint(0, A, (B,), device=dev, generator=g, dtype=th.int32)
    lam = th.full((1,), 0.3, device=dev)
    ops.td_mse_priority(q, act, rn(B * W, D), th.rand(W, D, device=dev, generator=g), 0.0, B, W, ops.ROWS_BMAJOR, lambda_dev=lam)
    qn = rn(2, B, A, D)
    ops.critic_min_td(qn, th.rand(B, D, device=dev, generator=g), rn(B, D), th.zeros(B, device=dev), 0.99)
    ops.gpi_envelope(rn(2, B, 5, A, D), th.rand(B, D, device=dev, generator=g))
    act2 = th.randint(0, A, (B // 2,), device=dev, generator=g, dtype=th.int32)
    ops.td_huber_priority(rn(2, B, A, D, scale=0.02), act2, rn(B, D, scale=0.02), rn(B, D, scale=0.02), th.rand(B, D, device=dev, generator=g), 0.01, B // 2)
    ops.actor_critic_td(rn(2, B, D), th.rand(D, device=dev, generator=g), rn(B, D), th.zeros(B, 1, device=dev), rn(B, 1), 0.2, 0.99, ops.AC_SCALAR_MIN)
    alpha, log_alpha = th.full((1,), 0.2, device=dev), th.full((1,), -0.5, device=dev)
    for n_nets, Nd, Ad in [(2, 300, 6), (1, 40, 256)]:  # two blocks with a ragged tail; the widest action count
        qd, ld, wd = rn(n_nets, Nd, Ad, D), rn(Nd, Ad), th.rand(D, device=dev, generator=g)
        ops.discrete_sac_target(qd, ld, wd, rn(Nd, D), th.zeros(Nd, device=dev), alpha, 0.99)
        ops.discrete_sac_actor_loss(ld, qd, wd, alpha, log_alpha, 0.9)
    th.cuda.synchronize()
    print("td ok")

if "gemm" in groups:
    for fmt in (ops.FMT_F16X2, ops.FMT_BF16X3):
        sa = ops.scale_tensor(8.0, dev) if fmt == ops.FMT_F16X2 else None
        sw = ops.scale_tensor(512.0, dev) if fmt == ops.FMT_F16X2 else None
        for M in (100, 700):  # 1-CTA kernel / CTA-pair kernel with a ragged last tile
            a, b, bias = rn(M, 128), rn(64, 128, scale=1 / 8), rn(64)
            ap, bp = ops.split_planes(a, fmt, scale=sa), ops.split_planes(b, fmt, scale=sw)
            for split in (True, False):
                bits = ops.empty_relu_bits(M, dev)
                c, cp = ops.gemm_planes(ap, bp, 64, bias=bias, relu=True, out_f32=True, out_planes=True, a_scale=sa, b_scale=sw, c_scale=sa, split_acc=split,
                                        relu_bits_out=bits)
                ops.gemm_planes(ap, bp, 64, relu_bits_in=bits, out_f32=True, a_scale=sa, b_scale=sw, split_acc=split, reverse_tiles=True)
                ref = (a.double() @ b.double().t() + bias.double()).clamp_min(0)
                assert float((c.double() - ref).abs().max()) < 1e-4
                # the planes the TMA bulk store wrote hold the same values as the fp32 output of the same call: they WERE written, whatever
                # initcheck reports about later reads of them (it does not track cp.async.bulk.tensor stores; see DESIGN 5b)
                back = sum(cp[i].double() for i in range(cp.shape[0])) / (8.0 if sa is not None else 1.0)
                assert float((back - c.double()).abs().max()) <= 2.0**-20 * float(c.abs().max())
                assert bool(th.equal(ops.unpack_relu_bits(bits, 64), c > 0))
        G, H = rn(600, 24, scale=1e-3), rn(600, 128).relu_()
        sg = ops.scale_tensor(2.0**16, dev) if fmt == ops.FMT_F16X2 else None
        Gp, Hp = ops.split_planes(G, fmt, ldp=64, scale=sg), ops.split_planes(H, fmt, scale=sa)
        cs = th.empty(24, device=dev)
        dW = ops.gemm_planes_mn(Gp, 24, Hp, 128, colsum=cs, g_scale=sg, h_scale=sa)
        assert float((dW.double() - G.double().t() @ H.double()).abs().max()) < 1e-4
        ops.pairs_grad_reduce(ops.split_planes(rn(6 * 5, 64), fmt, scale=sa), 6, 5, scale=sa)
        ops.pairs_grad_reduce(ops.split_planes(rn(3 * 70, 64), fmt, scale=sa), 3, 70, scale=sa)
        ops.pairs_relu_split(rn(6, 64), rn(5, 64), fmt=fmt, scale=sa, relu_bits_out=ops.empty_relu_bits(30, dev))
        w1, w2 = rn(64, 64, scale=0.1), rn(24, 64)
        o = [ops.empty_planes(fmt, 64, 64, dev), ops.empty_planes(fmt, 64, 64, dev), ops.empty_planes(fmt, 32, 64, dev)]
        s1, s2 = ops.scale_tensor(1.0, dev), ops.scale_tensor(1.0, dev)
        te = 14 if fmt == ops.FMT_F16X2 else None
        ops.split_planes_multi([(w1, o[0], False, s1, te), (w1, o[1], True, s1, te), (w2, o[2], False, s2, te)], fmt)
        ops.split_planes(rn(50, 13), fmt, ldp=32, scale=sa)
    out, ws = th.zeros(1, device=dev), th.zeros(2, device=dev, dtype=th.int32)
    ops.amax_scale(rn(5000, scale=1e-5), 9, out, ws)
    th.cuda.synchronize()
    assert ops.plane_overflow_count() == 0
    print("gemm ok")

if "layer1" in groups:
    feats, wset, W1, b1 = rn(37, 11), th.rand(5, 2, device=dev, generator=g), rn(64, 13), rn(64)
    u, v = ops.pair_layer1_uv(feats, wset, W1, b1)
    ops.pair_layer1_grad(rn(37, 64), rn(5, 64), feats, wset)
    th.cuda.synchronize()
    print("layer1 ok")

if "optim" in groups:
    from morl_baselines_b200.common.fused_adam import FusedClipAdam

    ps = [th.nn.Parameter(rn(64, 35)), th.nn.Parameter(rn(64))]
    opt = FusedClipAdam(ps, lr=1e-3)
    for _ in range(2):
        for p in ps:
            p.grad = th.randn_like(p)
        opt.step_fused(1.0)
    ts = [rn(64, 35), rn(64)]
    ops.PolyakPlan([p.data for p in ps], ts).run(0.5)
    th.cuda.synchronize()
    print("optim ok")

if "pareto" in groups:
    pts = th.randn(700, 3, device=dev, generator=g, dtype=th.float64)
    keep = ops.pareto_mask(pts, True, raw=True)
    ops.pareto_mask(pts.float(), False)
    rec = th.empty(1 + 64 * 3 + 2, dtype=th.float64, device=dev)
    ops.front_pack(pts, keep, 64, rec, th.ones(2, dtype=th.float64, device=dev))
    gathered = th.stack([rec, rec]).contiguous()
    ops.front_unpack(gathered, 2, 3, 64, 2, th.empty(128, 3, dtype=th.float64, device=dev), th.empty(2, 3, dtype=th.float64, device=dev))
    th.cuda.synchronize()
    print("pareto ok")

if "replay" in groups:
    N, B = 300, 32
    obs, nobs = rn(N, 7), rn(N, 7)
    act = th.randint(0, 4, (N, 1), device=dev, generator=g, dtype=th.uint8)
    rew, done = rn(N, 3), th.zeros(N, 1, device=dev)
    idx = th.randint(0, N, (B,), device=dev, generator=g)
    ops.replay_gather(obs, nobs, act, rew, done, idx)
    th.cuda.synchronize()
    print("replay ok")
if "qhead" in groups:
    # fused output layers + envelope + Bellman (csrc/qhead_envelope.cu): several tiles per CTA are not needed for the protocol (ring and
    # accumulator phases wrap within 5 tiles of one CTA when the grid is capped) -- MORL has no grid cap switch, so a shape with more tiles
    # than SMs (B*W/128 = 160) exercises the wrap, and a W = 32 shape the four-transitions-per-tile path with ragged N = 18 rows
    for (B, W, A, D, K) in [(320, 64, 8, 3, 64), (24, 32, 6, 3, 128)]:
        M, N = B * W, A * D
        s_a, s_w = ops.scale_tensor(2.0, dev), ops.scale_tensor(1024.0, dev)
        a_on = ops.split_planes(rn(M, K).relu_(), ops.FMT_F16X2, rows_pad=M, ldp=K, scale=s_a)
        a_tg = ops.split_planes(rn(M, K).relu_(), ops.FMT_F16X2, rows_pad=M, ldp=K, scale=s_a)
        p_on = ops.split_planes(rn(N, K, scale=0.1), ops.FMT_F16X2, rows_pad=32, ldp=K, scale=s_w)
        p_tg = ops.split_planes(rn(N, K, scale=0.1), ops.FMT_F16X2, rows_pad=32, ldp=K, scale=s_w)
        b_on, b_tg, wset, rew, done = rn(N), rn(N), th.rand(W, D, device=dev, generator=g), rn(B, D), th.zeros(B, device=dev)
        q1, _ = ops.gemm_planes(a_on, p_on, N, bias=b_on, a_scale=s_a, b_scale=s_w)
        q2, _ = ops.gemm_planes(a_tg, p_tg, N, bias=b_tg, a_scale=s_a, b_scale=s_w)
        ref = ops.envelope_td(q1.view(B, W, A, D), q2.view(B, W, A, D), wset, rew, done, 0.99)
        qo, qt = th.zeros(M, N, device=dev), th.zeros(M, N, device=dev)
        out = ops.qhead_envelope_td(a_on, a_tg, p_on, p_tg, b_on, b_tg, wset, rew, done, 0.99, B, W, A, D, a_scale_on=s_a, a_scale_tg=s_a, w_scale_on=s_w,
                                    w_scale_tg=s_w, want_indices=True, q_on_out=qo, q_tg_out=qt)
        th.cuda.synchronize()
        assert th.equal(qo, q1) and th.equal(qt, q2) and all(th.equal(x, y) for x, y in zip(out, ref)), (B, W, A, D, K)
    print("qhead ok")

if "dyna" in groups:
    E, N, O = 5, 77, 35
    raw = rn(E, N, 2 * O, scale=3.0)
    idx = th.randint(0, E, (N,), device=dev, generator=g, dtype=th.int32)
    smp, var, unc = ops.ensemble_sample(raw, th.zeros(O, device=dev), th.full((O,), -5.0, device=dev), idx, rn(E, N, O), rn(N, O - 3), 3)
    th.cuda.synchronize()
    assert bool(th.isfinite(smp).all()) and bool((var > 0).all()) and bool((unc > 0).all())
    # fused commit: N = 77 leaves a partial last tile, ptr near the end of a 50-slot ring with every row kept wraps it; every rule
    S, A, cap = O - 3, 4, 50
    stores = tuple(th.zeros(cap, c, device=dev) for c in (S, S, A, 3, 1))
    na, unc_c, counts = th.empty(N, S, device=dev), th.empty(N, device=dev), th.empty(2, dtype=th.int32, device=dev)
    obs_c, act_c = rn(N, S), rn(N, A)
    for rule in (ops.TERM_NONE, ops.TERM_HOPPER, ops.TERM_HUMANOID, ops.TERM_MOUNTAINCAR, ops.TERM_LUNARLANDER):
        for thr in (1e30, float(unc.median())):
            ops.dyna_commit(raw, th.zeros(O, device=dev), th.full((O,), -5.0, device=dev), idx, rn(E, N, O), obs_c, act_c, 3, rule, thr, stores, cap - 3,
                            na, unc_c, counts)
    th.cuda.synchronize()
    assert int(counts[0]) == int((unc_c < thr).sum()) and 0 <= int(counts[1]) <= N
    print("dyna ok")
if "chain" in groups:
    # chained hidden layers (gemm_chain_kernel): 2 chains x 2 layers on 5 tiles (groups of 2 + a ragged last group), then a 1-chain dX chain with masks
    M, H = 1200, 256
    sa, sw = ops.scale_tensor(2.0, dev), ops.scale_tensor(1024.0, dev)
    acts, ws, bs, sws, bits = [], [], [], [], []
    for c in range(2):
        acts.append([ops.split_planes(rn(M, H).relu_(), ops.FMT_F16X2, rows_pad=M, ldp=H, scale=sa)] + [ops.empty_planes(ops.FMT_F16X2, M, H, dev) for _ in range(2)])
        ws.append([ops.split_planes(rn(H, H, scale=0.06), ops.FMT_F16X2, rows_pad=H, ldp=H, scale=sw) for _ in range(2)])
        bs.append([rn(H, scale=0.1) for _ in range(2)])
        sws.append([sw, sw])
        bits.append([ops.empty_relu_bits(M, dev) for _ in range(2)])
    ops.GemmChain(acts, ws, bs, sws, bits, act_scale=sa)()
    for c in range(2):
        a = acts[c][0]
        for l in range(2):
            _, a = ops.gemm_planes(a, ws[c][l], H, bias=bs[c][l], relu=True, out_f32=False, out_planes=True, a_scale=sa, b_scale=sw, c_scale=sa)
            assert th.equal(a.view(th.int16), acts[c][l + 1].view(th.int16)), (c, l)
    gb = [acts[0][2]] + [ops.empty_planes(ops.FMT_F16X2, M, H, dev) for _ in range(2)]
    ops.GemmChain([gb], [ws[0]], None, [sws[0]], None, act_scale=sa, relu=False, bits_in=[bits[0]])()
    th.cuda.synchronize()
    print("chain ok")
if "corners" in groups:
    # corner-weight enumeration (csrc/linear_support.cu): every dimension template, a degenerate integer set, and a launch whose count
    # exceeds its buffer (the writes past cap must be skipped)
    for d, n in [(2, 7), (3, 9), (4, 6), (5, 5), (6, 4), (7, 3), (8, 3)]:
        V = th.randint(0, 3, (n, d), device=dev, generator=g).double()
        ops.corner_weights(V, cap=1)
    th.cuda.synchronize()
    print("corners ok")
if "ppo" in groups:
    # vector GAE (csrc/ppo.cu): more steps than one shared-memory chunk, env counts that leave a CTA partly idle, both modes; the loss:
    # more rows than threads, A at its limit, both value-loss forms, and a device learning rate for the Adam that follows it
    for T, E, D in [(130, 5, 3), (1, 1, 8), (64, 33, 1)]:
        for gae in (True, False):
            ops.vector_gae(rn(T, E, D), rn(T, E, D), (th.rand(T, E, device=dev, generator=g) < 0.1).float(), rn(E, D), th.ones(E, device=dev),
                           th.rand(D, device=dev, generator=g), 0.99, 0.95, gae)
    stats = th.zeros(6, device=dev)
    for M, A, D, cv in [(300, 32, 2, True), (2, 1, 1, False), (257, 6, 3, True)]:
        ops.ppo_loss(rn(M, A), rn(A, scale=0.3), rn(M, D), rn(M, A), rn(M), rn(M), rn(M, D), rn(M, D), 0.2, 0.01, 0.5, True, cv, stats)
    th.cuda.synchronize()
    print("ppo ok")
if "pcn" in groups:
    # PCN (csrc/pcn.cu): a ragged last tile, one row, the largest hidden width, both action kinds; the forward on device and pinned rows
    from morl_baselines_b200.multi_policy.pcn import pcn as pcn_mod

    for S, d, H, A, B, cont in [(7, 3, 64, 6, 37, False), (3, 8, 256, 32, 1, False), (11, 3, 32, 3, 20, True)]:
        m = (pcn_mod.ContinuousActionsDefaultModel if cont else pcn_mod.DiscreteActionsDefaultModel)(S, A, d, np.ones(d + 1, np.float32), H).to(dev)
        ts = pcn_mod.default_model_tensors(m)
        N, ld = 64, S + d + (A if cont else 1)
        store = rn(N, ld)
        if not cont:
            store[:, S + d] = th.randint(0, A, (N,), device=dev, generator=g).int().view(th.float32)
        rows, hor = th.randint(0, N, (B,), device=dev, generator=g).int(), th.randint(1, 50, (B,), device=dev, generator=g).int()
        stats, pred = th.zeros(2, device=dev), th.zeros(B, A, device=dev)
        ops.pcn_update(ops.pcn_pointer_table(ts), ops.pcn_pointer_table([th.empty_like(t) for t in ts]), m.scaling_factor, store, S, d, rows, hor,
                       B, H, A, cont, stats[0:1], stats[1:2], pred, ops.pcn_workspace(S, d, H, A, B, dev))
        out, am = th.zeros(B, A, device=dev), th.zeros(B, dtype=th.int32, device=dev)
        ops.pcn_forward(ops.pcn_pointer_table(ts), m.scaling_factor, rn(B, S), rn(B, d), th.ones(B, device=dev), H, not cont, out, am)
        pin_out = th.zeros(1, A).pin_memory()
        ops.pcn_forward(ops.pcn_pointer_table(ts), m.scaling_factor, th.ones(1, S).pin_memory(), th.ones(1, d).pin_memory(), th.ones(1).pin_memory(),
                        H, not cont, pin_out)
    th.cuda.synchronize()
    print("pcn ok")
if "eupg" in groups:
    # EUPG (csrc/eupg.cu): a ragged last tile, T = 1, a T that gives each CTA several tiles (> 128 * 16 rows), width 50 and 256, one
    # action, a scalar v; the returns kernel over several chunks; the probabilities on device and pinned rows
    from morl_baselines_b200.single_policy.esr.eupg import PolicyNet, policy_tensors

    for arch, S, d, A, T in [([50], 1, 2, 2, 37), ([50], 3, 2, 4, 1), ([256], 8, 3, 32, 5000), ([17, 5], 2, 2, 1, 20), ([256, 50, 3, 7], 4, 8, 5, 70)]:
        net = PolicyNet((S,), A, d, arch).to(dev)
        ts = policy_tensors(net)
        knet = ops.EupgNet(S, d, arch, A, ts, [th.empty_like(t) for t in ts])
        ld = S + 2 * d + 1
        block = rn(T, ld)
        block[:, :S] = th.randint(-3, 4, (T, S), device=dev, generator=g).int().view(th.float32)
        block[:, S + d] = th.randint(0, A, (T,), device=dev, generator=g).int().view(th.float32)
        fwd = ops.eupg_returns(block[:, S + d + 1:], 0.99)
        v = fwd.sum(1) if T > 1 else fwd.sum().reshape(())
        ops.eupg_update(knet, block[:, :S].view(th.int32), block[:, S:S + d], block[:, S + d].view(th.int32), v, th.zeros(1, device=dev),
                        knet.workspace(dev))
        out = th.zeros(7, A, device=dev)
        ops.eupg_probs(knet, rn(7, S + d), out)
        pin_out = th.zeros(1, A).pin_memory()
        ops.eupg_probs(knet, th.ones(1, S + d).pin_memory(), pin_out)
    th.cuda.synchronize()
    print("eupg ok")

if "nl_ppo" in groups:
    # non-linear MO-PPO (csrc/nl_ppo.cu, the objective GAE of csrc/ppo.cu): M = 2, a ragged last tile, M = 4096 (each CTA several tiles),
    # Dp 0 and d, K = 256, A = 32; the forward on device and pinned rows; one commit step
    from morl_baselines_b200 import nl_ppo_ops
    from morl_baselines_b200.single_policy.ser.nl_mo_ppo import Agent
    from tests.nl_ppo_standin import RingVecEnv

    for S, d, Dp, A, M in [(2, 2, 2, 4, 2), (7, 3, 0, 6, 37), (240, 8, 8, 32, 4096)]:
        ts = list(Agent(RingVecEnv(1, obs_dim=S, n_actions=A, d=d), d, Dp).to(dev).parameters())
        knet = nl_ppo_ops.NlPpoNet(S, d, Dp, A, ts, [th.empty_like(t) for t in ts], rn(Dp) if Dp else None)
        B = M + 5
        perm = th.randperm(B, device=dev)[:M].contiguous()
        nl_ppo_ops.nl_ppo_update(knet, rn(B, S), rn(B, d), th.randint(0, A, (B,), device=dev), rn(B), rn(B, d), rn(B, d), rn(B, d), perm, rn(d),
                                 0.2, 0.01, 0.5, True, True, th.zeros(6, device=dev), knet.workspace(dev))
        nl_ppo_ops.nl_ppo_forward(knet, rn(19, S), rn(19, d), th.zeros(19, A, device=dev), th.zeros(19, d, device=dev),
                                  th.zeros(19, dtype=th.int32, device=dev))
        nl_ppo_ops.nl_ppo_forward(knet, th.ones(1, S).pin_memory(), th.ones(1, d).pin_memory(), argmax_out=th.zeros(1, dtype=th.int32).pin_memory())
        T, E = 3, 5
        nl_ppo_ops.vector_gae_objectives(rn(T, E, d), rn(T, E, d), th.zeros(T, E, device=dev), rn(E, d), th.zeros(E, device=dev), 0.99, 0.95)
        nl_ppo_ops.nl_ppo_commit(rn(E, S + d + 2), rn(E, A), th.randint(0, A, (E,), device=dev), 1, 0.99, rn(T, E, S), rn(T, E, d), rn(T, E),
                                 rn(T, E, d), th.zeros(T, E, dtype=th.int64, device=dev), rn(T, E), rn(E, S), rn(E, d), th.zeros(E, device=dev),
                                 th.zeros(E, dtype=th.int32, device=dev))
    th.cuda.synchronize()
    print("nl_ppo ok")
if "hv_batch" in groups:
    # batched exact hypervolume (csrc/pareto.cu): every d, an empty base, base alone, one and several candidates, the d = 4 cap
    from morl_baselines_b200 import hv_ops

    for d, n_base, n_cand in [(1, 0, 3), (2, 17, 0), (3, 33, 5), (3, 2048, 1), (4, 9, 4), (4, 512, 1)]:
        base = th.rand(n_base, d, device=dev, dtype=th.float64, generator=g)
        cand = th.rand(n_cand, d, device=dev, dtype=th.float64, generator=g) if n_cand else None
        hv_ops.hypervolume_batch(base, cand, th.zeros(d, device=dev, dtype=th.float64))
    th.cuda.synchronize()
    print("hv_batch ok")
if "pql" in groups:
    # Pareto Q-learning's set table (csrc/pql.cu): an update with s' == s, one with an overflow, both score modes at d 2 and 4, cardinality
    # at d 8, the A = 16 range
    from morl_baselines_b200 import pql_ops

    for S, A, K, d in [(3, 4, 8, 2), (3, 16, 64, 4), (3, 2, 4, 8)]:
        t = pql_ops.PqlTable(S, A, K, d, dev)
        t.nd.copy_(th.rand(S, A, K, d, device=dev, dtype=th.float64, generator=g))
        t.nd_count.fill_(K)
        pql_ops.pql_update(t, 0, A - 1, 0, np.ones(d), 0.9)
        pql_ops.pql_update(t, 1, 0, 2, np.ones(d), 1.0)
        pql_ops.pql_score(t, 0, pql_ops.CARDINALITY, 0.9)
        if d <= 4:
            pql_ops.pql_score(t, 1, pql_ops.HYPERVOLUME, 0.9, np.zeros(d))
    th.cuda.synchronize()
    print("pql ok")
if "moq" in groups:
    # multi-policy MO Q-learning (csrc/moq.cu): GPI and own-policy rows with state -1, a prioritised step with 70 Dyna updates (two launches)
    # and s' == s, a uniform step
    from morl_baselines_b200 import moq_ops

    for A, d, prio in [(4, 2, True), (16, 8, False)]:
        t = moq_ops.MoqTable(A, d, dev, True, S=8, P=3, M=8, K=2)
        flags = moq_ops.GPI | moq_ops.MODEL | (moq_ops.PRIORITIZE if prio else 0)
        moq_ops.moq_step(t, 3, 1, 0, A - 1, 0, False, np.ones(d) / d, np.ones(d), flags, 0.9, 0.1, pair=0, outcome=1, n_pairs=1,
                         pick=[0] * 70, u=[0.5] * 70, choice=[0.3] * 70)
        moq_ops.moq_act(t, 3, [0, -1, 7], [-1, 0, 2], np.ones((3, d)))
    th.cuda.synchronize()
    print("moq ok")
print("sanitize run ok")
