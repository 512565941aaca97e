"""GPI-PD's no-grad policy-set evaluations on the tensor-core plan (tc_mlp.TCProductMlp) against the library-GEMM path, in one call.

    python scripts/bench_gpi_tc.py [--reps 20]

  * GPIPD._envelope_target at B = 1024 observations x |M| = 64 support weights (65,536 pair rows x 2 target nets);
  * GPIPD._reset_priorities over 65,536 stored transitions with |M| = 16 (q_nets[0] on the chunk + the envelope target);
    both with use_tensor_cores False and True, net_arch [256] * 4, drop_rate 0.01, layer_norm True (GPIPD's defaults, nets in train mode);
  * the hidden-layer GEMM alone at 65,536 x 256 x 256 (f16x2): ReLU only (morl_gemm_planes_f32) against LayerNorm and against LayerNorm +
    dropout (morl_gemm_planes_ln_f32): the cost of the epilogue.  Each configuration is 20 back-to-back launches captured in one CUDA graph
    (no host work between the kernels), timed per replay; --rounds rounds alternate the three configurations and the median, min and max of
    the per-launch time over the rounds are reported.
Pass times are CUDA events around each call, medians over --reps calls after warm-up.  The card's name and power limit are read in the same
call and printed with the numbers (one JSON object on stdout)."""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch as th


def event_ms(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    th.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else th.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bench_gpi_tc.py needs a CUDA device")
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.weights import equally_spaced_weights
    from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import GPIPD
    from morl_baselines_b200.testing import FakeEnv

    dev = th.device("cuda:0")
    out = {"card": card(), "torch": th.__version__}
    th.manual_seed(0)
    rng = np.random.default_rng(0)
    OBS, A, D, N = 8, 6, 3, 65536
    agents = {}
    for tc in (False, True):
        th.manual_seed(0)
        ag = GPIPD(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), net_arch=[256] * 4, drop_rate=0.01, layer_norm=True, dyna=False, per=True,
                   buffer_size=N, log=False, seed=0, device=dev, use_tensor_cores=tc)
        rb = ag.replay_buffer
        rb.obs[:] = rng.standard_normal((N, OBS)).astype(np.float32)
        rb.next_obs[:] = rng.standard_normal((N, OBS)).astype(np.float32)
        rb.actions[:] = rng.integers(0, A, (N, 1)).astype(rb.actions.dtype)
        rb.rewards[:] = rng.standard_normal((N, D)).astype(np.float32)
        rb.dones[:] = (rng.random((N, 1)) < 0.02).astype(np.float32)
        rb.size, rb.ptr = N, 0
        rb.mark_all_dirty()
        agents[tc] = ag
    w = th.tensor(equally_spaced_weights(D, 64)[7], device=dev, dtype=th.float32)
    obs = th.randn(1024, OBS, device=dev)
    for tc, ag in agents.items():
        name = "tensor_cores" if tc else "library"
        ag.set_weight_support(equally_spaced_weights(D, 64))
        M = ag._support_matrix()
        ms = event_ms(lambda: ag._envelope_target(obs, w.reshape(1, D), M), args.reps)
        out[f"_envelope_target B=1024 |M|=64 {name}"] = {"ms": ms, "pair_rows_per_s": 1024 * 64 * 2 / ms * 1e3}
        ag.set_weight_support(equally_spaced_weights(D, 16))
        ms = event_ms(lambda: ag._reset_priorities(w), max(3, args.reps // 4), warm=1)
        out[f"_reset_priorities N=65536 |M|=16 {name}"] = {"ms": ms}
    for what in ("_envelope_target B=1024 |M|=64", "_reset_priorities N=65536 |M|=16"):
        out[f"{what} speed-up"] = out[f"{what} library"]["ms"] / out[f"{what} tensor_cores"]["ms"]

    # the epilogue alone: 65,536 x 256 x 256, f16x2, planes out
    Mr, Nn, K = 65536, 256, 256
    x, wt = th.randn(Mr, K, device=dev), th.randn(Nn, K, device=dev) / 16
    b, gm, bt = th.randn(Nn, device=dev) * 0.1, 1 + 0.1 * th.randn(Nn, device=dev), 0.1 * th.randn(Nn, device=dev)
    sx, sw = ops.scale_tensor(2.0, dev), ops.scale_tensor(1024.0, dev)
    xp, wp = ops.split_planes(x, ops.FMT_F16X2, scale=sx), ops.split_planes(wt, ops.FMT_F16X2, scale=sw)
    cp = ops.empty_planes(ops.FMT_F16X2, Mr, Nn, dev)
    seed, off = th.tensor([1], dtype=th.int64, device=dev), th.zeros(1, dtype=th.int32, device=dev)
    flop = 2.0 * Mr * Nn * K
    gemm = {
        "relu": lambda: ops.gemm_planes(xp, wp, Nn, bias=b, relu=True, out_f32=False, out_planes=True, c_planes=cp, a_scale=sx, b_scale=sw, c_scale=sx),
        "layernorm": lambda: ops.gemm_planes_ln(xp, wp, Nn, bias=b, ln_weight=gm, ln_bias=bt, ln_eps=1e-5, c_planes=cp, a_scale=sx, b_scale=sw, c_scale=sx),
        "layernorm+dropout": lambda: ops.gemm_planes_ln(xp, wp, Nn, bias=b, ln_weight=gm, ln_bias=bt, ln_eps=1e-5, drop_p=0.01, drop_seed=seed,
                                                        drop_offset=off, c_planes=cp, a_scale=sx, b_scale=sw, c_scale=sx),
    }
    per_graph = 20
    graphs = {}
    for k, fn in gemm.items():
        side = th.cuda.Stream()
        side.wait_stream(th.cuda.current_stream())
        with th.cuda.stream(side):
            for _ in range(3):
                fn()
        th.cuda.current_stream().wait_stream(side)
        g = th.cuda.CUDAGraph()
        with th.cuda.graph(g):
            for _ in range(per_graph):
                fn()
        graphs[k] = g
    samples = {k: [] for k in gemm}
    for _ in range(args.rounds):
        for k, g in graphs.items():
            samples[k].append(event_ms(g.replay, 10, warm=2) * 1e3 / per_graph)
    for k, us in samples.items():
        med = float(np.median(us))
        out[f"gemm 65536x256x256 f16x2 {k}"] = {"us_per_launch_median": med, "us_min": float(min(us)), "us_max": float(max(us)),
                                                "fp32_equiv_tflops": flop / med / 1e6}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
