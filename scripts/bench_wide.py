"""Throughput of the Envelope update at the shapes the tensor-core path gained: 512-wide hidden layers and more than 64 weight vectors
per update (a measurement of its own; bench.py is untouched):

    python scripts/bench_wide.py [--steps 30] [--warmup 3] [--skip-validation]

Prints the card's name and power limit, then one line per configuration: Envelope.update() updates/s with the replay store and the
sum-tree on the device and the update captured in a CUDA graph (B = 1024, obs 32, |A| 8, d 3), for
    4x256 |W| 64 (bench.py's shape), 4x512 |W| 64, 4x256 |W| 128, 4x256 |W| 256,
through the tensor-core path and through the library-GEMM validation path (use_tensor_cores=False).  Each configuration runs in a
fresh subprocess (its own CUDA context; a validation run whose graph capture is refused is repeated without the graph and says so).
Then the per-launch time and issued tensor-core TFLOP/s of the per-layer K-major kernel at 65,536 x 512 x 512 (bias + ReLU + plane
re-split epilogue) and of the weight-gradient kernel at 65,536 rows with G and H 512 wide (bias gradient fused), both as 16 launches in
one CUDA graph between CUDA events, four rotating operand sets (> 50 MB L2).  Needs a GPU; changes no device setting; every child has
exited when it returns."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBS, A, D, B, STORE = 32, 8, 3, 1024, 65536
CONFIGS = [("4x256", [256] * 4, 64), ("4x512", [512] * 4, 64), ("4x256", [256] * 4, 128), ("4x256", [256] * 4, 256)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi query failed)"


def child_update(net, W, tc, graph, steps, warmup):
    """One configuration in this process: updates/s over `steps` updates after `warmup`."""
    import numpy as np
    import torch as th

    sys.path.insert(0, ROOT)
    from morl_baselines_b200.multi_policy.envelope.envelope import Envelope
    from morl_baselines_b200.testing import FakeEnv, synthetic_store

    dev = th.device("cuda", 0)
    np.random.seed(1000)
    th.manual_seed(1000)
    agent = Envelope(FakeEnv(obs_dim=OBS, n_actions=A, reward_dim=D), batch_size=B, num_sample_w=W, per=True, buffer_size=STORE, net_arch=net,
                     log=False, seed=0, device=dev, replay_on_device=True, use_cuda_graph=graph, use_tensor_cores=tc)
    store = synthetic_store(STORE, OBS, A, D, seed=0)
    rb = agent.replay_buffer
    rb.obs[:], rb.next_obs[:], rb.actions[:], rb.rewards[:], rb.dones[:] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
    rb.size, rb.ptr = STORE, 0
    rb.mark_all_dirty()
    rb.tree.batch_set(np.arange(STORE), np.full(STORE, rb.min_priority))
    rb.flush()
    agent.global_step = 1
    for _ in range(warmup):
        agent.update()
    th.cuda.synchronize()
    e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        agent.update()
    e1.record()
    th.cuda.synchronize()
    loss = float(agent.last_loss_host())
    return {"updates_per_s": steps / (e0.elapsed_time(e1) * 1e-3), "loss": loss, "finite": bool(np.isfinite(loss)),
            "fused_head": bool(getattr(agent, "fused_head_active", False))}


def _graph_time(launch, per_graph=16, replays=8):
    import torch as th

    side = th.cuda.Stream()
    side.wait_stream(th.cuda.current_stream())
    with th.cuda.stream(side):
        for i in range(8):
            launch(i)
    th.cuda.current_stream().wait_stream(side)
    graph = th.cuda.CUDAGraph()
    with th.cuda.graph(graph):
        for i in range(per_graph):
            launch(i)
    for _ in range(3):
        graph.replay()
    th.cuda.synchronize()
    e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        graph.replay()
    e1.record()
    th.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / (replays * per_graph)


def child_kernels():
    import torch as th

    sys.path.insert(0, ROOT)
    from morl_baselines_b200 import ops

    dev = th.device("cuda", 0)
    fmt, nprod = ops.FMT_F16X2, 3
    M, H = 65536, 512
    g = th.Generator(device=dev).manual_seed(2)
    sa, sw, sg = ops.scale_tensor(8.0, dev), ops.scale_tensor(2048.0, dev), ops.scale_tensor(2.0**20, dev)
    wp = ops.split_planes(th.randn(H, H, device=dev, generator=g) / 16.0, fmt, scale=sw)
    bias = th.randn(H, device=dev, generator=g) * 0.1
    a_sets = [ops.split_planes(th.randn(M, H, device=dev, generator=g).relu_(), fmt, scale=sa) for _ in range(4)]
    c_sets = [th.empty_like(a_sets[0]) for _ in range(4)]
    bits = [ops.empty_relu_bits(M, dev, H) for _ in range(4)]
    t_layer = _graph_time(lambda i: ops.gemm_planes(a_sets[i % 4], wp, H, bias=bias, relu=True, out_f32=False, out_planes=True, c_planes=c_sets[i % 4],
                                                   a_scale=sa, b_scale=sw, c_scale=sa, relu_bits_out=bits[i % 4]))
    g_sets = [ops.split_planes(th.randn(M, H, device=dev, generator=g) * 1e-4, fmt, scale=sg) for _ in range(4)]
    ws = ops.gemm_mn_workspace(M, H, H, dev)
    dW, db = th.empty(H, H, device=dev), th.empty(H, device=dev)
    t_mn = _graph_time(lambda i: ops.gemm_planes_mn(g_sets[i % 4], H, a_sets[i % 4], H, out=dW, workspace=ws, colsum=db, g_scale=sg, h_scale=sa))
    flops = nprod * 2 * M * H * H
    return {"layer_us": t_layer * 1e6, "layer_tflops": flops / t_layer * 1e-12, "mn_us": t_mn * 1e6, "mn_tflops": flops / t_mn * 1e-12}


def run_child(kind, **kw):
    code = (f"import json, sys; sys.path.insert(0, {ROOT!r}); sys.argv = ['bench_wide']; import runpy; "
            f"m = runpy.run_path({os.path.abspath(__file__)!r}); print('RESULT ' + json.dumps(m['child_{kind}'](**{kw!r})))")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    if r.returncode != 0 or not lines:
        return None, (r.stdout[-1500:] + r.stderr[-3000:])
    return json.loads(lines[-1][7:]), None


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-validation", action="store_true")
    args = ap.parse_args()
    import torch as th

    if not th.cuda.is_available():
        raise SystemExit("bench_wide.py measures on a GPU; no CUDA device is visible")
    print(f"# card: {card()} (name, power limit, max SM clock)", flush=True)
    print(f"# Envelope.update(): B {B}, obs {OBS}, |A| {A}, d {D}, PER with the store and sum-tree on the device, {args.steps} timed updates "
          f"after {args.warmup}", flush=True)
    rows = []
    for name, net, W in CONFIGS:
        tc, err = run_child("update", net=net, W=W, tc=True, graph=True, steps=args.steps, warmup=args.warmup)
        if tc is None:
            raise SystemExit(f"tensor-core update {name} |W| {W} failed:\n{err}")
        line = f"{name} |W| {W:3d}: tensor cores {tc['updates_per_s']:8.1f} updates/s (fused head {tc['fused_head']}, loss finite {tc['finite']})"
        val = None
        if not args.skip_validation:
            val, err = run_child("update", net=net, W=W, tc=False, graph=True, steps=max(3, args.steps // 3), warmup=args.warmup)
            how = "graph"
            if val is None:
                val, err2 = run_child("update", net=net, W=W, tc=False, graph=False, steps=max(3, args.steps // 3), warmup=args.warmup)
                how = "eager (graph capture refused)"
            if val is None:
                line += f" | validation path failed: {err2.strip().splitlines()[-1] if err2 else '?'}"
            else:
                line += f" | validation path ({how}) {val['updates_per_s']:7.1f} updates/s -> x{tc['updates_per_s'] / val['updates_per_s']:.2f}"
        print(line, flush=True)
        rows.append({"config": f"{name} |W| {W}", "tensor_cores": tc, "validation": val})
    k, err = run_child("kernels")
    if k is None:
        raise SystemExit(f"kernel timing failed:\n{err}")
    print(f"per-layer K-major kernel 65536 x 512 x 512 (f16x2, bias + ReLU + planes + bits): {k['layer_us']:.1f} us/launch, "
          f"{k['layer_tflops']:.0f} TFLOP/s issued", flush=True)
    print(f"weight-gradient kernel 65536 rows, G 512 x H 512 (f16x2, bias gradient fused, + reduction): {k['mn_us']:.1f} us/launch, "
          f"{k['mn_tflops']:.0f} TFLOP/s issued", flush=True)
    print(json.dumps({"card": card(), "updates": rows, "kernels": k}))


if __name__ == "__main__":
    main()
