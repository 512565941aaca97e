"""A/B of the three envelope-TD paths (MORL_ENVELOPE_PATH = v1 | v3 | tc): bit-exact agreement on a sweep of shapes and value
patterns, then CUDA-event timing at the north-star shape on 16 rotating input sets (> L2).  Development aid, not the bench."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch as th

from morl_baselines_b200 import ops

dev = th.device("cuda:0")


def run(path, *a, **k):
    os.environ["MORL_ENVELOPE_PATH"] = path
    try:
        return ops.envelope_td(*a, **k)
    finally:
        os.environ.pop("MORL_ENVELOPE_PATH", None)


def make(B, W, A, D, kind, seed):
    g = th.Generator(device=dev).manual_seed(seed)
    if kind == "ties":
        q_on = th.randint(-2, 3, (B, W, A, D), device=dev, generator=g).float()
        wset = th.randint(1, 4, (W, D), device=dev, generator=g).float() / 8.0
    elif kind == "neartie":
        q_on = th.randn(B, W, A, D, device=dev, generator=g)
        q_on = q_on[:, :1].repeat(1, W, 1, 1) * (1.0 + 1e-7 * th.randn(B, W, A, D, device=dev, generator=g))
        wset = th.rand(W, D, device=dev, generator=g)
    elif kind == "signed":
        q_on = th.randn(B, W, A, D, device=dev, generator=g) * 100.0
        wset = th.randn(W, D, device=dev, generator=g)
    elif kind == "special":
        q_on = th.randn(B, W, A, D, device=dev, generator=g)
        q_on[0].fill_(float("nan"))
        if B > 1:
            q_on[1, 0, 0, 0] = float("inf")
        if B > 2:
            q_on[2].fill_(-float("inf"))
        if B > 3:
            q_on[3].fill_(0.0)
        if B > 4:
            q_on[4] *= 1e38
        if B > 5:
            q_on[5] *= 1e-38
        wset = th.rand(W, D, device=dev, generator=g)
    else:
        q_on = th.randn(B, W, A, D, device=dev, generator=g) * 3.0
        wset = th.rand(W, D, device=dev, generator=g)
        wset = wset / wset.sum(1, keepdim=True)
    q_tg = q_on + 0.05 * th.randn(B, W, A, D, device=dev, generator=g)
    rew = th.randn(B, D, device=dev, generator=g)
    done = (th.rand(B, device=dev, generator=g) < 0.1).float()
    return q_on, q_tg, wset, rew, done


def same(a, b):
    return bool((a.view(th.int32) == b.view(th.int32)).all()) if a.dtype == th.float32 else bool((a == b).all())


bad = 0
shapes = [(1024, 64, 8, 3), (256, 32, 6, 3), (64, 8, 8, 3), (96, 16, 4, 2), (128, 16, 8, 3), (33, 50, 8, 3), (7, 64, 8, 1), (300, 2, 8, 3),
          (17, 64, 4, 2), (5, 16, 1, 3), (1, 64, 8, 3), (600, 62, 8, 3)]
for shape in shapes:
    for kind in ["plain", "ties", "neartie", "signed", "special"]:
        for mode in (ops.DOT_UNFUSED, ops.DOT_FMA, ops.DOT_PAIRFMA):
            for order in (ops.ROWS_BMAJOR, ops.ROWS_REFERENCE):
                if (mode != ops.DOT_UNFUSED or order != ops.ROWS_BMAJOR) and kind not in ("plain", "ties"):
                    continue
                inp = make(*shape, kind, seed=sum(shape) + len(kind))
                ref = run("v1", *inp, 0.99, mode, order)
                for path in (["tc", "wp"] if shape[1] > 32 else ["tc"]):
                    got = run(path, *inp, 0.99, mode, order)
                    th.cuda.synchronize()
                    ok = all(same(r, g) for r, g in zip(ref, got))
                    if not ok:
                        bad += 1
                        nt = int((ref[0].view(th.int32) != got[0].view(th.int32)).any(1).sum())
                        np_ = int((ref[1] != got[1]).sum())
                        na = int((ref[2] != got[2]).sum())
                        print(f"MISMATCH path={path} shape={shape} kind={kind} mode={mode} order={order}: target rows {nt}, pref {np_}, act {na} of {ref[1].numel()}", flush=True)
print("agreement sweep:", "OK" if bad == 0 else f"{bad} FAILED", flush=True)

# ---- timing at the north-star shape ----
# 16 rotating input sets (> L2).  Two clocks: a python launch loop (includes the host's per-call cost: ctypes + checks, which can
# exceed the kernel) and a CUDA-graph replay of the same 16 launches (back-to-back GPU time, what the update's graph sees).
def timed(path, B, W, A, D, sets, out):
    os.environ["MORL_ENVELOPE_PATH"] = path
    call = lambda i: ops.envelope_td(*sets[i % 16], 0.99, ops.DOT_UNFUSED, ops.ROWS_BMAJOR, want_indices=False, out=out)
    for i in range(32):
        call(i)
    th.cuda.synchronize()
    e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(400):
        call(i)
    e1.record()
    th.cuda.synchronize()
    t_loop = e0.elapsed_time(e1) * 1e-3 / 400
    side = th.cuda.Stream()
    side.wait_stream(th.cuda.current_stream())
    with th.cuda.stream(side):
        for i in range(16):
            call(i)
    th.cuda.current_stream().wait_stream(side)
    g = th.cuda.CUDAGraph()
    with th.cuda.graph(g):
        for i in range(16):
            call(i)
    for _ in range(3):
        g.replay()
    th.cuda.synchronize()
    e0.record()
    for _ in range(25):
        g.replay()
    e1.record()
    th.cuda.synchronize()
    os.environ.pop("MORL_ENVELOPE_PATH", None)
    return t_loop, e0.elapsed_time(e1) * 1e-3 / 400


for (B, W, A, D) in [(1024, 64, 8, 3), (132, 64, 8, 3), (2048, 64, 8, 3)]:
    sets = [make(B, W, A, D, "plain", 100 + i) for i in range(16)]
    out = th.empty(W * B, D, device=dev)
    alg = 2 * B * W * A * D * 4 + W * D * 4 + B * D * 4 + B * 4 + W * B * D * 4
    for path in ["v3", "wp", "tc", "v3", "wp"]:
        t_loop, t_graph = timed(path, B, W, A, D, sets, out)
        print(f"B={B} path {path}: python loop {t_loop * 1e6:.2f} us/launch, graph replay {t_graph * 1e6:.2f} us/launch = {alg / t_graph / 1e9:.0f} GB/s algorithmic",
              flush=True)
