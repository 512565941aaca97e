"""Per-role cycle accounting of the K-major split-operand GEMM (MORL_GEMM_STATS=1): where does the MMA thread wait?
usage: gemm_stats.py [f16x2|bf16x3]"""
import ctypes, os, sys
os.environ["MORL_GEMM_STATS"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch as th
from morl_baselines_b200 import ops, _lib
dev = th.device("cuda:0")
g = th.Generator(device=dev).manual_seed(0)
M, N, K = 65536, 256, 256
lib = _lib.load()
fmt = ops.FMT_BF16X3 if (len(sys.argv) > 1 and sys.argv[1] == "bf16x3") else ops.FMT_F16X2
sa = ops.scale_tensor(8.0, dev) if fmt == ops.FMT_F16X2 else None
sb = ops.scale_tensor(2048.0, dev) if fmt == ops.FMT_F16X2 else None
bp = ops.split_planes(th.randn(N, K, device=dev, generator=g) / 16, fmt, scale=sb)
bias = th.randn(N, device=dev, generator=g)
sets = [ops.split_planes(th.randn(M, K, device=dev, generator=g).relu_(), fmt, scale=sa) for _ in range(3)]
outs = [th.empty_like(sets[0]) for _ in range(3)]
def run(n):
    for i in range(n):
        ops.gemm_planes(sets[i % 3], bp, N, bias=bias, relu=True, out_f32=False, out_planes=True, c_planes=outs[i % 3], a_scale=sa, b_scale=sb, c_scale=sa)
run(6)
buf = (ctypes.c_ulonglong * 8)()
lib.morl_debug_gemm_stats(buf, 1)
n = 30
e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
e0.record(); run(n); e1.record(); th.cuda.synchronize()
lib.morl_debug_gemm_stats(buf, 1)
us = e0.elapsed_time(e1) / n * 1e3
sm = ops.sm_count()
ctas = min(sm, (M + 127) // 128)
tiles = (M + 127) // 128 / ctas  # tiles per CTA and launch
# GemmArgs::stats: [0] consumer cycles waiting for TMA, [1] consumer loop total, [2] producer waiting for a free stage, [3] epilogue busy;
# [0], [1], [3] are written by consumer warp 0 of every CTA, [2] by the producer thread
wait_tma, total, wait_free, epi = (float(buf[i]) / ctas / n for i in range(4))
print(f"format {'bf16x3' if fmt == ops.FMT_BF16X3 else 'f16x2'}, accumulators {'split' if os.environ.get('MORL_GEMM_SPLIT_ACC') == '1' else 'single'}, "
      f"{th.cuda.get_device_name(0)}")
print(f"launch {us:.1f} us on {ctas} CTAs, {tiles:.2f} tiles per CTA (the counters add a little overhead)")
print(f"consumer warp (per CTA, per launch): total {total:.0f} cyc = {total / tiles:.0f} per tile; waiting for TMA {wait_tma:.0f} = {wait_tma / tiles:.0f} per tile "
      f"({wait_tma / total:.2f}); epilogue busy {epi:.0f} = {epi / tiles:.0f} per tile ({epi / total:.2f}); "
      f"issuing / waiting for MMAs {(total - wait_tma - epi) / tiles:.0f} per tile ({(total - wait_tma - epi) / total:.2f})")
print(f"producer thread (per CTA, per launch): waiting for a free stage {wait_free:.0f} cyc = {wait_free / tiles:.0f} per tile ({wait_free / total:.2f} of the consumer total)")
