"""Quick probe of the wgmma split-operand GEMM on an H100: correctness on one shape + timing vs cuBLAS fp32 (CUDA events), both
operand formats.  Also a profiler target (`-k regex:gemm_planes`)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch as th
from morl_baselines_b200 import ops
dev = th.device("cuda:0")
g = th.Generator(device=dev).manual_seed(0)
M, N, K = 65536, 256, 256
a = th.randn(M, K, device=dev, generator=g).relu_(); b = th.randn(N, K, device=dev, generator=g) / 16; bias = th.randn(N, device=dev, generator=g)
def timeit(fn, n=20):
    for _ in range(3): fn()
    th.cuda.synchronize(); e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); th.cuda.synchronize(); return e0.elapsed_time(e1) / n * 1e3
fl = 2.0 * M * N * K
fmts = [(ops.FMT_F16X2, "f16x2", 3)] + ([(ops.FMT_BF16X3, "bf16x3", 6)] if "--all" in sys.argv else [])
for fmt, name, nprod in fmts:
    sa = ops.scale_tensor(8.0, dev) if fmt == ops.FMT_F16X2 else None
    sb = ops.scale_tensor(2048.0, dev) if fmt == ops.FMT_F16X2 else None
    ap, bp = ops.split_planes(a, fmt, scale=sa), ops.split_planes(b, fmt, scale=sb)
    c, cp = ops.gemm_planes(ap, bp, N, bias=bias, relu=True, out_f32=True, out_planes=True, a_scale=sa, b_scale=sb, c_scale=sa)
    th.cuda.synchronize()
    ref = (a[:4096].double() @ b.double().t() + bias.double()).clamp_min(0)
    print(name, "max abs err", float((c[:4096].double() - ref).abs().max()), "ref max", float(ref.abs().max()))
    t1 = timeit(lambda: ops.gemm_planes(ap, bp, N, bias=bias, relu=True, out_f32=False, out_planes=True, c_planes=cp, a_scale=sa, b_scale=sb, c_scale=sa))
    t2 = timeit(lambda: ops.gemm_planes(ap, bp, N, bias=bias, relu=True, out_f32=True, out_planes=False, c_f32=c, a_scale=sa, b_scale=sb))
    print(f"wgmma {name} -> planes: {t1:.1f} us ({nprod*fl/t1/1e6:.0f} TFLOP/s issued, {fl/t1/1e6:.1f} fp32-equivalent); -> f32: {t2:.1f} us")
t3 = timeit(lambda: th.relu(th.addmm(bias, a, b.t())))
print(f"cuBLAS fp32 addmm+relu: {t3:.1f} us")
