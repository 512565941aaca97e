"""Error statistics of the tensor-core split-operand GEMMs against float64 on a north-star layer (65,536 x 256 x 256), next to cuBLAS fp32:
    bias  = mean of (c - ref) / (|A| . |B|^T)      (a systematic component: the tensor cores' fp32 accumulation TRUNCATES)
    rms   = rms of the same ratio
and the error of a whole 4 x 256 Q-network forward (TCPairMlp) against a float64 forward of the same parameters.
usage: gemm_error_probe.py [single|split]   (accumulator mode of the GEMMs and of the network's layers; default single)"""
import os
import sys

import torch as th

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from morl_baselines_b200 import ops  # noqa: E402
from morl_baselines_b200.tc_mlp import TCPairMlp  # noqa: E402

dev = th.device("cuda:0")
g = th.Generator(device=dev).manual_seed(0)
M, N, K = 65536, 256, 256
a = th.randn(M, K, device=dev, generator=g).relu_()
b = th.randn(N, K, device=dev, generator=g) / 16
ref = a.double() @ b.double().t()
mag = a.abs().double() @ b.abs().double().t()
split = len(sys.argv) > 1 and sys.argv[1] == "split"
print("accumulators:", "split" if split else "single")


def stats(name, c):
    r = (c.double() - ref) / mag
    rel = (c.double() - ref).abs().max() / ref.abs().max()
    print(f"  {name:10s} bias {float(r.mean()):+.3e}  rms {float(r.pow(2).mean().sqrt()):.3e}  max|err|/max|ref| {float(rel):.3e}")


stats("cublas", a @ b.t())
for fmt, name in ((ops.FMT_F16X2, "f16x2"), (ops.FMT_BF16X3, "bf16x3")):
    sa = ops.scale_tensor(8.0, dev) if fmt == ops.FMT_F16X2 else None
    sb = ops.scale_tensor(4096.0, dev) if fmt == ops.FMT_F16X2 else None
    c, _ = ops.gemm_planes(ops.split_planes(a, fmt, scale=sa), ops.split_planes(b, fmt, scale=sb), N, a_scale=sa, b_scale=sb, split_acc=split)
    stats(name, c)

# whole-network forward on the pair batch
from morl_baselines_b200.common.networks import mlp  # noqa: E402

th.manual_seed(0)
B, W, F, D, A = 1024, 64, 32, 3, 8
net = mlp(F + D, A * D, [256, 256, 256, 256]).to(dev)
for m in net:
    if isinstance(m, th.nn.Linear):
        th.nn.init.orthogonal_(m.weight)
        th.nn.init.normal_(m.bias, std=0.1)
feats = th.randn(B, F, device=dev, generator=g)
wset = th.rand(W, D, device=dev, generator=g)
wset = wset / wset.sum(1, keepdim=True)
x = th.cat([feats.repeat_interleave(W, 0), wset.repeat(B, 1)], dim=1)
with th.no_grad():
    q64 = net.double()(x.double())
    net.float()
    q32 = net(x)
    print(f"  network forward vs float64: cublas fp32 max rel {float((q32.double() - q64).abs().max() / q64.abs().max()):.3e} "
          f"mean signed rel {float(((q32.double() - q64) / q64.abs().clamp_min(1e-3)).mean()):+.3e}")
    for fmt, name in ((ops.FMT_F16X2, "f16x2"), (ops.FMT_BF16X3, "bf16x3")):
        plan = TCPairMlp(net, F, B, W, fmt=fmt, split_acc=split)
        plan.refresh_weights()
        q = plan.forward_pairs(feats, wset)
        e = q.double() - q64
        print(f"  network forward vs float64: {name:7s} max rel {float(e.abs().max() / q64.abs().max()):.3e} "
              f"mean signed rel {float((e * q64.sign() / q64.abs().clamp_min(1e-3)).mean()):+.3e}  rms {float(e.pow(2).mean().sqrt() / q64.pow(2).mean().sqrt()):.3e}")
print("overflow flags:", ops.plane_overflow_count())
