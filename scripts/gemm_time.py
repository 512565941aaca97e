"""In-graph launch time of the dominant GEMM (bench.time_gemm_kernel) under the environment switches given on the command line, one
subprocess per variant:
    python scripts/gemm_time.py "" MORL_GEMM_STAGES=2 "MORL_GEMM_SPLIT_ACC=1 MORL_GEMM_STAGES=2"
"""
import os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = ("import torch as th, bench\n"
        "dev = th.device('cuda:0')\n"
        "t = [bench.time_gemm_kernel(dev, iters=320)[0] for _ in range(3)]\n"
        "print('US', ' '.join('%.2f' % (x * 1e6) for x in t))\n")
for variant in (sys.argv[1:] or [""]):
    env = dict(os.environ, PYTHONPATH=ROOT)
    for kv in variant.split():
        k, v = kv.split("=")
        env[k] = v
    r = subprocess.run([sys.executable, "-c", CODE], env=env, capture_output=True, text=True, cwd=ROOT)
    line = [l for l in r.stdout.splitlines() if l.startswith("US")]
    print(f"{variant or 'default':50s} {line[0] if line else 'FAILED ' + r.stderr[-400:]}")
