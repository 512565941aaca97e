"""In-graph launch time of the dominant GEMM (bench.time_gemm_kernel), measured three times:
    python scripts/gemm_time.py
"""
import os, sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch as th  # noqa: E402

import bench  # noqa: E402

t = [bench.time_gemm_kernel(th.device("cuda:0"), iters=320)[0] for _ in range(3)]
print("US", " ".join("%.2f" % (x * 1e6) for x in t))
