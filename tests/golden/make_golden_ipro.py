"""Golden vectors for IPRO and IPRO-2D's outer loop, produced by the unmodified reference on CPU (needs the reference's source tree and
``sortedcontainers``, so it is run by hand, not by the tests):
    python tests/golden/make_golden_ipro.py   ->  tests/golden/ipro.npz

Each case of ``tests/ipro_standin.CASES`` runs the reference's ``IPRO`` / ``IPRO2D`` with its learner replaced by the scripted oracle of
tests/ipro_standin.py, and records every iteration's referent, fronts, points or boxes, volumes, coverage, error and callback arguments,
then the final front and Pareto set, under ``<case>/...``.  pymoo is not needed: its ``Config`` and ``Hypervolume`` are replaced by
stand-ins, the latter backed by the exact sweep of oracle/hv_oracle.py.  A rerun writes the same bytes.
"""

from __future__ import annotations

import io
import os
import sys
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402
from oracle.hv_oracle import hypervolume_min  # noqa: E402
from tests.ipro_standin import CASES, run_case  # noqa: E402


class Hypervolume:
    """pymoo.indicators.hv.Hypervolume stand-in (minimisation form) on the exact host sweep."""

    def __init__(self, ref_point):
        self.ref_point = np.asarray(ref_point, dtype=np.float64)

    def __call__(self, points):
        return hypervolume_min(np.asarray(points, dtype=np.float64), self.ref_point)


def install_pymoo_standins():
    rh.install_stubs()
    cfg = sys.modules.setdefault("pymoo.config", types.ModuleType("pymoo.config"))
    cfg.Config = type("Config", (), {"warnings": {}})
    sys.modules["pymoo.indicators.hv"].Hypervolume = Hypervolume


def main():
    install_pymoo_standins()
    ipro = rh.import_reference("morl_baselines.multi_policy.ipro.ipro")
    ipro2d = rh.import_reference("morl_baselines.multi_policy.ipro.ipro_2d")
    classes = {"IPRO": ipro.IPRO, "IPRO2D": ipro2d.IPRO2D}
    out = {}
    for name in CASES:
        res = run_case(name, classes, device="cpu")
        its, replays = int(res["final/counters"][0]), int(res["final/counters"][1])
        print(f"{name}: {its} iterations, {replays} replays, |pf| = {len(res['final/pf'])}")
        out.update({f"{name}/{k}": v for k, v in res.items()})
    # fixed member order and timestamps, so a rerun gives the same bytes
    path = os.path.join(HERE, "ipro.npz")
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(out[k]), allow_pickle=False)
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(zi, buf.getvalue())
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
