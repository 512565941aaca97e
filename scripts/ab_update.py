"""A/B of two builds of libmorl_b200.so on the Envelope update that bench.py measures (a measurement of its own; bench.py is untouched):

    python scripts/ab_update.py LIB_A LIB_B [--rounds 3] [--steps 200] [--warmup 5] [--dump-dir DIR]

Runs bench.py's envelope workload in fresh subprocesses, alternating A, B, A, B, ... with morl_baselines_b200._lib.LIB_PATH pointed at
the given library, and prints per run `value`, `e2e.value`, the chained launch (`roofline.us_per_launch`), the per-layer launch
(`roofline_gemm_layer.us_per_launch`), the envelope operator as the update runs it (`roofline_envelope.us_per_launch`: the fused head at
the north-star shape) and standalone on Q tensors in HBM (`roofline_envelope_operator.us_per_launch`), and the clocks / throttle reasons
bench.py samples; then median and min-max per side, next to the
card's name and power limit.  With --dump-dir the first run of each side writes its outputs (bench.py --dump-outputs) and the script
reports whether every array is bit-identical between the sides.  Needs a GPU: there is nothing to fall back to.  Changes no device
setting; every child has exited when it returns."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# child: point the loader at the library under test, then run bench.py as __main__
CHILD = (
    "import runpy, sys\n"
    "sys.path.insert(0, {root!r})\n"
    "from morl_baselines_b200 import _lib\n"
    "_lib.LIB_PATH = {lib!r}\n"
    "sys.argv = ['bench.py'] + {argv!r}\n"
    "runpy.run_path({bench!r}, run_name='__main__')\n"
)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi query failed)"


def run_once(lib, steps, warmup, dump):
    argv = ["--gpus", "1", "--steps", str(steps), "--warmup", str(warmup)] + (["--dump-outputs", dump] if dump else [])
    code = CHILD.format(root=ROOT, lib=os.path.abspath(lib), argv=argv, bench=os.path.join(ROOT, "bench.py"))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, MORL_SKIP_CPU_BASELINE="1"), capture_output=True, text=True, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise SystemExit(f"bench.py failed with {lib} (exit {r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    d = json.loads(lines[-1])
    return {"value": d["value"], "e2e": d["e2e"]["value"], "chain_us": d["roofline"]["us_per_launch"], "layer_us": d["roofline_gemm_layer"]["us_per_launch"],
            "env_us": d["roofline_envelope"]["us_per_launch"], "env_op_us": d["roofline_envelope_operator"]["us_per_launch"], "clocks": d.get("clocks")}


def same_dumps(dir_a, dir_b):
    import numpy as np

    names = sorted(os.listdir(dir_a))
    if names != sorted(os.listdir(dir_b)) or not names:
        return False, ["different sets of arrays"]
    diff = [n for n in names if not np.array_equal(np.load(os.path.join(dir_a, n)), np.load(os.path.join(dir_b, n)))]
    return not diff, diff


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dump-dir", default=None)
    args = ap.parse_args()
    for lib in (args.lib_a, args.lib_b):
        if not os.path.exists(lib):
            raise SystemExit(f"{lib}: no such library")
    import torch as th

    if not th.cuda.is_available():
        raise SystemExit("ab_update.py measures on a GPU; no CUDA device is visible")
    print(f"# card: {card()} (name, power limit, max SM clock); {args.rounds} rounds A, B of bench.py --steps {args.steps} --warmup {args.warmup}", flush=True)
    sides = {"A": (args.lib_a, []), "B": (args.lib_b, [])}
    for rnd in range(args.rounds):
        for name, (lib, runs) in sides.items():
            dump = os.path.join(args.dump_dir, name) if (args.dump_dir and rnd == 0) else None
            res = run_once(lib, args.steps, args.warmup, dump)
            runs.append(res)
            print(f"{name} round {rnd}: value {res['value']:.1f} updates/s  e2e {res['e2e']:.1f}  chain {res['chain_us']:.1f} us  layer {res['layer_us']:.1f} us  "
                  f"envelope {res['env_us']:.2f} us  envelope operator {res['env_op_us']:.2f} us  clocks {res['clocks']}", flush=True)
    for name, (lib, runs) in sides.items():
        print(f"# {name} = {lib}")
        for key in ("value", "e2e", "chain_us", "layer_us", "env_us", "env_op_us"):
            v = [r[key] for r in runs]
            print(f"#   {key:9s} median {statistics.median(v):.2f}  min {min(v):.2f}  max {max(v):.2f}")
    va, vb = ([r["value"] for r in sides[s][1]] for s in "AB")
    ca, cb = (statistics.median(r["chain_us"] for r in sides[s][1]) for s in "AB")
    print(f"# B / A: value median x{statistics.median(vb) / statistics.median(va):.3f}, min(B) {'>' if min(vb) > max(va) else '<='} max(A); "
          f"chained launch median {100 * (cb / ca - 1):+.1f} %")
    if args.dump_dir:
        ok, diff = same_dumps(os.path.join(args.dump_dir, "A"), os.path.join(args.dump_dir, "B"))
        print("# outputs of the last timed update (loss, priorities, q_net.*): " + ("bit-identical" if ok else f"DIFFERENT: {diff}"))
        if not ok:
            raise SystemExit(1)


if __name__ == "__main__":
    main()
