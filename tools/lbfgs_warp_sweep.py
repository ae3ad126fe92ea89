#!/usr/bin/env python
"""tools/lbfgs_warp_sweep.py -- throughput of the persistent L-BFGS kernel against the warps resident per SM.

Builds copies of libcno.so with build.NVCC_FLAGS plus -DCNO_LBFGS_MAX_WARPS=w (a cap on the warp count of every
L-BFGS plan) as cppnumericalsolvers_b200/libcno_w<w>.so, then times, for each copy in a subprocess of its own
(CNO_LIB=libcno_w<w>.so):
  c2  Rosenbrock d=128 fp64, L-BFGS m=10 (bench_configs.run_config("c2"), bench.py's workload)
  m5  the same workload with m=5
and reports kernel iterations per second, B * mean_iterations / kernel_ms.  The copies are run in alternation,
`--repeats` rounds, so that a drift of the card's clock lands on every warp count alike.  One JSON line per run,
then one summary line per (config, warps): the median rate and its ratio to the smallest warp count.

    python tools/lbfgs_warp_sweep.py [--c2-warps 6,8,10,11] [--m5-warps 16,20] [--repeats 3] [--scale 1]
                                     [--build-only]

If the kernel is latency-bound, c2's rate grows close to in proportion to the warps (11/8 = 1.375 between 8 and 11).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cppnumericalsolvers_b200 import build as cno_build  # noqa: E402


def lib_name(w: int) -> str:
    return f"libcno_w{w}.so"


def build_all(warps):
    """Compiles the capped copies in parallel (skips a copy newer than every source)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    deps = [os.path.join(cno_build.CSRC, f) for f in os.listdir(cno_build.CSRC)]
    deps.append(os.path.join(ROOT, "include", "cno.h"))
    procs = []
    for w in warps:
        target = os.path.join(cno_build.HERE, lib_name(w))
        if os.path.exists(target) and all(os.path.getmtime(d) <= os.path.getmtime(target) for d in deps):
            continue
        procs.append(subprocess.Popen([nvcc, *cno_build.NVCC_FLAGS, f"-DCNO_LBFGS_MAX_WARPS={w}", "-o", target,
                                       *cno_build.sources(), "-ldl"]))
    for p in procs:
        if p.wait() != 0:
            raise subprocess.CalledProcessError(p.returncode, p.args)


def child(configs, scale: int, reps: int):
    """Runs in the subprocess: times each config with the library CNO_LIB names."""
    import torch

    import bench_configs
    import cppnumericalsolvers_b200 as cn
    for c in configs:
        if c == "c2":
            rec = bench_configs.run_config("c2", scale, reps)
        else:  # m5: c2's inputs, Lbfgs<F, 5>
            B = (1 << 20) >> scale
            x0 = torch.empty(B, 128, dtype=torch.float64, device="cuda")
            cn.fill_uniform(x0, 0, 12345, -2.0, 2.0)
            rec = bench_configs.run("m5 lbfgs(m=5) rosenbrock d128 f64", cn.Lbfgs(m=5), cn.Rosenbrock(128), x0,
                                    bench_configs.lbfgs_bytes(8, 128, m=5), reps)
        rec["iterations_per_s"] = rec["batch"] * rec["mean_iterations"] / rec["kernel_ms"] * 1e3
        rec["short"] = c
        rec["lib"] = os.environ.get("CNO_LIB", "libcno.so")
        print(json.dumps(rec), flush=True)
        torch.cuda.empty_cache()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c2-warps", default="6,8,10,11")
    ap.add_argument("--m5-warps", default="16,20")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--scale", type=int, default=1, help="batch = 2^(20 - scale)")
    ap.add_argument("--reps", type=int, default=2, help="timed solves per run (after one warm-up solve)")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child.split(","), args.scale, args.reps)

    c2 = [int(w) for w in args.c2_warps.split(",") if w]
    m5 = [int(w) for w in args.m5_warps.split(",") if w]
    warps = sorted(set(c2) | set(m5))
    build_all(warps)
    if args.build_only:
        return 0
    print(json.dumps({"card": card(), "columns": "name, power.limit, clocks.max.sm"}), flush=True)
    rates = {}
    for _ in range(args.repeats):
        for w in warps:
            configs = (["c2"] if w in c2 else []) + (["m5"] if w in m5 else [])
            env = dict(os.environ, CNO_LIB=lib_name(w))
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", ",".join(configs),
                                  "--scale", str(args.scale), "--reps", str(args.reps)],
                                 env=env, cwd=ROOT, check=True, capture_output=True, text=True).stdout
            for line in out.splitlines():
                rec = json.loads(line)
                rec["cap"] = w
                print(json.dumps(rec), flush=True)
                rates.setdefault((rec["short"], rec["warps_per_cta"]), []).append(rec["iterations_per_s"])
    for c in ("c2", "m5"):
        keys = sorted(k for k in rates if k[0] == c)
        if not keys:
            continue
        base = statistics.median(rates[keys[0]])
        for k in keys:
            med = statistics.median(rates[k])
            print(json.dumps({"summary": c, "warps_per_cta": k[1], "median_iterations_per_s": med,
                              "min": min(rates[k]), "max": max(rates[k]), "runs": len(rates[k]),
                              "vs_fewest_warps": med / base, "warps_ratio": k[1] / keys[0][1]}), flush=True)
    print(json.dumps({"card": card()}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
