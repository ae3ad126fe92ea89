#!/usr/bin/env python
"""tools/lbfgs_phase_clocks.py -- where the cycles of a steady-state L-BFGS iteration go, phase by phase.

Builds a copy of libcno.so with build.NVCC_FLAGS plus -DCNO_LBFGS_PHASE_CLOCKS as
cppnumericalsolvers_b200/libcno_phase.so (the phase probe of lbfgs_minimize_kernel, cno_lbfgs.cuh), then, in a
subprocess with CNO_LIB=libcno_phase.so, runs bench_configs.run_config("c2", scale) -- Rosenbrock d = 128 fp64,
L-BFGS m = 10, bench.py's workload -- and reads the probe's counters.  Prints one JSON line per phase (cycles per
counted iteration; the line-search phases also per evaluation), their sum, and the kernel's own cycles per
warp-iteration from its event time, SM clock x SMs x warps per CTA x kernel time / iterations, with the card's name,
power limit and SM clock read in the same run.

    python tools/lbfgs_phase_clocks.py [--scale 1] [--reps 2] [--lib libcno_phase.so] [--build-only]

--lib names an already built probe library under cppnumericalsolvers_b200/ (for instance one built from an earlier
commit) and skips the build.  The probe's clock reads cost cycles of their own and take a few registers, so the
phase sum and the kernel figure of the probe build are both a little above those of the plain library.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cppnumericalsolvers_b200 import build as cno_build  # noqa: E402

LIB = "libcno_phase.so"
# the slots of cno_lbfgs_phase_clocks, in the order of enum LbfgsPhase (cno_lbfgs.cuh)
PHASES = ["recursion", "direction", "first_trial", "more_trials", "pair_update", "progress", "loop_back"]
SLOTS = PHASES + ["iterations", "extra_evals", "loop_backs"]


def build():
    """Compiles the probe copy (skipped when it is newer than every source)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    deps = [os.path.join(cno_build.CSRC, f) for f in os.listdir(cno_build.CSRC)]
    deps.append(os.path.join(ROOT, "include", "cno.h"))
    target = os.path.join(cno_build.HERE, LIB)
    if os.path.exists(target) and all(os.path.getmtime(d) <= os.path.getmtime(target) for d in deps):
        return
    subprocess.run([nvcc, *cno_build.NVCC_FLAGS, "-DCNO_LBFGS_PHASE_CLOCKS", "-o", target, *cno_build.sources(),
                    "-ldl"], check=True)


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def take(lib):
    buf = (ctypes.c_ulonglong * len(SLOTS))()
    rc = lib.cno_lbfgs_phase_clocks_take(buf, len(SLOTS))
    if rc != 0:
        raise RuntimeError(f"cno_lbfgs_phase_clocks_take: {rc}")
    return dict(zip(SLOTS, buf))


def child(scale: int, reps: int):
    """Runs in the subprocess: one c2 run with the library CNO_LIB names, then its counters."""
    import torch

    import bench_configs
    from cppnumericalsolvers_b200 import _lib
    lib = _lib.lib()
    if not hasattr(lib, "cno_lbfgs_phase_clocks_take"):
        raise RuntimeError(f"{_lib.LIB_PATH} was built without -DCNO_LBFGS_PHASE_CLOCKS")
    torch.cuda.synchronize()
    take(lib)  # zero
    rec = bench_configs.run_config("c2", scale, reps)
    torch.cuda.synchronize()
    clocks = take(lib)
    sm_clock = smi("clocks.sm")  # right after the last solve, before the card idles down
    print(json.dumps({"record": rec, "clocks": clocks, "sm_clock_after": sm_clock,
                      "sms": torch.cuda.get_device_properties(0).multi_processor_count}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=1, help="batch = 2^(20 - scale)")
    ap.add_argument("--reps", type=int, default=2, help="timed solves (after one warm-up solve)")
    ap.add_argument("--lib", default=None, help="an already built probe library under cppnumericalsolvers_b200/")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.scale, args.reps)
    name = args.lib or LIB
    if args.lib is None:
        build()
    if args.build_only:
        return 0
    card = smi("name,power.limit,clocks.max.sm")
    env = dict(os.environ, CNO_LIB=name)
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--scale", str(args.scale),
                          "--reps", str(args.reps)], env=env, cwd=ROOT, check=True, capture_output=True,
                         text=True).stdout
    res = json.loads(out.strip().splitlines()[-1])
    rec, c = res["record"], res["clocks"]
    it = max(c["iterations"], 1)
    for p in PHASES:
        n = max(c["loop_backs"], 1) if p == "loop_back" else it
        line = {"phase": p, "cycles_per_iteration": c[p] / n}
        if p == "more_trials":
            line["extra_evals_per_iteration"] = c["extra_evals"] / it
        print(json.dumps(line), flush=True)
    phase_sum = sum(c[p] / (max(c["loop_backs"], 1) if p == "loop_back" else it) for p in PHASES)
    # the kernel's own figure: every resident warp busy for the whole kernel time (the tail of the batch aside)
    mhz = float(card.split(",")[2].split()[0]) if card else float("nan")
    warp_iters = rec["batch"] * rec["mean_iterations"]
    kernel_cycles = rec["kernel_ms"] * 1e-3 * mhz * 1e6 * res["sms"] * rec["warps_per_cta"] / warp_iters
    print(json.dumps({"lib": name, "phase_sum_cycles_per_iteration": phase_sum,
                      "kernel_cycles_per_warp_iteration_at_max_sm_clock": kernel_cycles,
                      "steady_iterations_counted": c["iterations"], "all_iterations": warp_iters * (args.reps + 1),
                      "kernel_ms": rec["kernel_ms"], "instances_per_s": rec["instances_per_s"],
                      "mean_iterations": rec["mean_iterations"], "warps_per_cta": rec["warps_per_cta"],
                      "card": card, "columns": "name, power.limit, clocks.max.sm",
                      "sm_clock_after_run": res["sm_clock_after"]}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
