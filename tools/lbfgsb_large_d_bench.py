"""Throughput of Lbfgsb on Rosenbrock fp64 at d = 256, 512 and 1024 (csrc/cno_lbfgsb_group.cuh, through
cno_lbfgsb_minimize), on three workloads per d:

  shared_box       the box [-0.5, 0.8]^d for every instance
  instance_boxes   per-instance random boxes: lower U(-1.5, -0.2), upper = lower + U(0.3, 2.0)
  unbounded        no box, the Lbfgsb() preset with an iteration limit of 200

Starts are seeded U(-2.5, 2.5) (cno_fill_uniform).  The batch is sized for about `--seconds` of kernel time; after a
warm-up, `--runs` runs are timed with CUDA events around the kernel (cno_launch_info_t::kernel_ms) and the median is
reported with instances/s and the mean iterations and evaluations per instance.  For context only, the same workloads
on a sample of instances through the reference's own lbfgsb.h on the CPU (oracle/_ref, as build() made it, spread
over the host's threads) give a CPU rate: that is the reference header on the Eigen-API shim, not a tuned CPU solver.
The card name and power limit come from `nvidia-smi --query-gpu` (read-only) in the same call.  One JSON line on
stdout.  Needs a GPU.

    python tools/lbfgsb_large_d_bench.py [--d 256 512 1024] [--seconds 2] [--runs 3] [--cpu-sample 64]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KEYS = ("x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta", "gradient_norm")
WORKLOADS = ("shared_box", "instance_boxes", "unbounded")
UNBOUNDED_ITERATIONS = 200


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [s.strip() for s in q.split(",")]
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--seconds", type=float, default=2.0, help="kernel time per run to size the batch for")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=64, help="instances solved by the reference header (0: none)")
    a = ap.parse_args()

    import torch

    from cppnumericalsolvers_b200 import _lib
    from oracle import oracle_binding as ob
    if not torch.cuda.is_available():
        raise SystemExit("lbfgsb_large_d_bench.py needs a GPU")
    name, limit = card()
    L = _lib.lib()
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev).cuda_stream
    ws = torch.zeros(256, dtype=torch.uint8, device=dev)
    threads = os.cpu_count() or 1
    results = {"card": name, "power_limit": limit, "runs": a.runs, "d": {},
               "cpu_reference": f"the reference's own lbfgsb.h on the Eigen-API shim (oracle/_ref), {threads} host threads"}

    def stop_for(workload):
        s = _lib.Stop()
        L.cno_lbfgsb_default_stop(C.byref(s))
        if workload == "unbounded":
            s.num_iterations = UNBOUNDED_ITERATIONS
        return s

    def starts(B, d):
        x0 = torch.empty(B, d, dtype=torch.float64, device=dev)
        L.cno_fill_uniform(_lib.F64, C.c_void_p(x0.data_ptr()), C.c_int64(0), C.c_int64(x0.numel()),
                           C.c_uint64(2025), C.c_double(-2.5), C.c_double(2.5), C.c_void_p(stream))
        return x0

    def box(workload, B, d):
        if workload == "shared_box":
            return (torch.full((d,), -0.5, dtype=torch.float64, device=dev),
                    torch.full((d,), 0.8, dtype=torch.float64, device=dev))
        if workload == "instance_boxes":
            g = torch.Generator(device=dev).manual_seed(d)
            lo = -1.5 + 1.3 * torch.rand(B, d, dtype=torch.float64, device=dev, generator=g)
            return lo, lo + 0.3 + 1.7 * torch.rand(B, d, dtype=torch.float64, device=dev, generator=g)
        return None, None

    def run(x0, lo, hi, stop):
        B, d = x0.shape
        t = dict(x=torch.empty(B, d, dtype=torch.float64, device=dev),
                 value=torch.empty(B, dtype=torch.float64, device=dev),
                 gradient=torch.empty(B, d, dtype=torch.float64, device=dev),
                 num_iterations=torch.empty(B, dtype=torch.int32, device=dev),
                 status=torch.empty(B, dtype=torch.int8, device=dev),
                 nfev=torch.empty(B, dtype=torch.int32, device=dev),
                 x_delta=torch.empty(B, dtype=torch.float64, device=dev),
                 f_delta=torch.empty(B, dtype=torch.float64, device=dev),
                 gradient_norm=torch.empty(B, dtype=torch.float64, device=dev))
        out = _lib.BatchOut(*[t[k].data_ptr() for k in KEYS])
        bounds = _lib.Bounds(None if lo is None else lo.data_ptr(), None if hi is None else hi.data_ptr(),
                             d if (lo is not None and lo.dim() == 2) else 0)
        prob = _lib.Problem(family=0, dtype=_lib.F64, d=d, policy=_lib.POLICY_DMMA_TREE)
        info = _lib.LaunchInfo()
        _lib.check(L.cno_lbfgsb_minimize(C.byref(prob), C.byref(bounds), B, x0.data_ptr(), C.byref(stop),
                                         C.byref(out), ws.data_ptr(), ws.numel(), stream, C.byref(info)),
                   "cno_lbfgsb_minimize")
        torch.cuda.synchronize()
        return t, info.kernel_ms

    for d in a.d:
        row = {}
        for workload in WORKLOADS:
            stop = stop_for(workload)
            probe = starts(1024, d)
            run(probe, *box(workload, 1024, d), stop)                # warm-up
            _, ms = run(probe, *box(workload, 1024, d), stop)       # batch sizing
            B = int(min(max(1024 * a.seconds * 1e3 / max(ms, 1e-3), 1024), 1 << 18))
            x0 = starts(B, d)
            lo, hi = box(workload, B, d)
            times = []
            for _ in range(a.runs):
                t, ms = run(x0, lo, hi, stop)
                times.append(ms)
            times.sort()
            med = times[len(times) // 2]
            it = t["num_iterations"].double()
            nf = t["nfev"].double()
            r = {"batch": B, "kernel_ms_median": round(med, 2), "kernel_ms_min": round(times[0], 2),
                 "kernel_ms_max": round(times[-1], 2), "instances_per_s": round(B / (med * 1e-3), 1),
                 "iterations_per_instance": round(it.mean().item(), 2),
                 "evaluations_per_instance": round(nf.mean().item(), 2)}
            if a.cpu_sample > 0 and ob.ref_available():
                n = min(a.cpu_sample, B)
                xs = x0[:n].cpu().numpy()
                los = None if lo is None else (lo.cpu().numpy() if lo.dim() == 1 else lo[:n].cpu().numpy())
                his = None if hi is None else (hi.cpu().numpy() if hi.dim() == 1 else hi[:n].cpu().numpy())
                cs = ob.Stop()
                C.memmove(C.byref(cs), C.byref(stop), C.sizeof(cs))
                o = ob.ref_lbfgsb_minimize(ob.FN_ROSENBROCK, xs, los, his, stop=cs, threads=threads)
                same = all(np.array_equal(np.asarray(o[k]).view(np.uint8),
                                          t[k][:n].cpu().numpy().astype(o[k].dtype).view(np.uint8)) for k in KEYS)
                r["cpu_reference_instances_per_s"] = round(n / o["seconds"], 1)
                r["cpu_reference_sample"] = n
                r["sample_bit_identical"] = same
            row[workload] = r
            print(f"d={d} {workload}: {json.dumps(r)}", file=sys.stderr)
        results["d"][str(d)] = row
    print(json.dumps(results))


if __name__ == "__main__":
    main()
