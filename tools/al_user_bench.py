"""Kernel time of AugmentedLagrangian on the `bench_configs.py al` workload (Rosenbrock d = 128 fp64, a sphere
equality t - x.x = 0 at t = 16 and a halfspace inequality sum(x) + 1 >= 0, B = 2^15, outer limit 20) two ways:

  rows      cno_al_minimize on [a | t] rows (the built-in constraint set, csrc/cno_auglag.cuh: AlRows)
  functors  cno_<tag>_al_minimize from CNO_INSTANTIATE_CONSTRAINED with the SqNormRow / AffineRow functors of
            tests/cpp/al_user_problems.cuh (problem 5) reading the same rows (AlFunctors)

The functor library is compiled here into a temporary directory.  The two are alternated, `--runs` times each after one
warm-up, and must agree bit for bit on every cno_al_out_t array.  Reports the median, min and max of the device time
each call records (cno_launch_info_t::kernel_ms: every launch of the call plus the per-outer-iteration read-back), and
the card name and power limit from `nvidia-smi --query-gpu` (read-only) in the same call.  One JSON line on stdout.
Needs a GPU.

    python tools/al_user_bench.py [--runs 3] [--scale k]   (--scale k divides the batch by 2^k)
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [s.strip() for s in q.split(",")]
    return name, limit


def build_functors(tmp):
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib = os.path.join(ROOT, "cppnumericalsolvers_b200")
    out = os.path.join(tmp, "libcno_al_user.so")
    subprocess.run([os.environ.get("NVCC", f"{cuda}/bin/nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                    "-std=c++17", "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false", "-shared",
                    "-Xcompiler", "-fPIC", os.path.join(ROOT, "tests", "cpp", "al_user_functions.cu"),
                    "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(lib, "csrc"),
                    "-I" + os.path.join(ROOT, "tests", "cpp"), "-o", out, f"-L{lib}", "-lcno", "-Xlinker",
                    f"-rpath={lib}"], check=True)
    return C.CDLL(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scale", type=int, default=0)
    args = ap.parse_args()

    import numpy as np
    import torch

    import cppnumericalsolvers_b200 as cn
    from cppnumericalsolvers_b200 import _lib
    import al_user_ref as ar
    from oracle import oracle_binding as ob

    dev = "cuda:0"
    B, d = (1 << 15) >> args.scale, 128
    x0 = torch.empty(B, d, dtype=torch.float64, device=dev)
    cn.fill_uniform(x0, 0, 12345, -1.5, 1.5)
    rows = torch.zeros(2, d + 1, dtype=torch.float64, device=dev)
    rows[0, d] = 16.0           # t - x.x = 0  (equality: on the sphere of radius 4)
    rows[1, :d] = 1.0           # sum(x) + 1 >= 0
    rows[1, d] = -1.0

    problem = cn.ConstrainedOptimizationProblem(cn.Rosenbrock(d), [ob.CON_SQNORM, ob.CON_AFFINE], rows, 1)
    solver = cn.AugmentedLagrangian(problem)
    solver.stopping_progress.num_iterations = 20

    def run_rows():
        st, pr = solver.Minimize(cn.AugmentedLagrangeState(x0))
        torch.cuda.synchronize()
        out = dict(x=st.x, equality_multipliers=st.equality_multipliers,
                   inequality_multipliers=st.inequality_multipliers, penalty=st.penalty, max_violation=st.max_violation,
                   max_lagrangian_gradient=st.max_lagrangian_gradient, num_iterations=pr.num_iterations,
                   status=pr.status, nfev=pr.nfev, x_delta=pr.x_delta, f_delta=pr.f_delta,
                   gradient_norm=pr.gradient_norm)
        return {k: v.cpu().numpy() for k, v in out.items()}, pr.launch.kernel_ms, pr.launch.kernel_launches

    with tempfile.TemporaryDirectory() as tmp:
        alu = build_functors(tmp)
        nbytes = C.c_size_t(0)
        assert alu.cno_test_al_user(ar.AL_P_ROWS, 0, d, None, C.c_int64(0), C.c_int64(B), *([None] * 8), None,
                                    C.c_size_t(0), None, None, C.byref(nbytes)) == 0
        ws = torch.zeros(nbytes.value + 256, dtype=torch.uint8, device=dev)
        shapes = ar.out_arrays(B, d, 1, 1, np.float64)
        tdt = {np.dtype(np.float64): torch.float64, np.dtype(np.uint32): torch.int32, np.dtype(np.int8): torch.int8}
        t = {k: torch.zeros(a.shape, dtype=tdt[a.dtype], device=dev) for k, a in shapes.items()}
        out = ob.AlOut(*[t[k].data_ptr() for k in ar.OUT_KEYS])
        stop = ob.al_default_stop()
        stop.num_iterations = 20

        def run_functors():
            info = _lib.LaunchInfo()
            rc = alu.cno_test_al_user(ar.AL_P_ROWS, 0, d, C.c_void_p(rows.data_ptr()), C.c_int64(0), C.c_int64(B),
                                      C.c_void_p(x0.data_ptr()), None, None, None, C.byref(ob.default_stop()),
                                      C.byref(stop), C.byref(ob.al_default_config()), C.byref(out),
                                      C.c_void_p(ws.data_ptr()), C.c_size_t(nbytes.value),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(info), None)
            torch.cuda.synchronize()
            assert rc == 0, rc
            r = {k: v.cpu().numpy() for k, v in t.items()}
            r["num_iterations"] = r["num_iterations"].astype(np.uint32)
            r["nfev"] = r["nfev"].astype(np.uint32)
            return r, info.kernel_ms, info.kernel_launches

        name, limit = card()
        run_rows()
        run_functors()  # warm-up: module load of both libraries
        ms = {"rows": [], "functors": []}
        launches = {}
        identical = True
        for _ in range(args.runs):
            a, ms_a, launches["rows"] = run_rows()
            b, ms_b, launches["functors"] = run_functors()
            ms["rows"].append(ms_a)
            ms["functors"].append(ms_b)
            identical &= all(np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8))
                             for k in ar.OUT_KEYS)

    rec = {"workload": "al rosenbrock d128 f64 sphere+halfspace (outer limit 20)", "batch": B, "card": name,
           "power_limit": limit, "runs": args.runs, "bitwise_identical": bool(identical),
           "kernel_launches": launches, "mean_outer_iterations": float(a["num_iterations"].mean())}
    for k, v in ms.items():
        rec[f"{k}_kernel_ms_median"] = float(np.median(v))
        rec[f"{k}_kernel_ms_min"] = float(np.min(v))
        rec[f"{k}_kernel_ms_max"] = float(np.max(v))
    rec["functors_over_rows"] = rec["functors_kernel_ms_median"] / rec["rows_kernel_ms_median"]
    print(json.dumps(rec), flush=True)
    return 0 if identical else 1


if __name__ == "__main__":
    sys.exit(main())
