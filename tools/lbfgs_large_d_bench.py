"""Throughput of Lbfgs on Rosenbrock fp64 at d = 512 and 1024: the group kernel (csrc/cno_lbfgs_group.cuh, the
built-in family through cno_minimize) against the one-warp kernel (csrc/cno_lbfgs.cuh) on the same objective as a user
functor (tests/cpp/one_warp_rosenbrock.cu, compiled here into a temporary directory).

Both solve the same seeded U(-2, 2) starts (cno_fill_uniform) and must agree bit for bit on every output.  Per d and
kernel: instances/s and kernel ms over `--runs` alternated runs (median, min, max), iterations and evaluations per
instance, and a MODEL figure for the memory traffic -- 8 d (2 k + 6) bytes per iteration at k = m = 10 pairs, what an
implementation that streamed the history and the vectors through HBM would move -- as a share of the card's HBM
bandwidth.  The card name and power limit come from `nvidia-smi --query-gpu` (read-only) in the same call.  One JSON
line on stdout.  Needs a GPU.

    python tools/lbfgs_large_d_bench.py [--d 512 1024] [--seconds 2] [--runs 3]

A d needs a row of the dispatch table (csrc/cno_api.cu); d = 256 has none (see DESIGN.md 2.10).
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

KEYS = ("x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta", "gradient_norm")
HBM_BYTES_PER_S = 3.35e12  # H100 SXM5 80 GB HBM3, the datasheet figure


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [s.strip() for s in q.split(",")]
    return name, limit


def build_one_warp(tmp):
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib = os.path.join(ROOT, "cppnumericalsolvers_b200")
    out = os.path.join(tmp, "libcno_one_warp.so")
    subprocess.run([os.environ.get("NVCC", f"{cuda}/bin/nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                    "-std=c++17", "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false", "-shared",
                    "-Xcompiler", "-fPIC", os.path.join(ROOT, "tests", "cpp", "one_warp_rosenbrock.cu"),
                    "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(lib, "csrc"), "-o", out, f"-L{lib}",
                    "-lcno", "-Xlinker", f"-rpath={lib}"], check=True)
    return C.CDLL(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--seconds", type=float, default=2.0, help="kernel time per run to size the batch for")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()

    import torch

    from cppnumericalsolvers_b200 import _lib
    if not torch.cuda.is_available():
        raise SystemExit("lbfgs_large_d_bench.py needs a GPU")
    name, limit = card()
    L = _lib.lib()
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev).cuda_stream
    ws = torch.zeros(256, dtype=torch.uint8, device=dev)
    stop = _lib.Stop()
    L.cno_default_stop(C.byref(stop))
    results = {"card": name, "power_limit": limit, "runs": a.runs, "d": {}}
    with tempfile.TemporaryDirectory() as tmp:
        one_warp = build_one_warp(tmp)

        def outputs(B, d):
            t = dict(x=torch.empty(B, d, dtype=torch.float64, device=dev),
                     value=torch.empty(B, dtype=torch.float64, device=dev),
                     gradient=torch.empty(B, d, dtype=torch.float64, device=dev),
                     num_iterations=torch.empty(B, dtype=torch.int32, device=dev),
                     status=torch.empty(B, dtype=torch.int8, device=dev),
                     nfev=torch.empty(B, dtype=torch.int32, device=dev),
                     x_delta=torch.empty(B, dtype=torch.float64, device=dev),
                     f_delta=torch.empty(B, dtype=torch.float64, device=dev),
                     gradient_norm=torch.empty(B, dtype=torch.float64, device=dev))
            return t, _lib.BatchOut(*[t[k].data_ptr() for k in KEYS])

        def run(kernel, x0):
            B, d = x0.shape
            t, out = outputs(B, d)
            info = _lib.LaunchInfo()
            if kernel == "group":
                prob = _lib.Problem(family=0, dtype=_lib.F64, d=d, policy=_lib.POLICY_DMMA_TREE)
                _lib.check(L.cno_minimize(_lib.LBFGS, C.byref(prob), B, x0.data_ptr(), C.byref(stop), C.byref(out),
                                          ws.data_ptr(), ws.numel(), stream, C.byref(info)), "cno_minimize")
            else:
                rc = one_warp.cno_one_warp_rosenbrock_minimize(d, C.c_int64(B), C.c_void_p(x0.data_ptr()),
                                                               C.byref(stop), C.byref(out), C.c_void_p(ws.data_ptr()),
                                                               C.c_size_t(256), C.c_void_p(stream), C.byref(info))
                _lib.check(rc, "one-warp minimize")
            torch.cuda.synchronize()
            return t, info.kernel_ms

        for d in a.d:
            probe = torch.empty(4096, d, dtype=torch.float64, device=dev)
            L.cno_fill_uniform(_lib.F64, C.c_void_p(probe.data_ptr()), C.c_int64(0), C.c_int64(probe.numel()),
                               C.c_uint64(2024), C.c_double(-2.0), C.c_double(2.0), C.c_void_p(stream))
            _, ms = run("group", probe)  # (warm-up and batch sizing)
            run("one_warp", probe)
            B = int(min(max(4096 * a.seconds * 1e3 / max(ms, 1e-3), 4096), 1 << 20))
            x0 = torch.empty(B, d, dtype=torch.float64, device=dev)
            L.cno_fill_uniform(_lib.F64, C.c_void_p(x0.data_ptr()), C.c_int64(0), C.c_int64(x0.numel()),
                               C.c_uint64(2024), C.c_double(-2.0), C.c_double(2.0), C.c_void_p(stream))
            times = {"group": [], "one_warp": []}
            outs = {}
            for _ in range(a.runs):
                for kernel in ("group", "one_warp"):
                    t, ms = run(kernel, x0)
                    times[kernel].append(ms)
                    outs[kernel] = t
            identical = all(torch.equal(outs["group"][k].view(torch.uint8), outs["one_warp"][k].view(torch.uint8))
                            for k in KEYS)
            assert identical, f"d = {d}: the group and one-warp kernels differ"
            it = outs["group"]["num_iterations"].double()
            nf = outs["group"]["nfev"].double()
            row = {"batch": B, "bit_identical": identical, "iterations_per_instance": round(it.mean().item(), 2),
                   "evaluations_per_instance": round(nf.mean().item(), 2)}
            model_bytes = 8.0 * d * (2 * 10 + 6) * it.sum().item()
            for kernel, ts in times.items():
                ms = sorted(ts)
                med = ms[len(ms) // 2]
                row[kernel] = {"kernel_ms_median": round(med, 2), "kernel_ms_min": round(ms[0], 2),
                               "kernel_ms_max": round(ms[-1], 2),
                               "instances_per_s": round(B / (med * 1e-3), 1),
                               "hbm_model_share": round(model_bytes / (med * 1e-3) / HBM_BYTES_PER_S, 4)}
            row["group_over_one_warp"] = round(row["one_warp"]["kernel_ms_median"] / row["group"]["kernel_ms_median"], 3)
            results["d"][str(d)] = row
            print(f"d={d}: {json.dumps(row)}", file=sys.stderr)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
