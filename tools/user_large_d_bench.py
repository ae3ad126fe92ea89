"""Throughput of Lbfgs on user objectives at d = 1024: the group kernel (csrc/cno_lbfgs_group.cuh, what
CNO_INSTANTIATE_FUNCTION routes a functor with the group form to) against the one-warp kernel (csrc/cno_lbfgs.cuh) on
the same type, for the functors and composites of tests/cpp/user_group_functions.cu (built by build()).

Per objective, one seeded U(-2, 2) batch (cno_fill_uniform) sized for about `--seconds` of kernel time on the group
kernel, at most `--max-batch` rows; `--runs` runs of each kernel, alternated; instances/s and kernel ms (median, min,
max); the outputs of the two kernels compared bit for bit.  The card name and power limit come from `nvidia-smi --query-gpu` (read-only) in the
same call.  A table on stderr, one JSON line on stdout.  Needs a GPU.

    python tools/user_large_d_bench.py [--tags rph1024 ...] [--seconds 2] [--runs 3] [--max-batch 131072]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

TAGS = ("gbowl1024", "rph1024", "pen1024", "zmul1024", "prodrosen1024", "rosen1024")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [s.strip() for s in q.split(",")]
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tags", nargs="+", default=list(TAGS))
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--runs", type=int, default=3)
    # objectives that converge in tens of iterations would need millions of rows for 2 s; x0, x and the gradient of
    # each kernel's result are held on the host, 8 KB per row each
    ap.add_argument("--max-batch", type=int, default=131072)
    a = ap.parse_args()

    import numpy as np
    import torch

    import test_user_group_gpu as ug
    from oracle import oracle_binding as ob

    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = []
    for tag in a.tags:
        ug.run(tag, ob.fill_uniform((sms, ug.D), 0, 1, -2.0, 2.0))  # warm-up (module load, smem attribute)
        probe = ug.run(tag, ob.fill_uniform((8 * sms, ug.D), 0, 2, -2.0, 2.0))
        B = max(sms, min(a.max_batch, int(8 * sms * a.seconds * 1e3 / max(probe["launch"].kernel_ms, 1e-3))))
        x0 = ob.fill_uniform((B, ug.D), 0, 12345, -2.0, 2.0)
        ms = {ug.GROUP: [], ug.ONE_WARP: []}
        outs = {}
        for _ in range(a.runs):
            for path in (ug.GROUP, ug.ONE_WARP):
                r = ug.run(tag, x0, path=path)
                assert r["rc"] == 0, (tag, path, r["rc"])
                ms[path].append(r["launch"].kernel_ms)
                if path in outs:
                    ug.same(r, outs[path])  # run to run
                outs[path] = r
        identical = all(np.array_equal(np.asarray(outs[0][k]).view(np.uint8), np.asarray(outs[1][k]).view(np.uint8))
                        for k in ug.KEYS)
        row = {"tag": tag, "batch": B, "bitwise_identical": identical,
               "iterations_mean": float(outs[0]["num_iterations"].mean())}
        for path, key in ((ug.GROUP, "group"), (ug.ONE_WARP, "one_warp")):
            m = sorted(ms[path])
            row[key] = {"kernel_ms_median": statistics.median(m), "kernel_ms_min": m[0], "kernel_ms_max": m[-1],
                        "instances_per_s": B / (statistics.median(m) * 1e-3)}
        row["speedup"] = row["one_warp"]["kernel_ms_median"] / row["group"]["kernel_ms_median"]
        rows.append(row)
        print(f"{tag:14s} B={B:6d} it={row['iterations_mean']:7.1f}  group {row['group']['instances_per_s']:8.0f}/s "
              f"[{row['group']['kernel_ms_min']:.1f}, {row['group']['kernel_ms_max']:.1f}] ms  one-warp "
              f"{row['one_warp']['instances_per_s']:8.0f}/s [{row['one_warp']['kernel_ms_min']:.1f}, "
              f"{row['one_warp']['kernel_ms_max']:.1f}] ms  x{row['speedup']:.2f}  identical={identical}",
              file=sys.stderr)
    print(json.dumps({"card": name, "power_limit": limit, "runs": a.runs, "rows": rows}))


if __name__ == "__main__":
    main()
