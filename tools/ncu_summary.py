#!/usr/bin/env python
"""tools/ncu_summary.py <report.ncu-rep> [iterations] -- text summary of one ncu --set full
capture (raw + source pages).  `iterations` = solver iterations executed by
the profiled launch (to normalise instruction counts)."""
import collections
import csv
import io
import subprocess
import sys


def page(rep, name):
    out = subprocess.run(["ncu", "-i", rep, "--page", name, "--csv"], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    rep = sys.argv[1]
    iters = float(sys.argv[2]) if len(sys.argv) > 2 and not sys.argv[2].startswith("--") else None
    rows = page(rep, "raw")
    d = {h: (u, v) for h, u, v in zip(rows[0], rows[1], rows[2])}
    keys = [
        "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.per_cycle_active",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__warps_eligible.avg.per_cycle_active",
        "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    ]
    print(f"# ncu summary of {rep}")
    for k in keys:
        if k in d:
            print(f"{k:85s} {d[k][1]} {d[k][0]}")
    print("\n# warp stall reasons (warps stalled per issue-active cycle)")
    for k in sorted(d):
        if "issue_stalled" in k and "per_issue_active" in k:
            print(f"  {k.split('stalled_')[1].split('_per')[0]:22s} {float(d[k][1]):.3f}")
    rows = page(rep, "source")
    hdr, body = rows[1], rows[2:]
    iS, iE, iSamp = hdr.index("Source"), hdr.index("Instructions Executed"), hdr.index("# Samples")
    byop, samp, tot = collections.Counter(), collections.Counter(), 0
    for r in body:
        try:
            n, s = int(r[iE]), int(r[iSamp])
        except ValueError:
            continue
        toks = r[iS].split()
        op = toks[1] if toks[0].startswith("@") else toks[0]
        op = op.split(".")[0]
        byop[op] += n
        samp[op] += s
        tot += n
    print(f"\n# executed warp instructions: {tot}  (SASS lines {len(body)})")
    if iters:
        print(f"# per solver iteration ({iters:.0f} iterations in this launch): {tot / iters:.1f}")
    for op, n in byop.most_common(16):
        per = f"{n / iters:8.1f}/iter" if iters else ""
        print(f"  {op:8s} {n:14d} {per}  samples {samp[op]}")
    # FP64-datapath work: every D* opcode issues to the FP64 pipe (DADD DMUL DFMA DSETP ...); DMMA is the
    # FP64 tensor-core MMA, which occupies the same datapath (tools/fp64_pipe_probe.cu) for 16 cycles
    fp64 = sum(n for op, n in byop.items() if op.startswith("D") and op not in ("DMMA", "DEPBAR"))
    dmma = byop.get("DMMA", 0)
    if iters:
        print(f"# FP64-pipe warp instructions/iter {fp64 / iters:.1f}, DMMA/iter {dmma / iters:.1f}, "
              f"FP64-datapath cycles/iter = 2*fp64 + 16*dmma = {(2 * fp64 + 16 * dmma) / iters:.0f}")
    if "--mix-json" in sys.argv and iters:
        import json
        path = sys.argv[sys.argv.index("--mix-json") + 1]
        json.dump({"kernel": "lbfgs_minimize_kernel<RosenbrockFn<double,128>,10>", "report": rep,
                   "iterations_in_profiled_launch": iters, "instr_per_iteration": tot / iters,
                   "fp64_per_iteration": fp64 / iters, "dmma_per_iteration": dmma / iters}, open(path, "w"), indent=1)


if __name__ == "__main__":
    main()
