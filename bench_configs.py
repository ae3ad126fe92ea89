#!/usr/bin/env python
"""bench_configs.py -- device timing of the BASELINE.json configs that are NOT
bench.py's headline (configs[2..4]) plus the headline for reference.  These are
parity-test cases per the contract; this script only reports their throughput
and the SURVEY.md 8(d) algorithmic-byte roofline next to it.  One JSON object
per config on stdout.  Usage: python bench_configs.py [c2 c3 c4 c5] [--scale k]
(--scale k divides the batch by 2^k)."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import cppnumericalsolvers_b200 as cn  # noqa: E402

DEV = "cuda"


def peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    return float(json.load(open(p))["hbm_gbs"]) if os.path.exists(p) else 3350.0  # H100 SXM data sheet


def run(name, solver, fn, x0, bytes_fn, reps=3, extra=None):
    ms = []
    for _ in range(reps + 1):
        st, pr = solver.Minimize(fn, cn.BatchedFunctionState(x0), timed=True)
        ms.append(pr.launch.kernel_ms)
    ms = float(np.mean(ms[1:]))
    it = pr.num_iterations.cpu().numpy().astype(np.int64)
    nf = pr.nfev.cpu().numpy().astype(np.int64)
    B = x0.shape[0]
    alg = float(bytes_fn(it, nf))
    out = {"config": name, "batch": B, "kernel_ms": ms, "instances_per_s": B / ms * 1e3,
           "mean_iterations": float(it.mean()), "mean_nfev": float(nf.mean()),
           "status_histogram": np.bincount(pr.status.cpu().numpy().astype(np.int64) + 1).tolist(),
           "algorithmic_GBps": alg / ms / 1e6, "hbm_peak_GBps": peak(),
           "frac_of_hbm_roofline": alg / ms / 1e6 / peak(),
           "grid": pr.launch.grid, "warps_per_cta": pr.launch.warps_per_cta,
           "dynamic_smem": pr.launch.dynamic_smem}
    out.update(extra or {})
    return out


def lbfgs_bytes(w, d, m=10):
    def f(it, nf):
        full = np.maximum(it - m, 0)
        ramp = np.minimum(it, m)
        pairs = full * m + ramp * (ramp - 1) // 2
        return (w * d * (6 * it + 2 * pairs)).sum()
    return f


def _gen():
    g = torch.Generator(device=DEV)
    g.manual_seed(0)
    return g


def run_config(which: str, scale: int = 0, reps: int = 3) -> dict:
    """Builds the synthetic inputs of one config, times it on the current device and returns the record."""
    gen = _gen()
    if which == "c2":  # Rosenbrock d=128 fp64 L-BFGS, B = 2^20
        B = (1 << 20) >> scale
        x0 = torch.empty(B, 128, dtype=torch.float64, device=DEV)
        cn.fill_uniform(x0, 0, 12345, -2.0, 2.0)
        return run("c2 lbfgs rosenbrock d128 f64", cn.Lbfgs(), cn.Rosenbrock(128), x0, lbfgs_bytes(8, 128), reps)
    if which == "c3":  # logistic n=256 d=64 fp32 L-BFGS, B = 2^18
        B, n, d, lam = (1 << 18) >> scale, 256, 64, 1e-2
        data = torch.empty(B, d * n + n, dtype=torch.float32, device=DEV)
        chunk = 1 << 14
        for lo in range(0, B, chunk):
            hi = min(B, lo + chunk)
            X = torch.rand(hi - lo, n, d, device=DEV, generator=gen) * 2 - 1
            ws = torch.randn(hi - lo, d, device=DEV, generator=gen)
            y = torch.sign(torch.einsum("bnd,bd->bn", X, ws) + 0.1 * torch.randn(hi - lo, n, device=DEV, generator=gen))
            y[y == 0] = 1
            data[lo:hi, : d * n] = X.transpose(1, 2).reshape(hi - lo, -1)
            data[lo:hi, d * n:] = y
            del X, ws, y
        x0 = torch.zeros(B, d, dtype=torch.float32, device=DEV)
        lb = lbfgs_bytes(4, d)
        return run("c3 lbfgs logistic n256 d64 f32", cn.Lbfgs(), cn.Logistic(data, n, d, lam), x0,
                   lambda it, nf: lb(it, nf) + (nf * 4 * (n * d + n)).sum(), reps)
    if which == "c4":  # BFGS Rosenbrock d=32 fp64, B = 2^19
        B = (1 << 19) >> scale
        x0 = torch.empty(B, 32, dtype=torch.float64, device=DEV)
        cn.fill_uniform(x0, 0, 12345, -2.0, 2.0)
        return run("c4 bfgs rosenbrock d32 f64", cn.Bfgs(), cn.Rosenbrock(32), x0,
                   lambda it, nf: (8 * (2 * 32 * 32 + 4 * 32) * it).sum(), reps)
    if which in ("c5", "c5t"):  # NewtonDescent dense quadratic d=64 fp64, B = 2^17; c5t = CNO_POLICY_DMMA_LU (tensor core)
        B, d = (1 << 17) >> scale, 64
        data = torch.empty(B, d * d + d, dtype=torch.float64, device=DEV)
        chunk = 1 << 13
        eye = torch.eye(d, dtype=torch.float64, device=DEV)
        for lo in range(0, B, chunk):
            hi = min(B, lo + chunk)
            M = torch.rand(hi - lo, d, d, dtype=torch.float64, device=DEV, generator=gen) * 2 - 1
            A = torch.bmm(M.transpose(1, 2), M) / d + eye
            A = (A + A.transpose(1, 2)) / 2
            data[lo:hi, : d * d] = A.transpose(1, 2).reshape(hi - lo, -1)
            data[lo:hi, d * d:] = torch.rand(hi - lo, d, dtype=torch.float64, device=DEV, generator=gen) * 2 - 1
        x0 = torch.empty(B, d, dtype=torch.float64, device=DEV)
        cn.fill_uniform(x0, 0, 12345, -2.0, 2.0)
        flops = lambda it: float(((2.0 / 3.0) * d ** 3 + 4.0 * d * d) * it.sum())  # noqa: E731  SURVEY.md 8(d)
        tensor = which == "c5t"
        rec = run(("c5t newton dense quadratic d64 f64 policy=dmma_lu (FP64 tensor-core factorisation)" if tensor
                   else "c5 newton dense quadratic d64 f64"),
                  cn.NewtonDescent(), cn.DenseQuadratic(data, d, policy=cn._lib.POLICY_DMMA_LU if tensor else None), x0,
                  lambda it, nf: (8 * (d * d + 3 * d) * it).sum(), reps)
        rec["algorithmic_TFLOPs"] = flops(np.full(B, rec["mean_iterations"])) / rec["kernel_ms"] / 1e9
        return rec
    if which in ("gd", "cg"):
        # Rosenbrock d=128 fp64, B = 2^18, iteration limit (these solvers crawl on Rosenbrock: the limit fixes
        # the work per instance).  Algorithmic bytes as in SURVEY.md 8(d): every evaluation the kernel makes
        # reads x and writes g; an iteration touches x, g, d once more.
        solver, limit = (cn.GradientDescent, 200) if which == "gd" else (cn.ConjugatedGradientDescent, 100)
        B, d = (1 << 18) >> scale, 128
        x0 = torch.empty(B, d, dtype=torch.float64, device=DEV)
        cn.fill_uniform(x0, 0, 12345, -2.0, 2.0)
        prog = cn.DefaultStoppingSolverProgress()
        prog.num_iterations = limit
        return run(f"{which} rosenbrock d128 f64 (iteration limit {limit})", solver(prog), cn.Rosenbrock(d), x0,
                   lambda it, nf: (8 * d * (2 * (nf - 3 * it) + 6 * it)).sum(), reps)
    if which == "hz":  # Lbfgs<F, 10, HagerZhang>, same workload as c2 at B = 2^18
        B = (1 << 18) >> scale
        x0 = torch.empty(B, 128, dtype=torch.float64, device=DEV)
        cn.fill_uniform(x0, 0, 12345, -2.0, 2.0)
        return run("hz lbfgs(HagerZhang) rosenbrock d128 f64", cn.Lbfgs(linesearch=cn.HagerZhang), cn.Rosenbrock(128),
                   x0, lbfgs_bytes(8, 128), reps)
    if which == "al":  # AugmentedLagrangian: Rosenbrock d=128 on a sphere (equality) + a halfspace
        B, d = (1 << 15) >> scale, 128
        x0 = torch.empty(B, d, dtype=torch.float64, device=DEV)
        cn.fill_uniform(x0, 0, 12345, -1.5, 1.5)
        rows = torch.zeros(2, d + 1, dtype=torch.float64, device=DEV)
        rows[0, d] = 16.0           # t - x.x = 0  (equality: on the sphere of radius 4)
        rows[1, :d] = 1.0           # sum(x) + 1 >= 0
        rows[1, d] = -1.0
        problem = cn.ConstrainedOptimizationProblem(cn.Rosenbrock(d), [1, 0], rows, 1)
        solver = cn.AugmentedLagrangian(problem)
        solver.stopping_progress.num_iterations = 20
        ms = []
        for _ in range(3):
            st, pr = solver.Minimize(cn.AugmentedLagrangeState(x0))
            ms.append(pr.launch.total_ms)
        return {"config": "al rosenbrock d128 f64 sphere+halfspace (outer limit 20)", "batch": B,
                "total_ms": float(np.mean(ms[1:])), "instances_per_s": B / float(np.mean(ms[1:])) * 1e3,
                "kernel_launches": pr.launch.kernel_launches,
                "mean_outer_iterations": float(pr.num_iterations.float().mean()),
                "mean_objective_evaluations": float(pr.nfev.float().mean()),
                "status_histogram": np.bincount(pr.status.cpu().numpy().astype(np.int64) + 1).tolist(),
                "max_violation_max": float(st.max_violation.max())}
    raise ValueError(f"unknown config {which!r}")


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    scale = int(sys.argv[sys.argv.index("--scale") + 1]) if "--scale" in sys.argv else 0
    which = args or ["c2", "c3", "c4", "c5"]  # "gd", "cg", "hz", "al": the SURVEY.md 8(f) rows, on request
    for w in which:
        if w.isdigit():  # (the value of --scale)
            continue
        print(json.dumps(run_config(w, scale)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
