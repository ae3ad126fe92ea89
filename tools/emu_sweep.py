#!/usr/bin/env python
"""tools/emu_sweep.py -- sweeps the DEVICE SOURCE, run on the CPU under the warp emulation of tests/emu,
against the oracle on edge-case inputs the GPU parity tests do not cover (NaN / Inf / huge / tiny starts,
starts at the minimiser, degenerate constraints).  A NaN must be a NaN on both sides (its sign / payload is
not part of the contract); everything else must agree bit for bit.

    python tools/emu_sweep.py [solvers] [headline] [al] [newton] [modes]      (default: all)

This is how the GradientDescent-HagerZhang failure-path defect was found (DESIGN.md 2.7)."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import oracle_binding as ob  # noqa: E402
import test_device_emulated as T  # noqa: E402

subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu")], check=True)
emu = C.CDLL(os.path.join(ROOT, "tests", "emu", "libcno_emu.so"))


def differing(a, b, keys):
    bad = []
    for k in keys:
        u, v = a[k], b[k]
        if u.dtype.kind == "f":
            nan = np.isnan(u)
            if not np.array_equal(nan, np.isnan(v)):
                bad.append(k + ":nan-pattern")
                continue
            u, v = np.where(nan, 0, u), np.where(nan, 0, v)
        if not np.array_equal(u.view(np.uint8), v.view(np.uint8)):
            bad.append(k)
    return bad


def run_solver(solver, hz, x0, limit):
    B = x0.shape[0]
    dtype = x0.dtype.type
    stop = ob.default_stop()
    stop.num_iterations = limit
    prob = T._problem(ob.FN_ROSENBROCK, x0)
    r = dict(x=np.zeros_like(x0), value=np.zeros(B, dtype), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B, dtype), f_delta=np.zeros(B, dtype), gradient_norm=np.zeros(B, dtype))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_minimize(solver, hz, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                            C.byref(out)) == 0
    o = ob.minimize(solver, ob.FN_ROSENBROCK, x0, stop=stop, linesearch=hz)
    return differing(r, o, T.SOLVER_KEYS), o


def poison(x0, trial, rng):
    if trial % 5 == 0:
        x0[0, int(rng.integers(0, x0.shape[1]))] = np.nan
    if trial % 7 == 0:
        x0[1, int(rng.integers(0, x0.shape[1]))] = np.inf
    if trial % 9 == 0:
        x0[0] = 1.0  # the minimiser: zero gradient


def sweep_solvers(trials=30):
    rng = np.random.default_rng(7)
    n = bad_n = 0
    for trial in range(trials):
        scale = float(rng.choice([0.05, 2.0, 30.0, 300.0, 1e6, 1e150]))
        for solver, hz, d, dt in ((ob.BFGS, 0, 8, np.float64), (ob.BFGS, 1, 8, np.float64), (ob.LBFGS, 0, 37, np.float32),
                                  (ob.LBFGS, 1, 37, np.float64), (ob.GRADIENT_DESCENT, 0, 37, np.float32),
                                  (ob.GRADIENT_DESCENT, 1, 8, np.float64), (ob.CONJUGATED_GRADIENT_DESCENT, 0, 2, np.float64)):
            with np.errstate(over="ignore"):
                x0 = rng.uniform(-scale, scale, (2, d)).astype(dt)
            poison(x0, trial, rng)
            bad, o = run_solver(solver, hz, x0, 8)
            n += 1
            if bad:
                bad_n += 1
                print("MISMATCH solver", solver, "hz", hz, "d", d, dt.__name__, "scale", scale, bad, flush=True)
    return n, bad_n


def sweep_headline(trials=36):
    rng = np.random.default_rng(21)
    n = bad_n = 0
    for trial in range(trials):
        scale = float(rng.choice([1e-3, 0.05, 2.0, 30.0, 300.0, 1e6, 1e100]))
        x0 = rng.uniform(-scale, scale, (2, 128))
        poison(x0, trial, rng)
        for hz in (0, 1):
            bad, o = run_solver(ob.LBFGS, hz, x0, 30)
            n += 1
            if bad:
                bad_n += 1
                print("MISMATCH headline shape, hz", hz, "scale", scale, bad, flush=True)
    return n, bad_n


def sweep_al(trials=24):
    rng = np.random.default_rng(11)
    n = bad_n = 0
    for trial in range(trials):
        d, B = 8, 2
        ne, ni = int(rng.integers(0, 4)), int(rng.integers(0, 4))
        kinds = [int(rng.integers(0, 2)) for _ in range(ne + ni)]
        scale = float(rng.choice([0.5, 1.5, 30.0]))
        x0 = rng.uniform(-scale, scale, (B, d))
        rows = rng.uniform(-1, 1, (B, ne + ni, d + 1))
        for i, k in enumerate(kinds):
            if k == ob.CON_SQNORM:
                rows[:, i, d] = rng.uniform(0.5, 4.0, B)
        if trial % 6 == 0:
            x0[0, 3] = np.nan
        if trial % 8 == 0 and ne + ni:
            rows[1] = 0.0
        stop = ob.al_default_stop()
        stop.num_iterations = 5
        kw = dict(outer_stop=stop, penalty0=None if trial % 3 else float(rng.choice([1e-9, 1.0, 1e6])),
                  eq0=None if trial % 4 else 0.3)
        fam = ob.FN_ROSENBROCK if trial % 2 else ob.FN_HALF_SQUARED_NORM
        o = ob.al_minimize(fam, x0, kinds, rows, ne, **kw)
        for device_inner in (False, True):
            r = T.emulated_al_minimize(emu, fam, x0, kinds, rows, ne, device_inner=device_inner, **kw)
            bad = differing(r, o, T.KEYS)
            n += 1
            if bad:
                bad_n += 1
                print("MISMATCH AugmentedLagrangian trial", trial, "device inner", device_inner, bad, flush=True)
    return n, bad_n


def sweep_newton(trials=24):
    """NewtonDescent on dense quadratics: well-conditioned, nearly singular, indefinite, rank-deficient,
    NaN / Inf entries -- the pivoted LU at d = 64 fp64 and at other shapes."""
    rng = np.random.default_rng(31)
    n = bad_n = 0
    for trial in range(trials):
        d, dt = ((64, np.float64), (12, np.float64), (64, np.float32))[trial % 3]
        B = 2
        M = rng.uniform(-1, 1, (B, d, d))
        A = np.einsum("bij,bkj->bik", M, M) / d
        kind = trial % 6
        if kind == 0:
            A = A + np.eye(d)                      # well conditioned
        elif kind == 1:
            A = A + 1e-12 * np.eye(d)              # nearly singular: the 1e-5 shift decides
        elif kind == 2:
            A = A - 0.5 * np.eye(d)                # indefinite
        elif kind == 3:
            A[:, :, d // 2] = 0.0                  # a zero column / row: rank deficient
            A[:, d // 2, :] = 0.0
        elif kind == 4:
            A = A + np.eye(d)
            A[0, 3, 5] = A[0, 5, 3] = np.nan
        else:
            A = (A + np.eye(d)) * 1e150 if dt == np.float64 else (A + np.eye(d)) * 1e30
        A = (A + A.transpose(0, 2, 1)) / 2
        b = rng.uniform(-1, 1, (B, d))
        with np.errstate(over="ignore", invalid="ignore"):
            data = np.concatenate([A.transpose(0, 2, 1).reshape(B, -1), b], 1).astype(dt)
        x0 = rng.uniform(-2, 2, (B, d)).astype(dt)
        prob = ob.Problem(ob.FN_DENSE_QUADRATIC, ob._np_dtype(x0), d, 0, 0.0, data.ctypes.data, data.shape[1],
                          ob.device_policy(x0.dtype), 0)
        stop = ob.default_stop()
        stop.num_iterations = 6
        r = dict(x=np.zeros_like(x0), value=np.zeros(B, dt), gradient=np.zeros_like(x0),
                 num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
                 x_delta=np.zeros(B, dt), f_delta=np.zeros(B, dt), gradient_norm=np.zeros(B, dt))
        out = ob.BatchOut(*[r[k].ctypes.data for k, _ in ob.BatchOut._fields_])
        assert emu.emu_newton(C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop), C.byref(out)) == 0
        o = ob.minimize(ob.NEWTON, ob.FN_DENSE_QUADRATIC, x0, data=data, stop=stop)
        bad = differing(r, o, T.SOLVER_KEYS)
        n += 1
        if bad:
            bad_n += 1
            print("MISMATCH newton d", d, dt.__name__, "kind", kind, bad, o["status"], o["num_iterations"], flush=True)
    return n, bad_n


def sweep_modes(trials=24):
    """Lbfgs on a Second-mode function (diagonal preconditioner, lbfgs.h:116-139) and the Eigen-SSE2 parity policy."""
    rng = np.random.default_rng(5)
    n = bad_n = 0
    for trial in range(trials):
        scale = float(rng.choice([1e-3, 2.0, 30.0, 300.0, 1e6, 1e100]))
        for d, mode, policy in ((37, 2, ob.POLICY_DMMA_TREE), (128, 2, ob.POLICY_DMMA_TREE), (128, 0, ob.POLICY_EIGEN_SSE2)):
            x0 = rng.uniform(-scale, scale, (2, d))
            poison(x0, trial, rng)
            stop = ob.default_stop()
            stop.num_iterations = 25
            prob = ob.Problem(ob.FN_ROSENBROCK, 0, d, 0, 0.0, None, 0, policy, mode)
            r = dict(x=np.zeros_like(x0), value=np.zeros(2), gradient=np.zeros_like(x0), num_iterations=np.zeros(2, np.uint32),
                     status=np.zeros(2, np.int8), nfev=np.zeros(2, np.uint32), x_delta=np.zeros(2), f_delta=np.zeros(2),
                     gradient_norm=np.zeros(2))
            out = ob.BatchOut(*[r[k].ctypes.data for k, _ in ob.BatchOut._fields_])
            assert emu.emu_minimize(ob.LBFGS, 0, C.byref(prob), C.c_longlong(2), C.c_void_p(x0.ctypes.data), C.byref(stop),
                                    C.byref(out)) == 0
            o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop, policy=policy, mode=mode)
            bad = differing(r, o, T.SOLVER_KEYS)
            n += 1
            if bad:
                bad_n += 1
                print("MISMATCH d", d, "mode", mode, "policy", policy, "scale", scale, bad, flush=True)
    return n, bad_n


def main():
    which = sys.argv[1:] or ["solvers", "headline", "al", "newton", "modes"]
    for name, fn in (("solvers", sweep_solvers), ("headline", sweep_headline), ("al", sweep_al), ("newton", sweep_newton),
                     ("modes", sweep_modes)):
        if name in which:
            t0 = time.time()
            n, bad = fn()
            print(f"{name}: {n} cases, {bad} mismatches, {time.time() - t0:.0f} s", flush=True)


if __name__ == "__main__":
    main()
