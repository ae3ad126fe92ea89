"""DEVICE SOURCE executed on the CPU (no GPU needed).

csrc/cno_auglag.cuh (the composite functor AugLagFn and the auto-scale / outer-step / finalize
kernels) and the solver kernels (csrc/cno_lbfgs.cuh, cno_bfgs.cuh, cno_descent.cuh with
cno_linesearch.cuh) are compiled by g++ against tests/emu/warp_emu.h -- 32 lock-step threads per
warp, the warp intrinsics as publish/barrier/read, the FP64 tensor-core reduction restated with the
arithmetic of tools/dmma_probe.cu -- and driven through the outer loop of csrc/cno_api.cu::al_run,
restated here in numpy.  The inner solve is either the oracle's L-BFGS on the composite or the fused
device kernel itself under emulation.  Everything must equal the oracle -- which equals the
reference's own headers -- bit for bit; the GPU-validated kernels are run too, to show that the
emulation reproduces what the GPU computes.

The same paths run on the GPU in tests/test_al_gpu.py; this is their `-m "not gpu"` counterpart."""
import ctypes as C
import glob
import os
import subprocess

import edge_sums as es
import numpy as np
import pytest

from oracle import oracle_binding as ob

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(HERE, "emu")
GOLDEN = os.path.join(HERE, "golden")
KEYS = ("num_iterations", "status", "nfev", "x", "equality_multipliers", "inequality_multipliers", "penalty",
        "max_violation", "max_lagrangian_gradient", "x_delta", "f_delta", "gradient_norm")
COMPOSITE, AUTOSCALE, OUTER_STEP, FINALIZE, INNER = range(5)


class EmuArrays(C.Structure):  # tests/emu/emu_auglag.cc
    _fields_ = [(n, C.c_void_p) for n in (
        "x", "x_work", "lam", "mu", "penalty", "prev_penalty", "max_violation", "max_lagrangian_gradient",
        "num_iterations", "status", "nfev", "inner_nfev", "x_delta", "f_delta", "gradient_norm", "best_recorded",
        "best_x", "best_lambda", "best_mu", "best_penalty", "best_objective", "best_violation", "best_kkt",
        "remaining")]


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    return C.CDLL(os.path.join(EMU_DIR, "libcno_emu.so"))


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def _problem(family, x0, policy=None, data=None):
    return ob.Problem(family, ob._np_dtype(x0), x0.shape[1], 0, 0.0, data.ctypes.data if data is not None else None,
                      data.shape[1] if data is not None else 0, ob.device_policy(x0.dtype) if policy is None else policy, 0)


def emulated_al_minimize(emu, family, x0, kinds, rows, n_eq, *, outer_stop=None, config=None, inner_stop=None,
                         eq0=None, ineq0=None, penalty0=None, device_inner=False):
    """csrc/cno_api.cu::al_run with the kernels of csrc/cno_auglag.cuh run under the warp emulation."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    dt = x0.dtype
    prob = _problem(family, x0)
    k, keep = ob._constraints(kinds, rows, n_eq, dt, B, d)
    ne, ni = k.n_eq, k.n_ineq
    cfg = config if config is not None else ob.al_default_config()
    ostop = outer_stop if outer_stop is not None else ob.al_default_stop()
    istop = inner_stop if inner_stop is not None else ob.default_stop()
    full = lambda v, n: np.ascontiguousarray(np.broadcast_to(np.asarray(0.0 if v is None else v, dt), (B, n)))  # noqa: E731
    s = dict(x=x0.copy(), x_work=np.zeros_like(x0), lam=full(eq0, ne).copy(), mu=full(ineq0, ni).copy(),
             penalty=np.ascontiguousarray(np.broadcast_to(np.asarray(0.0 if penalty0 is None else penalty0, dt), (B,))).copy(),
             max_violation=np.zeros(B, dt), max_lagrangian_gradient=np.zeros(B, dt),
             num_iterations=np.zeros(B, np.uint32), status=np.full(B, -1, np.int8), nfev=np.zeros(B, np.uint32),
             inner_nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B, dt), f_delta=np.zeros(B, dt),
             gradient_norm=np.zeros(B, dt), best_recorded=np.zeros(B, np.int8), best_x=np.zeros_like(x0),
             best_lambda=np.zeros((B, ne), dt), best_mu=np.zeros((B, ni), dt), best_penalty=np.zeros(B, dt),
             best_objective=np.zeros(B, dt), best_violation=np.zeros(B, dt), best_kkt=np.zeros(B, dt),
             remaining=np.zeros(1, np.int32))
    s["prev_penalty"] = s["penalty"].copy()
    arr = EmuArrays(*[_ptr(s[n]) for n, _ in EmuArrays._fields_])

    def kernel(op):
        rc = emu.emu_al(op, C.byref(prob), C.byref(k), C.c_longlong(B), C.byref(arr), C.byref(cfg), C.byref(ostop),
                        None, None, None)
        assert rc == 0

    outer = 0
    while True:
        outer += 1
        if outer == 1 and cfg.auto_scale_initial_penalty:
            kernel(AUTOSCALE)
        inner = ob.Stop.from_buffer_copy(istop)  # working copy of the template, ConfigureInnerSubproblem
        inner.f_delta = 0.0
        if outer == 1 and (ne > 0 or ni > 0) and cfg.warmup_max_inner_iterations > 0:
            inner.num_iterations = cfg.warmup_max_inner_iterations
            inner.gradient_norm = float(dt.type(cfg.warmup_inner_gradient_tolerance))
        active = (s["status"] == 0) | (s["status"] == -1)  # AugLagFn::active: the inner kernel skips the rest
        idx = np.nonzero(active)[0]
        if device_inner:  # the fused L-BFGS kernel itself on the composite, incl. its active() skip hook
            assert emu.emu_al(INNER, C.byref(prob), C.byref(k), C.c_longlong(B), C.byref(arr), C.byref(cfg),
                              C.byref(ostop), C.byref(inner), None, None) == 0
        elif idx.size:
            xw = np.zeros((idx.size, d), dt)
            nf = np.zeros(idx.size, np.uint32)
            rows_a = np.ascontiguousarray(keep[1][idx]) if keep[1].ndim == 3 else keep[1]
            ka, keep_a = ob._constraints(keep[0], rows_a, n_eq, dt, idx.size, d)
            xa, la, ma, pa = (np.ascontiguousarray(s[n][idx]) for n in ("x", "lam", "mu", "penalty"))  # kept alive
            rc = ob.oracle_lib().cno_al_oracle_inner_minimize(
                C.byref(prob), C.byref(ka), C.c_int64(idx.size), C.c_void_p(xa.ctypes.data),
                C.c_void_p(_ptr(la)), C.c_void_p(_ptr(ma)), C.c_void_p(pa.ctypes.data), C.byref(inner),
                C.c_void_p(xw.ctypes.data), C.c_void_p(nf.ctypes.data), 0)
            assert rc == 0
            s["x_work"][idx] = xw
            s["inner_nfev"][idx] = nf
            del keep_a
        s["remaining"][0] = 0
        kernel(OUTER_STEP)
        if s["remaining"][0] == 0:
            break
    kernel(FINALIZE)
    return dict(x=s["x"], equality_multipliers=s["lam"], inequality_multipliers=s["mu"], penalty=s["penalty"],
                max_violation=s["max_violation"], max_lagrangian_gradient=s["max_lagrangian_gradient"],
                num_iterations=s["num_iterations"], status=s["status"], nfev=s["nfev"], x_delta=s["x_delta"],
                f_delta=s["f_delta"], gradient_norm=s["gradient_norm"])


def _assert_same(a, b):
    for key in KEYS:
        assert np.array_equal(a[key].view(np.uint8), b[key].view(np.uint8)), f"{key} differs"


@pytest.mark.parametrize("family,dtype,d", [(ob.FN_ROSENBROCK, np.float64, 8), (ob.FN_ROSENBROCK, np.float64, 37),
                                            (ob.FN_ROSENBROCK, np.float64, 128), (ob.FN_ROSENBROCK, np.float32, 8),
                                            (ob.FN_HALF_SQUARED_NORM, np.float64, 8)])
def test_device_composite_functor_equals_oracle(emu, family, dtype, d):
    """AugLagFn::operator() == ToAugmentedLagrangian(...)(x, &grad) of the oracle: value and gradient, all bits;
    zero / positive / inactive-side multipliers, penalty 0 (no penalty and no inequality part) and > 0."""
    rng = np.random.default_rng(d)
    B = 12
    x = rng.uniform(-1.5, 1.5, (B, d)).astype(dtype)
    kinds = [ob.CON_AFFINE, ob.CON_SQNORM, ob.CON_AFFINE, ob.CON_SQNORM]
    rows = rng.uniform(-1, 1, (B, 4, d + 1)).astype(dtype)
    rows[:, 3, d] = d / 2.0  # t - x.x > mu / rho for some instances (inactive side), not for others
    lam = rng.uniform(-1, 1, (B, 2)).astype(dtype)
    lam[::3, 0] = 0.0  # the MulExpression c == 0 short cut
    mu = rng.uniform(0, 2, (B, 2)).astype(dtype)
    rho = rng.uniform(0.5, 3, B).astype(dtype)
    rho[1::4] = 0.0
    prob = _problem(family, x)
    k, keep = ob._constraints(kinds, rows, 2, x.dtype, B, d)
    arr = EmuArrays()
    arr.lam, arr.mu, arr.penalty = lam.ctypes.data, mu.ctypes.data, rho.ctypes.data
    v, g = np.zeros(B, dtype), np.zeros_like(x)
    cfg, stop = ob.al_default_config(), ob.al_default_stop()
    assert emu.emu_al(COMPOSITE, C.byref(prob), C.byref(k), C.c_longlong(B), C.byref(arr), C.byref(cfg), C.byref(stop),
                      C.c_void_p(x.ctypes.data), C.c_void_p(v.ctypes.data), C.c_void_p(g.ctypes.data)) == 0
    vo, go = ob.al_evaluate(family, x, kinds, rows, 2, lam, mu, rho)
    assert np.array_equal(v.view(np.uint8), vo.view(np.uint8))
    assert np.array_equal(g.view(np.uint8), go.view(np.uint8))


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "al_*.npz"))))
def test_emulated_device_loop_matches_reference_fixtures(emu, path):
    """The committed outputs of the reference's own headers (tests/golden/make_golden_al.py)."""
    z = np.load(path)
    n = min(4, z["x0"].shape[0])  # the emulation runs 32 threads per warp: keep it to a few instances
    stop = ob.al_default_stop()
    stop.num_iterations = int(z["outer_limit"])
    r = emulated_al_minimize(emu, int(z["family"]), z["x0"][:n], z["kinds"], z["rows"][:n], int(z["n_eq"]), outer_stop=stop)
    for key in KEYS:
        assert np.array_equal(r[key].view(np.uint8), z[key][:n].view(np.uint8)), key


@pytest.mark.parametrize("family,dtype,d,n_eq,per_instance", [
    (ob.FN_ROSENBROCK, np.float64, 2, 1, False), (ob.FN_ROSENBROCK, np.float64, 8, 3, True),
    (ob.FN_ROSENBROCK, np.float64, 37, 0, True), (ob.FN_ROSENBROCK, np.float32, 8, 1, True),
    (ob.FN_HALF_SQUARED_NORM, np.float64, 8, 2, False)])
def test_emulated_device_loop_equals_oracle(emu, family, dtype, d, n_eq, per_instance):
    B = 5
    rng = np.random.default_rng(200 + d)
    x0 = ob.fill_uniform((B, d), 0, 31 + d, -1.5, 1.5, dtype)
    kinds = [ob.CON_AFFINE, ob.CON_SQNORM, ob.CON_AFFINE]
    shape = (B, 3, d + 1) if per_instance else (3, d + 1)
    rows = rng.uniform(-1, 1, shape).astype(dtype)
    rows[..., 1, d] = 2.0 + rng.uniform(0, 1, shape[:-2])
    stop = ob.al_default_stop()
    stop.num_iterations = 8
    _assert_same(emulated_al_minimize(emu, family, x0, kinds, rows, n_eq, outer_stop=stop),
                 ob.al_minimize(family, x0, kinds, rows, n_eq, outer_stop=stop))
    # user-set multipliers / penalty (no auto-scaling), non-default config and inner preset
    cfg = ob.al_default_config()
    cfg.warmup_max_inner_iterations, cfg.violation_shrink_ratio, cfg.multiplier_max = 0, 0.5, 5.0
    kw = dict(outer_stop=stop, config=cfg, inner_stop=ob.conservative_stop(), eq0=0.25, ineq0=0.5, penalty0=2.0)
    _assert_same(emulated_al_minimize(emu, family, x0, kinds, rows, n_eq, **kw),
                 ob.al_minimize(family, x0, kinds, rows, n_eq, **kw))


def test_emulated_device_loop_known_answers(emu):
    """augmented_lagrangian_test.cc:492-539 (EqualityOnlyQuadratic), :627-692 (FeasibleStart, NoConstraints)."""
    r = emulated_al_minimize(emu, ob.FN_HALF_SQUARED_NORM, np.array([[5.0, 5.0]]), [ob.CON_AFFINE], [[1.0, 0.0, 1.0]], 1,
                             penalty0=1.0)
    assert abs(r["x"][0, 0] - 1.0) <= 1e-3 and abs(r["x"][0, 1]) <= 1e-3
    assert abs(r["equality_multipliers"][0, 0] + 1.0) <= 1e-2
    _assert_same(r, ob.al_minimize(ob.FN_HALF_SQUARED_NORM, np.array([[5.0, 5.0]]), [ob.CON_AFFINE], [[1.0, 0.0, 1.0]], 1,
                                   penalty0=1.0))
    r = emulated_al_minimize(emu, ob.FN_HALF_SQUARED_NORM, np.array([[0.0, 0.0]]), [ob.CON_AFFINE], [[0.0, 0.0, 0.0]], 1,
                             penalty0=1.0)
    assert r["status"][0] == 6 and r["num_iterations"][0] <= 5
    r = emulated_al_minimize(emu, ob.FN_HALF_SQUARED_NORM, np.array([[5.0, 5.0]]), [], np.zeros((0, 3)), 0, penalty0=1.0)
    assert r["status"][0] == 6 and np.all(np.abs(r["x"][0]) <= 1e-3)


# ---- the fused inner kernel too: the whole device path of the row under emulation ----------------
@pytest.mark.parametrize("family,dtype,d,n_eq", [(ob.FN_ROSENBROCK, np.float64, 128, 1), (ob.FN_ROSENBROCK, np.float32, 8, 1)])
def test_emulated_device_loop_with_the_device_inner_kernel(emu, family, dtype, d, n_eq):
    """lbfgs_minimize_kernel<AugLagFn<Obj>> (with its active() skip of finished instances) + the outer-loop
    kernels, all device source, all under emulation == the oracle, bit for bit."""
    B = 2  # 32 lock-step threads per warp: a few instances keep this to seconds
    rng = np.random.default_rng(300 + d)
    x0 = ob.fill_uniform((B, d), 0, 57 + d, -1.5, 1.5, dtype)
    kinds = [ob.CON_AFFINE, ob.CON_SQNORM, ob.CON_AFFINE]
    rows = rng.uniform(-1, 1, (B, 3, d + 1)).astype(dtype)
    rows[:, 1, d] = 2.0 + rng.uniform(0, 1, B)
    stop = ob.al_default_stop()
    stop.num_iterations = 2 if dtype == np.float32 else 3  # (fp64 d = 8 / 37 and the half norm: the host-loop test below)
    _assert_same(emulated_al_minimize(emu, family, x0, kinds, rows, n_eq, outer_stop=stop, device_inner=True),
                 ob.al_minimize(family, x0, kinds, rows, n_eq, outer_stop=stop))


# ---- fidelity of the emulation itself: GPU-validated kernels under emulation == oracle --------------
SOLVER_KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")


@pytest.mark.parametrize("solver,hz,dtype,d,limit", [
    (ob.LBFGS, 0, np.float64, 2, 10000), (ob.LBFGS, 0, np.float64, 37, 40), (ob.LBFGS, 0, np.float32, 37, 20),
    (ob.LBFGS, 0, np.float64, 128, 50), (ob.LBFGS, 1, np.float64, 128, 25),  # the headline shape
    (ob.LBFGS, 1, np.float64, 8, 10000), (ob.BFGS, 0, np.float64, 8, 10000), (ob.BFGS, 1, np.float64, 2, 10000),
    (ob.GRADIENT_DESCENT, 0, np.float64, 8, 40), (ob.GRADIENT_DESCENT, 1, np.float64, 8, 40),
    (ob.CONJUGATED_GRADIENT_DESCENT, 0, np.float64, 8, 8)])
def test_emulation_reproduces_gpu_validated_kernels(emu, solver, hz, dtype, d, limit):
    """The L-BFGS / BFGS / descent kernels (MoreThuente and HagerZhang) are bit-identical to the oracle on the
    GPU; run under the emulation they must be too -- that is what makes the emulated AugmentedLagrangian
    results above evidence about the device code rather than about the emulator."""
    B = 2
    x0 = ob.fill_uniform((B, d), 0, 900 + d, -2.0, 2.0, dtype)
    stop = ob.default_stop()
    stop.num_iterations = limit
    prob = _problem(ob.FN_ROSENBROCK, x0)
    r = dict(x=np.zeros_like(x0), value=np.zeros(B, dtype), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B, dtype), f_delta=np.zeros(B, dtype), gradient_norm=np.zeros(B, dtype))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_minimize(solver, hz, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                            C.byref(out)) == 0
    o = ob.minimize(solver, ob.FN_ROSENBROCK, x0, stop=stop, linesearch=hz)
    for key in SOLVER_KEYS:
        assert np.array_equal(r[key].view(np.uint8), o[key].view(np.uint8)), key


@pytest.mark.parametrize("solver,hz,dtype,d", [
    (ob.LBFGS, 0, np.float64, 8), (ob.LBFGS, 1, np.float64, 8), (ob.LBFGS, 0, np.float32, 37), (ob.BFGS, 0, np.float64, 8),
    (ob.GRADIENT_DESCENT, 0, np.float64, 8), (ob.CONJUGATED_GRADIENT_DESCENT, 0, np.float64, 8)])
def test_emulated_kernels_follow_progress_update_under_random_settings(emu, solver, hz, dtype, d):
    """The device progress_update (csrc/cno_progress.cuh: the order of Progress::Update's tests, the allowed-violation
    counters, relative thresholds, the past-f ring and its square-root-free plateau pre-test) against the oracle under
    six random Progress settings per kernel family -- every output bit for bit."""
    rng = np.random.default_rng(77 + 10 * solver + hz + d)
    B = 3
    seen = set()
    for k in range(6):
        stop = ob.default_stop()
        stop.num_iterations = int(rng.choice([3, 7, 25, 40]))
        stop.x_delta = float(rng.choice([0.0, 1e-9, 1e-4, 1e-2]))
        stop.x_delta_violations = int(rng.integers(1, 4))
        stop.f_delta = float(rng.choice([0.0, 0.0, 1e-8, 1e-3, 1e-1]))
        stop.f_delta_violations = int(rng.integers(1, 4))
        stop.f_delta_relative = int(rng.integers(0, 2))
        stop.gradient_norm = float(rng.choice([0.0, 1e-5, 1e-2, 1.0]))
        stop.gradient_norm_relative = int(rng.integers(0, 2))
        stop.past = int(rng.integers(0, 9))
        stop.past_delta = float(rng.choice([1e-10, 1e-6, 1e-2]))
        x0 = ob.fill_uniform((B, d), 31 * k, 808 + d, -2.0, 2.0, dtype)
        prob = _problem(ob.FN_ROSENBROCK, x0)
        r = dict(x=np.zeros_like(x0), value=np.zeros(B, dtype), gradient=np.zeros_like(x0),
                 num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
                 x_delta=np.zeros(B, dtype), f_delta=np.zeros(B, dtype), gradient_norm=np.zeros(B, dtype))
        out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
        assert emu.emu_minimize(solver, hz, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                                C.byref(out)) == 0
        o = ob.minimize(solver, ob.FN_ROSENBROCK, x0, stop=stop, linesearch=hz)
        for key in SOLVER_KEYS:
            assert np.array_equal(r[key].view(np.uint8), o[key].view(np.uint8)), (k, key, [getattr(stop, f[0]) for f in ob.Stop._fields_])
        seen.update(int(v) for v in r["status"])
    if solver == ob.LBFGS and d == 8:
        assert len(seen) >= 2, seen   # (the sweep is not all iteration limits)


def test_gradient_descent_hager_zhang_failed_search_rebuilds_point_from_step(emu):
    """Found by sweeping the emulated kernels against the oracle: when HagerZhang fails (non-finite
    evaluations) GradientDescent's next point is x - rate * g with rate = 0 (gradient_descent.h:72), i.e. NaN
    wherever g is not finite -- not the start state the search leaves behind.  NaN / Inf / huge starts."""
    x0 = np.array([[np.nan, 1.0, -0.5, 2.0, 0.3, -1.2, 0.8, 0.1], [0.4, -0.7, 1.1, 0.2, -0.9, 0.6, 1.3, np.inf],
                   [3e5, -2e5, 1e5, 4e5, -3e5, 2e5, -1e5, 5e5]])
    B, d = x0.shape
    stop = ob.default_stop()
    stop.num_iterations = 10
    prob = _problem(ob.FN_ROSENBROCK, x0)
    r = dict(x=np.zeros_like(x0), value=np.zeros(B), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B), f_delta=np.zeros(B), gradient_norm=np.zeros(B))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_minimize(ob.GRADIENT_DESCENT, 1, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data),
                            C.byref(stop), C.byref(out)) == 0
    o = ob.minimize(ob.GRADIENT_DESCENT, ob.FN_ROSENBROCK, x0, stop=stop, linesearch=ob.LS_HAGER_ZHANG)
    for key in SOLVER_KEYS:
        u, v = r[key], o[key]
        if u.dtype.kind == "f":  # a NaN must be a NaN in both; its sign / payload is not part of the contract
            nan = np.isnan(u)
            assert np.array_equal(nan, np.isnan(v)), key
            u, v = np.where(nan, 0, u), np.where(nan, 0, v)
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8)), key
    assert np.isnan(o["x"][0]).sum() > 1  # the oracle (= reference) really spreads the NaN through 0 * g


def _spd_data(B, d, seed, dtype=np.float64):
    rng = np.random.default_rng(seed)
    M = rng.uniform(-1, 1, (B, d, d))
    A = np.einsum("bij,bkj->bik", M, M) / d + np.eye(d)
    A = (A + A.transpose(0, 2, 1)) / 2
    b = rng.uniform(-1, 1, (B, d))
    return np.concatenate([A.transpose(0, 2, 1).reshape(B, -1), b], 1).astype(dtype)


@pytest.mark.parametrize("family,dtype,d", [(ob.FN_DENSE_QUADRATIC, np.float64, 64), (ob.FN_DENSE_QUADRATIC, np.float32, 64),
                                            (ob.FN_DENSE_QUADRATIC, np.float64, 12), (ob.FN_ROSENBROCK, np.float64, 2)])
def test_emulation_reproduces_the_newton_kernel(emu, family, dtype, d):
    """newton_minimize_kernel under emulation (the TMA bulk copy as a memcpy) == the oracle, as on the GPU."""
    B = 2
    x0 = ob.fill_uniform((B, d), 0, 5, -2.0, 2.0, dtype)
    data = _spd_data(B, d, 9, dtype) if family == ob.FN_DENSE_QUADRATIC else None
    prob = ob.Problem(family, ob._np_dtype(x0), d, 0, 0.0, data.ctypes.data if data is not None else None,
                      data.shape[1] if data is not None else 0, ob.device_policy(x0.dtype), 0)
    stop = ob.default_stop()
    r = dict(x=np.zeros_like(x0), value=np.zeros(B, dtype), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B, dtype), f_delta=np.zeros(B, dtype), gradient_norm=np.zeros(B, dtype))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_newton(C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop), C.byref(out)) == 0
    o = ob.minimize(ob.NEWTON, family, x0, data=data, stop=stop)
    for key in SOLVER_KEYS:
        assert np.array_equal(r[key].view(np.uint8), o[key].view(np.uint8)), key


@pytest.mark.parametrize("family,dtype,d", [(ob.FN_DENSE_QUADRATIC, np.float64, 64), (ob.FN_DENSE_QUADRATIC, np.float32, 64),
                                            (ob.FN_DENSE_QUADRATIC, np.float64, 12), (ob.FN_ROSENBROCK, np.float64, 8),
                                            (ob.FN_ROSENBROCK, np.float64, 2)])
def test_emulation_condition_hessian_kernel_equals_the_oracle(emu, family, dtype, d):
    """condition_hessian_kernel (Progress::condition_hessian on request, progress.h:203-210) under emulation == the
    oracle == the reference's own Progress::Update (tests/test_oracle_pins.py) bit for bit: the Frobenius sums in the
    policy's order, the inverse as d re-solves with one factorisation."""
    B = 3
    x = ob.fill_uniform((B, d), 0, 6, -2.0, 2.0, dtype)
    data = _spd_data(B, d, 10, dtype) if family == ob.FN_DENSE_QUADRATIC else None
    prob = ob.Problem(family, ob._np_dtype(x), d, 0, 0.0, data.ctypes.data if data is not None else None,
                      data.shape[1] if data is not None else 0, ob.device_policy(x.dtype), 2)
    out = np.zeros(B, dtype)
    assert emu.emu_condition_hessian(C.byref(prob), C.c_longlong(B), C.c_void_p(x.ctypes.data), C.c_void_p(out.ctypes.data)) == 0
    o = ob.condition_hessian(family, x, data=data)
    assert np.array_equal(out.view(np.uint8), o.view(np.uint8))
    assert np.all(out >= d * 0.99)  # ||H|| ||H^-1|| >= ||I||_F^2 / ... : at least d for the Frobenius norm


def _newton_pivot_cases(d=64, B=8):
    """Symmetric indefinite matrices (pivots move in every panel), exact ties, a zero row / column, a NaN entry, an
    anti-diagonal permutation matrix."""
    rng = np.random.default_rng(17)
    A = np.zeros((B, d, d))
    for b in range(B):
        M = rng.uniform(-1, 1, (d, d))
        S = (M + M.T) / 2
        if b == 1:
            S = np.round(S * 4) / 4
        if b == 2:
            S[:, 5] = 0.0
            S[5, :] = 0.0
        if b == 3:
            S[7, 9] = S[9, 7] = np.nan
        if b == 4:
            S = np.eye(d)[::-1].copy()
        A[b] = S
    bvec = rng.uniform(-1, 1, (B, d))
    return np.ascontiguousarray(np.concatenate([A.transpose(0, 2, 1).reshape(B, -1), bvec], axis=1))


@pytest.mark.parametrize("store", ["shared_memory"])
@pytest.mark.parametrize("case", ["spd", "pivoting", "huge", "tiny"])
def test_emulation_tensor_core_newton_equals_the_fused_oracle(emu, case, store):
    """csrc/cno_newton_dmma.cuh (CNO_POLICY_DMMA_LU) under emulation, DMMA.8x8x4 as the FMA chain of tools/dmma_probe.cu:
    the BLOCKED elimination (register panels, U12 in the B-fragment layout, tensor-core trailing update, blocked
    substitutions) equals the oracle's UNBLOCKED lu_solve with fused multiply-subtracts bit for bit."""
    d = 64
    if case == "spd":
        B, data = 3, _spd_data(3, d, 9)
    else:
        data = _newton_pivot_cases(d) * {"pivoting": 1.0, "huge": 1e150, "tiny": 1e-150}[case]
        B = data.shape[0]
    x0 = ob.fill_uniform((B, d), 0, 5, -2.0, 2.0, np.float64)
    # (the matrix lives in the emulated warp's shared memory, in fragment order)
    prob = ob.Problem(ob.FN_DENSE_QUADRATIC, ob._np_dtype(x0), d, 0, 0.0,
                      data.ctypes.data, data.shape[1], ob.POLICY_DMMA_LU, 0)
    stop = ob.default_stop()
    stop.num_iterations = 4
    r = dict(x=np.zeros_like(x0), value=np.zeros(B), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B), f_delta=np.zeros(B), gradient_norm=np.zeros(B))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_newton(C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop), C.byref(out)) == 0
    o = ob.minimize(ob.NEWTON, ob.FN_DENSE_QUADRATIC, x0, data=data, stop=stop, policy=ob.POLICY_DMMA_LU)
    for key in SOLVER_KEYS:
        u, v = r[key], o[key]
        if u.dtype.kind == "f":  # (a NaN's sign / payload is not part of the contract)
            nan = np.isnan(u)
            assert np.array_equal(nan, np.isnan(v)), key
            u, v = np.where(nan, 0, u), np.where(nan, 0, v)
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8)), key
    if case == "spd":  # the policy changes the rounding, not the answer
        o0 = ob.minimize(ob.NEWTON, ob.FN_DENSE_QUADRATIC, x0, data=data, stop=stop)
        assert not np.array_equal(o0["x"].view(np.uint64), o["x"].view(np.uint64))
        assert np.allclose(o0["x"], o["x"], rtol=1e-9, atol=1e-12)


def test_emulation_reproduces_the_logistic_kernel(emu):
    """L-BFGS on the logistic-regression functor (csrc/cno_logistic.cuh): per-instance data staged by a TMA bulk
    copy into shared memory -- under emulation a memcpy -- and evaluated by a TEAM of two warps (solver warp + helper warp, 64 lock-step threads meeting at the named
    barrier; emu::run_team).  Three instances through one team: the data are re-staged and the helper re-armed."""
    B, n, d, lam = 3, 256, 64, 1e-2
    rng = np.random.default_rng(3)
    X = rng.uniform(-1, 1, (B, n, d)).astype(np.float32)
    wstar = rng.normal(size=(B, d)).astype(np.float32)
    y = np.sign(np.einsum("bnd,bd->bn", X, wstar) + 0.1 * rng.normal(size=(B, n))).astype(np.float32)
    y[y == 0] = 1
    data = np.ascontiguousarray(np.concatenate([X.transpose(0, 2, 1).reshape(B, -1), y], axis=1))
    x0 = np.zeros((B, d), np.float32)
    prob = ob.Problem(ob.FN_LOGISTIC, ob._np_dtype(x0), d, n, lam, data.ctypes.data, data.shape[1],
                      ob.device_policy(x0.dtype), 0)
    stop = ob.default_stop()
    r = dict(x=np.zeros_like(x0), value=np.zeros(B, np.float32), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B, np.float32), f_delta=np.zeros(B, np.float32), gradient_norm=np.zeros(B, np.float32))
    out = ob.BatchOut(*[r[k].ctypes.data for k, _ in ob.BatchOut._fields_])
    assert emu.emu_logistic(C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop), C.byref(out)) == 0
    o = ob.minimize(ob.LBFGS, ob.FN_LOGISTIC, x0, data=data, n=n, param=lam)
    for key in SOLVER_KEYS:
        assert np.array_equal(r[key].view(np.uint8), o[key].view(np.uint8)), key


def test_emulated_logistic_team_evaluates_like_the_oracle(emu):
    """The functor alone, through both commands of its helper warp (value only / value + gradient), at points chosen
    to reach every branch of the shared exp / log1p kernels: small weights, margins of a few tens, and margins beyond
    the clamp (|m| > 87: exp returns 0) and just inside it (2^k with k near -126: the scaling is one multiplication on
    the device side, ldexpf in the oracle)."""
    B, n, d, lam = 6, 256, 64, 1e-2
    rng = np.random.default_rng(11)
    X = rng.uniform(-1, 1, (B, n, d)).astype(np.float32)
    y = np.sign(rng.normal(size=(B, n))).astype(np.float32)
    data = np.ascontiguousarray(np.concatenate([X.transpose(0, 2, 1).reshape(B, -1), y], axis=1))
    scales = np.array([0.0, 0.1, 1.0, 5.0, 19.0, 40.0], np.float32)   # |m| up to ~ 4 scale sqrt(d / 3)
    x = (rng.normal(size=(B, d)).astype(np.float32) * scales[:, None]).astype(np.float32)
    prob = ob.Problem(ob.FN_LOGISTIC, ob._np_dtype(x), d, n, lam, data.ctypes.data, data.shape[1],
                      ob.device_policy(x.dtype), 0)
    fo, go = ob.evaluate(ob.FN_LOGISTIC, x, data=data, n=n, param=lam)
    m = y * np.einsum("bnd,bd->bn", X.astype(np.float64), x.astype(np.float64))
    assert np.abs(m).max() > 100 and ((np.abs(m) > 80) & (np.abs(m) < 87)).any()   # the clamp and the 2^-126 neighbourhood are hit
    f = np.zeros(B, np.float32)
    g = np.zeros((B, d), np.float32)
    emu.emu_logistic_evaluate.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    assert emu.emu_logistic_evaluate(C.byref(prob), B, x.ctypes.data, f.ctypes.data, g.ctypes.data) == 0
    assert np.array_equal(f.view(np.uint32), np.asarray(fo, np.float32).view(np.uint32))
    assert np.array_equal(g.view(np.uint32), np.asarray(go, np.float32).view(np.uint32))
    f2 = np.zeros(B, np.float32)
    assert emu.emu_logistic_evaluate(C.byref(prob), B, x.ctypes.data, f2.ctypes.data, None) == 0   # value-only command
    assert np.array_equal(f2.view(np.uint32), f.view(np.uint32))


# ---- the host side of cno_al_minimize itself (csrc/cno_auglag_host.h) with an emulation backend ------------
def emulated_cno_al_minimize(emu, family, x0, kinds, rows, n_eq, *, outer_stop=None, config=None, inner_stop=None,
                             eq0=None, ineq0=None, penalty0=None, data=None):
    """cno::al_outer_loop -- the code csrc/cno_api.cu::al_run runs with the CUDA backend -- with memcpy / memset
    and emulated kernel launches as the backend, carving its scratch out of cno::AlLayout."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    dt = x0.dtype
    prob = _problem(family, x0, data=data)
    k, keep = ob._constraints(kinds, rows, n_eq, dt, B, d)
    ne, ni = k.n_eq, k.n_ineq
    cfg = config if config is not None else ob.al_default_config()
    ostop = outer_stop if outer_stop is not None else ob.al_default_stop()
    istop = inner_stop if inner_stop is not None else ob.default_stop()
    opt = lambda v, shape: None if v is None else np.ascontiguousarray(np.broadcast_to(np.asarray(v, dt), shape))  # noqa: E731
    e0, i0, p0 = opt(eq0, (B, ne)), opt(ineq0, (B, ni)), opt(penalty0, (B,))
    r = dict(x=np.zeros_like(x0), equality_multipliers=np.zeros((B, ne), dt), inequality_multipliers=np.zeros((B, ni), dt),
             penalty=np.zeros(B, dt), max_violation=np.zeros(B, dt), max_lagrangian_gradient=np.zeros(B, dt),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B, dt), f_delta=np.zeros(B, dt), gradient_norm=np.zeros(B, dt))
    out = ob.AlOut(*[_ptr(r[n]) for n, _ in ob.AlOut._fields_])
    launches = C.c_int(0)
    rc = emu.emu_al_minimize(C.byref(prob), C.byref(k), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.c_void_p(_ptr(e0)),
                             C.c_void_p(_ptr(i0)), C.c_void_p(_ptr(p0)), C.byref(istop), C.byref(ostop), C.byref(cfg),
                             C.byref(out), C.byref(launches))
    assert rc == 0
    del keep
    r["launches"] = launches.value
    return r


@pytest.mark.parametrize("family,dtype,d,n_eq,per_instance", [
    (ob.FN_ROSENBROCK, np.float64, 8, 1, True), (ob.FN_ROSENBROCK, np.float64, 37, 0, False),
    (ob.FN_HALF_SQUARED_NORM, np.float64, 8, 2, True)])
def test_host_loop_of_cno_al_minimize_under_emulation(emu, family, dtype, d, n_eq, per_instance):
    """Initial state, auto-scale on iteration 1, warm-up inner limits, termination on the remaining-counter,
    best-iterate epilogue, scratch layout: the shared host loop + every kernel == the oracle, bit for bit."""
    B = 2
    rng = np.random.default_rng(400 + d)
    x0 = ob.fill_uniform((B, d), 0, 71 + d, -1.5, 1.5, dtype)
    kinds = [ob.CON_AFFINE, ob.CON_SQNORM, ob.CON_AFFINE]
    shape = (B, 3, d + 1) if per_instance else (3, d + 1)
    rows = rng.uniform(-1, 1, shape).astype(dtype)
    rows[..., 1, d] = 2.0 + rng.uniform(0, 1, shape[:-2])
    stop = ob.al_default_stop()
    stop.num_iterations = 3 if d > 8 else 5
    r = emulated_cno_al_minimize(emu, family, x0, kinds, rows, n_eq, outer_stop=stop)
    o = ob.al_minimize(family, x0, kinds, rows, n_eq, outer_stop=stop)
    _assert_same(r, o)
    # launches = 1 (auto-scale) + 2 per outer iteration of the slowest instance + 1 (finalize)
    assert r["launches"] == 2 + 2 * int(o["num_iterations"].max())
    if d > 8:
        return
    cfg = ob.al_default_config()
    cfg.warmup_max_inner_iterations, cfg.auto_scale_initial_penalty = 0, 0
    kw = dict(outer_stop=stop, config=cfg, eq0=0.25, ineq0=0.5, penalty0=2.0)
    _assert_same(emulated_cno_al_minimize(emu, family, x0, kinds, rows, n_eq, **kw),
                 ob.al_minimize(family, x0, kinds, rows, n_eq, **kw))


@pytest.mark.parametrize("d,every", [(2, 3), (128, 7)])
def test_emulation_reproduces_the_stepwise_kernel(emu, d, every):
    """cno_minimize_steps (lbfgs_minimize_kernel<Fn, M, kResume = true>): rounds of `every` iterations with the
    solver state parked in between == the fused solve of the oracle, bit for bit, incl. a NaN start."""
    B = 3
    x0 = ob.fill_uniform((B, d), 0, 33 + d, -2.0, 2.0)
    x0[2, 0] = np.nan
    stop = ob.default_stop()
    stop.num_iterations = 30
    prob = _problem(ob.FN_ROSENBROCK, x0)
    r = dict(x=np.zeros_like(x0), value=np.zeros(B), gradient=np.zeros_like(x0), num_iterations=np.zeros(B, np.uint32),
             status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B), f_delta=np.zeros(B),
             gradient_norm=np.zeros(B))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    rounds = C.c_int(0)
    assert emu.emu_minimize_steps(C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop), C.byref(out),
                                  every, C.byref(rounds)) == 0
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop)
    for key in SOLVER_KEYS:
        u, v = r[key], o[key]
        if u.dtype.kind == "f":
            nan = np.isnan(u)
            assert np.array_equal(nan, np.isnan(v)), key
            u, v = np.where(nan, 0, u), np.where(nan, 0, v)
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8)), key
    assert rounds.value == -(-int(o["num_iterations"].max()) // every)


# ---- the First-mode dense quadratic functor (csrc/cno_functors.cuh: DenseQuadraticGlobalFn) ------------------
def _quadratic(center, scale):
    """scale/2 |x - center|^2 up to a constant, as a DenseQuadratic data row [A col-major | b]."""
    d = len(center)
    return np.array([list((scale * np.eye(d)).T.ravel()) + [scale * c for c in center]])


@pytest.mark.parametrize("d", [8, 64])
def test_emulated_lbfgs_on_dense_quadratics_equals_oracle(emu, d):
    B = 2
    x0 = ob.fill_uniform((B, d), 0, 17 + d, -2.0, 2.0)
    data = _spd_data(B, d, 21)
    prob = _problem(ob.FN_DENSE_QUADRATIC, x0, data=data)
    stop = ob.default_stop()
    r = dict(x=np.zeros_like(x0), value=np.zeros(B), gradient=np.zeros_like(x0), num_iterations=np.zeros(B, np.uint32),
             status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B), f_delta=np.zeros(B),
             gradient_norm=np.zeros(B))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_minimize(ob.LBFGS, 0, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                            C.byref(out)) == 0
    o = ob.minimize(ob.LBFGS, ob.FN_DENSE_QUADRATIC, x0, data=data, stop=stop)
    for key in SOLVER_KEYS:
        assert np.array_equal(r[key].view(np.uint8), o[key].view(np.uint8)), key
    # A x* = b
    A = data[:, :d * d].reshape(B, d, d).transpose(0, 2, 1)
    assert np.abs(np.einsum("bij,bj->bi", A, r["x"]) - data[:, d * d:]).max() < 1e-4


def test_emulated_al_reference_kkt_known_answers_on_the_device_path(emu):
    """src/test/augmented_lagrangian_test.cc:541-625 on the device source (quadratic objectives through
    DenseQuadraticGlobalFn): InequalityActiveRecoversMultiplier and BothEqualityAndInequalityActive."""
    kw = dict(penalty0=1.0)
    data = _quadratic([2.0, 0.0], 1.0)  # QuadraticAt20
    r = emulated_cno_al_minimize(emu, ob.FN_DENSE_QUADRATIC, np.array([[5.0, 5.0]]), [ob.CON_AFFINE], [[-1.0, 0.0, -1.0]], 0,
                                 data=data, **kw)
    x, mu = r["x"][0], r["inequality_multipliers"][0, 0]
    assert abs(x[0] - 1.0) <= 1e-3 and abs(x[1]) <= 1e-3 and 1.0 - x[0] >= -1e-5 and abs(mu - 1.0) <= 1e-2
    _assert_same(r, ob.al_minimize(ob.FN_DENSE_QUADRATIC, np.array([[5.0, 5.0]]), [ob.CON_AFFINE], [[-1.0, 0.0, -1.0]], 0,
                                   data=data, **kw))
    data = _quadratic([1.0, 2.0], 2.0)  # QuadraticAt12
    args = (ob.FN_DENSE_QUADRATIC, np.array([[1.0, 1.0]]), [ob.CON_AFFINE, ob.CON_AFFINE], [[1.0, 0.0, 0.5], [-1.0, -1.0, -2.0]], 1)
    r = emulated_cno_al_minimize(emu, *args, data=data, **kw)
    x = r["x"][0]
    assert abs(x[0] - 0.5) <= 1e-3 and abs(x[1] - 1.5) <= 1e-3 and 2.0 - (x[0] + x[1]) >= -1e-5
    assert r["inequality_multipliers"][0, 0] >= -1e-2
    _assert_same(r, ob.al_minimize(*args, data=data, **kw))


def emulated_evaluate(emu, family, x, data=None, value=True, gradient=True):
    """cno_evaluate's kernel (csrc/cno_evaluate.cuh: evaluate_kernel) under emulation; unrequested outputs are None."""
    x = np.ascontiguousarray(x)
    B = x.shape[0]
    prob = _problem(family, x, data=data)
    f = np.zeros(B, x.dtype) if value else None
    g = np.zeros_like(x) if gradient else None
    emu.emu_evaluate.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    assert emu.emu_evaluate(C.byref(prob), B, x.ctypes.data, _ptr(f), _ptr(g)) == 0
    return f, g


@pytest.mark.parametrize("case", es.probe_cases(), ids=lambda c: c[0])
def test_emulated_evaluate_edge_vectors_equal_model_and_oracle(emu, case):
    """The summation edges of tests/test_evaluate_gpu.py (subnormal partials and results, overflow in each stage of the
    tensor-core tree, absorption, +-Inf, a NaN in every lane, -0.0; fp32 Rosenbrock with a subnormal gradient, an
    overflowing value, NaN starts) on the device source under emulation: emulated kernel == numpy model of the
    specification == oracle, bit for bit (NaN: NaN-ness only).  A later difference on the GPU is then the hardware's."""
    name, family, x, data, names, (fm, gm) = case
    fo, go = ob.evaluate(family, x, data=data)
    f, g = emulated_evaluate(emu, family, x, data)
    for i, vec in enumerate(names):
        assert es.same_bits(f[i], fm[i]) and es.same_bits(fo[i], fm[i]), (vec, f[i], fm[i], fo[i])
        assert es.same_bits(g[i], gm[i]) and es.same_bits(go[i], gm[i]), vec
    ok = es.chain_finite(family, x, data)
    assert ok.any()
    es.check_exact(family, x[ok], None if data is None else data[ok], f[ok], g[ok], x.dtype.type)
    if name.startswith("rosenbrock"):
        k = names.index("subnormal_gradient")
        assert g[k, -1] == es.SUBNORMAL_G != 0 and abs(g[k, -1]) < np.finfo(np.float32).tiny
        k = names.index("huge")
        assert f[k] == np.inf and np.isfinite(g[k]).all()
    f1, _ = emulated_evaluate(emu, family, x, data, gradient=False)
    _, g1 = emulated_evaluate(emu, family, x, data, value=False)
    assert es.same_bits(f1, f) and es.same_bits(g1, g)


@pytest.mark.parametrize("d,B,hz", [(37, 4, 0), (128, 2, 0), (37, 3, 1)])
def test_emulated_bfgs_shared_memory_inverse_hessian_equals_oracle(emu, d, B, hz):
    """bfgs_smem_minimize_kernel (csrc/cno_bfgs.cuh: Bfgs above d = 32, H in the warp's shared-memory slice)."""
    x0 = ob.fill_uniform((B, d), 0, 5 + d, -2.0, 2.0)
    stop = ob.default_stop()
    stop.num_iterations = 40
    prob = _problem(ob.FN_ROSENBROCK, x0)
    r = dict(x=np.zeros_like(x0), value=np.zeros(B), gradient=np.zeros_like(x0), num_iterations=np.zeros(B, np.uint32),
             status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B), f_delta=np.zeros(B),
             gradient_norm=np.zeros(B))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_minimize(ob.BFGS, hz, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                            C.byref(out)) == 0
    o = ob.minimize(ob.BFGS, ob.FN_ROSENBROCK, x0, stop=stop, linesearch=hz)
    for key in SOLVER_KEYS:
        assert np.array_equal(r[key].view(np.uint8), o[key].view(np.uint8)), key
