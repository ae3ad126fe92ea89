"""ctypes binding of the CPU ORACLE (oracle/libcno_oracle.so, oracle/_ref).

TEST INFRASTRUCTURE: import this only from tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  Never from the product.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_LIB = os.path.join(HERE, "libcno_oracle.so")
REF_LIB = os.path.join(HERE, "_ref", "libcno_ref.so")

LBFGS, BFGS, NEWTON, GRADIENT_DESCENT, CONJUGATED_GRADIENT_DESCENT = 0, 1, 2, 3, 4
FN_ROSENBROCK, FN_DIAG_QUADRATIC, FN_HALF_SQUARED_NORM, FN_LOGISTIC, FN_DENSE_QUADRATIC = range(5)
POLICY_WARP_TREE, POLICY_EIGEN_SSE2, POLICY_DMMA_TREE, POLICY_DMMA_LU = 0, 1, 2, 3


def device_policy(dtype) -> int:
    """The reduction policy the CUDA kernels of this dtype implement."""
    return POLICY_DMMA_TREE if np.dtype(dtype) == np.float64 else POLICY_WARP_TREE


class Stop(C.Structure):
    _fields_ = [
        ("num_iterations", C.c_uint64), ("x_delta", C.c_double),
        ("x_delta_violations", C.c_int32), ("f_delta", C.c_double),
        ("f_delta_violations", C.c_int32), ("f_delta_relative", C.c_int32),
        ("gradient_norm", C.c_double), ("gradient_norm_relative", C.c_int32),
        ("condition_hessian", C.c_double), ("past", C.c_int32),
        ("past_delta", C.c_double),
    ]


def default_stop() -> "Stop":
    """solver/progress.h:353-431 (DefaultStoppingSolverProgress)."""
    return Stop(10000, 1e-9, 1, 0.0, 1, 0, 1e-5, 1, 0.0, 3, 1e-6)


def conservative_stop() -> "Stop":
    """solver/progress.h:456-464 (ConservativeStoppingSolverProgress)."""
    s = default_stop()
    s.gradient_norm, s.past, s.past_delta = 5e-6, 5, 1e-10
    return s


class Problem(C.Structure):
    _fields_ = [
        ("family", C.c_int32), ("dtype", C.c_int32), ("d", C.c_int32), ("n", C.c_int32),
        ("param", C.c_double), ("data", C.c_void_p), ("data_stride", C.c_int64),
        ("policy", C.c_int32), ("mode", C.c_int32), ("lbfgs_m", C.c_int32), ("reserved_", C.c_int32),
    ]


class BatchOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "x", "value", "gradient", "num_iterations", "status", "nfev",
        "x_delta", "f_delta", "gradient_norm")]


def build(reference: str = "/root/reference") -> None:
    """Compiles the oracle (and oracle/_ref when the reference tree is present)."""
    subprocess.run(["make", "-s", "-C", HERE, "all", f"REFERENCE={reference}"], check=True)


_oracle = None
_ref = None


def oracle_lib() -> C.CDLL:
    global _oracle
    if _oracle is None:
        if not os.path.exists(ORACLE_LIB):
            build()
        _oracle = C.CDLL(ORACLE_LIB, mode=C.RTLD_GLOBAL)
        _oracle.cno_oracle_reduce_sum_f64.restype = C.c_double
        _oracle.cno_oracle_reduce_sum_f32.restype = C.c_float
    return _oracle


def ref_available() -> bool:
    return os.path.exists(REF_LIB)


def ref_lib() -> C.CDLL:
    global _ref
    if _ref is None:
        oracle_lib()
        _ref = C.CDLL(REF_LIB)
    return _ref


def _np_dtype(a):
    return 0 if a.dtype == np.float64 else 1


LS_MORE_THUENTE, LS_HAGER_ZHANG = 0, 1


def _batch_out(x0: np.ndarray):
    B, dt = x0.shape[0], x0.dtype
    r = dict(x=np.zeros_like(x0), value=np.zeros(B, dt), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8),
             nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B, dt), f_delta=np.zeros(B, dt),
             gradient_norm=np.zeros(B, dt))
    return r, BatchOut(*[r[k].ctypes.data for k, _ in BatchOut._fields_])


def minimize(solver: int, family: int, x0: np.ndarray, *, policy: int | None = None, stop: Stop | None = None,
             data: np.ndarray | None = None, n: int = 0, param: float = 0.0, threads: int = 0,
             impl: str = "oracle", mode: int = 0, linesearch: int = LS_MORE_THUENTE, lbfgs_m: int = 0) -> dict:
    """Runs the CPU oracle ("oracle") or the reference-headers build ("ref").  linesearch = the
    LineSearch template parameter of Lbfgs / Bfgs / GradientDescent (HagerZhang: oracle only)."""
    x0 = np.ascontiguousarray(x0)
    assert x0.dtype in (np.float64, np.float32) and x0.ndim == 2
    B, d = x0.shape
    dt = x0.dtype
    if policy is None:
        policy = device_policy(dt)
    if data is not None:
        data = np.ascontiguousarray(data, dtype=dt)
    p = Problem(family, _np_dtype(x0), d, n, param,
                data.ctypes.data if data is not None else None,
                data.shape[1] if data is not None else 0, policy, mode, lbfgs_m)
    r, o = _batch_out(x0)
    fn = oracle_lib().cno_oracle_minimize_ls if impl == "oracle" else ref_lib().cno_ref_minimize_ls
    t0 = time.perf_counter()
    rc = fn(solver, C.byref(p), C.c_int64(B), C.c_void_p(x0.ctypes.data),
            C.byref(stop) if stop is not None else None, C.byref(o), threads, linesearch)
    r["seconds"] = time.perf_counter() - t0
    if rc != 0:
        raise RuntimeError(f"oracle minimize failed: {rc}")
    return r


MAX_M = 32  # CNO_ORACLE_MAX_M


def lbfgs_paths(family: int, x0: np.ndarray, *, stop: Stop | None = None, lbfgs_m: int = 0,
                policy: int | None = None, threads: int = 0) -> tuple[dict, dict]:
    """minimize(LBFGS, family, x0) with MoreThuente, plus how often each instance took the rare branches of
    OptimizationStep (cno_lbfgs_paths_t): skipped [B, 2, 3] (k < m / k == m; position 0, 1, >= 2 from the newest
    pair), rejected [B], fallback [B, MAX_M + 1] and nonfinite [B, MAX_M + 1] (by mem_count)."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    p = Problem(family, _np_dtype(x0), d, 0, 0.0, None, 0, device_policy(x0.dtype) if policy is None else policy, 0,
                lbfgs_m)
    r, o = _batch_out(x0)
    n = MAX_M + 1
    raw = np.zeros((B, 7 + 2 * n), np.uint64)
    rc = oracle_lib().cno_oracle_lbfgs_paths(C.byref(p), C.c_int64(B), C.c_void_p(x0.ctypes.data),
                                             C.byref(stop) if stop is not None else None, C.byref(o),
                                             C.c_void_p(raw.ctypes.data), threads)
    if rc != 0:
        raise RuntimeError(f"oracle lbfgs_paths failed: {rc}")
    paths = dict(skipped=raw[:, :6].reshape(B, 2, 3), rejected=raw[:, 6], fallback=raw[:, 7:7 + n],
                 nonfinite=raw[:, 7 + n:])
    return r, paths


BFGS_PATHS = ("reset_positive", "reset_nan", "refused_fresh", "refused_updated", "curvature_fallback_false",
              "curvature_fallback_true", "nonfinite", "small_direction")  # the fields of cno_bfgs_paths_t


def bfgs_paths(family: int, x0: np.ndarray, *, stop: Stop | None = None, linesearch: int = LS_MORE_THUENTE,
               policy: int | None = None, threads: int = 0) -> tuple[dict, dict]:
    """minimize(BFGS, family, x0, linesearch=linesearch), plus how often each instance took the rare branches of
    OptimizationStep (cno_bfgs_paths_t): one [B] count per name of BFGS_PATHS."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    p = Problem(family, _np_dtype(x0), d, 0, 0.0, None, 0, device_policy(x0.dtype) if policy is None else policy, 0, 0)
    r, o = _batch_out(x0)
    raw = np.zeros((B, len(BFGS_PATHS)), np.uint64)
    rc = oracle_lib().cno_oracle_bfgs_paths(C.byref(p), C.c_int64(B), C.c_void_p(x0.ctypes.data),
                                            C.byref(stop) if stop is not None else None, C.byref(o),
                                            C.c_void_p(raw.ctypes.data), threads, linesearch)
    if rc != 0:
        raise RuntimeError(f"oracle bfgs_paths failed: {rc}")
    return r, {k: raw[:, i] for i, k in enumerate(BFGS_PATHS)}


def evaluate(family: int, x: np.ndarray, *, policy: int | None = None, data=None, n: int = 0,
             param: float = 0.0, hessian: bool = False):
    x = np.ascontiguousarray(x)
    B, d = x.shape
    dt = x.dtype
    if policy is None:
        policy = device_policy(dt)
    if data is not None:
        data = np.ascontiguousarray(data, dtype=dt)
    p = Problem(family, _np_dtype(x), d, n, param,
                data.ctypes.data if data is not None else None,
                data.shape[1] if data is not None else 0, policy, 0)
    f = np.zeros(B, dt)
    g = np.zeros_like(x)
    H = np.zeros((B, d, d), dt) if hessian else None
    rc = oracle_lib().cno_oracle_evaluate(C.byref(p), C.c_int64(B), C.c_void_p(x.ctypes.data),
                                          C.c_void_p(f.ctypes.data), C.c_void_p(g.ctypes.data),
                                          C.c_void_p(H.ctypes.data) if hessian else None)
    if rc != 0:
        raise RuntimeError(f"oracle evaluate failed: {rc}")
    return (f, g, H) if hessian else (f, g)


def fill_uniform(shape, first: int, seed: int, lo: float, hi: float, dtype=np.float64) -> np.ndarray:
    a = np.zeros(shape, dtype)
    rc = oracle_lib().cno_oracle_fill_uniform(0 if dtype == np.float64 else 1,
                                              C.c_void_p(a.ctypes.data), C.c_int64(first),
                                              C.c_int64(a.size), C.c_uint64(seed),
                                              C.c_double(lo), C.c_double(hi))
    assert rc == 0
    return a


def cstep(io, brackt: int, info: int = 0, impl: str = "oracle"):
    """MoreThuente::cstep; io = [stx, fx, dx, sty, fy, dy, stp, fp, dp, stpmin, stpmax]."""
    arr = (C.c_double * 11)(*io)
    b, i, r = C.c_int(brackt), C.c_int(info), C.c_int(0)
    fn = oracle_lib().cno_oracle_cstep if impl == "oracle" else ref_lib().cno_ref_cstep
    fn(arr, C.byref(b), C.byref(i), C.byref(r))
    return list(arr), b.value, i.value, r.value


def num_threads() -> int:
    return oracle_lib().cno_oracle_num_threads()


# ---- AugmentedLagrangian oracle (cno_al_oracle.h; SURVEY.md 8(f) rank 1, no device path yet) ----
CON_AFFINE, CON_SQNORM = 0, 1


class Constraints(C.Structure):
    _fields_ = [("n_eq", C.c_int32), ("n_ineq", C.c_int32), ("kinds", C.c_void_p),
                ("data", C.c_void_p), ("data_stride", C.c_int64)]


class AlConfig(C.Structure):
    _fields_ = [("penalty_growth_factor", C.c_double), ("violation_shrink_ratio", C.c_double),
                ("auto_scale_initial_penalty", C.c_int32), ("penalty_auto_objective_scale", C.c_double),
                ("penalty_auto_min", C.c_double), ("penalty_auto_max", C.c_double),
                ("warmup_max_inner_iterations", C.c_int32),
                ("warmup_inner_gradient_tolerance", C.c_double), ("multiplier_max", C.c_double),
                ("kkt_gradient_tolerance", C.c_double)]


class AlStop(C.Structure):
    _fields_ = [("num_iterations", C.c_uint64), ("constraint_threshold", C.c_double),
                ("kkt_stationarity_threshold", C.c_double)]


class AlOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "x", "equality_multipliers", "inequality_multipliers", "penalty", "max_violation",
        "max_lagrangian_gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta",
        "gradient_norm")]


def al_default_config() -> AlConfig:
    c = AlConfig()
    oracle_lib().cno_al_oracle_default_config(C.byref(c))
    return c


def al_default_stop() -> AlStop:
    s = AlStop()
    oracle_lib().cno_al_oracle_default_stop(C.byref(s))
    return s


def _constraints(kinds, rows, n_eq, dt, B, d):
    """rows: [n_con, d+1] shared by the batch, or [B, n_con, d+1] per instance."""
    kinds = np.ascontiguousarray(kinds, dtype=np.int32)
    rows = np.ascontiguousarray(rows, dtype=dt)
    n_con = kinds.shape[0]
    assert rows.shape[-2:] == (n_con, d + 1) or n_con == 0
    stride = 0 if rows.ndim == 2 else n_con * (d + 1)
    assert rows.ndim == 2 or rows.shape[0] == B
    k = Constraints(n_eq, n_con - n_eq, kinds.ctypes.data if n_con else None,
                    rows.ctypes.data if n_con else None, stride)
    return k, (kinds, rows)


def al_minimize(family: int, x0: np.ndarray, kinds, rows, n_eq: int, *, eq0=None, ineq0=None,
                penalty0=None, inner_stop: Stop | None = None, outer_stop: AlStop | None = None,
                config: AlConfig | None = None, policy: int | None = None, data=None, threads: int = 0,
                impl: str = "oracle") -> dict:
    """AugmentedLagrangian<Problem, Lbfgs>::Minimize per instance: the C restatement ("oracle")
    or the reference's own headers on the Eigen-API shim ("ref")."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    dt = x0.dtype
    if policy is None:
        policy = device_policy(dt)
    if data is not None:
        data = np.ascontiguousarray(data, dtype=dt)
    p = Problem(family, _np_dtype(x0), d, 0, 0.0, data.ctypes.data if data is not None else None,
                data.shape[1] if data is not None else 0, policy, 0)
    k, keep = _constraints(kinds, rows, n_eq, dt, B, d)
    ne, ni = k.n_eq, k.n_ineq
    arr = lambda a, n: None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, dt), (B, n)))  # noqa: E731
    eq0, ineq0 = arr(eq0, ne), arr(ineq0, ni)
    pen = None if penalty0 is None else np.ascontiguousarray(np.broadcast_to(np.asarray(penalty0, dt), (B,)))
    r = dict(x=np.zeros_like(x0), equality_multipliers=np.zeros((B, ne), dt),
             inequality_multipliers=np.zeros((B, ni), dt), penalty=np.zeros(B, dt),
             max_violation=np.zeros(B, dt), max_lagrangian_gradient=np.zeros(B, dt),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8),
             nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B, dt), f_delta=np.zeros(B, dt),
             gradient_norm=np.zeros(B, dt))
    o = AlOut(*[r[n].ctypes.data for n, _ in AlOut._fields_])
    fn = oracle_lib().cno_al_oracle_minimize if impl == "oracle" else ref_lib().cno_ref_al_minimize
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    t0 = time.perf_counter()
    rc = fn(C.byref(p), C.byref(k), C.c_int64(B), C.c_void_p(x0.ctypes.data), ptr(eq0), ptr(ineq0), ptr(pen),
            C.byref(inner_stop) if inner_stop is not None else None,
            C.byref(outer_stop) if outer_stop is not None else None,
            C.byref(config) if config is not None else None, C.byref(o), threads)
    r["seconds"] = time.perf_counter() - t0
    del keep
    if rc != 0:
        raise RuntimeError(f"al minimize failed: {rc}")
    return r


def al_evaluate(family: int, x: np.ndarray, kinds, rows, n_eq: int, eq, ineq, penalty, *,
                policy: int | None = None, data=None):
    """ToAugmentedLagrangian(problem, multipliers, penalty)(x, &grad) -> (value [B], grad [B,d])."""
    x = np.ascontiguousarray(x)
    B, d = x.shape
    dt = x.dtype
    if policy is None:
        policy = device_policy(dt)
    if data is not None:
        data = np.ascontiguousarray(data, dtype=dt)
    p = Problem(family, _np_dtype(x), d, 0, 0.0, data.ctypes.data if data is not None else None,
                data.shape[1] if data is not None else 0, policy, 0)
    k, keep = _constraints(kinds, rows, n_eq, dt, B, d)
    eq = np.ascontiguousarray(np.broadcast_to(np.asarray(eq, dt), (B, k.n_eq)))
    ineq = np.ascontiguousarray(np.broadcast_to(np.asarray(ineq, dt), (B, k.n_ineq)))
    pen = np.ascontiguousarray(np.broadcast_to(np.asarray(penalty, dt), (B,)))
    v, g = np.zeros(B, dt), np.zeros_like(x)
    rc = oracle_lib().cno_al_oracle_evaluate(C.byref(p), C.byref(k), C.c_int64(B), C.c_void_p(x.ctypes.data),
                                             C.c_void_p(eq.ctypes.data), C.c_void_p(ineq.ctypes.data),
                                             C.c_void_p(pen.ctypes.data), C.c_void_p(v.ctypes.data),
                                             C.c_void_p(g.ctypes.data))
    del keep
    if rc != 0:
        raise RuntimeError(f"al evaluate failed: {rc}")
    return v, g


def hz_search_poly(coef, x0: float, alpha_init: float, impl: str = "oracle"):
    """HagerZhang<F,1>::Search on the quartic (((c4 v + c3) v + c2) v + c1) v + c0 along s = +1
    (RunSearch of src/test/hager_zhang_test.cc:87-99).  Returns (alpha, f_at, x_at, nfev)."""
    k = (C.c_double * 5)(*[float(v) for v in coef])
    a, f, x, n = C.c_double(0), C.c_double(0), C.c_double(0), C.c_int(0)
    fn = oracle_lib().cno_oracle_hz_search_poly if impl == "oracle" else ref_lib().cno_ref_hz_search_poly
    fn(k, C.c_double(x0), C.c_double(alpha_init), C.byref(a), C.byref(f), C.byref(x), C.byref(n))
    return a.value, f.value, x.value, n.value


# ---- function composition: the reference's own operators over the ref functors (ref_driver.cc EXPR_*) ----
(EXPR_BOWL, EXPR_ROSEN_PLUS_HALF, EXPR_PROD, EXPR_SUB, EXPR_PENALTY, EXPR_ZERO_MUL, EXPR_SECOND_SUM,
 EXPR_SECOND_PROD, EXPR_DOWNGRADE) = range(9)


def condition_hessian(family: int, x: np.ndarray, *, policy: int | None = None, data=None, impl: str = "oracle"):
    """progress.condition_hessian (solver/progress.h:203-210) = H(x).norm() * H(x).inverse().norm() per instance:
    impl="oracle" the C restatement, impl="ref" the reference's own Progress::Update (oracle/_ref)."""
    x = np.ascontiguousarray(x)
    B, d = x.shape
    dt = x.dtype
    if policy is None:
        policy = device_policy(dt)
    if data is not None:
        data = np.ascontiguousarray(data, dtype=dt)
    prob = Problem(family, _np_dtype(x), d, 0, 0.0, data.ctypes.data if data is not None else None,
                   data.shape[1] if data is not None else 0, policy, 2)
    out = np.zeros(B, dt)
    fn = oracle_lib().cno_oracle_condition_hessian if impl == "oracle" else ref_lib().cno_ref_condition_hessian
    rc = fn(C.byref(prob), C.c_int64(B), C.c_void_p(x.ctypes.data), C.c_void_p(out.ctypes.data))
    if rc != 0:
        raise RuntimeError(f"condition_hessian failed: {rc}")
    return out


def ref_minimize_expr(expr: int, solver: int, x0: np.ndarray, *, param: float = 0.0, stop: Stop | None = None,
                      linesearch: int = LS_MORE_THUENTE, policy: int | None = None, threads: int = 0,
                      lbfgs_m: int = 0) -> dict:
    """Solver<decltype(composite)>::Minimize per instance, the composite built with the reference's own
    operator+ - * / MinZero / MaxZero (function_expressions.h) -- oracle/_ref only."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    dt = x0.dtype
    if policy is None:
        policy = device_policy(dt)
    r = dict(x=np.zeros_like(x0), value=np.zeros(B, dt), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8),
             nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B, dt), f_delta=np.zeros(B, dt),
             gradient_norm=np.zeros(B, dt))
    o = BatchOut(*[r[k].ctypes.data for k in (
        "x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta", "gradient_norm")])
    rc = ref_lib().cno_ref_minimize_expr(expr, C.c_double(param), solver, linesearch, _np_dtype(x0), d, policy,
                                         C.c_int64(B), C.c_void_p(x0.ctypes.data),
                                         C.byref(stop) if stop is not None else None, C.byref(o), threads, lbfgs_m)
    if rc != 0:
        raise RuntimeError(f"ref minimize_expr failed: {rc}")
    return r


def ref_evaluate_expr(expr: int, x: np.ndarray, *, param: float = 0.0, policy: int | None = None):
    x = np.ascontiguousarray(x)
    B, d = x.shape
    if policy is None:
        policy = device_policy(x.dtype)
    f, g = np.zeros(B, x.dtype), np.zeros_like(x)
    rc = ref_lib().cno_ref_evaluate_expr(expr, C.c_double(param), _np_dtype(x), d, policy, C.c_int64(B),
                                         C.c_void_p(x.ctypes.data), C.c_void_p(f.ctypes.data), C.c_void_p(g.ctypes.data))
    if rc != 0:
        raise RuntimeError(f"ref evaluate_expr failed: {rc}")
    return f, g


# ---- Lbfgsb (solver/lbfgsb.h): box constraints; oracle/_ref only (the reference's own header on the shim) ----
def lbfgsb_stop() -> Stop:
    """The Lbfgsb() constructor's preset (lbfgsb.h:78-81): the default + f_delta = 2.22e-9, relative."""
    s = default_stop()
    s.f_delta = 2.22e-9
    s.f_delta_relative = 1
    return s


def ref_lbfgsb_minimize(family: int, x0: np.ndarray, lower=None, upper=None, *, stop: Stop | None = None,
                        data=None, policy: int | None = None, threads: int = 0, m: int = 0) -> dict:
    """Lbfgsb<F, m>::Minimize per instance with SetBounds(lower, upper); lower / upper: [d] (one box) or [B, d];
    m = 0 / 5: the reference's default, 10: Lbfgsb<F, 10> (Rosenbrock)."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    dt = x0.dtype
    if policy is None:
        policy = device_policy(dt)
    if data is not None:
        data = np.ascontiguousarray(data, dtype=dt)
    p = Problem(family, _np_dtype(x0), d, 0, 0.0, data.ctypes.data if data is not None else None,
                data.shape[1] if data is not None else 0, policy, 0, m)
    lo = None if lower is None else np.ascontiguousarray(lower, dtype=dt)
    hi = None if upper is None else np.ascontiguousarray(upper, dtype=dt)
    stride = 0
    for a in (lo, hi):
        if a is not None and a.ndim == 2:
            stride = d
    r = dict(x=np.zeros_like(x0), value=np.zeros(B, dt), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8),
             nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B, dt), f_delta=np.zeros(B, dt),
             gradient_norm=np.zeros(B, dt))
    o = BatchOut(*[r[k].ctypes.data for k in (
        "x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta", "gradient_norm")])
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    t0 = time.perf_counter()
    rc = ref_lib().cno_ref_lbfgsb_minimize(C.byref(p), C.c_int64(B), C.c_void_p(x0.ctypes.data), ptr(lo), ptr(hi),
                                           C.c_int64(stride), C.byref(stop) if stop is not None else None, C.byref(o),
                                           threads)
    r["seconds"] = time.perf_counter() - t0
    if rc != 0:
        raise RuntimeError(f"ref lbfgsb minimize failed: {rc}")
    return r
