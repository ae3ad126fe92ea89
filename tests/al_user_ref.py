"""ctypes binding of oracle/_ref/libcno_ref_al_user.so (oracle/ref_al_user.cc, built by oracle/ref_al_user.mk): the
reference's own AugmentedLagrangian, functors and operators on the functor-constrained test problems whose device twins
are tests/cpp/al_user_problems.cuh.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import oracle_binding as ob

LIB = os.path.join(os.path.dirname(ob.REF_LIB), "libcno_ref_al_user.so")
# problem ids: keep in step with tests/cpp/al_user_problems.cuh and oracle/ref_al_user.cc
(AL_P_HS029, AL_P_SIMPLE, AL_P_COMPOSITE_CONS, AL_P_COMPOSITES, AL_P_BALL_OF_INSTANCE, AL_P_ROWS, AL_P_BOWL,
 AL_P_DOWNGRADE) = range(8)
# problem id -> (n_eq, n_ineq)
COUNTS = {AL_P_HS029: (0, 1), AL_P_SIMPLE: (1, 1), AL_P_COMPOSITE_CONS: (1, 1), AL_P_COMPOSITES: (1, 1),
          AL_P_BALL_OF_INSTANCE: (0, 1), AL_P_ROWS: (1, 1), AL_P_BOWL: (0, 0), AL_P_DOWNGRADE: (1, 0)}
OUT_KEYS = tuple(n for n, _ in ob.AlOut._fields_)

_lib = None


def available() -> bool:
    return os.path.exists(LIB)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        ob.oracle_lib()
        _lib = C.CDLL(LIB)
    return _lib


def out_arrays(B: int, d: int, ne: int, ni: int, dt) -> dict:
    """Zeroed host arrays of every cno_al_out_t output."""
    return dict(x=np.zeros((B, d), dt), equality_multipliers=np.zeros((B, ne), dt),
                inequality_multipliers=np.zeros((B, ni), dt), penalty=np.zeros(B, dt), max_violation=np.zeros(B, dt),
                max_lagrangian_gradient=np.zeros(B, dt), num_iterations=np.zeros(B, np.uint32),
                status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32), x_delta=np.zeros(B, dt),
                f_delta=np.zeros(B, dt), gradient_norm=np.zeros(B, dt))


def minimize(problem: int, x0: np.ndarray, *, data=None, eq0=None, ineq0=None, penalty0=None,
             inner_stop: ob.Stop | None = None, outer_stop: ob.AlStop | None = None, config: ob.AlConfig | None = None,
             threads: int = 0) -> dict:
    """AugmentedLagrangian<ConstrainedOptimizationProblem, Lbfgs<FunctionExpr>>::Minimize per instance on test problem
    `problem` (AL_P_*).  data: the radii [B] of AL_P_BALL_OF_INSTANCE."""
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    dt = x0.dtype
    n_eq, n_ineq = COUNTS[problem]
    arr = lambda a, n: None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, dt), (B, n)))  # noqa: E731
    eq0, ineq0 = arr(eq0, n_eq), arr(ineq0, n_ineq)
    pen = None if penalty0 is None else np.ascontiguousarray(np.broadcast_to(np.asarray(penalty0, dt), (B,)))
    data = None if data is None else np.ascontiguousarray(data, dtype=dt)
    r = out_arrays(B, d, n_eq, n_ineq, dt)
    o = ob.AlOut(*[r[n].ctypes.data for n in OUT_KEYS])
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib().cno_ref_al_minimize_expr(problem, 0 if dt == np.float64 else 1, d, ptr(data), C.c_int64(B),
                                        C.c_void_p(x0.ctypes.data), ptr(eq0), ptr(ineq0), ptr(pen),
                                        C.byref(inner_stop) if inner_stop is not None else None,
                                        C.byref(outer_stop) if outer_stop is not None else None,
                                        C.byref(config) if config is not None else None, C.byref(o), threads)
    if rc != 0:
        raise RuntimeError(f"cno_ref_al_minimize_expr failed: {rc}")
    return r
