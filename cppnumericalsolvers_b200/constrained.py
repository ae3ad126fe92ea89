"""Host-side mirror of cppoptlib's constrained interface with a batch axis
(function_problem.h:38-60 ConstrainedOptimizationProblem, solver/augmented_lagrangian.h:63-449
AugmentedLagrangianConfig / AugmentedLagrangeState / AugmentedLagrangian) over the C ABI of
include/cno_al.h.

The algorithm is pinned on the CPU (oracle/cno_al_oracle.h, tests/test_al_oracle.py); the device path
equals it bit for bit on the GPU (tests/test_al_gpu.py)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from .function import Function
from .solver import Lbfgs, Progress


@dataclass
class ConstrainedOptimizationProblem:
    """objective + constraints.  A constraint is a row [a (d) | t] of one of two families:
    AFFINE c(x) = a.x - t, SQNORM c(x) = t - x.x; equalities c(x) == 0 first, then inequalities
    c(x) >= 0.  rows: [n_con, d+1] shared by the batch, or [B, n_con, d+1] per instance."""
    objective: Function
    kinds: Sequence[int]
    rows: torch.Tensor
    n_eq: int

    @property
    def n_ineq(self) -> int:
        return len(self.kinds) - self.n_eq


@dataclass
class AugmentedLagrangianConfig:  # solver/augmented_lagrangian.h:63-239
    penalty_growth_factor: float = 10.0
    violation_shrink_ratio: float = 0.25
    auto_scale_initial_penalty: bool = True
    penalty_auto_objective_scale: float = 10.0
    penalty_auto_min: float = 1e-8
    penalty_auto_max: float = 1e8
    warmup_max_inner_iterations: int = 10
    warmup_inner_gradient_tolerance: float = 1e-2
    multiplier_max: float = 1e20
    kkt_gradient_tolerance: float = 1e-4

    def to_c(self) -> _lib.AlConfig:
        return _lib.AlConfig(self.penalty_growth_factor, self.violation_shrink_ratio,
                             int(self.auto_scale_initial_penalty), self.penalty_auto_objective_scale,
                             self.penalty_auto_min, self.penalty_auto_max, self.warmup_max_inner_iterations,
                             self.warmup_inner_gradient_tolerance, self.multiplier_max,
                             self.kkt_gradient_tolerance)


@dataclass
class AugmentedLagrangeState:  # solver/augmented_lagrangian.h:241-276, one row per instance
    x: torch.Tensor
    equality_multipliers: Optional[torch.Tensor] = None
    inequality_multipliers: Optional[torch.Tensor] = None
    penalty: Optional[torch.Tensor] = None  # None / 0 = auto-scale (:312-318)
    max_violation: Optional[torch.Tensor] = None
    max_lagrangian_gradient: Optional[torch.Tensor] = None


@dataclass
class ConstrainedProgress:
    """The outer loop's per-instance Progress values."""
    num_iterations: torch.Tensor
    status: torch.Tensor
    nfev: torch.Tensor
    x_delta: torch.Tensor
    f_delta: torch.Tensor
    gradient_norm: torch.Tensor
    launch: Optional[_lib.LaunchInfo] = None


@dataclass
class ConstrainedStop:
    """The fields of the outer stopping_progress the constrained branch of Progress::Update reads
    (progress.h:112-126, 212-252)."""
    num_iterations: int = 10000
    constraint_threshold: float = 1e-5
    kkt_stationarity_threshold: float = 1e-4


class AugmentedLagrangian:
    """AugmentedLagrangian<Problem, Lbfgs<FunctionExpr>> (solver/augmented_lagrangian.h:278-449)."""

    def __init__(self, problem: ConstrainedOptimizationProblem, unconstrained_solver: Optional[Lbfgs] = None,
                 config: Optional[AugmentedLagrangianConfig] = None):
        self.problem = problem
        self.unconstrained_solver = unconstrained_solver if unconstrained_solver is not None else Lbfgs()
        self.config = config if config is not None else AugmentedLagrangianConfig()
        self.stopping_progress = ConstrainedStop()

    def _c_problem(self, B: int):
        p = self.problem
        fn = p.objective
        d = fn.Dimension
        kinds = torch.tensor(list(p.kinds), dtype=torch.int32, device=p.rows.device)
        rows = p.rows.contiguous()
        if rows.dtype != fn.ScalarType:
            raise ValueError("constraint rows must have the objective's scalar type")
        n_con = len(p.kinds)
        if n_con and rows.shape[-2:] != (n_con, d + 1):
            raise ValueError("rows must be [n_con, d+1] or [B, n_con, d+1]")
        if rows.dim() == 3 and rows.shape[0] != B:
            raise ValueError("per-instance rows must have B leading entries")
        stride = 0 if rows.dim() == 2 else n_con * (d + 1)
        k = _lib.Constraints(p.n_eq, p.n_ineq, kinds.data_ptr() if n_con else None,
                             rows.data_ptr() if n_con else None, stride)
        return fn.problem(), k, (kinds, rows)

    def supported(self) -> bool:
        prob, k, keep = self._c_problem(1 if self.problem.rows.dim() == 2 else self.problem.rows.shape[0])
        ok = _lib.lib().cno_al_supported(C.byref(prob), C.byref(k)) == _lib.OK
        del keep
        return ok

    def Minimize(self, state: AugmentedLagrangeState) -> Tuple[AugmentedLagrangeState, ConstrainedProgress]:
        if not state.x.is_cuda:
            raise RuntimeError("Minimize needs CUDA tensors (there is no CPU fallback)")
        return self._minimize(state, torch.cuda.current_stream(state.x.device).cuda_stream)

    def _minimize(self, state: AugmentedLagrangeState, stream: int):
        x0 = state.x
        fn = self.problem.objective
        if x0.dtype != fn.ScalarType or x0.dim() != 2 or x0.shape[1] != fn.Dimension:
            raise ValueError("x0 must be [B, d] of the objective's scalar type")
        x0 = x0.contiguous()
        B, d = x0.shape
        dev, dt = x0.device, x0.dtype
        prob, k, keep = self._c_problem(B)
        ne, ni = k.n_eq, k.n_ineq
        L = _lib.lib()

        def opt(t, n):
            if t is None:
                return None
            t = torch.as_tensor(t, dtype=dt, device=dev)
            return t.expand(B, n).contiguous() if n is not None else t.expand(B).contiguous()

        eq0, ineq0, pen0 = opt(state.equality_multipliers, ne), opt(state.inequality_multipliers, ni), opt(state.penalty, None)
        r = AugmentedLagrangeState(
            x=torch.empty_like(x0), equality_multipliers=torch.empty(B, ne, dtype=dt, device=dev),
            inequality_multipliers=torch.empty(B, ni, dtype=dt, device=dev),
            penalty=torch.empty(B, dtype=dt, device=dev), max_violation=torch.empty(B, dtype=dt, device=dev),
            max_lagrangian_gradient=torch.empty(B, dtype=dt, device=dev))
        pr = ConstrainedProgress(
            num_iterations=torch.empty(B, dtype=torch.int32, device=dev),
            status=torch.empty(B, dtype=torch.int8, device=dev), nfev=torch.empty(B, dtype=torch.int32, device=dev),
            x_delta=torch.empty(B, dtype=dt, device=dev), f_delta=torch.empty(B, dtype=dt, device=dev),
            gradient_norm=torch.empty(B, dtype=dt, device=dev), launch=_lib.LaunchInfo())
        out = _lib.AlOut(r.x.data_ptr(), r.equality_multipliers.data_ptr() if ne else None,
                         r.inequality_multipliers.data_ptr() if ni else None, r.penalty.data_ptr(),
                         r.max_violation.data_ptr(), r.max_lagrangian_gradient.data_ptr(),
                         pr.num_iterations.data_ptr(), pr.status.data_ptr(), pr.nfev.data_ptr(),
                         pr.x_delta.data_ptr(), pr.f_delta.data_ptr(), pr.gradient_norm.data_ptr())
        nbytes = C.c_size_t(0)
        _lib.check(L.cno_al_workspace_bytes(C.byref(prob), C.byref(k), B, C.byref(nbytes)), "cno_al_workspace_bytes")
        ws = torch.empty(max(nbytes.value, 256) + 256, dtype=torch.uint8, device=dev)
        ws_ptr = (ws.data_ptr() + 255) & ~255  # the scratch layout wants 256-byte alignment
        inner = self.unconstrained_solver.stopping_progress.to_c()
        sp = self.stopping_progress
        outer = _lib.AlStop(sp.num_iterations, sp.constraint_threshold, sp.kkt_stationarity_threshold)
        cfg = self.config.to_c()
        ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
        _lib.check(L.cno_al_minimize(
            C.byref(prob), C.byref(k), C.c_int64(B), C.c_void_p(x0.data_ptr()), ptr(eq0), ptr(ineq0), ptr(pen0),
            C.byref(inner), C.byref(outer), C.byref(cfg), C.byref(out), C.c_void_p(ws_ptr),
            C.c_size_t(ws.numel() - 256), C.c_void_p(stream), C.byref(pr.launch)), "cno_al_minimize")
        del keep
        return r, pr
