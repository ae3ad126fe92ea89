"""Host-side mirror of the reference's solver interface with a batch axis.

  reference                                     here
  --------------------------------------------  ----------------------------------
  solver/progress.h:37-47   Status              Status
  solver/progress.h:82-140  Progress            Progress (thresholds) /
                                                BatchedProgress (per-instance)
  solver/progress.h:353-431 DefaultStopping...  DefaultStoppingSolverProgress()
  solver/progress.h:456-464 Conservative...     ConservativeStoppingSolverProgress()
  solver/solver.h:156-231   Solver<F,State>     Solver (stopping_progress, Minimize)
  solver/lbfgs.h            Lbfgs<F, m=10>      Lbfgs
  solver/bfgs.h             Bfgs<F>             Bfgs
  solver/newton_descent.h   NewtonDescent<F>    NewtonDescent

`Minimize(function, state)` returns `(BatchedFunctionState, BatchedProgress)`
like the reference returns `tuple<State, Progress>`.  All compute happens in
libcno.so's CUDA kernels; PyTorch only owns device memory and streams.

`SetCallback(cb, every=K)` (solver/solver.h:163-176): with the whole loop fused on
the device a host callback cannot run inside it, so Minimize then proceeds in
rounds of K iterations (`cno_minimize_steps`: the solver's members are parked in
device memory between rounds) and calls `cb(function, state, progress)` on the
device-resident snapshot after every round -- bit for bit the same trajectory as
the one-shot solve.  `every=1` is the reference's per-iteration callback.
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass, field
from typing import Optional, Tuple

import torch

from . import _lib
from .function import BatchedFunctionState, Function


class Status(enum.IntEnum):  # solver/progress.h:37-47
    NotStarted = -1
    Continue = 0
    IterationLimit = 1
    XDeltaViolation = 2
    FDeltaViolation = 3
    GradientNormViolation = 4
    HessianConditionViolation = 5
    Finished = 6


@dataclass
class Progress:
    """Stopping thresholds (the fields of solver::Progress a preset sets)."""
    num_iterations: int = 0
    x_delta: float = 0.0
    x_delta_violations: int = 0
    f_delta: float = 0.0
    f_delta_violations: int = 0
    f_delta_relative: bool = False
    gradient_norm: float = 0.0
    gradient_norm_relative: bool = True
    condition_hessian: float = 0.0
    past: int = 0
    past_delta: float = 1e-6

    def to_c(self) -> _lib.Stop:
        return _lib.Stop(self.num_iterations, self.x_delta, self.x_delta_violations,
                         self.f_delta, self.f_delta_violations, int(self.f_delta_relative),
                         self.gradient_norm, int(self.gradient_norm_relative),
                         self.condition_hessian, self.past, self.past_delta)

    @staticmethod
    def from_c(s: _lib.Stop) -> "Progress":
        return Progress(s.num_iterations, s.x_delta, s.x_delta_violations, s.f_delta,
                        s.f_delta_violations, bool(s.f_delta_relative), s.gradient_norm,
                        bool(s.gradient_norm_relative), s.condition_hessian, s.past,
                        s.past_delta)


def DefaultStoppingSolverProgress() -> Progress:  # solver/progress.h:353-431
    s = _lib.Stop()
    _lib.lib().cno_default_stop(C.byref(s))
    return Progress.from_c(s)


def ConservativeStoppingSolverProgress() -> Progress:  # solver/progress.h:456-464
    s = _lib.Stop()
    _lib.lib().cno_conservative_stop(C.byref(s))
    return Progress.from_c(s)


@dataclass
class BatchedProgress:
    """Per-instance Progress values returned by Minimize."""
    num_iterations: torch.Tensor  # uint32 stored as int32 tensor view
    status: torch.Tensor          # int8, Status values
    nfev: torch.Tensor
    x_delta: torch.Tensor
    f_delta: torch.Tensor
    gradient_norm: torch.Tensor
    launch: Optional[_lib.LaunchInfo] = None

    def done_bitmap(self) -> torch.Tensor:
        """Per-GPU convergence bitmap (1 bit / instance) for the global stop test."""
        b = self.status.shape[0]
        words = torch.zeros((b + 31) // 32, dtype=torch.int32, device=self.status.device)
        _lib.check(_lib.lib().cno_done_bitmap(
            self.status.data_ptr(), b, words.data_ptr(),
            torch.cuda.current_stream(self.status.device).cuda_stream), "cno_done_bitmap")
        return words


def ConditionHessian(function: Function, x: torch.Tensor) -> torch.Tensor:
    """Progress::condition_hessian (solver/progress.h:203-210) on request: H(x).norm() * H(x).inverse().norm() for every
    row of x [B, d] -- what the reference's Progress::Update computes at each iteration of a Second-mode function
    (and no preset tests).  Called on the x a solve returned it is the reference's final progress.condition_hessian."""
    if not x.is_cuda or x.dim() != 2 or x.dtype != function.ScalarType or x.shape[1] != function.Dimension:
        raise ValueError("x must be a CUDA tensor [B, d] of the function's scalar type")
    x = x.contiguous()
    out = torch.empty(x.shape[0], dtype=x.dtype, device=x.device)
    ws = torch.zeros(256, dtype=torch.uint8, device=x.device)
    prob = function.problem()
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().cno_condition_hessian(C.byref(prob), x.shape[0], x.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                                    ws.numel(), torch.cuda.current_stream(x.device).cuda_stream),
                   "cno_condition_hessian")
    return out


class Solver:
    """solver/solver.h:156-231 with a batch axis."""
    _solver_id = -1

    def __init__(self, progress: Optional[Progress] = None):
        self.stopping_progress = progress if progress is not None else DefaultStoppingSolverProgress()
        self._workspace: Optional[torch.Tensor] = None
        self._callback = None
        self._callback_every = 1

    def SetCallback(self, callback, every: int = 1) -> None:
        """solver/solver.h:176.  callback(function, BatchedFunctionState, BatchedProgress)
        runs on the host after every `every` iterations (None removes it)."""
        self._callback = callback
        self._callback_every = max(1, int(every))

    def _problem(self, function: Function):
        """cno_problem_t of `function` as this solver uses it (Lbfgs adds its template parameter m)."""
        return function.problem()

    def supports_steps(self, function: Function) -> bool:
        p = self._problem(function)
        n = C.c_size_t(0)
        return _lib.lib().cno_state_bytes(self._solver_id, C.byref(p), 1, C.byref(n)) == _lib.OK

    def supported(self, function: Function) -> bool:
        p = self._problem(function)
        return _lib.lib().cno_supported(self._solver_id, C.byref(p)) == _lib.OK

    def Minimize(self, function: Function, state: BatchedFunctionState,
                 timed: bool = False) -> Tuple[BatchedFunctionState, BatchedProgress]:
        x0 = state.x
        if not x0.is_cuda:
            raise RuntimeError("Minimize needs CUDA tensors (there is no CPU fallback); "
                               "use MinimizeHost for host buffers")
        if x0.dtype != function.ScalarType or x0.dim() != 2 or x0.shape[1] != function.Dimension:
            raise ValueError("x0 must be [B, d] of the function's scalar type")
        x0 = x0.contiguous()
        dev, dt, B, d = x0.device, x0.dtype, x0.shape[0], x0.shape[1]
        L = _lib.lib()
        prob = self._problem(function)
        with torch.cuda.device(dev):
            x = torch.empty_like(x0)
            g = torch.empty_like(x0)
            f = torch.empty(B, dtype=dt, device=dev)
            xd = torch.empty(B, dtype=dt, device=dev)
            fd = torch.empty(B, dtype=dt, device=dev)
            gn = torch.empty(B, dtype=dt, device=dev)
            it = torch.empty(B, dtype=torch.int32, device=dev)
            nf = torch.empty(B, dtype=torch.int32, device=dev)
            st = torch.empty(B, dtype=torch.int8, device=dev)
            nbytes = C.c_size_t(0)
            _lib.check(L.cno_workspace_bytes(self._solver_id, C.byref(prob), B, C.byref(nbytes)),
                       "cno_workspace_bytes")
            if self._workspace is None or self._workspace.numel() < nbytes.value or \
                    self._workspace.device != dev:
                self._workspace = torch.empty(max(nbytes.value, 256), dtype=torch.uint8, device=dev)
            out = _lib.BatchOut(x.data_ptr(), f.data_ptr(), g.data_ptr(), it.data_ptr(),
                                st.data_ptr(), nf.data_ptr(), xd.data_ptr(), fd.data_ptr(),
                                gn.data_ptr())
            stop = self.stopping_progress.to_c()
            info = _lib.LaunchInfo() if timed else None
            if self._callback is not None:
                return self._minimize_steps(function, prob, x0, stop, out,
                                            (x, f, g, it, st, nf, xd, fd, gn))
            _lib.check(L.cno_minimize(
                self._solver_id, C.byref(prob), B, x0.data_ptr(), C.byref(stop), C.byref(out),
                self._workspace.data_ptr(), self._workspace.numel(),
                torch.cuda.current_stream(dev).cuda_stream,
                C.byref(info) if info is not None else None), "cno_minimize")
        return (BatchedFunctionState(x, f, g),
                BatchedProgress(it, st, nf, xd, fd, gn, info))

    def _minimize_steps(self, function, prob, x0, stop, out, arrays, stop_test=None):
        """Rounds of `every` iterations with the host callback (and, if given, a global
        stop test) in between; the device keeps every instance's solver state parked."""
        x, f, g, it, st, nf, xd, fd, gn = arrays
        L = _lib.lib()
        B, dev = x0.shape[0], x0.device
        nbytes = C.c_size_t(0)
        _lib.check(L.cno_state_bytes(self._solver_id, C.byref(prob), B, C.byref(nbytes)), "cno_state_bytes")
        state = torch.empty(max(nbytes.value, 16), dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        first, launches = 1, 0
        while True:
            _lib.check(L.cno_minimize_steps(
                self._solver_id, C.byref(prob), B, x0.data_ptr(), C.byref(stop), C.byref(out),
                state.data_ptr(), state.numel(), self._callback_every, first,
                self._workspace.data_ptr(), self._workspace.numel(), stream, None), "cno_minimize_steps")
            first, launches = 0, launches + 1
            snapshot_state = BatchedFunctionState(x, f, g)
            snapshot_prog = BatchedProgress(it, st, nf, xd, fd, gn, None)
            if self._callback is not None:
                self._callback(function, snapshot_state, snapshot_prog)
            done = bool((st != 0).all().item()) if stop_test is None else stop_test(snapshot_prog)
            if done:
                break
        info = _lib.LaunchInfo()
        info.kernel_launches = launches
        return snapshot_state, BatchedProgress(it, st, nf, xd, fd, gn, info)

    def MinimizeSharded(self, function: Function, state: BatchedFunctionState, global_batch: int,
                        every: int = 64) -> Tuple[BatchedFunctionState, BatchedProgress]:
        """Multi-GPU solve with the GLOBAL stop test every `every` iterations (SURVEY.md 8(e)):
        this rank's shard advances `every` iterations (cno_minimize_steps), its convergence
        bitmap is all-gathered (one NCCL collective per round), and all ranks stop together
        once every instance of every shard has terminated.  `state.x` is this rank's shard
        (distributed.shard_range); with one process it degenerates to a local loop."""
        from . import distributed as cd
        saved = (self._callback, self._callback_every)
        self._callback_every = max(1, int(every))
        x0 = state.x.contiguous()
        dev, dt, B = x0.device, x0.dtype, x0.shape[0]
        prob = self._problem(function)
        with torch.cuda.device(dev):
            x, g = torch.empty_like(x0), torch.empty_like(x0)
            f, xd, fd, gn = (torch.empty(B, dtype=dt, device=dev) for _ in range(4))
            it, nf = (torch.empty(B, dtype=torch.int32, device=dev) for _ in range(2))
            st = torch.empty(B, dtype=torch.int8, device=dev)
            if self._workspace is None or self._workspace.device != dev:
                self._workspace = torch.empty(256, dtype=torch.uint8, device=dev)
            out = _lib.BatchOut(x.data_ptr(), f.data_ptr(), g.data_ptr(), it.data_ptr(), st.data_ptr(),
                                nf.data_ptr(), xd.data_ptr(), fd.data_ptr(), gn.data_ptr())
            stop = self.stopping_progress.to_c()

            def stop_test(prog):
                return cd.all_done(cd.gather_done_bitmaps(prog.done_bitmap()), global_batch)
            try:
                return self._minimize_steps(function, prob, x0, stop, out,
                                            (x, f, g, it, st, nf, xd, fd, gn), stop_test=stop_test)
            finally:
                self._callback, self._callback_every = saved

    def MinimizeHost(self, function: Function, x0: torch.Tensor
                     ) -> Tuple[BatchedFunctionState, BatchedProgress]:
        """Same call with host tensors (pinned for full-speed copies): H2D, solve,
        D2H inside libcno.so (cno_minimize_host)."""
        if x0.is_cuda:
            raise ValueError("MinimizeHost takes host tensors")
        x0 = x0.contiguous()
        B, dt = x0.shape[0], x0.dtype
        pin = x0.is_pinned()
        key = (tuple(x0.shape), dt, pin)
        if getattr(self, "_host_out_key", None) != key:
            # (pinned) result buffers are allocated once per shape and reused by later calls:
            # the tensors a call returns are overwritten by the next MinimizeHost of this solver
            mk = lambda *s, dtype=dt: torch.empty(*s, dtype=dtype, pin_memory=pin)
            self._host_out = (mk(*x0.shape), mk(*x0.shape), mk(B), mk(B), mk(B), mk(B),
                              mk(B, dtype=torch.int32), mk(B, dtype=torch.int32), mk(B, dtype=torch.int8))
            self._host_out_key = key
        x, g, f, xd, fd, gn, it, nf, st = self._host_out
        out = _lib.BatchOut(x.data_ptr(), f.data_ptr(), g.data_ptr(), it.data_ptr(),
                            st.data_ptr(), nf.data_ptr(), xd.data_ptr(), fd.data_ptr(),
                            gn.data_ptr())
        prob = self._problem(function)
        stop = self.stopping_progress.to_c()
        info = _lib.LaunchInfo()
        _lib.check(_lib.lib().cno_minimize_host(
            self._solver_id, C.byref(prob), B, x0.data_ptr(), C.byref(stop), C.byref(out),
            C.byref(info)), "cno_minimize_host")
        return (BatchedFunctionState(x, f, g), BatchedProgress(it, st, nf, xd, fd, gn, info))


class MoreThuente:
    """linesearch/more_thuente.h: the default LineSearch policy."""


class HagerZhang:
    """linesearch/hager_zhang.h:54-552: the alternative LineSearch policy."""


class _LineSearchSolver(Solver):
    """Solvers with a LineSearch template parameter (lbfgs.h:41, bfgs.h:40, gradient_descent.h:38):
    `Lbfgs(progress, linesearch=HagerZhang)` mirrors `Lbfgs<F, 10, linesearch::HagerZhang>`."""
    _solver_ids = {}

    def __init__(self, progress: Optional[Progress] = None, linesearch=MoreThuente):
        super().__init__(progress)
        if linesearch not in self._solver_ids:
            raise ValueError("linesearch must be MoreThuente or HagerZhang")
        self.linesearch = linesearch
        self._solver_id = self._solver_ids[linesearch]


class Lbfgs(_LineSearchSolver):
    """solver/lbfgs.h:40-324: Lbfgs<F, m = 10, LineSearch = MoreThuente>; `m` = pairs kept (compiled: 5, 10, 20)."""
    _solver_id = _lib.LBFGS
    _solver_ids = {MoreThuente: _lib.LBFGS, HagerZhang: _lib.LBFGS_HAGER_ZHANG}

    def __init__(self, progress: Optional[Progress] = None, linesearch=MoreThuente, m: int = 10):
        super().__init__(progress, linesearch)
        self.m = int(m)

    def _problem(self, function: Function):
        p = function.problem()
        p.lbfgs_m = self.m
        return p


class Lbfgsb(Solver):
    """solver/lbfgsb.h:44-538: Lbfgsb<F, m = 5, MoreThuente> -- L-BFGS-B, box constraints lower <= x <= upper.
    `Lbfgsb()` carries the reference constructor's preset (default + f_delta = 2.22e-9 relative, :78-81);
    `SetBounds(lower, upper)` (:88-92) takes CUDA tensors [d] (one box for the batch) or [B, d] (None = unbounded
    on that side).  The stop test on `gradient_norm` uses the sup-norm of the box-projected gradient (:238-286)."""

    def __init__(self, progress: Optional[Progress] = None, m: int = 5):
        if progress is None:
            s = _lib.Stop()
            _lib.lib().cno_lbfgsb_default_stop(C.byref(s))
            progress = Progress.from_c(s)
        super().__init__(progress)
        # Lbfgsb<F, m>: pairs kept (compiled: 5 for every built-in, 10 for Rosenbrock d = 8 / 37 / 128); Rosenbrock fp64
        # at d = 256 / 512 / 1024 runs on the group kernel (m = 5)
        self.m = int(m)
        self.lower_bound: Optional[torch.Tensor] = None
        self.upper_bound: Optional[torch.Tensor] = None

    def SetBounds(self, lower_bound: Optional[torch.Tensor], upper_bound: Optional[torch.Tensor]) -> None:
        self.lower_bound, self.upper_bound = lower_bound, upper_bound

    def supported(self, function: Function) -> bool:
        p = function.problem()
        p.lbfgs_m = self.m
        return _lib.lib().cno_lbfgsb_supported(C.byref(p)) == _lib.OK

    def Minimize(self, function: Function, state: BatchedFunctionState,
                 timed: bool = False) -> Tuple[BatchedFunctionState, BatchedProgress]:
        x0 = state.x
        if not x0.is_cuda:
            raise RuntimeError("Minimize needs CUDA tensors (there is no CPU fallback)")
        if x0.dtype != function.ScalarType or x0.dim() != 2 or x0.shape[1] != function.Dimension:
            raise ValueError("x0 must be [B, d] of the function's scalar type")
        x0 = x0.contiguous()
        dev, dt, B, d = x0.device, x0.dtype, x0.shape[0], x0.shape[1]
        stride = 0
        keep = []
        ptrs = []
        for t in (self.lower_bound, self.upper_bound):
            if t is None:
                ptrs.append(None)
                continue
            if t.dtype != dt or t.device != dev or t.shape[-1] != d or t.dim() not in (1, 2):
                raise ValueError("bounds must be CUDA tensors [d] or [B, d] of the function's scalar type")
            if t.dim() == 2:
                if t.shape[0] != B:
                    raise ValueError("per-instance bounds must be [B, d]")
                stride = d
            t = t.contiguous()
            keep.append(t)
            ptrs.append(t.data_ptr())
        if stride and any(t.dim() == 1 for t in keep):
            raise ValueError("lower and upper must both be [d] or both be [B, d]")
        prob = function.problem()
        prob.lbfgs_m = self.m
        with torch.cuda.device(dev):
            x, g = torch.empty_like(x0), torch.empty_like(x0)
            f, xd, fd, gn = (torch.empty(B, dtype=dt, device=dev) for _ in range(4))
            it, nf = (torch.empty(B, dtype=torch.int32, device=dev) for _ in range(2))
            st = torch.empty(B, dtype=torch.int8, device=dev)
            if self._workspace is None or self._workspace.device != dev:
                self._workspace = torch.empty(256, dtype=torch.uint8, device=dev)
            out = _lib.BatchOut(x.data_ptr(), f.data_ptr(), g.data_ptr(), it.data_ptr(), st.data_ptr(), nf.data_ptr(),
                                xd.data_ptr(), fd.data_ptr(), gn.data_ptr())
            bounds = _lib.Bounds(ptrs[0], ptrs[1], stride)
            stop = self.stopping_progress.to_c()
            info = _lib.LaunchInfo() if timed else None
            _lib.check(_lib.lib().cno_lbfgsb_minimize(
                C.byref(prob), C.byref(bounds), B, x0.data_ptr(), C.byref(stop), C.byref(out),
                self._workspace.data_ptr(), self._workspace.numel(), torch.cuda.current_stream(dev).cuda_stream,
                C.byref(info) if info is not None else None), "cno_lbfgsb_minimize")
        del keep
        return BatchedFunctionState(x, f, g), BatchedProgress(it, st, nf, xd, fd, gn, info)


class Bfgs(_LineSearchSolver):
    """solver/bfgs.h:39-145 (LineSearch = MoreThuente unless given)."""
    _solver_id = _lib.BFGS
    _solver_ids = {MoreThuente: _lib.BFGS, HagerZhang: _lib.BFGS_HAGER_ZHANG}


class NewtonDescent(Solver):
    """solver/newton_descent.h:38-85 (Armijo<F,2>)."""
    _solver_id = _lib.NEWTON


class GradientDescent(_LineSearchSolver):
    """solver/gradient_descent.h:37-75 (LineSearch = MoreThuente, the reference's default, unless given)."""
    _solver_id = _lib.GRADIENT_DESCENT
    _solver_ids = {MoreThuente: _lib.GRADIENT_DESCENT, HagerZhang: _lib.GRADIENT_DESCENT_HAGER_ZHANG}


class ConjugatedGradientDescent(Solver):
    """solver/conjugated_gradient_descent.h:38-92 (Fletcher-Reeves, Armijo<F,1>); fp64 only."""
    _solver_id = _lib.CONJUGATED_GRADIENT_DESCENT


def _eigen_row(v) -> str:
    """`stream << vector.transpose()` with Eigen's default IOFormat on a default stream: every
    coefficient printed with 6 significant digits, right-aligned to the widest one, one space apart."""
    cells = ["%g" % float(c) for c in v]
    width = max((len(c) for c in cells), default=0)
    return " ".join(c.rjust(width) for c in cells)


def PrintProgressCallback(output_stream=None, instance: int = 0):
    """solver/solver.h:59-130 with a batch axis: prints the reference's per-iteration block for
    ONE instance of the batch (`instance`), followed by one line summarising the whole batch.
    Use with `solver.SetCallback(PrintProgressCallback(sys.stdout), every=K)`; each call costs a
    device->host read of that instance's row."""
    import sys
    out = output_stream if output_stream is not None else sys.stdout
    label_width, num_width = 18, 15

    def callback(function, state, progress):
        i = instance
        num = lambda v: ("%.6f" % float(v)).rjust(num_width)  # noqa: E731  std::fixed << setprecision(6)
        lines = ["--- Iteration: %5d ---" % int(progress.num_iterations[i])]
        if state.value is not None:
            lines.append("  Value:".ljust(label_width) + num(state.value[i]))
        lines.append("  X:".ljust(label_width) + " " + _eigen_row(state.x[i].tolist()))
        if state.gradient is not None:
            lines.append("  Gradient:".ljust(label_width) + " " + _eigen_row(state.gradient[i].tolist()))
            lines.append("  Gradient Norm:".ljust(label_width) + num(progress.gradient_norm[i]))
        lines.append("  X Delta:".ljust(label_width) + num(progress.x_delta[i]))
        lines.append("  F Delta:".ljust(label_width) + num(progress.f_delta[i]))
        if function.Differentiability == 2:
            lines.append("  Hessian Cond.:".ljust(label_width) + "N/A".rjust(num_width))  # not computed (DESIGN.md 2.3)
        running = int((progress.status == int(Status.Continue)).sum())
        lines.append("  Batch:".ljust(label_width) + " %d of %d instances still running" % (running, state.x.shape[0]))
        lines.append("-------------------------")
        out.write("\n".join(lines) + "\n")
        out.flush()

    return callback


def fill_uniform(t: torch.Tensor, first: int, seed: int, lo: float, hi: float) -> torch.Tensor:
    """Counter-based start generator on the device (SURVEY.md 8(d))."""
    assert t.is_cuda and t.is_contiguous()
    dt = _lib.F64 if t.dtype == torch.float64 else _lib.F32
    _lib.check(_lib.lib().cno_fill_uniform(dt, t.data_ptr(), first, t.numel(), seed, lo, hi,
                                           torch.cuda.current_stream(t.device).cuda_stream),
               "cno_fill_uniform")
    return t
