"""Lbfgsb<Rosenbrock, 5> fp64 at d = 256, 512 and 1024 (csrc/cno_lbfgsb_group.cuh: one group of d / 128 warps per
instance), on the CPU: the group kernel's device source under the CPU warp emulation against the reference's own
lbfgsb.h (oracle/_ref) on every output, with proof that the rare starts reach their branches; the compacted sum against
the specification's order; and the kernel's plan and register use.  The GPU side is tests/test_lbfgsb_group_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle_binding as ob

HERE = os.path.dirname(__file__)
EMU_DIR = os.path.join(HERE, "emu")
CSRC = os.path.join(HERE, "..", "cppnumericalsolvers_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
DS = (256, 512, 1024)
# d -> (groups per CTA, warps per group, dynamic shared memory per CTA) of LbfgsbGroupPlan<double, d, 5>
PLAN = {256: (4, 2, 131904), 512: (2, 4, 131872), 1024: (1, 8, 131856)}
needs_ref = pytest.mark.skipif(not ob.ref_available(), reason="oracle/_ref not built")


def bitwise_equal(a, b, nan_ok=False):
    """Every output bit for bit; with nan_ok a NaN only has to be a NaN on both sides (its sign and payload follow
    the operand that produced it, which differs between the reference's and the kernel's operation order)."""
    for k in KEYS:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if nan_ok and x.dtype.kind == "f":
            assert np.array_equal(np.isnan(x), np.isnan(y)), k
            x, y = np.where(np.isnan(x), 0, x), np.where(np.isnan(y), 0, y)
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), k


def rosenbrock_grad(x):
    """The gradient of the chained Rosenbrock function (only its signs and rough size are used here)."""
    g = np.zeros_like(x)
    g[:, :-1] = -2 * (1 - x[:, :-1]) - 400 * x[:, :-1] * (x[:, 1:] - x[:, :-1] ** 2)
    g[:, 1:] += 200 * (x[:, 1:] - x[:, :-1] ** 2)
    return g


def first_cauchy_point(x, g, lo, hi):
    """GetGeneralizedCauchyPoint (lbfgsb.h:322-446) at the first iteration, where the history is empty (theta = 1, W
    empty): the projected steepest-descent path with f' = -|d|^2 and f'' = |d|^2.  Returns (number of positive
    breakpoints, number of free variables at the Cauchy point) for one instance; in floating point, not bit for bit
    (the cases below are far from the boundaries of these counts)."""
    d = -g.copy()
    t = np.where(g < 0, (x - hi) / np.where(g == 0, 1, g), (x - lo) / np.where(g == 0, 1, g))
    t = np.where(g == 0, np.finfo(float).max, t)
    d[t == 0] = 0
    positive = int((t > 0).sum())
    if positive == 0:
        xc = x.copy()  # every d_i is 0: the Cauchy point is x, on the faces it started on
    else:
        fp, fpp = -d @ d, d @ d
        fpp = max(1e-12, fpp)
        fpp0 = fpp
        dt_min, t_old = -fp / fpp, 0.0
        xc = x.copy()
        visited = np.zeros(x.shape, bool)
        for b in sorted(np.flatnonzero(t > 0), key=lambda i: (t[i], i)):
            dt = t[b] - t_old
            if dt_min < dt:
                break
            zb = (hi[b] if d[b] > 0 else lo[b]) - x[b]
            fp += dt * fpp + g[b] ** 2 + g[b] * zb
            fpp = max(1e-12 * fpp0, fpp - g[b] ** 2)
            xc[b] = x[b] + zb
            d[b] = 0
            visited[b] = True
            dt_min, t_old = -fp / fpp, t[b]
        dt_min = max(dt_min, 0.0)
        xc = np.where(visited, xc, x + (t_old + dt_min) * d)
    free = int(((xc != hi) & (xc != lo)).sum())
    return positive, free


# ---------------------------------------------------------------- the starts ----

# iteration caps of the emulated cases (the emulation runs 32 d / 128 threads per group on the CPU): none at d = 256
CAP = {256: 0, 512: 3, 1024: 2}


def case(d, kind, cap=None):
    """(x0 [B, d], lower, upper, stop) of one case.  Boxes: [d] shared or [B, d] per instance, or None.  cap: the
    iteration limit (0 = none; default CAP[d])."""
    stop = ob.lbfgsb_stop()
    stop.num_iterations = CAP[d] if cap is None else cap
    if kind == "shared_box":  # U(-2.5, 2.5): most coordinates start outside [-0.5, 0.8] and are projected first
        return ob.fill_uniform((2, d), 0, 40 + d, -2.5, 2.5), np.full(d, -0.5), np.full(d, 0.8), stop
    if kind == "instance_boxes":
        rng = np.random.default_rng(d)
        lo = rng.uniform(-1.5, -0.2, (2, d))
        hi = lo + rng.uniform(0.3, 2.0, (2, d))
        return ob.fill_uniform((2, d), 0, 41 + d, -2.5, 2.5), lo, hi, stop
    if kind == "unbounded_capped":
        stop.num_iterations = stop.num_iterations or 12
        return ob.fill_uniform((1, d), 0, 42 + d, -2.5, 2.5), None, None, stop
    if kind == "nan_row":
        x0 = ob.fill_uniform((1, d), 0, 43 + d, -0.4, 0.7)
        x0[0, d // 3] = np.nan
        return x0, np.full(d, -0.5), np.full(d, 0.8), stop
    if kind == "no_positive_breakpoint":
        # each coordinate sits on the face its negative gradient points out of: every t_i is +-0
        x0 = ob.fill_uniform((1, d), 0, 44 + d, -1.5, 1.5)
        g = rosenbrock_grad(x0)
        lo = np.where(g > 0, x0, x0 - 1.0)
        hi = np.where(g < 0, x0, x0 + 1.0)
        return x0, lo, hi, stop
    if kind == "nfree_zero":
        # a box of half-width 1e-3 around the start: every breakpoint is crossed before the model's minimum
        x0 = ob.fill_uniform((1, d), 0, 45 + d, -1.5, 1.5)
        return x0, x0 - 1e-3, x0 + 1e-3, stop
    raise AssertionError(kind)


KINDS = ("shared_box", "instance_boxes", "unbounded_capped", "nan_row", "no_positive_breakpoint", "nfree_zero")


def assert_case_reached(kind, x0, lo, hi):
    if kind not in ("no_positive_breakpoint", "nfree_zero"):
        return
    d = x0.shape[1]
    for b in range(x0.shape[0]):
        l = np.broadcast_to(lo, x0.shape)[b]
        h = np.broadcast_to(hi, x0.shape)[b]
        x = np.minimum(np.maximum(x0[b], l), h)
        assert np.array_equal(x, x0[b]), "the start is inside its box, so the first projection keeps it"
        g = rosenbrock_grad(x[None])[0]
        assert (np.abs(g) > 1e-2).all()
        positive, free = first_cauchy_point(x, g, l, h)
        if kind == "no_positive_breakpoint":
            assert positive == 0
        else:
            assert positive == d and free == 0


# ---------------------------------------------------------------- emulation ----

def build_emu(out_dir):
    """tests/emu/emu_lbfgsb_group.cc compiled with the flags of tests/emu/Makefile into `out_dir`."""
    out = os.path.join(str(out_dir), "libcno_emu_lbfgsb_group.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-pthread",
                    "-DCNO_WARP_EMULATION", "-Wno-unknown-pragmas", "-Wno-attributes", "-shared", "-I", EMU_DIR,
                    "-I", CSRC, "-I", os.path.join(HERE, "..", "include"), "-x", "c++",
                    os.path.join(EMU_DIR, "emu_lbfgsb_group.cc"), "-o", out], check=True)
    lib = C.CDLL(out)
    lib.emu_compacted_sum.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emu(tmp_path_factory.mktemp("emu_lbfgsb_group"))


def emulated(emu, x0, lo, hi, stop):
    x0 = np.ascontiguousarray(x0)
    B, d = x0.shape
    prob = ob.Problem(ob.FN_ROSENBROCK, 0, d, 0, 0.0, None, 0, ob.POLICY_DMMA_TREE, 0, 0)
    r, out = ob._batch_out(x0)
    lo_a = None if lo is None else np.ascontiguousarray(lo, dtype=np.float64)
    hi_a = None if hi is None else np.ascontiguousarray(hi, dtype=np.float64)
    stride = d if any(a is not None and a.ndim == 2 for a in (lo_a, hi_a)) else 0
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    assert emu.emu_lbfgsb_group(C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), ptr(lo_a), ptr(hi_a),
                                C.c_longlong(stride), C.byref(stop), C.byref(out)) == 0
    return r


@needs_ref
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", DS)
def test_emulated_group_kernel_equals_reference(emu, d, kind):
    """lbfgsb_group_minimize_kernel<GroupRosenbrockFn<double, d>, 5> under the warp emulation (one group of d / 128
    warps draining the queue) == the reference's own Lbfgsb<F, 5> (oracle/_ref), every output bit for bit."""
    x0, lo, hi, stop = case(d, kind)
    if d > 256:  # one instance per case past d = 256 (the emulation's cost grows with the group)
        x0, lo, hi = x0[:1], (lo[:1] if lo is not None and lo.ndim == 2 else lo), (hi[:1] if hi is not None and hi.ndim == 2 else hi)
    assert_case_reached(kind, x0, lo, hi)
    o = ob.ref_lbfgsb_minimize(ob.FN_ROSENBROCK, x0, lo, hi, stop=stop)
    r = emulated(emu, x0, lo, hi, stop)
    bitwise_equal(r, o, nan_ok=(kind == "nan_row"))
    if lo is not None and kind != "nan_row":
        assert (r["x"] >= lo).all() and (r["x"] <= hi).all()
    if kind == "unbounded_capped":
        assert (o["num_iterations"] == stop.num_iterations + 1).all() and (o["status"] == 1).all()
    if kind == "shared_box":
        assert (x0 < -0.5).any() and (x0 > 0.8).any()
        assert (r["x"] == 0.8).any() or stop.num_iterations > 0


def test_rare_starts_reach_their_branches():
    """The two rare starts, checked on their own (also without oracle/_ref): no positive breakpoint, and a first
    Cauchy point with no free variable."""
    for d in DS:
        for kind in ("no_positive_breakpoint", "nfree_zero"):
            x0, lo, hi, _ = case(d, kind)
            assert_case_reached(kind, x0, lo, hi)


def _oracle_sum(t):
    t = np.ascontiguousarray(t)
    return ob.oracle_lib().cno_oracle_reduce_sum_f64(C.c_void_p(t.ctypes.data), t.shape[0], ob.POLICY_DMMA_TREE)


@pytest.mark.parametrize("d", DS)
def test_compacted_sum_equals_specification(emu, d):
    """The masked group sum over a compacted vector of every length n = 1 .. d == reduce_dmma_tree on that vector:
    random terms over several magnitudes, then all terms -0 with +0 at the padded positions.  Absent positions (past
    E' in a lane's run) hold 1e300 in the emulation, so adding one would show."""
    rng = np.random.default_rng(7 + d)
    ob.oracle_lib().cno_oracle_reduce_sum_f64.restype = C.c_double
    for label, terms in (("random", rng.uniform(-1, 1, (d, d)) * 10.0 ** rng.integers(-20, 20, (d, d))),
                         ("negative zeros", np.full((d, d), -0.0))):
        terms = np.ascontiguousarray(terms)
        got, pad = np.zeros(d), np.zeros(d)
        ns = np.arange(1, d + 1, dtype=np.int32)
        assert emu.emu_compacted_sum(d, ns.ctypes.data, d, terms.ctypes.data, pad.ctypes.data, got.ctypes.data) == 0
        want = np.array([_oracle_sum(terms[n - 1, :n]) for n in ns])
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), label


# ---------------------------------------------------------------- the plan and the registers ----

def _nvcc(*args):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    return subprocess.run([NVCC, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC,
                           "-I", os.path.join(HERE, "..", "include"), *args], check=True, capture_output=True, text=True)


def test_plan_program_prints_the_plan(tmp_path):
    """A host-only program prints LbfgsbGroupPlan<double, d, 5>: groups (= resident instances) per CTA, warps per
    group and bytes, as the launcher hands them to launch_persistent."""
    lines = [f'  printf("%d|%d|%d|%d|%zu\\n", {d}, LbfgsbGroupPlan<double, {d}, 5>::kWarps, '
             f"LbfgsbGroupPlan<double, {d}, 5>::kGroupWarps, LbfgsbGroupPlan<double, {d}, 5>::kThreads, "
             f"LbfgsbGroupPlan<double, {d}, 5>::kBytes);" for d in DS]
    prog = tmp_path / "plan.cu"
    prog.write_text('#include <cstdio>\n#include "cno_lbfgsb_group.cuh"\nusing namespace cno;\nint main() {\n'
                    + "\n".join(lines) + "\n}\n")
    _nvcc(str(prog), "-o", str(tmp_path / "plan"))
    out = subprocess.run([str(tmp_path / "plan")], check=True, capture_output=True, text=True).stdout
    got = {}
    for line in out.splitlines():
        d, groups, warps, threads, nbytes = map(int, line.split("|"))
        assert threads == 32 * groups * warps <= 256 and nbytes <= 227 * 1024
        got[d] = (groups, warps, nbytes)
    assert got == PLAN


def test_group_kernels_keep_everything_in_registers(tmp_path):
    """ptxas -v: no stack frame and no spills in the three group Lbfgsb kernels, and no local-memory instruction in
    their SASS."""
    src = tmp_path / "k.cu"
    inst = "\n".join(
        f"template __global__ void cno::lbfgsb_group_minimize_kernel<cno::GroupRosenbrockFn<double, {d}>, 5>("
        f"cno::GroupRosenbrockFn<double, {d}>, const double*, long long, cno::StopParams<double>, "
        f"cno::BatchOut<double>, unsigned long long*, cno::BoundsArgs<double>);" for d in DS)
    src.write_text('#include "cno_lbfgsb_group.cuh"\n' + inst + "\n")
    cubin = tmp_path / "k.cubin"
    r = _nvcc("-O3", "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false", "-Xptxas", "-v", "-cubin",
              str(src), "-o", str(cubin))
    props = re.findall(r"lbfgsb_group_minimize_kernel.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    assert len(props) == 3, r.stderr
    assert all(p == ("0", "0", "0") for p in props), props
    sass = subprocess.run([CUOBJDUMP, "-sass", str(cubin)], check=True, capture_output=True, text=True).stdout
    assert sass.count("Function : ") == 3
    assert not re.search(r"\b(LDL|STL)\b", sass)
