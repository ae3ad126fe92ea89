"""Lbfgs on Rosenbrock fp64 at d = 256, 512 and 1024 (csrc/cno_lbfgs_group.cuh: one group of d / 128 warps per
instance), on the CPU: the oracle against the reference's own headers and the committed fixtures, the group kernel's
device source under the CPU warp emulation against the oracle, the group sum against the specification's order, and
the kernel's plan and register use.  The GPU side is tests/test_lbfgs_group_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import edge_sums as es
from oracle import oracle_binding as ob

HERE = os.path.dirname(__file__)
EMU_DIR = os.path.join(HERE, "emu")
GOLDEN = os.path.join(HERE, "golden")
CSRC = os.path.join(HERE, "..", "cppnumericalsolvers_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
DS = (256, 512, 1024)
# d -> (groups per CTA, warps per group, dynamic shared memory per CTA) of LbfgsGroupPlan<double, d, 10>
PLAN = {256: (4, 2, 186176), 512: (2, 4, 186144), 1024: (1, 8, 186128)}


def bitwise_equal(a, b, rows=slice(None)):
    for k in KEYS:
        assert np.array_equal(np.asarray(a[k])[rows].view(np.uint8), np.asarray(b[k])[rows].view(np.uint8)), k


def starts(d, kind):
    """[B, d] starts: "uniform" = the seeded U(-2, 2) of cno_fill_uniform; "near" = 1 + U(-0.1, 0.1), which converge in
    a hundred-odd iterations; "nan" = a NaN coordinate; "minimiser" = x = 1 (g = 0 at the start); "spike" = [-2, 2]
    with every 64th coordinate scaled by 10^13.5, whose second step fails the descent test and takes the +g fallback."""
    if kind == "uniform":
        return ob.fill_uniform((2, d), 0, 1, -2.0, 2.0)
    if kind == "near":
        return 1.0 + ob.fill_uniform((2, d), 0, 3, -0.1, 0.1)
    if kind == "nan":
        x = ob.fill_uniform((1, d), 0, 4, -2.0, 2.0)
        x[0, d // 3] = np.nan
        return x
    if kind == "minimiser":
        return np.ones((1, d))
    if kind == "spike":
        x = ob.fill_uniform((8, d), 0, 21, -2.0, 2.0)
        x[:, ::64] *= 10.0 ** 13.5
        return x[:1]
    raise AssertionError(kind)


def stop_after(iterations):
    s = ob.default_stop()
    s.num_iterations = iterations
    return s


# ---------------------------------------------------------------- the oracle (CPU) ----

@pytest.mark.parametrize("d", DS)
def test_oracle_equals_reference_at_large_d(d):
    """The oracle's L-BFGS against the reference's lbfgs.h / more_thuente.h on the Eigen-API shim, to convergence."""
    if not ob.ref_available():
        pytest.skip("oracle/_ref not built")
    x0 = starts(d, "uniform")
    bitwise_equal(ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, impl="ref"), ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0))


@pytest.mark.parametrize("d", (512, 1024))
def test_oracle_reproduces_fixture(d):
    z = np.load(os.path.join(GOLDEN, f"lbfgs_rosenbrock_d{d}_f64.npz"))
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, z["x0"])
    bitwise_equal(o, {k: z[k] for k in KEYS})
    assert (z["status"] != 0).all() and (z["num_iterations"] > 100).all()


# ---------------------------------------------------------------- emulation (CPU) ----

def build_emu_group(out_dir):
    """tests/emu/emu_lbfgs_group.cc compiled with the flags of tests/emu/Makefile into `out_dir`."""
    out = os.path.join(str(out_dir), "libcno_emu_group.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-pthread",
                    "-DCNO_WARP_EMULATION", "-Wno-unknown-pragmas", "-Wno-attributes", "-shared", "-I", EMU_DIR,
                    "-I", CSRC, "-I", os.path.join(HERE, "..", "include"), "-x", "c++",
                    os.path.join(EMU_DIR, "emu_lbfgs_group.cc"), "-o", out], check=True)
    lib = C.CDLL(out)
    lib.emu_group_sum.argtypes = [C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emu_group(tmp_path_factory.mktemp("emu_group"))


def _emulated(emu, x0, stop):
    B, d = x0.shape
    prob = ob.Problem(ob.FN_ROSENBROCK, 0, d, 0, 0.0, None, 0, ob.POLICY_DMMA_TREE, 0, 0)
    r, out = ob._batch_out(x0)
    assert emu.emu_lbfgs_group(C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                               C.byref(out)) == 0
    return r


EMU_CASES = [(256, "near", 10000), (512, "uniform", 12), (1024, "uniform", 4), (256, "nan", 20),
             *[(256, kind, 10000) for kind in ("minimiser", "spike")]]


@pytest.mark.parametrize("d,kind,iterations", EMU_CASES, ids=[f"d{d}-{k}-{i}" for d, k, i in EMU_CASES])
def test_emulated_group_kernel_equals_oracle(emu, d, kind, iterations):
    """lbfgs_group_minimize_kernel<GroupRosenbrockFn<double, d>, 10> under the warp emulation (one group of d / 128
    warps draining the queue): every output bit for bit."""
    x0 = np.ascontiguousarray(starts(d, kind))
    stop = stop_after(iterations)
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop)
    if kind == "spike":
        _, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop)
        assert paths["fallback"][:, 1:].sum() > 0, "the spiked start must take the fallback with a non-empty history"
    if kind == "near":
        assert (o["num_iterations"] > 10).all() and (o["status"] != 0).all() and (o["num_iterations"] < iterations).all()
    if iterations < 100 and kind != "nan":
        assert (o["num_iterations"] == iterations + 1).all()
    bitwise_equal(_emulated(emu, x0, stop), o)


def _group_sums(emu, d, terms):
    terms = np.ascontiguousarray(terms, np.float64)
    sums = np.zeros(terms.shape[0])
    assert emu.emu_group_sum(d, terms.shape[0], terms.ctypes.data, sums.ctypes.data) == 0
    return sums


def _oracle_sum(t):
    return ob.oracle_lib().cno_oracle_reduce_sum_f64(C.c_void_p(np.ascontiguousarray(t).ctypes.data), t.shape[0],
                                                     ob.POLICY_DMMA_TREE)


@pytest.mark.parametrize("d", DS)
def test_emulated_group_sum_equals_specification(emu, d):
    """The group sum (warp_sum_p on a GroupCtx) against the oracle's reduce_dmma_tree and the numpy model of the
    specification, on random vectors over several magnitudes and on the edge partials of tests/edge_sums.py, each
    spread over the d / 32 elements of its lane (the edge value in one element, zeros and cancelling pairs around it)."""
    rng = np.random.default_rng(d)
    rows = [rng.uniform(-1, 1, d) * 10.0 ** rng.integers(-300, 300, d) for _ in range(8)]
    rows += [rng.standard_normal(d) for _ in range(8)]
    E = d // 32
    for i, p in enumerate(es.edge_partials().values()):
        t = np.zeros(d)
        for lane in range(32):
            j = (i + lane) % E
            t[lane * E + j] = p[lane]
        rows.append(t)
    terms = np.array(rows)
    got = _group_sums(emu, d, terms)
    want = np.array([_oracle_sum(t) for t in terms])
    assert es.same_bits(got, want)
    with np.errstate(all="ignore"):
        assert es.same_bits(got, es.warp_sum(terms))


# ---------------------------------------------------------------- the plan and the registers (CPU) ----

def _nvcc(*args):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    return subprocess.run([NVCC, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC,
                           "-I", os.path.join(HERE, "..", "include"), *args], check=True, capture_output=True, text=True)


def test_plan_program_prints_the_plan(tmp_path):
    """A host-only program prints LbfgsGroupPlan<double, d, 10>: groups (= resident instances) per CTA, warps per
    group and bytes, as the launcher hands them to launch_persistent."""
    lines = [f'  printf("%d|%d|%d|%d|%zu\\n", {d}, LbfgsGroupPlan<double, {d}, 10>::kWarps, '
             f"LbfgsGroupPlan<double, {d}, 10>::kGroupWarps, LbfgsGroupPlan<double, {d}, 10>::kThreads, "
             f"LbfgsGroupPlan<double, {d}, 10>::kBytes);" for d in DS]
    prog = tmp_path / "plan.cu"
    prog.write_text('#include <cstdio>\n#include "cno_lbfgs_group.cuh"\nusing namespace cno;\nint main() {\n'
                    + "\n".join(lines) + "\n}\n")
    _nvcc(str(prog), "-o", str(tmp_path / "plan"))
    out = subprocess.run([str(tmp_path / "plan")], check=True, capture_output=True, text=True).stdout
    got = {}
    for line in out.splitlines():
        d, groups, warps, threads, nbytes = map(int, line.split("|"))
        assert threads == 32 * groups * warps and nbytes <= 227 * 1024
        got[d] = (groups, warps, nbytes)
    assert got == PLAN


def test_group_kernels_keep_everything_in_registers(tmp_path):
    """ptxas -v: no stack frame and no spills in the three group kernels, and no local-memory instruction in their
    SASS."""
    src = tmp_path / "k.cu"
    inst = "\n".join(
        f"template __global__ void cno::lbfgs_group_minimize_kernel<cno::GroupRosenbrockFn<double, {d}>, 10>("
        f"cno::GroupRosenbrockFn<double, {d}>, const double*, long long, cno::StopParams<double>, "
        f"cno::BatchOut<double>, unsigned long long*);" for d in DS)
    src.write_text('#include "cno_lbfgs_group.cuh"\n' + inst + "\n")
    cubin = tmp_path / "k.cubin"
    r = _nvcc("-O3", "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false", "-Xptxas", "-v", "-cubin",
              str(src), "-o", str(cubin))
    props = re.findall(r"lbfgs_group_minimize_kernel.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stderr)
    assert len(props) == 3, r.stderr
    assert all(p == ("0", "0", "0") for p in props), props
    sass = subprocess.run([CUOBJDUMP, "-sass", str(cubin)], check=True, capture_output=True, text=True).stdout
    assert sass.count("Function : ") == 3
    assert not re.search(r"\b(LDL|STL)\b", sass)
