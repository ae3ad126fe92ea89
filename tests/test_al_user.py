"""AugmentedLagrangian on user functors and composite constraints (ConstrainedOptimizationProblem<Objective,
Equalities<...>, Inequalities<...>>, cno_<tag>_al_minimize), on the CPU: the reference's own solver on the test
problems of tests/cpp/al_user_problems.cuh against its known answers and the committed fixtures; the device source
under the CPU warp emulation against the reference bit for bit; the GPU test library compiles for sm_90a.  The GPU side
is tests/test_al_user_gpu.py."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import al_user_ref as ar
from oracle import oracle_binding as ob

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU_DIR = os.path.join(HERE, "emu")
CSRC = os.path.join(ROOT, "cppnumericalsolvers_b200", "csrc")
GOLDEN = os.path.join(HERE, "golden")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FIXTURES = ("user_al_hs029_d2_f64", "user_al_composites_d8_f64")
COUNTS = ar.COUNTS


def needs_ref():
    if not ar.available():
        pytest.skip("oracle/_ref/libcno_ref_al_user.so not built")


def bitwise_equal(a, b):
    for k in ar.OUT_KEYS:
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


def outer_stop(limit):
    s = ob.al_default_stop()
    s.num_iterations = limit
    return s


def test_ref_hs029_meets_the_reference_tolerances():
    """augmented_lagrangian_test.cc:1106-1154 (Hs029EllipseEscapesOrigin) from (1, 1), penalty 0 (auto-scale)."""
    needs_ref()
    r = ar.minimize(ar.AL_P_HS029, np.array([[1.0, 1.0]]), penalty0=0.0)
    x = r["x"][0]
    assert abs(x[0] - 2 * math.sqrt(6)) <= 0.2 and abs(x[1] - 2 * math.sqrt(3)) <= 0.2
    assert abs(-x[0] * x[1] - (-12 * math.sqrt(2))) <= 0.5


def test_ref_constrained_simple_reaches_the_optimum():
    """src/examples/constrained_simple.cc: x* = (0.5, 1.5) from (1, 1), penalty 1."""
    needs_ref()
    r = ar.minimize(ar.AL_P_SIMPLE, np.array([[1.0, 1.0]]), penalty0=1.0)
    assert np.all(np.abs(r["x"][0] - [0.5, 1.5]) <= 1e-3)


@pytest.mark.parametrize("name", FIXTURES)
def test_ref_reproduces_fixture(name):
    needs_ref()
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    r = ar.minimize(int(z["problem"]), z["x0"], penalty0=float(z["penalty0"]),
                    outer_stop=outer_stop(int(z["outer_limit"])))
    bitwise_equal(r, {k: z[k] for k in ar.OUT_KEYS})


# ---------------------------------------------------------------- emulation ----

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/emu/emu_al_user.cc compiled with the flags of tests/emu/Makefile into a temporary directory."""
    out = tmp_path_factory.mktemp("emu_al_user") / "libcno_emu_al_user.so"
    subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-pthread",
                    "-DCNO_WARP_EMULATION", "-Wno-unknown-pragmas", "-Wno-attributes", "-shared", "-I", EMU_DIR,
                    "-I", CSRC, "-I", os.path.join(ROOT, "include"), "-I", os.path.join(HERE, "cpp"), "-x", "c++",
                    os.path.join(EMU_DIR, "emu_al_user.cc"), "-o", str(out)], check=True)
    return C.CDLL(str(out))


def emulated(emu, problem, x0, *, data=None, stride=0, penalty0=None, limit=10000):
    B, d = x0.shape
    ne, ni = COUNTS[problem]
    dt = x0.dtype
    r = ar.out_arrays(B, d, ne, ni, dt)
    o = ob.AlOut(*[r[n].ctypes.data for n in ar.OUT_KEYS])
    pen = None if penalty0 is None else np.full(B, penalty0, dt)
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    launches = C.c_int(0)
    rc = emu.emu_al_user_minimize(problem, 0 if dt == np.float64 else 1, d, ptr(data), C.c_longlong(stride),
                                  C.c_longlong(B), C.c_void_p(x0.ctypes.data), None, None, ptr(pen),
                                  C.byref(ob.default_stop()), C.byref(outer_stop(limit)),
                                  C.byref(ob.al_default_config()), C.byref(o), C.byref(launches))
    assert rc == 0
    r["launches"] = launches.value
    return r


EMU_CASES = [(ar.AL_P_HS029, 2, 0.0, 10000), (ar.AL_P_SIMPLE, 2, 1.0, 10000), (ar.AL_P_COMPOSITES, 8, None, 8)]


@pytest.mark.parametrize("problem,d,penalty0,limit", EMU_CASES, ids=["hs029", "constrained_simple", "composites_d8"])
def test_emulated_device_source_equals_reference(emu, problem, d, penalty0, limit):
    """AugLagFn<Obj, AlFunctors<...>>, the AL kernels and the fused L-BFGS kernel under the warp emulation, driven by
    al_outer_loop: all 12 cno_al_out_t arrays equal the reference's own solver bit for bit."""
    needs_ref()
    x0 = np.concatenate([[[1.0] * d], ob.fill_uniform((5, d), 0, 50 + d, -1.5, 1.5)])
    e = emulated(emu, problem, x0, penalty0=penalty0, limit=limit)
    bitwise_equal(e, ar.minimize(problem, x0, penalty0=penalty0, outer_stop=outer_stop(limit)))
    # auto-scale (on by default; it skips nonzero penalties) + (inner + outer step) per outer iteration + finalize
    assert e["launches"] == 2 * int(e["num_iterations"].max()) + 2


def test_emulated_row_functors_equal_the_row_composite(emu):
    """Problem 5's SqNormRow / AffineRow functors read [a | t] rows as cno_al_minimize does: its composite equals the
    row path's ToAugmentedLagrangian (the pinned C oracle, itself bit-identical to the device row path)."""
    B, d = 16, 8
    rng = np.random.default_rng(3)
    x = ob.fill_uniform((B, d), 0, 61, -1.5, 1.5)
    rows = rng.uniform(-1, 1, (B, 2, d + 1))
    rows[:, 0, d] = 2.0 + rng.uniform(0, 1, B)
    lam, mu, pen = rng.uniform(-1, 1, (B, 1)), rng.uniform(0, 1, (B, 1)), rng.uniform(0.5, 5, B)
    lam[0] = 0.0  # (the c == 0 short cut of the Lagrangian term)
    v, g = np.zeros(B), np.zeros((B, d))
    assert emu.emu_al_user_composite(ar.AL_P_ROWS, 0, d, C.c_void_p(rows.ctypes.data), C.c_longlong(2 * (d + 1)),
                                     C.c_longlong(B), C.c_void_p(x.ctypes.data), C.c_void_p(lam.ctypes.data),
                                     C.c_void_p(mu.ctypes.data), C.c_void_p(pen.ctypes.data), C.c_void_p(v.ctypes.data),
                                     C.c_void_p(g.ctypes.data)) == 0
    ov, og = ob.al_evaluate(ob.FN_ROSENBROCK, x, [ob.CON_SQNORM, ob.CON_AFFINE], rows, 1, lam, mu, pen)
    assert np.array_equal(v.view(np.uint64), ov.view(np.uint64))
    assert np.array_equal(g.view(np.uint64), og.view(np.uint64))


def test_test_library_compiles_for_sm90a(tmp_path):
    """tests/cpp/al_user_functions.cu (CNO_DECLARE_CONSTRAINED + CNO_INSTANTIATE_CONSTRAINED on every problem)
    cross-compiles for sm_90a with no stack in the new AL kernels at d <= 37."""
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                        "-prec-div=true", "-prec-sqrt=true", "-ftz=false", "-Xptxas", "-v", "-c",
                        os.path.join(HERE, "cpp", "al_user_functions.cu"), "-I", os.path.join(ROOT, "include"),
                        "-I", CSRC, "-I", os.path.join(HERE, "cpp"), "-o", str(tmp_path / "al_user.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = r.stderr.split("Compiling entry function")[1:]
    assert len(blocks) >= 4 * 8  # autoscale, inner, outer step (+ finalize per (dtype, d)) for every problem
    for b in blocks:
        if "AlFunctors" in b and ("al_autoscale_kernel" in b or "al_outer_step_kernel" in b):
            assert "0 bytes stack frame" in b, b[:400]
