"""User objectives past d = 128 on the CPU: the group L-BFGS kernel's device source on user functors and composites at
d = 1024 under the warp emulation, against the reference's own FunctionCRTP functors and operators (oracle/_ref); and
the library of tests/cpp/user_group_functions.cu, where CNO_INSTANTIATE_FUNCTION compiles Rosenbrock at d = 512 and
1024, composites at 1024 and a functor without the group form, with the group kernels free of stack and spills.  The
GPU side is tests/test_user_group_gpu.py."""
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
LIB = os.path.join(HERE, "cpp", "build", "libcno_usergroup.so")
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
D = 1024
EXPR_PROD_ROSEN = 100  # (Rosenbrock + 1) (Rosenbrock + 1): tests/emu/emu_user_group.cc only


def bitwise_equal(a, b, keys=KEYS):
    for k in keys:
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


def stop_after(iterations):
    s = ob.default_stop()
    s.num_iterations = iterations
    return s


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("emu_user_group")), "libcno_emu_user_group.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-pthread",
                    "-DCNO_WARP_EMULATION", "-Wno-unknown-pragmas", "-Wno-attributes", "-shared", "-I", EMU_DIR,
                    "-I", CSRC, "-I", os.path.join(HERE, "..", "include"), "-x", "c++",
                    os.path.join(EMU_DIR, "emu_user_group.cc"), "-o", out], check=True)
    lib = C.CDLL(out)
    lib.emu_user_group.argtypes = [C.c_int, C.c_double, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _emulated(emu, expr, x0, stop, param=0.0):
    r, out = ob._batch_out(x0)
    assert emu.emu_user_group(expr, param, x0.shape[0], x0.ctypes.data, C.byref(stop), C.byref(out)) == 0
    return r


# (expr, param, iterations): Bowl converges within the limit; the others stop at it
CASES = [(ob.EXPR_BOWL, 0.5, 10000), (ob.EXPR_ROSEN_PLUS_HALF, 0.0, 5), (ob.EXPR_PENALTY, 0.0, 5),
         (ob.EXPR_ZERO_MUL, 0.0, 10000)]


@pytest.mark.parametrize("expr,param,iterations", CASES, ids=["bowl", "rosen_plus_half", "penalty", "zero_mul"])
def test_emulated_group_kernel_on_user_objectives_equals_reference(emu, expr, param, iterations):
    """lbfgs_group_minimize_kernel on a group-form functor and on composites of the mirror's group-form leaves, at
    d = 1024: every output bit for bit against Lbfgs<decltype(composite)>::Minimize of the reference's own headers."""
    if not ob.ref_available():
        pytest.skip("oracle/_ref not built")
    x0 = np.ascontiguousarray(ob.fill_uniform((2, D), 0, 7, -2.0, 2.0))
    stop = stop_after(iterations)
    ref = ob.ref_minimize_expr(expr, ob.LBFGS, x0, param=param, stop=stop)
    if iterations < 100:
        assert (ref["num_iterations"] == iterations + 1).all()
    else:
        assert (ref["status"] != 0).all() and (ref["num_iterations"] < iterations).all()
    # nfev only for a single functor: the reference's counter ticks once per leaf evaluation of a composite
    bitwise_equal(_emulated(emu, expr, x0, stop, param), ref,
                  KEYS if expr == ob.EXPR_BOWL else tuple(k for k in KEYS if k != "nfev"))


def test_emulated_two_exchanging_leaves(emu):
    """(Rosenbrock + 1) (Rosenbrock + 1) evaluates both leaves through the one exchange block: the value and gradient
    it returns equal (r + 1)^2 and 2 (r + 1) g_r formed from the oracle's Rosenbrock at the returned x, bit for bit."""
    x0 = np.ascontiguousarray(ob.fill_uniform((2, D), 0, 8, -2.0, 2.0))
    r = _emulated(emu, EXPR_PROD_ROSEN, x0, stop_after(3))
    assert (r["num_iterations"] == 4).all()
    fr, gr = ob.evaluate(ob.FN_ROSENBROCK, r["x"])
    f1 = fr + 1.0
    assert np.array_equal(r["value"].view(np.uint64), (f1 * f1).view(np.uint64))
    g = f1[:, None] * gr + f1[:, None] * gr  # ProdExpression: gx grad_f + fx grad_g
    assert np.array_equal(r["gradient"].view(np.uint64), g.view(np.uint64))


# ---------------------------------------------------------------- the compiled library (CPU) ----

def _library():
    if not os.path.exists(LIB):
        from cppnumericalsolvers_b200 import build
        build.build_cpp_tests()
    return LIB


def test_macro_instantiates_past_d128():
    """CNO_INSTANTIATE_FUNCTION defines every symbol for Rosenbrock at d = 512 and 1024, composites at 1024 and a
    functor at 1024 without the group form (the Bfgs case, whose inverse Hessian does not fit, returns
    CNO_ERR_UNSUPPORTED instead of failing to compile)."""
    syms = subprocess.run(["nm", "-D", "--defined-only", _library()], check=True, capture_output=True, text=True).stdout
    for tag in ("rosen512", "rosen1024", "rph1024", "zmul1024", "pen1024", "prodrosen1024", "gbowl1024", "bowl1024"):
        for op in ("minimize", "state_bytes", "minimize_steps", "evaluate", "condition_hessian"):
            assert re.search(rf"\bcno_{tag}_{op}\b", syms), (tag, op)


def test_user_group_kernels_keep_everything_in_registers():
    """cuobjdump -res-usage: the group kernels of the user objectives (one per d = 1024 functor with the group form)
    have no stack frame and no local memory, and the functor without the group form has none."""
    res = subprocess.run([CUOBJDUMP, "-res-usage", _library()], check=True, capture_output=True, text=True).stdout
    rows = re.findall(r"Function (\S*lbfgs_group_minimize_kernel\S*):\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)",
                      res)
    names = [r[0] for r in rows]
    assert len(rows) == 6, names  # GroupBowl, the three composites, ProdRosen, Rosenbrock<1024>
    assert not any("PlainBowl" in n or "RosenbrockIdLi512" in n for n in names)
    assert all(stack == "0" and local == "0" for _, _, stack, local in rows), rows
