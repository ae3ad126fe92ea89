"""Lbfgs on user objectives at d = 1024 through CNO_INSTANTIATE_FUNCTION on the GPU (tests/cpp/user_group_functions.cu):
functors with the group form run the group kernel (csrc/cno_lbfgs_group.cuh), bit for bit equal to the reference's own
operators and to the one-warp kernel on the same type; every case the routing leaves to the one-warp kernel gives the
one-warp kernel's bits; Bfgs past d = 128 is refused.  The CPU side is tests/test_user_group.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from cppnumericalsolvers_b200 import _lib
from oracle import oracle_binding as ob

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "cpp", "build", "libcno_usergroup.so")
KEYS = ("x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta", "gradient_norm")
D = 1024
GROUP = 0  # cno_<tag>_minimize
ONE_WARP = 1  # cno::user_lbfgs: the one-warp kernel
# tag -> (reference twin EXPR_* or None, Bowl's c)
TAGS = {"gbowl1024": (ob.EXPR_BOWL, 0.5), "rph1024": (ob.EXPR_ROSEN_PLUS_HALF, 0.0),
        "pen1024": (ob.EXPR_PENALTY, 0.0), "zmul1024": (ob.EXPR_ZERO_MUL, 0.0), "prodrosen1024": (None, 0.0),
        "rosen1024": (None, 0.0)}
SENTINEL = {"x": np.nan, "value": -7.0, "gradient": np.nan, "num_iterations": 77, "status": 99, "nfev": 55,
            "x_delta": -3.0, "f_delta": -3.0, "gradient_norm": -3.0}

_handle = None


def lib():
    global _handle
    if _handle is None:
        if not os.path.exists(LIB):
            from cppnumericalsolvers_b200 import build
            build.build_cpp_tests()
        _lib.lib()
        _handle = C.CDLL(LIB)
    return _handle


def run(tag, x0_np, *, path=GROUP, solver=0, stop=None, param=None, lbfgs_m=0, rows=None, skip=()):
    """ug_<tag> on a batch; `rows` > B allocates sentinel-filled rows past the batch; `skip` = outputs not requested."""
    x0 = torch.from_numpy(np.ascontiguousarray(x0_np)).cuda()
    B = x0.shape[0]
    R = rows or B
    t = {}
    for k in KEYS:
        shape = (R, D) if k in ("x", "gradient") else (R,)
        dt = {"num_iterations": torch.int32, "nfev": torch.int32, "status": torch.int8}.get(k, torch.float64)
        t[k] = torch.full(shape, SENTINEL[k], dtype=dt, device="cuda")
    out = _lib.BatchOut(*[0 if k in skip else t[k].data_ptr() for k in KEYS])
    ws = torch.zeros(256, dtype=torch.uint8, device="cuda")
    info = _lib.LaunchInfo()
    p = TAGS.get(tag, (None, 0.0))[1] if param is None else param
    fn = getattr(lib(), "ug_" + tag)
    rc = fn(path, solver, lbfgs_m, C.c_double(p), C.c_int64(B), C.c_void_p(x0.data_ptr()),
            C.byref(stop) if stop is not None else None, C.byref(out), C.c_void_p(ws.data_ptr()), C.c_size_t(256),
            C.byref(info))
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy() for k, v in t.items()}
    r["num_iterations"] = r["num_iterations"].astype(np.uint32)
    r["nfev"] = r["nfev"].astype(np.uint32)
    r["rc"], r["launch"] = rc, info
    return r


def same(a, b, keys=KEYS, rows=slice(None)):
    for k in keys:
        assert np.array_equal(np.asarray(a[k])[rows].view(np.uint8), np.asarray(b[k])[rows].view(np.uint8)), k


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def starts(B, seed):
    return ob.fill_uniform((B, D), 0, seed, -2.0, 2.0)


@pytest.mark.parametrize("tag", [t for t, (e, _) in TAGS.items() if e is not None])
def test_group_path_equals_reference(tag):
    """cno_<tag>_minimize at d = 1024 (the group kernel) against Lbfgs<decltype(composite)>::Minimize of the reference's
    own operators, every output bit for bit (nfev only for a single functor: the reference counts leaf calls)."""
    if not ob.ref_available():
        pytest.skip("oracle/_ref not built")
    expr, param = TAGS[tag]
    x0 = starts(6, 31)
    stop = ob.default_stop()
    stop.num_iterations = 40
    g = run(tag, x0, stop=stop)
    assert g["rc"] == 0
    ref = ob.ref_minimize_expr(expr, ob.LBFGS, x0, param=param, stop=stop, threads=ob.num_threads())
    same(g, ref, KEYS if expr == ob.EXPR_BOWL else tuple(k for k in KEYS if k != "nfev"))


@pytest.mark.parametrize("tag", list(TAGS))
def test_group_path_equals_one_warp_kernel(tag):
    """The group kernel and the one-warp kernel on the same type, to convergence, at B = 2 SMs + 3 (every CTA of the
    group kernel drains several instances): identical bits; the group launch has the built-in d = 1024 shape."""
    B = 2 * sms() + 3
    x0 = starts(B, 32)
    g = run(tag, x0)
    w = run(tag, x0, path=ONE_WARP)
    assert g["rc"] == 0 and w["rc"] == 0
    same(g, w)
    assert (g["status"] != 0).all()
    info = g["launch"]
    assert (info.block, info.warps_per_cta, info.dynamic_smem) == (256, 1, 186128)
    assert w["launch"].dynamic_smem != 186128


def test_isolation_nan_rows_iteration_limit_and_padding():
    """NaN starts next to normal rows, uneven iteration counts and the iteration limit, with rows past the batch and an
    unrequested output: each row equals its own solve, sentinels stay where nothing was asked for."""
    B = 2 * sms() + 3
    x0 = starts(B, 33)
    x0[::7, 100] = np.nan
    x0[3::11] = 1.0 + 1e-3 * x0[3::11]
    stop = ob.default_stop()
    stop.num_iterations = 150
    g = run("rph1024", x0, stop=stop, rows=B + 5, skip=("gradient_norm",))
    assert g["rc"] == 0
    w = run("rph1024", x0, path=ONE_WARP, stop=stop)
    same(g, w, tuple(k for k in KEYS if k != "gradient_norm"), rows=slice(0, B))
    its = g["num_iterations"][:B]
    assert (its == 151).any() and (its < 151).any() and len(np.unique(its)) > 3
    for k in KEYS:
        tail = g[k][B:]
        want = np.full_like(tail, SENTINEL[k])
        assert np.array_equal(tail.view(np.uint8), want.view(np.uint8)), k
    assert np.array_equal(g["gradient_norm"], np.full(B + 5, -3.0))
    nan_rows = np.isnan(x0).any(axis=1)
    one = run("rph1024", x0[~nan_rows][:3], stop=stop)  # the normal rows alone give the same bits
    same(one, {k: v[:B][~nan_rows][:3] for k, v in g.items() if k in KEYS}, tuple(k for k in KEYS if k != "gradient_norm"))


@pytest.mark.parametrize("case", ["no_group_form", "d512"])
def test_fallbacks_take_the_one_warp_path(case):
    """What the routing leaves to the one-warp kernel gives its bits: a functor without the group form, and d = 512."""
    if case == "no_group_form":
        x0 = starts(5, 34)
        g, w = run("bowl1024", x0), run("bowl1024", x0, path=ONE_WARP)
    else:
        x0 = ob.fill_uniform((5, 512), 0, 34, -2.0, 2.0)
        g, w = run_d(512, "rosen512", x0), run_d(512, "rosen512", x0, path=ONE_WARP)
    assert g["rc"] == 0 and w["rc"] == 0
    same(g, w)
    assert (g["launch"].block, g["launch"].dynamic_smem) == (w["launch"].block, w["launch"].dynamic_smem)


def test_other_solvers_and_m_keep_their_paths():
    """Lbfgs<F, m> for an m the tag was not compiled for is refused as before; HagerZhang runs the one-warp kernel."""
    x0 = starts(3, 37)
    assert run("rph1024", x0, lbfgs_m=7)["rc"] == _lib.ERR_UNSUPPORTED
    g = run("rph1024", x0, solver=_lib.LBFGS_HAGER_ZHANG)
    assert g["rc"] == 0 and g["launch"].dynamic_smem != 186128 and (g["status"] != 0).all()


def test_bfgs_and_newton_at_d1024_are_refused():
    """Bfgs (its inverse Hessian does not fit one SM) and NewtonDescent (no Hessian) on a d = 1024 functor return
    CNO_ERR_UNSUPPORTED."""
    x0 = starts(2, 35)
    for solver in (ob.BFGS, ob.NEWTON):
        assert run("rph1024", x0, solver=solver)["rc"] == _lib.ERR_UNSUPPORTED


def test_cpp_mirror_lbfgs_minimize():
    """cppoptlib::solver::Lbfgs<Rosenbrock + 0.5 HalfSquaredNorm at d = 1024>::Minimize from an nvcc translation unit:
    the same x, value and iterations as the symbol it binds to."""
    B = 4
    x0 = np.ascontiguousarray(starts(B, 36))
    x, v, it = np.zeros((B, D)), np.zeros(B), np.zeros(B, np.uint32)
    assert lib().ug_mirror_lbfgs_rph1024(C.c_int64(B), C.c_void_p(x0.ctypes.data), C.c_void_p(x.ctypes.data),
                                         C.c_void_p(v.ctypes.data), C.c_void_p(it.ctypes.data)) == 0
    g = run("rph1024", x0)
    assert np.array_equal(x.view(np.uint64), g["x"].view(np.uint64))
    assert np.array_equal(v.view(np.uint64), g["value"].view(np.uint64))
    assert np.array_equal(it, g["num_iterations"])


def run_d(d, tag, x0_np, path=GROUP):
    global D
    saved, D = D, d
    try:
        return run(tag, x0_np, path=path)
    finally:
        D = saved
