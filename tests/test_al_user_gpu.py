"""AugmentedLagrangian on user functors and composite constraints on the GPU (cno_<tag>_al_minimize from
CNO_INSTANTIATE_CONSTRAINED, the problems of tests/cpp/al_user_problems.cuh): every cno_al_out_t array bit for bit
against the reference's own solver (oracle/_ref), the committed fixtures, per-instance data, equivalence with
cno_al_minimize on the same rows, the launch count, argument errors and the C++ mirror."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import cppnumericalsolvers_b200 as cn
from cppnumericalsolvers_b200 import _lib
import al_user_ref as ar
from oracle import oracle_binding as ob

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
DEV = "cuda:0"
TDT = {np.dtype(np.float64): torch.float64, np.dtype(np.float32): torch.float32}
COUNTS = ar.COUNTS
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
LIBDIR = os.path.join(ROOT, "cppnumericalsolvers_b200")
DEV_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false", "-prec-div=true",
             "-prec-sqrt=true", "-ftz=false"]
INC = ["-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(LIBDIR, "csrc"), "-I" + os.path.join(HERE, "cpp")]


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def alu(tmp_path_factory):
    """tests/cpp/al_user_functions.cu built into a temporary directory."""
    out = tmp_path_factory.mktemp("al_user") / "libcno_al_user.so"
    subprocess.run([os.environ.get("NVCC", f"{CUDA}/bin/nvcc"), *DEV_FLAGS, "-shared", "-Xcompiler", "-fPIC",
                    os.path.join(HERE, "cpp", "al_user_functions.cu"), *INC, "-o", str(out), f"-L{LIBDIR}", "-lcno",
                    "-Xlinker", f"-rpath={LIBDIR}"], check=True)
    _lib.lib()
    return C.CDLL(str(out))


def outer_stop(limit):
    s = ob.al_default_stop()
    s.num_iterations = limit
    return s


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def gpu(alu, problem, x0_np, *, data=None, stride=0, penalty0=None, limit=10000, out_skip=(), x_offset=0,
        workspace_bytes=None):
    """cno_<tag>_al_minimize through cno_test_al_user; returns (rc, host outputs, launch info)."""
    B, d = x0_np.shape
    dt = TDT[x0_np.dtype]
    ne, ni = COUNTS[problem]
    dtype = 0 if x0_np.dtype == np.float64 else 1
    x0 = torch.zeros(B * d + 2, dtype=dt, device=DEV)
    x0[x_offset:x_offset + B * d] = torch.from_numpy(np.ascontiguousarray(x0_np)).reshape(-1).to(DEV)
    t = {k: torch.zeros(a.shape, dtype=TDT.get(a.dtype, {np.dtype(np.uint32): torch.int32,
                                                         np.dtype(np.int8): torch.int8}.get(a.dtype)), device=DEV)
         for k, a in ar.out_arrays(B, d, ne, ni, x0_np.dtype).items()}
    out = ob.AlOut(*[None if k in out_skip else t[k].data_ptr() for k in ar.OUT_KEYS])
    dev_data = None if data is None else torch.from_numpy(np.ascontiguousarray(data)).to(DEV)
    nbytes = C.c_size_t(0)
    assert alu.cno_test_al_user(problem, dtype, d, None, C.c_int64(0), C.c_int64(B), *([None] * 8), None, C.c_size_t(0),
                                None, None, C.byref(nbytes)) == 0
    ws = torch.zeros(max(nbytes.value, 256) + 256, dtype=torch.uint8, device=DEV)
    pen = None if penalty0 is None else torch.full((B,), penalty0, dtype=dt, device=DEV)
    info = _lib.LaunchInfo()
    rc = alu.cno_test_al_user(problem, dtype, d, _ptr(dev_data), C.c_int64(stride), C.c_int64(B),
                              C.c_void_p(x0.data_ptr() + x_offset * x0.element_size()), None, None, _ptr(pen),
                              C.byref(ob.default_stop()), C.byref(outer_stop(limit)), C.byref(ob.al_default_config()),
                              C.byref(out), C.c_void_p(ws.data_ptr()),
                              C.c_size_t(nbytes.value if workspace_bytes is None else workspace_bytes),
                              C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(info), None)
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy() for k, v in t.items()}
    r["num_iterations"] = r["num_iterations"].astype(np.uint32)
    r["nfev"] = r["nfev"].astype(np.uint32)
    return rc, r, info


def bitwise_equal(a, b, rows=slice(None)):
    for k in ar.OUT_KEYS:
        assert np.array_equal(np.asarray(a[k])[rows].view(np.uint8), np.asarray(b[k])[rows].view(np.uint8)), k


# (problem, dtype, d, outer limit, penalty0): the reference's runs of problems 3 and 4 meet the KKT test late, so
# their outer loop is cut short
CASES = [(ar.AL_P_HS029, np.float64, 2, 10000, 0.0), (ar.AL_P_SIMPLE, np.float64, 2, 10000, 1.0),
         (ar.AL_P_COMPOSITE_CONS, np.float64, 2, 10000, None), (ar.AL_P_COMPOSITES, np.float64, 8, 8, None),
         (ar.AL_P_COMPOSITES, np.float64, 128, 3, None), (ar.AL_P_COMPOSITES, np.float32, 37, 6, None),
         (ar.AL_P_BALL_OF_INSTANCE, np.float64, 37, 6, None), (ar.AL_P_BOWL, np.float64, 16, 10000, None),
         (ar.AL_P_DOWNGRADE, np.float64, 2, 10000, None)]


def radii(B):
    return 2.0 + ob.fill_uniform((B, 1), 0, 71, 0.0, 3.0)[:, 0]


@pytest.mark.parametrize("problem,dtype,d,limit,penalty0", CASES,
                         ids=[f"p{p}-{np.dtype(t).name}-d{d}" for p, t, d, _, _ in CASES])
@pytest.mark.parametrize("batch", ("1", "7", "full"))
def test_gpu_equals_reference(alu, problem, dtype, d, limit, penalty0, batch):
    needs_ref()
    B = {"1": 1, "7": 7, "full": 3 * sms() * 8 + 5}[batch]
    x0 = ob.fill_uniform((B, d), 0, 90 + problem * 7 + d, -1.5, 1.5, dtype)
    data = radii(B) if problem == ar.AL_P_BALL_OF_INSTANCE else None
    rc, g, info = gpu(alu, problem, x0, data=data, penalty0=penalty0, limit=limit)
    assert rc == 0
    bitwise_equal(g, ar.minimize(problem, x0, data=data, penalty0=penalty0, outer_stop=outer_stop(limit)))
    assert info.kernel_launches == 2 * int(g["num_iterations"].max()) + 2


def needs_ref():
    if not ar.available():
        pytest.skip("oracle/_ref/libcno_ref_al_user.so not built")


def test_gpu_hs029_meets_the_reference_tolerances(alu):
    """augmented_lagrangian_test.cc:1106-1154 from (1, 1)."""
    rc, g, _ = gpu(alu, ar.AL_P_HS029, np.array([[1.0, 1.0]]), penalty0=0.0)
    assert rc == 0
    x = g["x"][0]
    assert abs(x[0] - 2 * math.sqrt(6)) <= 0.2 and abs(x[1] - 2 * math.sqrt(3)) <= 0.2
    assert abs(-x[0] * x[1] + 12 * math.sqrt(2)) <= 0.5


@pytest.mark.parametrize("name", ("user_al_hs029_d2_f64", "user_al_composites_d8_f64"))
def test_gpu_reproduces_fixture(alu, name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    rc, g, _ = gpu(alu, int(z["problem"]), z["x0"], penalty0=float(z["penalty0"]), limit=int(z["outer_limit"]))
    assert rc == 0
    bitwise_equal(g, {k: z[k] for k in ar.OUT_KEYS})


def test_gpu_per_instance_data_isolated(alu):
    """Problem 4 reads its radius through ctx.instance: rows of a full batch equal the same rows solved alone."""
    B, d = 3 * sms() * 8 + 5, 37
    x0 = ob.fill_uniform((B, d), 0, 77, -1.5, 1.5)
    r = radii(B)
    _, full, _ = gpu(alu, ar.AL_P_BALL_OF_INSTANCE, x0, data=r, limit=6)
    for rows in (slice(0, 1), slice(B // 2, B // 2 + 3), slice(B - 2, B)):
        _, alone, _ = gpu(alu, ar.AL_P_BALL_OF_INSTANCE, x0[rows], data=r[rows], limit=6)
        bitwise_equal(alone, {k: v[rows] for k, v in full.items()})


def _rows_path(x0, rows, limit):
    """cno_al_minimize on [SQNORM, AFFINE] rows (one equality, one inequality), Rosenbrock."""
    B, d = x0.shape
    dt = TDT[x0.dtype]
    problem = cn.ConstrainedOptimizationProblem(cn.Rosenbrock(d, dt), [ob.CON_SQNORM, ob.CON_AFFINE],
                                                torch.from_numpy(rows).to(DEV), 1)
    solver = cn.AugmentedLagrangian(problem)
    solver.stopping_progress.num_iterations = limit
    st, pr = solver.Minimize(cn.AugmentedLagrangeState(torch.from_numpy(x0).to(DEV)))
    torch.cuda.synchronize()
    return dict(x=st.x.cpu().numpy(), equality_multipliers=st.equality_multipliers.cpu().numpy(),
                inequality_multipliers=st.inequality_multipliers.cpu().numpy(), penalty=st.penalty.cpu().numpy(),
                max_violation=st.max_violation.cpu().numpy(),
                max_lagrangian_gradient=st.max_lagrangian_gradient.cpu().numpy(),
                num_iterations=pr.num_iterations.cpu().numpy().astype(np.uint32), status=pr.status.cpu().numpy(),
                nfev=pr.nfev.cpu().numpy().astype(np.uint32), x_delta=pr.x_delta.cpu().numpy(),
                f_delta=pr.f_delta.cpu().numpy(), gradient_norm=pr.gradient_norm.cpu().numpy()), pr.launch


@pytest.mark.parametrize("dtype,d,per_instance", [(np.float64, 8, True), (np.float64, 128, False),
                                                  (np.float32, 8, True)])
def test_row_functors_equal_cno_al_minimize(alu, dtype, d, per_instance):
    """Problem 5: SqNormRow / AffineRow functors on the rows cno_al_minimize reads -- the functor path and the row
    path compute the same bits and launch the same number of kernels."""
    B = 3 * sms() * 8 + 5 if d == 8 else 256
    rng = np.random.default_rng(d)
    x0 = ob.fill_uniform((B, d), 0, 33 + d, -1.5, 1.5, dtype)
    shape = (B, 2, d + 1) if per_instance else (2, d + 1)
    rows = rng.uniform(-1, 1, shape).astype(dtype)
    rows[..., 0, d] = 2.0 + rng.uniform(0, 1, shape[:-2])
    rc, g, info = gpu(alu, ar.AL_P_ROWS, x0, data=rows, stride=2 * (d + 1) if per_instance else 0, limit=10)
    assert rc == 0
    r, launch = _rows_path(x0, rows, 10)
    bitwise_equal(g, r)
    assert info.kernel_launches == launch.kernel_launches


def test_argument_errors_match_cno_al_minimize(alu):
    """The checks of cno_al_minimize, in its order and with its codes."""
    x0 = ob.fill_uniform((4, 2), 0, 5, -1.5, 1.5)
    assert gpu(alu, ar.AL_P_SIMPLE, x0, out_skip=("nfev",))[0] == _lib.ERR_INVALID_ARGUMENT
    assert gpu(alu, ar.AL_P_SIMPLE, x0, out_skip=("equality_multipliers",))[0] == _lib.ERR_INVALID_ARGUMENT
    assert gpu(alu, ar.AL_P_HS029, x0, out_skip=("equality_multipliers",))[0] == _lib.OK  # (no equalities)
    assert gpu(alu, ar.AL_P_SIMPLE, x0, x_offset=1)[0] == _lib.ERR_INVALID_ARGUMENT  # 8-byte aligned x0
    assert gpu(alu, ar.AL_P_SIMPLE, x0, workspace_bytes=256)[0] == _lib.ERR_WORKSPACE
    # the same inputs through cno_al_minimize
    B, d = x0.shape
    xd = torch.from_numpy(x0).to(DEV)
    rows = torch.tensor([[1.0, 0.0, 0.5], [-1.0, -1.0, -2.0]], dtype=torch.float64, device=DEV)
    kinds = torch.tensor([0, 0], dtype=torch.int32, device=DEV)
    k = _lib.Constraints(1, 1, kinds.data_ptr(), rows.data_ptr(), 0)
    p = _lib.Problem(family=ob.FN_HALF_SQUARED_NORM, dtype=_lib.F64, d=2, policy=_lib.POLICY_DMMA_TREE)
    arrays = {k_: torch.zeros(a.shape, dtype={np.dtype(np.uint32): torch.int32, np.dtype(np.int8): torch.int8}.get(
        a.dtype, torch.float64), device=DEV) for k_, a in ar.out_arrays(B, d, 1, 1, np.float64).items()}

    def call(skip=(), x=xd.data_ptr(), wsb=None):
        out = _lib.AlOut(*[None if n in skip else arrays[n].data_ptr() for n in ar.OUT_KEYS])
        nb = C.c_size_t(0)
        _lib.check(_lib.lib().cno_al_workspace_bytes(C.byref(p), C.byref(k), C.c_int64(B), C.byref(nb)), "ws")
        ws = torch.zeros(nb.value + 256, dtype=torch.uint8, device=DEV)
        return _lib.lib().cno_al_minimize(C.byref(p), C.byref(k), C.c_int64(B), C.c_void_p(x), None, None, None, None,
                                          None, None, C.byref(out), C.c_void_p(ws.data_ptr()),
                                          C.c_size_t(nb.value if wsb is None else wsb), None, None)
    assert call(skip=("nfev",)) == _lib.ERR_INVALID_ARGUMENT
    assert call(skip=("equality_multipliers",)) == _lib.ERR_INVALID_ARGUMENT
    assert call(x=xd.data_ptr() + 8) == _lib.ERR_INVALID_ARGUMENT
    assert call(wsb=256) == _lib.ERR_WORKSPACE
    # B = 0
    info = _lib.LaunchInfo()
    assert alu.cno_test_al_user(ar.AL_P_SIMPLE, 0, 2, None, C.c_int64(0), C.c_int64(0), None, None, None, None, None,
                                None, None, C.byref(_lib.AlOut()), None, C.c_size_t(0), None, C.byref(info),
                                None) == _lib.OK
    assert info.kernel_launches == 0


def test_cpp_mirror_hs029(tmp_path):
    """tests/cpp/al_user_host.cu: the C++ mirror on augmented_lagrangian_test.cc's Hs029, written like that test."""
    exe = tmp_path / "al_user_host"
    subprocess.run([os.environ.get("NVCC", f"{CUDA}/bin/nvcc"), *DEV_FLAGS, os.path.join(HERE, "cpp", "al_user_host.cu"),
                    *INC, "-o", str(exe), f"-L{LIBDIR}", "-lcno", "-Xlinker", f"-rpath={LIBDIR}"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout + r.stderr
