"""Launch shape of every persistent solver kernel, through the C ABI (-m gpu): for each compiled entry of cno_minimize,
cno_minimize_steps and cno_lbfgsb_minimize, and for one user functor per solver, a small solve at B = 1, 37 and 4096
must report the kernel_launches / block / warps_per_cta / dynamic_smem recorded in SHAPES, and a grid of
min(ceil(B / warps), SMs) CTAs.  The data-block checks that run after the device check are pinned here as well."""
import ctypes as C

import numpy as np
import pytest
import torch

from cppnumericalsolvers_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BATCHES = (1, 37, 4096)
F64, F32 = _lib.F64, _lib.F32
RB, DQ, HN, LG, DENSE = range(5)  # families
DMMA, WARP, SSE2, LU = _lib.POLICY_DMMA_TREE, _lib.POLICY_WARP_TREE, _lib.POLICY_EIGEN_SSE2, _lib.POLICY_DMMA_LU

# (solver, family, dtype, d, lbfgs_m, policy, mode) of every cno_minimize entry
MINIMIZE = [
    *[(0, RB, F64, d, 0, DMMA, 0) for d in (2, 3, 8, 32, 37, 64, 128)],
    (0, RB, F64, 128, 0, SSE2, 0),
    *[(0, RB, F64, d, 0, DMMA, 2) for d in (2, 37, 128)],
    *[(0, RB, F64, d, m, DMMA, 0) for m in (5, 20) for d in (8, 37, 128)],
    (0, RB, F32, 37, 5, WARP, 0),
    *[(0, RB, F32, d, 0, WARP, 0) for d in (2, 37, 128)],
    (0, DQ, F64, 2, 0, DMMA, 0), (0, HN, F64, 2, 0, DMMA, 0), (0, HN, F64, 50, 0, DMMA, 0),
    (0, LG, F32, 64, 0, WARP, 0),
    *[(0, DENSE, F64, d, 0, DMMA, 0) for d in (2, 8, 64)],
    *[(1, RB, F64, d, 0, DMMA, 0) for d in (2, 8, 32, 37, 64, 128)],
    (1, RB, F32, 32, 0, WARP, 0), (1, RB, F32, 128, 0, WARP, 0), (1, DQ, F64, 2, 0, DMMA, 0), (1, HN, F64, 2, 0, DMMA, 0),
    (2, DENSE, F64, 64, 0, DMMA, 0), (2, DENSE, F64, 64, 0, LU, 0), (2, DENSE, F64, 12, 0, DMMA, 0),
    (2, DENSE, F32, 64, 0, WARP, 0), (2, RB, F64, 2, 0, DMMA, 0), (2, RB, F64, 8, 0, DMMA, 0),
    *[(s, RB, F64, d, 0, DMMA, 0) for s in (3, 4) for d in (2, 8, 37, 128)],
    (3, RB, F32, 37, 0, WARP, 0), (3, DQ, F64, 2, 0, DMMA, 0), (4, DQ, F64, 2, 0, DMMA, 0),
    *[(5, RB, F64, d, 0, DMMA, 0) for d in (2, 37, 128)], (5, RB, F32, 37, 0, WARP, 0),
    *[(6, RB, F64, d, 0, DMMA, 0) for d in (8, 32, 64)],
    *[(7, RB, F64, d, 0, DMMA, 0) for d in (8, 37)],
]
# (family, dtype, d) of every cno_minimize_steps entry (Lbfgs)
STEPS = [*[(RB, F64, d) for d in (2, 3, 8, 32, 37, 64, 128)], *[(RB, F32, d) for d in (2, 37, 128)],
         (DQ, F64, 2), (HN, F64, 2), (HN, F64, 50)]
# (family, dtype, d, lbfgs_m) of every cno_lbfgsb_minimize entry
LBFGSB = [*[(RB, F64, d, 10) for d in (8, 37, 128)], *[(RB, F64, d, 5) for d in (2, 8, 37, 64, 128)], (RB, F32, 37, 5),
          (DQ, F64, 2, 5), (HN, F64, 2, 5), (HN, F64, 8, 5), (DENSE, F64, 8, 5), (DENSE, F64, 64, 5)]
# (expr, solver, dtype, d, mode) of user functors (tests/cpp/user_functions.cu): one per solver, and both BFGS kernels
EXPR_BOWL, EXPR_SECOND_SUM = 0, 6
USER = [(EXPR_BOWL, s, F64, 16, 1) for s in (0, 1, 3, 4, 5, 6, 7)] + [
    (EXPR_BOWL, 1, F64, 64, 1), (EXPR_SECOND_SUM, 2, F64, 8, 2), (EXPR_SECOND_SUM, 0, F64, 8, 2)]
# (family, dtype, d) of every cno_condition_hessian entry
CONDITION = [(DENSE, F64, 64), (DENSE, F64, 12), (DENSE, F32, 64), (RB, F64, 2), (RB, F64, 8)]

# (kernel_launches, block, warps_per_cta, dynamic_smem) per case id
SHAPES = {
    'minimize-0-0-0-2-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-0-0-3-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-0-0-8-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-0-0-32-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-0-0-37-m0-p2-mode0': (1, 512, 16, 167424),
    'minimize-0-0-0-64-m0-p2-mode0': (1, 512, 16, 167424),
    'minimize-0-0-0-128-m0-p2-mode0': (1, 384, 12, 223872),
    'minimize-0-0-0-128-m0-p1-mode0': (1, 384, 12, 211200),
    'minimize-0-0-0-2-m0-p2-mode2': (1, 512, 16, 85504),
    'minimize-0-0-0-37-m0-p2-mode2': (1, 512, 16, 167424),
    'minimize-0-0-0-128-m0-p2-mode2': (1, 352, 11, 227744),
    'minimize-0-0-0-8-m5-p2-mode0': (1, 512, 16, 43520),
    'minimize-0-0-0-37-m5-p2-mode0': (1, 512, 16, 84480),
    'minimize-0-0-0-128-m5-p2-mode0': (1, 640, 20, 208000),
    'minimize-0-0-0-8-m20-p2-mode0': (1, 512, 16, 169984),
    'minimize-0-0-0-37-m20-p2-mode0': (1, 384, 12, 225408),
    'minimize-0-0-0-128-m20-p2-mode0': (1, 192, 6, 223296),
    'minimize-0-0-1-37-m5-p0-mode0': (1, 512, 16, 42240),
    'minimize-0-0-1-2-m0-p0-mode0': (1, 512, 16, 42752),
    'minimize-0-0-1-37-m0-p0-mode0': (1, 512, 16, 83712),
    'minimize-0-0-1-128-m0-p0-mode0': (1, 512, 16, 165632),
    'minimize-0-1-0-2-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-2-0-2-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-2-0-50-m0-p2-mode0': (1, 512, 16, 167424),
    'minimize-0-3-1-64-m0-p0-mode0': (1, 192, 3, 229296),
    'minimize-0-4-0-2-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-4-0-8-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-0-4-0-64-m0-p2-mode0': (1, 512, 16, 167424),
    'minimize-1-0-0-2-m0-p2-mode0': (1, 384, 12, 6912),
    'minimize-1-0-0-8-m0-p2-mode0': (1, 384, 12, 6912),
    'minimize-1-0-0-32-m0-p2-mode0': (1, 320, 10, 5760),
    'minimize-1-0-0-37-m0-p2-mode0': (1, 256, 8, 160256),
    'minimize-1-0-0-64-m0-p2-mode0': (1, 192, 6, 203136),
    'minimize-1-0-0-128-m0-p2-mode0': (1, 32, 1, 133184),
    'minimize-1-0-1-32-m0-p0-mode0': (1, 384, 12, 3456),
    'minimize-1-0-1-128-m0-p0-mode0': (1, 96, 3, 199776),
    'minimize-1-1-0-2-m0-p2-mode0': (1, 384, 12, 6912),
    'minimize-1-2-0-2-m0-p2-mode0': (1, 384, 12, 6912),
    'minimize-2-4-0-64-m0-p2-mode0': (1, 192, 6, 203328),
    'minimize-2-4-0-64-m0-p3-mode0': (1, 192, 6, 204672),
    'minimize-2-4-0-12-m0-p2-mode0': (1, 256, 8, 11520),
    'minimize-2-4-1-64-m0-p0-mode0': (1, 256, 8, 135552),
    'minimize-2-0-0-2-m0-p2-mode0': (1, 256, 8, 1280),
    'minimize-2-0-0-8-m0-p2-mode0': (1, 256, 8, 5888),
    'minimize-3-0-0-2-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-3-0-0-8-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-3-0-0-37-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-3-0-0-128-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-4-0-0-2-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-4-0-0-8-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-4-0-0-37-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-4-0-0-128-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-3-0-1-37-m0-p0-mode0': (1, 512, 16, 512),
    'minimize-3-1-0-2-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-4-1-0-2-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-5-0-0-2-m0-p2-mode0': (1, 512, 16, 85504),
    'minimize-5-0-0-37-m0-p2-mode0': (1, 512, 16, 167424),
    'minimize-5-0-0-128-m0-p2-mode0': (1, 352, 11, 227744),
    'minimize-5-0-1-37-m0-p0-mode0': (1, 512, 16, 83712),
    'minimize-6-0-0-8-m0-p2-mode0': (1, 384, 12, 6912),
    'minimize-6-0-0-32-m0-p2-mode0': (1, 320, 10, 5760),
    'minimize-6-0-0-64-m0-p2-mode0': (1, 192, 6, 203136),
    'minimize-7-0-0-8-m0-p2-mode0': (1, 512, 16, 1024),
    'minimize-7-0-0-37-m0-p2-mode0': (1, 512, 16, 1024),
    'steps-0-0-2': (1, 512, 16, 85504),
    'steps-0-0-3': (1, 512, 16, 85504),
    'steps-0-0-8': (1, 512, 16, 85504),
    'steps-0-0-32': (1, 512, 16, 85504),
    'steps-0-0-37': (1, 512, 16, 167424),
    'steps-0-0-64': (1, 512, 16, 167424),
    'steps-0-0-128': (1, 352, 11, 227744),
    'steps-0-1-2': (1, 512, 16, 42752),
    'steps-0-1-37': (1, 512, 16, 83712),
    'steps-0-1-128': (1, 512, 16, 165632),
    'steps-1-0-2': (1, 512, 16, 85504),
    'steps-2-0-2': (1, 512, 16, 85504),
    'steps-2-0-50': (1, 512, 16, 167424),
    'lbfgsb-0-0-8-m10': (1, 384, 12, 163200),
    'lbfgsb-0-0-37-m10': (1, 384, 12, 227712),
    'lbfgsb-0-0-128-m10': (1, 224, 7, 208096),
    'lbfgsb-0-0-2-m5': (1, 384, 12, 59520),
    'lbfgsb-0-0-8-m5': (1, 384, 12, 59520),
    'lbfgsb-0-0-37-m5': (1, 384, 12, 93312),
    'lbfgsb-0-0-64-m5': (1, 384, 12, 93312),
    'lbfgsb-0-0-128-m5': (1, 384, 12, 160896),
    'lbfgsb-0-1-37-m5': (1, 384, 12, 47232),
    'lbfgsb-1-0-2-m5': (1, 384, 12, 59520),
    'lbfgsb-2-0-2-m5': (1, 384, 12, 59520),
    'lbfgsb-2-0-8-m5': (1, 384, 12, 59520),
    'lbfgsb-4-0-8-m5': (1, 384, 12, 59520),
    'lbfgsb-4-0-64-m5': (1, 384, 12, 93312),
    'user-0-0-0-16-mode1': (1, 512, 16, 85504),
    'user-0-1-0-16-mode1': (1, 384, 12, 6912),
    'user-0-3-0-16-mode1': (1, 512, 16, 1024),
    'user-0-4-0-16-mode1': (1, 512, 16, 1024),
    'user-0-5-0-16-mode1': (1, 512, 16, 85504),
    'user-0-6-0-16-mode1': (1, 384, 12, 6912),
    'user-0-7-0-16-mode1': (1, 512, 16, 1024),
    'user-0-1-0-64-mode1': (1, 192, 6, 203136),
    'user-6-2-0-8-mode2': (1, 256, 8, 5888),
    'user-6-0-0-8-mode2': (1, 512, 16, 85504),
}


def min_id(c):
    return "minimize-%d-%d-%d-%d-m%d-p%d-mode%d" % c


def steps_id(c):
    return "steps-%d-%d-%d" % c


def lbfgsb_id(c):
    return "lbfgsb-%d-%d-%d-m%d" % c


def user_id(c):
    return "user-%d-%d-%d-%d-mode%d" % c


def tdt(dtype):
    return torch.float64 if dtype == F64 else torch.float32


def data_block(family, dtype, d, B, n=256):
    """[A | b] with A = 2 I (column-major), b = 1; logistic: [X^T | y] with y = +-1."""
    g = torch.Generator().manual_seed(7)
    if family == DENSE:
        blk = torch.zeros(B, d * d + d, dtype=tdt(dtype))
        blk[:, : d * d : d + 1] = 2.0
        blk[:, d * d:] = 1.0
    else:
        blk = torch.cat([torch.rand(B, d * n, generator=g, dtype=tdt(dtype)) - 0.5,
                         torch.sign(torch.rand(B, n, generator=g, dtype=tdt(dtype)) - 0.5)], 1)
    return blk.to(DEV)


def problem(family, dtype, d, m=0, policy=None, mode=0, data=None):
    if policy is None:
        policy = DMMA if dtype == F64 else WARP
    p = _lib.Problem(family=family, dtype=dtype, d=d, n=256, param=0.01, policy=policy, mode=mode, lbfgs_m=m)
    if data is not None:
        p.data, p.data_stride = data.data_ptr(), data.shape[1]
    return p


def stop(iterations=3):
    s = _lib.Stop()
    _lib.lib().cno_default_stop(C.byref(s))
    s.num_iterations = iterations
    return s


def x0_and_out(B, d, dtype):
    g = torch.Generator().manual_seed(B * 1000 + d)
    x0 = (torch.rand(B, d, generator=g, dtype=tdt(dtype)) * 2 - 1).to(DEV)
    t = dict(x=torch.empty_like(x0), value=torch.empty(B, dtype=x0.dtype, device=DEV), gradient=torch.empty_like(x0),
             num_iterations=torch.zeros(B, dtype=torch.int32, device=DEV),
             status=torch.zeros(B, dtype=torch.int8, device=DEV), nfev=torch.zeros(B, dtype=torch.int32, device=DEV),
             x_delta=torch.empty(B, dtype=x0.dtype, device=DEV), f_delta=torch.empty(B, dtype=x0.dtype, device=DEV),
             gradient_norm=torch.empty(B, dtype=x0.dtype, device=DEV))
    keys = ("x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta", "gradient_norm")
    return x0, t, _lib.BatchOut(*[t[k].data_ptr() for k in keys])


def run_minimize(c, B):
    solver, family, dtype, d, m, policy, mode = c
    data = data_block(family, dtype, d, B) if family in (LG, DENSE) else None
    p = problem(family, dtype, d, m, policy, mode, data)
    x0, t, out = x0_and_out(B, d, dtype)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    info = _lib.LaunchInfo()
    st = stop()
    rc = _lib.lib().cno_minimize(solver, C.byref(p), B, x0.data_ptr(), C.byref(st), C.byref(out), ws.data_ptr(), 256,
                                 None, C.byref(info))
    torch.cuda.synchronize()
    return rc, info


def run_steps(c, B):
    family, dtype, d = c
    p = problem(family, dtype, d)
    x0, t, out = x0_and_out(B, d, dtype)
    n = C.c_size_t(0)
    assert _lib.lib().cno_state_bytes(_lib.LBFGS, C.byref(p), B, C.byref(n)) == _lib.OK
    state = torch.zeros(n.value, dtype=torch.uint8, device=DEV)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    info = _lib.LaunchInfo()
    st = stop(0)
    rc = _lib.lib().cno_minimize_steps(_lib.LBFGS, C.byref(p), B, x0.data_ptr(), C.byref(st), C.byref(out),
                                       state.data_ptr(), n.value, 2, 1, ws.data_ptr(), 256, None, C.byref(info))
    torch.cuda.synchronize()
    return rc, info


def run_lbfgsb(c, B):
    family, dtype, d, m = c
    data = data_block(family, dtype, d, B) if family == DENSE else None
    p = problem(family, dtype, d, m, data=data)
    x0, t, out = x0_and_out(B, d, dtype)
    lo = torch.full((d,), -0.5, dtype=tdt(dtype), device=DEV)
    bounds = _lib.Bounds(lo.data_ptr(), None, 0)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    info = _lib.LaunchInfo()
    st = stop()
    rc = _lib.lib().cno_lbfgsb_minimize(C.byref(p), C.byref(bounds), B, x0.data_ptr(), C.byref(st), C.byref(out),
                                        ws.data_ptr(), 256, None, C.byref(info))
    torch.cuda.synchronize()
    return rc, info


def run_user(c, B):
    import usertest_binding as ub
    expr, solver, dtype, d, mode = c
    x0 = np.random.default_rng(B).uniform(-1, 1, (B, d))
    r = ub.minimize(expr, solver, x0, param=0.25, mode=mode, stop=stop(), dev=DEV)
    return _lib.OK, r["launch"]


RUNS = [(min_id(c), run_minimize, c) for c in MINIMIZE] + [(steps_id(c), run_steps, c) for c in STEPS] + \
       [(lbfgsb_id(c), run_lbfgsb, c) for c in LBFGSB] + [(user_id(c), run_user, c) for c in USER]


@pytest.mark.parametrize("case_id,run,case", RUNS, ids=[r[0] for r in RUNS])
def test_launch_shape(case_id, run, case):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for B in BATCHES:
        rc, info = run(case, B)
        assert rc == _lib.OK, (case_id, B, rc)
        assert (info.kernel_launches, info.block, info.warps_per_cta, info.dynamic_smem) == SHAPES[case_id], B
        assert info.grid == min(-(-B // info.warps_per_cta), sms), B


@pytest.mark.parametrize("case", CONDITION, ids=["condition-%d-%d-%d" % c for c in CONDITION])
def test_condition_hessian_runs(case):
    family, dtype, d = case
    for B in BATCHES:
        data = data_block(family, dtype, d, B) if family == DENSE else None
        p = problem(family, dtype, d, data=data)
        x = (torch.rand(B, d, dtype=tdt(dtype)) * 0.5).to(DEV)
        cond = torch.full((B,), -1.0, dtype=tdt(dtype), device=DEV)
        ws = torch.zeros(8, dtype=torch.uint8, device=DEV)
        rc = _lib.lib().cno_condition_hessian(C.byref(p), B, x.data_ptr(), cond.data_ptr(), ws.data_ptr(), 8, None)
        torch.cuda.synchronize()
        assert rc == _lib.OK
        assert bool(torch.isfinite(cond).all()) and bool((cond >= 1).all())


def test_user_condition_hessian_runs():
    import usertest_binding as ub
    for B in BATCHES:
        c = ub.condition_hessian(EXPR_SECOND_SUM, np.random.default_rng(B).uniform(-1, 1, (B, 8)))
        assert np.isfinite(c).all() and (c >= 1).all()


# ---- data-block checks that run after the device check: rejected before any launch --------------------------------
def _minimize_with_data(solver, family, dtype, d, policy, data, stride):
    p = problem(family, dtype, d, policy=policy)
    p.data, p.data_stride = data, stride
    x0, t, out = x0_and_out(4, d, dtype)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    return _lib.lib().cno_minimize(solver, C.byref(p), 4, x0.data_ptr(), None, C.byref(out), ws.data_ptr(), 256, None,
                                   None)


# (solver, family, dtype, d, policy, block elements, TMA-read)
DATA_ENTRIES = [(2, DENSE, F64, 64, DMMA, 64 * 65, True), (2, DENSE, F64, 64, LU, 64 * 65, True),
                (2, DENSE, F64, 12, DMMA, 12 * 13, True), (2, DENSE, F32, 64, WARP, 64 * 65, True),
                (0, LG, F32, 64, WARP, 64 * 256 + 256, True), (0, DENSE, F64, 8, DMMA, 72, False)]


@pytest.mark.parametrize("entry", DATA_ENTRIES, ids=["data-%d-%d-%d-%d-p%d" % e[:5] for e in DATA_ENTRIES])
def test_data_block_checks(entry):
    solver, family, dtype, d, policy, elems, tma = entry
    esz = 8 if dtype == F64 else 4
    buf = torch.zeros(4 * (elems + 8) + 16, dtype=tdt(dtype), device=DEV)
    base = buf.data_ptr()
    assert _minimize_with_data(solver, family, dtype, d, policy, None, elems) == _lib.ERR_INVALID_ARGUMENT
    assert _minimize_with_data(solver, family, dtype, d, policy, base, elems - 1) == _lib.ERR_INVALID_ARGUMENT
    if tma:
        assert _minimize_with_data(solver, family, dtype, d, policy, base + esz, elems) == _lib.ERR_INVALID_ARGUMENT
        odd = elems + (16 // esz) - 1 if (elems * esz) % 16 == 0 else elems
        assert (odd * esz) % 16 != 0
        assert _minimize_with_data(solver, family, dtype, d, policy, base, odd) == _lib.ERR_INVALID_ARGUMENT


def test_logistic_sample_count_is_checked():
    buf = torch.zeros(4 * (64 * 256 + 256), dtype=torch.float32, device=DEV)
    p = problem(LG, F32, 64)
    p.n, p.data, p.data_stride = 128, buf.data_ptr(), 64 * 256 + 256
    x0, t, out = x0_and_out(4, 64, F32)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    assert _lib.lib().cno_minimize(0, C.byref(p), 4, x0.data_ptr(), None, C.byref(out), ws.data_ptr(), 256, None,
                                   None) == _lib.ERR_INVALID_ARGUMENT


def test_lbfgsb_and_condition_data_block_checks():
    L = _lib.lib()
    x0, t, out = x0_and_out(4, 8, F64)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    for data, stride in ((None, 72), (x0.data_ptr(), 71)):
        p = problem(DENSE, F64, 8)
        p.data, p.data_stride = data, stride
        assert L.cno_lbfgsb_minimize(C.byref(p), None, 4, x0.data_ptr(), None, C.byref(out), ws.data_ptr(), 256, None,
                                     None) == _lib.ERR_INVALID_ARGUMENT
    buf = torch.zeros(4 * 64 * 65 + 16, dtype=torch.float64, device=DEV)
    x = torch.zeros(4, 64, dtype=torch.float64, device=DEV)
    cond = torch.zeros(4, dtype=torch.float64, device=DEV)
    for data, stride in ((None, 64 * 65), (buf.data_ptr(), 64 * 65 - 1), (buf.data_ptr() + 8, 64 * 65),
                         (buf.data_ptr(), 64 * 65 + 1)):
        p = problem(DENSE, F64, 64)
        p.data, p.data_stride = data, stride
        assert L.cno_condition_hessian(C.byref(p), 4, x.data_ptr(), cond.data_ptr(), ws.data_ptr(), 8,
                                       None) == _lib.ERR_INVALID_ARGUMENT
