"""cno_evaluate on the GPU (-m gpu): every compiled key against the oracle and against exact sums, the FP64 tensor-core
sum at the edges of the floating-point range, fp32 subnormals, and the FunctionState invariant of every solver.

(a) Every key of kEvalTable (csrc/cno_api.cu) at B = 1, 7 and 3 * SMs * 64 + 5 (three passes of evaluate_kernel's
    grid-stride loop), in each output mode (value and gradient, value only, gradient only): bit for bit the oracle,
    unrequested outputs and the rows past B untouched, and the first 16 instances within the exact-sum bound of
    tests/edge_sums.py (which also catches a term the kernel and the oracle drop or double alike).
(b) fp64 edge vectors of the cross-lane sum (subnormal partials, overflow in each stage of the two MMAs, +-Inf, a NaN
    in each lane, -0.0) through three probes with direct control over the 32 lane partials: GPU == numpy model of
    the specification == oracle, bit for bit (NaN: NaN-ness only), and within the exact bound where the model's
    chain is finite.  tests/test_device_emulated.py runs the same vectors through the device source on the CPU.
(c) fp32 Rosenbrock at d = 32, 37, 128 with a subnormal gradient component (a flush-to-zero build returns 0), an
    overflowing value and NaN starts.  The fp32 butterfly itself is never fed subnormal lane partials: the only fp32
    key is Rosenbrock, whose terms (1 - x_i)^2 + 100 t_i^2 are 0 or at least 2^-48 (1 - x_i is 0 or at least 2^-24
    in magnitude, and x_i = 1 makes t_i = x_{i+1} - 1 the same), so that path is out of scope.
(d) The FunctionState invariant: the value and gradient every solver returns are F at the returned x, bit for bit
    equal to cno_evaluate(x), for every solver entry whose (family, dtype, d) has an evaluate key."""
import ctypes as C
import itertools

import edge_sums as es
import numpy as np
import pytest
import torch
from test_dispatch_contract import DS, LBFGSB_SUPPORTED, STATE_STRIDE, SUPPORTED, expand

from cppnumericalsolvers_b200 import _lib
from oracle import oracle_binding as ob

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64, F32 = _lib.F64, _lib.F32
RB, DQ, HN, DENSE = _lib.FN_ROSENBROCK, _lib.FN_DIAG_QUADRATIC, _lib.FN_HALF_SQUARED_NORM, _lib.FN_DENSE_QUADRATIC
NP = {F64: np.float64, F32: np.float32}
TDT = {np.float64: torch.float64, np.float32: torch.float32}
SENTINEL = -1234.5

# (family, dtype, d) of every cno_evaluate key
EVAL_KEYS = {*[(RB, F64, d) for d in (2, 3, 8, 32, 37, 64, 128)], *[(RB, F32, d) for d in (2, 32, 37, 128)],
             (DQ, F64, 2), (HN, F64, 2), (HN, F64, 8), (HN, F64, 50), (DENSE, F64, 2), (DENSE, F64, 8), (DENSE, F64, 64)}
MODES = ((True, True), (True, False), (False, True))  # (value, gradient) requested


def _problem(family, dtype, d, data=None, policy=None):
    p = _lib.Problem(family=family, dtype=dtype, d=d,
                     policy=policy if policy is not None else (_lib.POLICY_DMMA_TREE if dtype == F64 else _lib.POLICY_WARP_TREE))
    if data is not None:
        p.data, p.data_stride = data.data_ptr(), data.shape[1]
    return p


def gpu_evaluate(family, x, data=None, value=True, gradient=True, guard=3):
    """cno_evaluate on device copies of x (and the data block); outputs pre-filled with a sentinel, `guard` rows past B.
    Checks that the unrequested output and the guard rows still hold the sentinel."""
    B, d = x.shape
    tdt = TDT[x.dtype.type]
    xt = torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    dt = torch.from_numpy(np.ascontiguousarray(data)).to(DEV) if data is not None else None
    f = torch.full((B + guard,), SENTINEL, dtype=tdt, device=DEV)
    g = torch.full((B + guard, d), SENTINEL, dtype=tdt, device=DEV)
    p = _problem(family, F64 if x.dtype == np.float64 else F32, d, dt)
    rc = _lib.lib().cno_evaluate(C.byref(p), B, xt.data_ptr(), f.data_ptr() if value else None,
                                 g.data_ptr() if gradient else None, None)
    torch.cuda.synchronize()
    assert rc == _lib.OK
    f, g = f.cpu().numpy(), g.cpu().numpy()
    assert (f[B:] == SENTINEL).all() and (g[B:] == SENTINEL).all()
    assert value or (f == SENTINEL).all()
    assert gradient or (g == SENTINEL).all()
    return f[:B], g[:B]


def _spd_blocks(n, d, seed):
    """[A col-major | b] with A symmetric positive definite (tests/test_device_emulated.py: _spd_data)."""
    rng = np.random.default_rng(seed)
    M = rng.uniform(-1, 1, (n, d, d))
    A = np.einsum("bij,bkj->bik", M, M) / d + np.eye(d)
    A = (A + A.transpose(0, 2, 1)) / 2
    return np.concatenate([A.transpose(0, 2, 1).reshape(n, -1), rng.uniform(-1, 1, (n, d))], 1)


def dense_data(B, d, seed):
    """Even instances: SPD blocks (16 distinct, repeated); odd instances: a non-symmetric A, so that reading A in
    the wrong order (row- instead of column-major) changes the result."""
    data = np.random.default_rng(seed + 1).uniform(-1, 1, (B, d * d + d))
    data[0::2] = _spd_blocks(16, d, seed)[np.arange((B + 1) // 2) % 16]
    return data


# ---- (a) every key ------------------------------------------------------------------------------------------------------
def test_evaluate_key_set():
    """The keys cno_evaluate accepts (batch 0: no launch) over family x dtype x the d values of the dispatch sweep."""
    buf = torch.zeros(16, dtype=torch.float64, device=DEV)
    got = set()
    for family, dtype, d in itertools.product(range(5), (F64, F32), DS):
        p = _problem(family, dtype, d)
        p.data, p.data_stride = buf.data_ptr(), d * d + d  # passes the data-block check of the dense quadratic
        rc = _lib.lib().cno_evaluate(C.byref(p), 0, buf.data_ptr(), buf.data_ptr(), buf.data_ptr(), None)
        assert rc in (_lib.OK, _lib.ERR_UNSUPPORTED), (family, dtype, d, rc)
        if rc == _lib.OK:
            got.add((family, dtype, d))
    assert got == EVAL_KEYS and len(got) == 18


@pytest.mark.parametrize("key", sorted(EVAL_KEYS), ids=lambda k: "f%d-t%d-d%d" % k)
def test_evaluate_equals_oracle_and_exact_sums(key):
    family, dtype, d = key
    T = NP[dtype]
    big = 3 * torch.cuda.get_device_properties(0).multi_processor_count * 64 + 5
    for B in (1, 7, big):
        x = ob.fill_uniform((B, d), 0, 1000 * d + B, -2.0, 2.0, T)
        data = dense_data(B, d, d + B) if family == DENSE else None
        fo, go = ob.evaluate(family, x, data=data)
        for value, gradient in MODES:
            f, g = gpu_evaluate(family, x, data, value, gradient)
            if value:
                assert es.same_bits(f, fo), (B, value, gradient)
            if gradient:
                assert es.same_bits(g, go), (B, value, gradient)
            if value and gradient:
                fg = f, g
    n = 16
    es.check_exact(family, x[:n], None if data is None else data[:n], fg[0][:n], fg[1][:n], T)


# ---- (b), (c) edge vectors ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", es.probe_cases(), ids=lambda c: c[0])
def test_evaluate_edge_vectors_equal_model_and_oracle(case):
    name, family, x, data, names, (fm, gm) = case
    fo, go = ob.evaluate(family, x, data=data)
    f, g = gpu_evaluate(family, x, data)
    for i, vec in enumerate(names):
        assert es.same_bits(f[i], fm[i]), (vec, f[i], fm[i])
        assert es.same_bits(g[i], gm[i]), (vec, g[i], gm[i])
        assert es.same_bits(fo[i], fm[i]) and es.same_bits(go[i], gm[i]), vec
    ok = es.chain_finite(family, x, data)
    assert ok.any()
    es.check_exact(family, x[ok], None if data is None else data[ok], f[ok], g[ok], x.dtype.type)
    if name.startswith("rosenbrock"):
        k = names.index("subnormal_gradient")
        assert g[k, -1] == es.SUBNORMAL_G != 0 and abs(g[k, -1]) < np.finfo(np.float32).tiny
        k = names.index("huge")
        assert f[k] == np.inf and np.isfinite(g[k]).all()
    f1, _ = gpu_evaluate(family, x, data, gradient=False)
    _, g1 = gpu_evaluate(family, x, data, value=False)
    assert es.same_bits(f1, f) and es.same_bits(g1, g)


# ---- (d) the FunctionState invariant ------------------------------------------------------------------------------------
def _default(dtype):
    return _lib.POLICY_DMMA_TREE if dtype == F64 else _lib.POLICY_WARP_TREE


def _minimize_entries():
    """(solver, family, dtype, d, lbfgs_m, policy, mode) of every cno_minimize entry with an evaluate key: the
    default policy, and NewtonDescent's tensor-core LU (its sums use the same tree).  Mode 1 repeats mode 0; only
    Lbfgs reads lbfgs_m, where 0 repeats 10 (the default)."""
    keys = []
    lbfgs = (_lib.LBFGS, _lib.LBFGS_HAGER_ZHANG)
    for key in sorted(expand(SUPPORTED, 4)):
        solver, family, dtype, d, m, policy, mode = key
        if (family, dtype, d) not in EVAL_KEYS or mode == 1 or (m == 0) == (solver in lbfgs):
            continue
        if policy == _default(dtype) or (solver == _lib.NEWTON and policy == _lib.POLICY_DMMA_LU):
            keys.append(key)
    return keys


def _starts(B, d, T, seed):
    """Random starts in [-2, 2], the Rosenbrock minimiser, a far start and a NaN start."""
    x = ob.fill_uniform((B, d), 0, seed, -2.0, 2.0, T)
    x[1] = 1.0
    x[2] *= 1e6
    x[3, 0] = np.nan
    return x


class _Out:
    def __init__(self, B, d, T):
        tdt = TDT[T]
        self.t = dict(x=torch.zeros(B, d, dtype=tdt, device=DEV), value=torch.zeros(B, dtype=tdt, device=DEV),
                      gradient=torch.zeros(B, d, dtype=tdt, device=DEV),
                      num_iterations=torch.zeros(B, dtype=torch.int32, device=DEV),
                      status=torch.zeros(B, dtype=torch.int8, device=DEV),
                      nfev=torch.zeros(B, dtype=torch.int32, device=DEV),
                      x_delta=torch.zeros(B, dtype=tdt, device=DEV), f_delta=torch.zeros(B, dtype=tdt, device=DEV),
                      gradient_norm=torch.zeros(B, dtype=tdt, device=DEV))
        self.out = _lib.BatchOut(*[self.t[k].data_ptr() for k, _ in _lib.BatchOut._fields_])

    def np(self, k):
        return self.t[k].cpu().numpy()


def _stop(iterations):
    s = _lib.Stop()
    _lib.lib().cno_default_stop(C.byref(s))
    s.num_iterations = iterations
    return s


def _assert_state_is_f_at_x(family, o, data):
    x, value, gradient = o.np("x"), o.np("value"), o.np("gradient")
    f, g = gpu_evaluate(family, x, data)
    for i in range(x.shape[0]):
        assert es.same_bits(value[i], f[i]) and es.same_bits(gradient[i], g[i]), (i, int(o.np("status")[i]))


B_INV = 64


@pytest.mark.parametrize("key", _minimize_entries(), ids=lambda k: "s%d-f%d-t%d-d%d-m%d-p%d-mode%d" % k)
def test_minimize_returns_f_at_x(key):
    solver, family, dtype, d, m, policy, mode = key
    T = NP[dtype]
    x0 = _starts(B_INV, d, T, 31 + d + solver)
    data = _spd_blocks(B_INV, d, d) if family == DENSE else None
    dt = torch.from_numpy(data).to(DEV) if data is not None else None
    p = _problem(family, dtype, d, dt, policy)
    p.lbfgs_m, p.mode = m, mode
    o = _Out(B_INV, d, T)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    st = _stop(200)  # bounds the descent solvers on Rosenbrock
    x0t = torch.from_numpy(x0).to(DEV)
    rc = _lib.lib().cno_minimize(solver, C.byref(p), B_INV, x0t.data_ptr(), C.byref(st), C.byref(o.out),
                                 ws.data_ptr(), 256, None, None)
    torch.cuda.synchronize()
    assert rc == _lib.OK
    _assert_state_is_f_at_x(family, o, data)


LBFGSB_ENTRIES = sorted({(f, t, d, m or 5) for f, t, d, m, policy, mode in expand(LBFGSB_SUPPORTED, 3)
                         if (f, t, d) in EVAL_KEYS})


@pytest.mark.parametrize("key", LBFGSB_ENTRIES, ids=lambda k: "f%d-t%d-d%d-m%d" % k)
def test_lbfgsb_returns_f_at_x(key):
    family, dtype, d, m = key
    T = NP[dtype]
    x0 = _starts(B_INV, d, T, 77 + d)
    data = _spd_blocks(B_INV, d, d) if family == DENSE else None
    dt = torch.from_numpy(data).to(DEV) if data is not None else None
    p = _problem(family, dtype, d, dt)
    p.lbfgs_m = m
    lo = torch.full((d,), -0.5, dtype=TDT[T], device=DEV)
    hi = torch.full((d,), 1.5, dtype=TDT[T], device=DEV)
    bounds = _lib.Bounds(lo.data_ptr(), hi.data_ptr(), 0)
    o = _Out(B_INV, d, T)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    st = _stop(200)
    x0t = torch.from_numpy(x0).to(DEV)
    rc = _lib.lib().cno_lbfgsb_minimize(C.byref(p), C.byref(bounds), B_INV, x0t.data_ptr(), C.byref(st), C.byref(o.out),
                                        ws.data_ptr(), 256, None, None)
    torch.cuda.synchronize()
    assert rc == _lib.OK
    _assert_state_is_f_at_x(family, o, data)


STEP_ENTRIES = sorted((f, t, d) for s, f, t, d in STATE_STRIDE if (f, t, d) in EVAL_KEYS)


@pytest.mark.parametrize("key", STEP_ENTRIES, ids=lambda k: "f%d-t%d-d%d" % k)
def test_minimize_steps_returns_f_at_x_after_every_call(key):
    """cno_minimize_steps parks the solver state between calls; the value and gradient of every call's output are F at
    that call's x -- for instances still running and for finished ones."""
    family, dtype, d = key
    T = NP[dtype]
    x0 = _starts(B_INV, d, T, 55 + d)
    p = _problem(family, dtype, d)
    n = C.c_size_t(0)
    assert _lib.lib().cno_state_bytes(_lib.LBFGS, C.byref(p), B_INV, C.byref(n)) == _lib.OK
    state = torch.zeros(n.value, dtype=torch.uint8, device=DEV)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    o = _Out(B_INV, d, T)
    st = _stop(60)
    x0t = torch.from_numpy(x0).to(DEV)
    for call in range(40):
        rc = _lib.lib().cno_minimize_steps(_lib.LBFGS, C.byref(p), B_INV, x0t.data_ptr(), C.byref(st), C.byref(o.out),
                                           state.data_ptr(), n.value, 7, int(call == 0), ws.data_ptr(), 256, None, None)
        torch.cuda.synchronize()
        assert rc == _lib.OK
        _assert_state_is_f_at_x(family, o, None)
        if (o.np("status") != 0).all():
            break
    assert (o.np("status") != 0).all()
