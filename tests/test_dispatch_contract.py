"""The dispatch contract of libcno.so, pinned without a GPU: which (solver, family, dtype, d, lbfgs_m, policy, mode)
keys each entry point accepts, the scratch sizes it asks for, and the exact return code of every input rejected
before the device is touched, in the order the checks run.  Inputs that get as far as the device check give
CNO_ERR_NO_DEVICE on a machine without one and are not run on a machine with one (their pointers are fake)."""
import ctypes as C
import itertools

import pytest
import torch

from cppnumericalsolvers_b200 import _lib

OK, INV, UNS, NODEV, WS = _lib.OK, _lib.ERR_INVALID_ARGUMENT, _lib.ERR_UNSUPPORTED, _lib.ERR_NO_DEVICE, _lib.ERR_WORKSPACE
HAVE_GPU = torch.cuda.is_available()
DS = (1, 2, 3, 4, 8, 12, 32, 37, 50, 64, 128, 129)  # every d of the tables, plus 1, 4 and 129
MS = (0, 5, 10, 20)

# Accepted keys.  One row: solver family dtype policy | lbfgs_m values | modes | d values.
SUPPORTED = """
0 0 0 1 | 0 10 | 0 1 | 128
0 0 0 2 | 0 5 10 20 | 0 1 | 8 37 128
0 0 0 2 | 0 10 | 0 1 | 3 32 64
0 0 0 2 | 0 10 | 0 1 2 | 2
0 0 0 2 | 0 10 | 2 | 37 128
0 0 1 0 | 0 5 10 | 0 1 | 37
0 0 1 0 | 0 10 | 0 1 | 2 128
0 1 0 2 | 0 10 | 0 1 | 2
0 2 0 2 | 0 10 | 0 1 | 2 50
0 3 1 0 | 0 10 | 0 1 | 64
0 4 0 2 | 0 10 | 0 1 | 2 8 64
1 0 0 2 | 0 5 10 20 | 0 1 2 | 2 8 32 37 64 128
1 0 1 0 | 0 5 10 20 | 0 1 2 | 32 128
1 1 0 2 | 0 5 10 20 | 0 1 2 | 2
1 2 0 2 | 0 5 10 20 | 0 1 2 | 2
2 0 0 2 | 0 5 10 20 | 0 1 2 | 2 8
2 4 0 2 | 0 5 10 20 | 0 1 2 | 12 64
2 4 0 3 | 0 5 10 20 | 0 1 2 | 64
2 4 1 0 | 0 5 10 20 | 0 1 2 | 64
3 0 0 2 | 0 5 10 20 | 0 1 | 2 8 37 128
3 0 1 0 | 0 5 10 20 | 0 1 | 37
3 1 0 2 | 0 5 10 20 | 0 1 | 2
4 0 0 2 | 0 5 10 20 | 0 1 | 2 8 37 128
4 1 0 2 | 0 5 10 20 | 0 1 | 2
5 0 0 2 | 0 10 | 0 1 | 2 37 128
5 0 1 0 | 0 10 | 0 1 | 37
6 0 0 2 | 0 5 10 20 | 0 1 | 8 32 64
7 0 0 2 | 0 5 10 20 | 0 1 | 8 37
"""
# Lbfgsb and AugmentedLagrangian: family dtype policy | lbfgs_m values | modes | d values.
LBFGSB_SUPPORTED = """
0 0 2 | 0 5 | 0 1 2 | 2 64
0 0 2 | 0 5 10 | 0 1 2 | 8 37 128
0 1 0 | 0 5 | 0 1 2 | 37
1 0 2 | 0 5 | 0 1 2 | 2
2 0 2 | 0 5 | 0 1 2 | 2 8
4 0 2 | 0 5 | 0 1 2 | 8 64
"""
AL_SUPPORTED = """
0 0 2 | 0 5 10 20 | 0 1 | 2 8 37 128
0 1 0 | 0 5 10 20 | 0 1 | 8
2 0 2 | 0 5 10 20 | 0 1 | 2 8
4 0 2 | 0 5 10 20 | 0 1 | 2 8
"""
# bytes of one parked instance (cno_state_bytes / batch) of every stepwise entry: (solver, family, dtype, d)
STATE_STRIDE = {
    (0, 0, 0, 2): 5328, (0, 0, 0, 3): 5328, (0, 0, 0, 8): 5328, (0, 0, 0, 32): 5328, (0, 0, 0, 37): 10448,
    (0, 0, 0, 64): 10448, (0, 0, 0, 128): 20688, (0, 0, 1, 2): 2688, (0, 0, 1, 37): 5248, (0, 0, 1, 128): 10368,
    (0, 1, 0, 2): 5328, (0, 2, 0, 2): 5328, (0, 2, 0, 50): 10448,
}
# cno_al_workspace_bytes at B = 1, 1000, 4096: (family, dtype, d, n_eq, n_ineq)
AL_WORKSPACE = {
    (0, 0, 8, 0, 0): (3328, 175104, 709632), (0, 0, 8, 1, 1): (3328, 190976, 774656),
    (0, 0, 8, 3, 0): (3328, 198912, 807680), (0, 0, 8, 32, 32): (3328, 686592, 2806272),
    (0, 1, 8, 0, 0): (3328, 90624, 365568), (0, 1, 8, 1, 1): (3328, 98304, 397824),
    (0, 1, 8, 3, 0): (3328, 102400, 414464), (0, 1, 8, 32, 32): (3328, 346112, 1413632),
    (4, 0, 2, 0, 0): (3328, 79360, 316416), (4, 0, 2, 1, 1): (3328, 95232, 381440),
    (4, 0, 2, 3, 0): (3328, 103168, 414464), (4, 0, 2, 32, 32): (3328, 590848, 2413056),
    (0, 0, 128, 0, 0): (4864, 2095104, 8573952), (0, 0, 128, 1, 1): (4864, 2110976, 8638976),
    (0, 0, 128, 3, 0): (4864, 2118912, 8672000), (0, 0, 128, 32, 32): (4864, 2606592, 10670592),
}


def expand(table, lead):
    keys = set()
    for row in table.strip().splitlines():
        head, ms, modes, ds = (list(map(int, f.split())) for f in row.split("|"))
        assert len(head) == lead
        for m, mode, d in itertools.product(ms, modes, ds):
            keys.add((*head[:-1], d, m, head[-1], mode))  # (..., d, lbfgs_m, policy, mode)
    return keys


def problem(family=0, dtype=0, d=8, m=0, policy=None, mode=0, n=256, data=None, stride=0):
    if policy is None:
        policy = _lib.POLICY_DMMA_TREE if dtype == _lib.F64 else _lib.POLICY_WARP_TREE
    return _lib.Problem(family=family, dtype=dtype, d=d, n=n, policy=policy, mode=mode, lbfgs_m=m, data=data,
                        data_stride=stride)


def sweep():
    for family, dtype, d, m, policy, mode in itertools.product(range(5), range(2), DS, MS, range(4), range(3)):
        yield (family, dtype, d, m, policy, mode), problem(family, dtype, d, m, policy, mode)


def test_supported_keys():
    L = _lib.lib()
    got = set()
    for (family, dtype, d, m, policy, mode), p in sweep():
        for solver in range(8):
            rc = L.cno_supported(solver, C.byref(p))
            assert rc in (OK, UNS)
            if rc == OK:
                got.add((solver, family, dtype, d, m, policy, mode))
    assert got == expand(SUPPORTED, 4)


def test_lbfgsb_and_al_supported_keys():
    L = _lib.lib()
    none = _lib.Constraints(0, 0, None, None, 0)
    lb, al = set(), set()
    for key, p in sweep():
        rc = L.cno_lbfgsb_supported(C.byref(p))
        assert rc in (OK, UNS)
        if rc == OK:
            lb.add(key)
        rc = L.cno_al_supported(C.byref(p), C.byref(none))
        assert rc in (OK, UNS)
        if rc == OK:
            al.add(key)
    assert lb == expand(LBFGSB_SUPPORTED, 3)
    assert al == expand(AL_SUPPORTED, 3)


def test_state_and_workspace_bytes():
    L = _lib.lib()
    stride = {}
    for key in expand(SUPPORTED, 4):
        solver, family, dtype, d, m, policy, mode = key
        p = problem(family, dtype, d, m, policy, mode)
        n = C.c_size_t(0)
        assert L.cno_workspace_bytes(solver, C.byref(p), 1000, C.byref(n)) == OK and n.value == 256
        assert L.cno_workspace_bytes(solver, C.byref(p), 1000, None) == INV
        rc = L.cno_state_bytes(solver, C.byref(p), 3, C.byref(n))
        if rc == OK:
            stride.setdefault((solver, family, dtype, d), set()).add(n.value // 3)
            assert n.value % 3 == 0
            assert L.cno_state_bytes(solver, C.byref(p), -1, C.byref(n)) == INV
            assert L.cno_state_bytes(solver, C.byref(p), 3, None) == INV
        else:
            assert rc == UNS
    assert stride == {k: {v} for k, v in STATE_STRIDE.items()}
    bad = problem(d=129)
    assert L.cno_state_bytes(_lib.LBFGS, C.byref(bad), 3, C.byref(n)) == UNS
    assert L.cno_workspace_bytes(_lib.LBFGS, C.byref(bad), 3, C.byref(n)) == UNS


def test_al_workspace_bytes():
    L = _lib.lib()
    rows = (C.c_int32 * 64)()
    for (family, dtype, d, ne, ni), sizes in AL_WORKSPACE.items():
        k = _lib.Constraints(ne, ni, C.addressof(rows), C.addressof(rows), 0)
        p = problem(family, dtype, d)
        got = []
        for B in (1, 1000, 4096):
            n = C.c_size_t(0)
            assert L.cno_al_workspace_bytes(C.byref(p), C.byref(k), B, C.byref(n)) == OK
            got.append(n.value)
        assert tuple(got) == sizes
        assert L.cno_al_workspace_bytes(C.byref(p), C.byref(k), -1, C.byref(n)) == INV
        assert L.cno_al_workspace_bytes(C.byref(p), C.byref(k), 4, None) == INV


# ---- return codes of rejected inputs --------------------------------------------------------------------------------
# Fake device addresses: never dereferenced before the device check.
A16, A8, A1 = 0x100000, 0x100008, 0x100001
DEV = "device"  # reaches the device check


def stop(past=3):
    s = _lib.Stop()
    _lib.lib().cno_default_stop(C.byref(s))
    s.past = past
    return s


def out(x=A16, gradient=A16, value=A16, status=A16, iters=A16):
    return _lib.BatchOut(x, value, gradient, iters, status, A16, A16, A16, A16)


def minimize(p=None, batch=4, x0=A16, st=None, o=..., ws=A16, wsb=256, solver=_lib.LBFGS):
    p = problem() if p is None else p
    o = out() if o is ... else o
    return _lib.lib().cno_minimize(solver, C.byref(p) if p else None, batch, x0, C.byref(st) if st else None,
                                   C.byref(o) if o else None, ws, wsb, None, None)


def steps(p=None, batch=4, x0=A16, st=None, o=..., state=A16, state_bytes=1 << 20, it=5, first=1, ws=A16, wsb=256):
    p = problem() if p is None else p
    o = out() if o is ... else o
    return _lib.lib().cno_minimize_steps(_lib.LBFGS, C.byref(p), batch, x0, C.byref(st) if st else None,
                                         C.byref(o) if o else None, state, state_bytes, it, first, ws, wsb, None, None)


def lbfgsb(p=None, bounds=None, batch=4, x0=A16, st=None, o=..., ws=A16, wsb=256):
    p = problem() if p is None else p
    o = out() if o is ... else o
    return _lib.lib().cno_lbfgsb_minimize(C.byref(p) if p else None, C.byref(bounds) if bounds else None, batch, x0,
                                          C.byref(st) if st else None, C.byref(o) if o else None, ws, wsb, None, None)


def host(p=None, batch=4, x0=A16, o=...):
    p = problem() if p is None else p
    o = out() if o is ... else o
    return _lib.lib().cno_minimize_host(_lib.LBFGS, C.byref(p), batch, x0, None, C.byref(o) if o else None, None)


def evaluate(p=None, batch=4, x=A16, value=A16, gradient=A16):
    p = problem() if p is None else p
    return _lib.lib().cno_evaluate(C.byref(p) if p else None, batch, x, value, gradient, None)


def condition(p=None, batch=4, x=A16, cond=A16, ws=A16, wsb=8):
    p = problem(family=_lib.FN_ROSENBROCK, d=8) if p is None else p
    return _lib.lib().cno_condition_hessian(C.byref(p) if p else None, batch, x, cond, ws, wsb, None)


def al(p=None, k=..., batch=4, x0=A16, st=None, o=..., ws=A16, wsb=1 << 24, mult=A16):
    L = _lib.lib()
    p = problem() if p is None else p
    if k is ...:
        k = _lib.Constraints(1, 1, A16, A16, 0)
    if o is ...:
        o = _lib.AlOut(*([A16] * 12))
        o.equality_multipliers = o.inequality_multipliers = mult
    return L.cno_al_minimize(C.byref(p) if p else None, C.byref(k) if k else None, batch, x0, None, None, None,
                             C.byref(st) if st else None, None, None, C.byref(o) if o else None, ws, wsb, None, None)


def cases():
    nul = _lib.BatchOut()
    return [
        # cno_minimize: problem, batch / out, batch == 0, x0, workspace, I/O alignment, past, device
        ("min null problem", lambda: minimize(p=False), INV),
        ("min bad solver", lambda: minimize(solver=8), INV),
        ("min bad dtype", lambda: minimize(p=problem(dtype=2)), INV),
        ("min d <= 0", lambda: minimize(p=problem(d=0)), INV),
        ("min unsupported", lambda: minimize(p=problem(d=129)), UNS),
        ("min batch < 0", lambda: minimize(batch=-1), INV),
        ("min null out", lambda: minimize(o=None), INV),
        ("min batch 0", lambda: minimize(batch=0, x0=None, ws=None), (DEV, OK)),
        ("min null x0", lambda: minimize(x0=None, ws=None), INV),
        ("min null workspace", lambda: minimize(ws=None, x0=A8), WS),
        ("min short workspace", lambda: minimize(wsb=255, x0=A8), WS),
        ("min misaligned workspace", lambda: minimize(ws=A16 + 4, x0=A8), WS),
        ("min misaligned x0", lambda: minimize(x0=A8, st=stop(-1)), INV),
        ("min misaligned out.x", lambda: minimize(o=out(x=A8)), INV),
        ("min misaligned out.gradient", lambda: minimize(o=out(gradient=A1)), INV),
        ("min past -1", lambda: minimize(st=stop(-1)), INV),
        ("min past max+1", lambda: minimize(st=stop(9)), INV),
        ("min null out.x/gradient", lambda: minimize(o=out(x=None, gradient=None)), (DEV, None)),
        ("min default stop", lambda: minimize(), (DEV, None)),
        ("min past max", lambda: minimize(st=stop(8)), (DEV, None)),
        # cno_minimize_steps: ... stepwise entry, batch / out / max_iterations, out arrays, batch == 0, x0, state,
        # workspace, I/O alignment, past, device
        ("steps unsupported", lambda: steps(p=problem(d=129)), UNS),
        ("steps no stepwise kernel", lambda: steps(p=problem(m=5)), UNS),
        ("steps batch < 0", lambda: steps(batch=-1), INV),
        ("steps null out", lambda: steps(o=None), INV),
        ("steps max_iterations 0", lambda: steps(it=0), INV),
        ("steps max_iterations < 0", lambda: steps(it=-3), INV),
        ("steps null out.value", lambda: steps(o=out(value=None), batch=0), INV),
        ("steps null out.status", lambda: steps(o=out(status=None)), INV),
        ("steps null out.num_iterations", lambda: steps(o=out(iters=None)), INV),
        ("steps batch 0", lambda: steps(batch=0, x0=None, state=None, ws=None), (DEV, OK)),
        ("steps null x0 first call", lambda: steps(x0=None, state=None), INV),
        ("steps null x0 later call", lambda: steps(x0=None, first=0, state=None), WS),
        ("steps null state", lambda: steps(state=None, ws=None), WS),
        ("steps short state", lambda: steps(state_bytes=4 * 5328 - 1, ws=None), WS),
        ("steps misaligned state", lambda: steps(state=A8, ws=None), WS),
        ("steps null workspace", lambda: steps(ws=None, x0=A8), WS),
        ("steps short workspace", lambda: steps(wsb=8, x0=A8), WS),
        ("steps misaligned x0", lambda: steps(x0=A8, st=stop(-1)), INV),
        ("steps misaligned out.x", lambda: steps(o=out(x=A1)), INV),
        ("steps misaligned out.gradient", lambda: steps(o=out(gradient=A8)), INV),
        ("steps past -1", lambda: steps(st=stop(-1)), INV),
        ("steps past max+1", lambda: steps(st=stop(9)), INV),
        ("steps exact state", lambda: steps(state_bytes=4 * 5328), (DEV, None)),
        # cno_minimize_host: problem, batch / x0 / out, then the device (before batch == 0 and past)
        ("host unsupported", lambda: host(p=problem(d=129)), UNS),
        ("host batch < 0", lambda: host(batch=-1), INV),
        ("host null x0", lambda: host(x0=None), INV),
        ("host null out", lambda: host(o=None), INV),
        ("host batch 0", lambda: host(batch=0), (DEV, OK)),
        # cno_lbfgsb_minimize: problem, batch / out, batch == 0, x0, bounds, workspace, I/O alignment, past, device
        ("lbfgsb null problem", lambda: lbfgsb(p=False), INV),
        ("lbfgsb unsupported", lambda: lbfgsb(p=problem(d=3)), UNS),
        ("lbfgsb lbfgs_m 20", lambda: lbfgsb(p=problem(m=20)), UNS),
        ("lbfgsb batch < 0", lambda: lbfgsb(batch=-1), INV),
        ("lbfgsb null out", lambda: lbfgsb(o=None), INV),
        ("lbfgsb batch 0", lambda: lbfgsb(batch=0, x0=None), (DEV, OK)),
        ("lbfgsb null x0", lambda: lbfgsb(x0=None, ws=None), INV),
        ("lbfgsb bounds stride < d", lambda: lbfgsb(bounds=_lib.Bounds(A16, A16, 7), ws=None), INV),
        ("lbfgsb null workspace", lambda: lbfgsb(bounds=_lib.Bounds(A16, A16, 8), ws=None, x0=A8), WS),
        ("lbfgsb short workspace", lambda: lbfgsb(wsb=0, x0=A8), WS),
        ("lbfgsb misaligned workspace", lambda: lbfgsb(ws=A16 + 2), WS),
        ("lbfgsb misaligned x0", lambda: lbfgsb(x0=A8, st=stop(9)), INV),
        ("lbfgsb misaligned out.x", lambda: lbfgsb(o=out(x=A8)), INV),
        ("lbfgsb misaligned out.gradient", lambda: lbfgsb(o=out(gradient=A8)), INV),
        ("lbfgsb past -1", lambda: lbfgsb(st=stop(-1)), INV),
        ("lbfgsb past max+1", lambda: lbfgsb(st=stop(9)), INV),
        ("lbfgsb one box", lambda: lbfgsb(bounds=_lib.Bounds(A16, None, 0)), (DEV, None)),
        ("lbfgsb default stop", lambda: lbfgsb(), (DEV, None)),
        # cno_evaluate: problem / batch, dtype, policy, table, device (the pointer checks run after it)
        ("eval null problem", lambda: evaluate(p=False), INV),
        ("eval batch < 0", lambda: evaluate(batch=-1), INV),
        ("eval bad dtype", lambda: evaluate(p=problem(dtype=5)), INV),
        ("eval policy", lambda: evaluate(p=problem(policy=_lib.POLICY_EIGEN_SSE2)), UNS),
        ("eval unsupported", lambda: evaluate(p=problem(family=_lib.FN_LOGISTIC, dtype=1, d=64)), UNS),
        ("eval null x", lambda: evaluate(x=None), (DEV, INV)),
        ("eval no outputs", lambda: evaluate(value=None, gradient=None), (DEV, INV)),
        ("eval batch 0", lambda: evaluate(batch=0), (DEV, OK)),
        # cno_condition_hessian: problem / batch, dtype, policy, table, batch == 0 (no device check), pointers
        ("cond null problem", lambda: condition(p=False), INV),
        ("cond batch < 0", lambda: condition(batch=-1), INV),
        ("cond bad dtype", lambda: condition(p=problem(dtype=2, d=8)), INV),
        ("cond policy", lambda: condition(p=problem(family=4, d=64, policy=_lib.POLICY_DMMA_LU)), UNS),
        ("cond unsupported", lambda: condition(p=problem(family=0, d=37)), UNS),
        ("cond batch 0", lambda: condition(batch=0, x=None, cond=None, ws=None), OK),
        ("cond null x", lambda: condition(x=None), INV),
        ("cond misaligned x", lambda: condition(x=A8), INV),
        ("cond null condition", lambda: condition(cond=None), INV),
        ("cond null workspace", lambda: condition(ws=None), INV),
        ("cond short workspace", lambda: condition(wsb=7), INV),
        ("cond misaligned workspace", lambda: condition(ws=A16 + 4), INV),
        ("cond 8-aligned workspace", lambda: condition(ws=A8), (DEV, None)),
        # cno_al_minimize: problem / constraints, batch / out, batch == 0, out arrays, multipliers, alignment,
        # workspace, inner past, device
        ("al null problem", lambda: al(p=False), INV),
        ("al null constraints", lambda: al(k=None), INV),
        ("al bad dtype", lambda: al(p=problem(dtype=3)), INV),
        ("al negative count", lambda: al(k=_lib.Constraints(-1, 0, A16, A16, 0)), INV),
        ("al too many", lambda: al(k=_lib.Constraints(0, 33, A16, A16, 0)), UNS),
        ("al null kinds", lambda: al(k=_lib.Constraints(1, 0, None, A16, 0)), INV),
        ("al unsupported", lambda: al(p=problem(d=64)), UNS),
        ("al batch < 0", lambda: al(batch=-1), INV),
        ("al null out", lambda: al(o=None), INV),
        ("al batch 0", lambda: al(batch=0, x0=None, ws=None), (DEV, OK)),
        ("al null x0", lambda: al(x0=None), INV),
        ("al null multipliers", lambda: al(mult=None), INV),
        ("al misaligned x0", lambda: al(x0=A8, ws=None), INV),
        ("al null workspace", lambda: al(ws=None, st=stop(-1)), WS),
        ("al short workspace", lambda: al(wsb=1024), WS),
        ("al misaligned workspace", lambda: al(ws=A16 + 128), WS),
        ("al past -1", lambda: al(st=stop(-1)), INV),
        ("al past max+1", lambda: al(st=stop(9)), INV),
        ("al no constraints", lambda: al(k=_lib.Constraints(0, 0, None, None, 0), mult=None), (DEV, None)),
        # cno_supported / cno_workspace_bytes
        ("supported null problem", lambda: _lib.lib().cno_supported(0, None), INV),
        ("supported bad solver", lambda: _lib.lib().cno_supported(-1, C.byref(problem())), INV),
        ("workspace null problem", lambda: _lib.lib().cno_workspace_bytes(0, None, 4, None), INV),
        ("lbfgsb supported null", lambda: _lib.lib().cno_lbfgsb_supported(None), INV),
        ("al supported null", lambda: _lib.lib().cno_al_supported(None, None), INV),
    ] + [("unused out struct", lambda: minimize(o=nul), (DEV, None))]


@pytest.mark.parametrize("name,call,expect", cases(), ids=[c[0] for c in cases()])
def test_return_code(name, call, expect):
    if isinstance(expect, tuple):  # reaches the device check
        if not HAVE_GPU:
            assert call() == NODEV
        elif expect[1] is not None:  # safe on a device: returns before any launch
            assert call() == expect[1]
        return
    assert call() == expect
