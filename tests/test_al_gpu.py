"""AugmentedLagrangian on the device (include/cno_al.h, csrc/cno_auglag.cuh) against the pinned CPU
oracle and the reference-headers fixtures tests/golden/al_*.npz, bit for bit."""
import glob
import os

import numpy as np
import pytest
import torch

import cppnumericalsolvers_b200 as cn
from oracle import oracle_binding as ob

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda:0"
TDT = {np.float64: torch.float64, np.float32: torch.float32}
KEYS = ("num_iterations", "status", "nfev", "x", "equality_multipliers", "inequality_multipliers", "penalty",
        "max_violation", "max_lagrangian_gradient", "x_delta", "f_delta", "gradient_norm")
FAMILY = {ob.FN_ROSENBROCK: cn.Rosenbrock, ob.FN_HALF_SQUARED_NORM: cn.HalfSquaredNorm}


def _gpu(family, x0_np, kinds, rows_np, n_eq, outer_limit=None, eq0=None, ineq0=None, penalty0=None,
         config=None, inner=None):
    d = x0_np.shape[1]
    fn = FAMILY[family](d, TDT[x0_np.dtype.type])
    problem = cn.ConstrainedOptimizationProblem(fn, list(kinds), torch.from_numpy(np.ascontiguousarray(rows_np)).to(DEV), n_eq)
    solver = cn.AugmentedLagrangian(problem, inner, config)
    assert solver.supported()
    if outer_limit is not None:
        solver.stopping_progress.num_iterations = outer_limit
    st, pr = solver.Minimize(cn.AugmentedLagrangeState(torch.from_numpy(x0_np).to(DEV), eq0, ineq0, penalty0))
    torch.cuda.synchronize()
    return dict(x=st.x.cpu().numpy(), equality_multipliers=st.equality_multipliers.cpu().numpy(),
                inequality_multipliers=st.inequality_multipliers.cpu().numpy(), penalty=st.penalty.cpu().numpy(),
                max_violation=st.max_violation.cpu().numpy(),
                max_lagrangian_gradient=st.max_lagrangian_gradient.cpu().numpy(),
                num_iterations=pr.num_iterations.cpu().numpy().astype(np.uint32), status=pr.status.cpu().numpy(),
                nfev=pr.nfev.cpu().numpy().astype(np.uint32), x_delta=pr.x_delta.cpu().numpy(),
                f_delta=pr.f_delta.cpu().numpy(), gradient_norm=pr.gradient_norm.cpu().numpy())


def _assert_same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), f"{k} differs"


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "al_*.npz"))))
def test_al_matches_reference_fixtures(path):
    """tests/golden/al_*.npz were produced by the reference's own headers (make_golden_al.py)."""
    z = np.load(path)
    r = _gpu(int(z["family"]), z["x0"], z["kinds"], z["rows"], int(z["n_eq"]), outer_limit=int(z["outer_limit"]))
    for k in KEYS:
        assert np.array_equal(r[k].view(np.uint8), z[k].view(np.uint8)), k


@pytest.mark.parametrize("family,dtype,d,n_eq,per_instance,B", [
    (ob.FN_ROSENBROCK, np.float64, 2, 1, False, 64), (ob.FN_ROSENBROCK, np.float64, 8, 1, True, 96),
    (ob.FN_ROSENBROCK, np.float64, 37, 0, True, 48), (ob.FN_ROSENBROCK, np.float64, 8, 3, False, 64),
    (ob.FN_ROSENBROCK, np.float32, 8, 1, True, 64), (ob.FN_ROSENBROCK, np.float64, 128, 1, True, 40),
    (ob.FN_HALF_SQUARED_NORM, np.float64, 8, 2, True, 64)])
def test_al_bitwise_equals_oracle(family, dtype, d, n_eq, per_instance, B):
    rng = np.random.default_rng(100 + d)
    x0 = ob.fill_uniform((B, d), 0, 31 + d, -1.5, 1.5, dtype)
    kinds = [ob.CON_AFFINE, ob.CON_SQNORM, ob.CON_AFFINE]
    shape = (B, 3, d + 1) if per_instance else (3, d + 1)
    rows = rng.uniform(-1, 1, shape).astype(dtype)
    rows[..., 1, d] = 2.0 + rng.uniform(0, 1, shape[:-2])
    stop = ob.al_default_stop()
    stop.num_iterations = 12
    _assert_same(_gpu(family, x0, kinds, rows, n_eq, outer_limit=12),
                 ob.al_minimize(family, x0, kinds, rows, n_eq, outer_stop=stop))


def test_al_reference_known_answers_and_user_state():
    """augmented_lagrangian_test.cc:492-539 (EqualityOnlyQuadratic), :627-692 (FeasibleStart,
    NoConstraints); user-set multipliers / penalty / config / inner preset."""
    r = _gpu(ob.FN_HALF_SQUARED_NORM, np.array([[5.0, 5.0]]), [ob.CON_AFFINE], np.array([[1.0, 0.0, 1.0]]), 1,
             penalty0=1.0)
    assert abs(r["x"][0, 0] - 1.0) <= 1e-3 and abs(r["x"][0, 1]) <= 1e-3
    assert abs(r["equality_multipliers"][0, 0] + 1.0) <= 1e-2
    _assert_same(r, ob.al_minimize(ob.FN_HALF_SQUARED_NORM, np.array([[5.0, 5.0]]), [ob.CON_AFFINE],
                                   [[1.0, 0.0, 1.0]], 1, penalty0=1.0))
    r = _gpu(ob.FN_HALF_SQUARED_NORM, np.array([[0.0, 0.0]]), [ob.CON_AFFINE], np.array([[0.0, 0.0, 0.0]]), 1,
             penalty0=1.0)
    assert r["status"][0] == 6 and r["num_iterations"][0] <= 5
    r = _gpu(ob.FN_HALF_SQUARED_NORM, np.array([[5.0, 5.0]]), [], np.zeros((0, 3)), 0, penalty0=1.0)
    assert r["status"][0] == 6 and np.all(np.abs(r["x"][0]) <= 1e-3)

    x0 = ob.fill_uniform((32, 8), 0, 77, -1.5, 1.5)
    rows = np.random.default_rng(5).uniform(-1, 1, (2, 9))
    rows[1, 8] = 2.5
    cfg = cn.AugmentedLagrangianConfig(warmup_max_inner_iterations=0, violation_shrink_ratio=0.5, multiplier_max=5.0)
    ocfg = ob.al_default_config()
    ocfg.warmup_max_inner_iterations, ocfg.violation_shrink_ratio, ocfg.multiplier_max = 0, 0.5, 5.0
    stop = ob.al_default_stop()
    stop.num_iterations = 10
    _assert_same(_gpu(ob.FN_ROSENBROCK, x0, [ob.CON_AFFINE, ob.CON_SQNORM], rows, 1, outer_limit=10, eq0=0.25,
                      ineq0=0.5, penalty0=2.0, config=cfg, inner=cn.Lbfgs(cn.ConservativeStoppingSolverProgress())),
                 ob.al_minimize(ob.FN_ROSENBROCK, x0, [ob.CON_AFFINE, ob.CON_SQNORM], rows, 1, outer_stop=stop,
                                config=ocfg, inner_stop=ob.conservative_stop(), eq0=0.25, ineq0=0.5, penalty0=2.0))


def test_al_cpp_mirror_equality_only_quadratic():
    """tests/cpp/al_host.cc: the C++ mirror (cppoptlib::solver::AugmentedLagrangian) on
    augmented_lagrangian_test.cc:492-539."""
    import subprocess
    from cppnumericalsolvers_b200 import build
    build.build_cpp_tests()
    exe = os.path.join(os.path.dirname(__file__), "cpp", "build", "al_host")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout + r.stderr


def _quadratic(center, scale):
    d = len(center)
    return np.array([list((scale * np.eye(d)).T.ravel()) + [scale * c for c in center]])


def test_lbfgs_first_mode_dense_quadratic_bitwise_equals_oracle():
    """DenseQuadraticGlobalFn (csrc/cno_functors.cuh), added after the last GPU session: Lbfgs on per-instance
    dense quadratics read from global memory."""
    for d, B in ((8, 64), (64, 32)):
        rng = np.random.default_rng(d)
        M = rng.uniform(-1, 1, (B, d, d))
        A = np.einsum("bij,bkj->bik", M, M) / d + np.eye(d)
        A = (A + A.transpose(0, 2, 1)) / 2
        data = np.concatenate([A.transpose(0, 2, 1).reshape(B, -1), rng.uniform(-1, 1, (B, d))], 1)
        x0 = ob.fill_uniform((B, d), 0, 17 + d, -2.0, 2.0)
        fn = cn.DenseQuadraticFirst(torch.from_numpy(data).to(DEV), d)
        assert cn.Lbfgs().supported(fn)
        st, pr = cn.Lbfgs().Minimize(fn, cn.BatchedFunctionState(torch.from_numpy(x0).to(DEV)))
        o = ob.minimize(ob.LBFGS, ob.FN_DENSE_QUADRATIC, x0, data=data)
        assert np.array_equal(st.x.cpu().numpy().view(np.uint8), o["x"].view(np.uint8))
        assert np.array_equal(pr.num_iterations.cpu().numpy().astype(np.uint32), o["num_iterations"])
        assert np.array_equal(pr.nfev.cpu().numpy().astype(np.uint32), o["nfev"])


def test_al_reference_kkt_known_answers_quadratic_objectives():
    """augmented_lagrangian_test.cc:541-625: InequalityActiveRecoversMultiplier, BothEqualityAndInequalityActive."""
    def gpu(data, x0, kinds, rows, n_eq):
        fn = cn.DenseQuadraticFirst(torch.from_numpy(data).to(DEV), 2)
        problem = cn.ConstrainedOptimizationProblem(fn, kinds, torch.tensor(rows, dtype=torch.float64, device=DEV), n_eq)
        st, pr = cn.AugmentedLagrangian(problem).Minimize(cn.AugmentedLagrangeState(torch.tensor(x0, dtype=torch.float64, device=DEV), penalty=1.0))
        return st, pr
    data = _quadratic([2.0, 0.0], 1.0)
    st, pr = gpu(data, [[5.0, 5.0]], [ob.CON_AFFINE], [[-1.0, 0.0, -1.0]], 0)
    o = ob.al_minimize(ob.FN_DENSE_QUADRATIC, np.array([[5.0, 5.0]]), [ob.CON_AFFINE], [[-1.0, 0.0, -1.0]], 0, data=data, penalty0=1.0)
    x = st.x.cpu().numpy()
    assert abs(x[0, 0] - 1.0) <= 1e-3 and abs(x[0, 1]) <= 1e-3
    assert abs(st.inequality_multipliers.cpu().numpy()[0, 0] - 1.0) <= 1e-2
    assert np.array_equal(x.view(np.uint8), o["x"].view(np.uint8))
    data = _quadratic([1.0, 2.0], 2.0)
    rows = [[1.0, 0.0, 0.5], [-1.0, -1.0, -2.0]]
    st, pr = gpu(data, [[1.0, 1.0]], [ob.CON_AFFINE, ob.CON_AFFINE], rows, 1)
    o = ob.al_minimize(ob.FN_DENSE_QUADRATIC, np.array([[1.0, 1.0]]), [ob.CON_AFFINE, ob.CON_AFFINE], rows, 1, data=data, penalty0=1.0)
    x = st.x.cpu().numpy()
    assert abs(x[0, 0] - 0.5) <= 1e-3 and abs(x[0, 1] - 1.5) <= 1e-3
    assert np.array_equal(x.view(np.uint8), o["x"].view(np.uint8))
