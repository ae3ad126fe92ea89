"""Independent models of the kernels' summation order, exact references and the edge vectors that
tests/test_evaluate_gpu.py (on the GPU) and tests/test_device_emulated.py (under the CPU warp emulation) share.

The arithmetic specification (csrc/cno_device.cuh, DESIGN.md section 3): every sum is an in-lane binary tree over
the E = ceil(d / 32) slots of a lane, then a cross-lane sum of the 32 lane partials p[0..31]:
  fp64: two FP64 tensor-core MMAs with A = ones, each element the FMA chain d = c; d = fma(1, b_k, d):
          S_n = (((0 + p[4n]) + p[4n+1]) + p[4n+2]) + p[4n+3]    n = 0..7
          T_j = S_2j + S_2j+1                                    j = 0..3
          sum = (((0 + T_0) + T_1) + T_2) + T_3
  fp32: xor butterfly over the offsets 16, 8, 4, 2, 1.
The models below restate that order with numpy's IEEE binary64 / binary32 operations, vectorised over the batch,
and restate each functor of csrc/cno_functors.cuh on top of it.  They are written from the specification, not from
the oracle, so the tests can hold GPU, emulated device source, model and oracle against each other.

Exact references: every functor value is sum_i term_i and every gradient component a short expression of the
inputs.  Evaluated in fractions.Fraction from the float inputs, the computed result must satisfy
  |computed - exact| <= gamma_k * abs + slack,   gamma_k = k u / (1 - k u)
where abs is the same expression evaluated exactly on |inputs| with every subtraction turned into an addition,
and k the rounding depth of the longest chain: a sum adds one to the deeper operand, a product adds one to the
sum of both operands' depths.  With no underflow this is the standard forward bound (Higham, Accuracy and
Stability of Numerical Algorithms, ch. 3); `slack` covers products that can land in the subnormal range, where
the rounding error is absolute (at most eta = half the smallest subnormal) instead of relative."""
from fractions import Fraction

import numpy as np

U = {np.float64: Fraction(1, 2 ** 53), np.float32: Fraction(1, 2 ** 24)}
ETA = {np.float64: Fraction(1, 2 ** 1075), np.float32: Fraction(1, 2 ** 150)}
F64_MAX = np.finfo(np.float64).max
SUB64 = np.float64(2.0 ** -1074)  # 5e-324, the smallest subnormal


def _quiet(f):  # overflow, Inf - Inf and NaN operands are the point of the edge vectors, not a warning
    def g(*a):
        with np.errstate(all="ignore"):
            return f(*a)
    return g


def gamma(k, dtype):
    u = U[dtype]
    return k * u / (1 - k * u)


def lane_depth(d):
    """Rounding depth of the in-lane binary tree: ceil(log2 E)."""
    E = (d + 31) // 32
    return (E - 1).bit_length()


def cross_depth(dtype):
    """4 + 1 + 4 for the tensor-core tree (first MMA chain, T_j, second MMA chain), 5 for the butterfly."""
    return 9 if dtype == np.float64 else 5


# ---- the summation order ----------------------------------------------------------------------------------------------
def lane_partials(t):
    """t: [..., d] terms -> [..., 32] lane partials (lane l owns slots l*E .. l*E+E-1, zero padded; binary tree)."""
    t = np.asarray(t)
    d = t.shape[-1]
    E = (d + 31) // 32
    v = np.zeros(t.shape[:-1] + (32 * E,), t.dtype)
    v[..., :d] = t
    v = v.reshape(t.shape[:-1] + (32, E)).copy()
    w = 1
    while w < E:
        for j in range(0, E - w, 2 * w):
            v[..., j] = v[..., j] + v[..., j + w]
        w *= 2
    return v[..., 0].copy()


def cross_lane_sum(p):
    """[..., 32] lane partials -> [...] the cross-lane sum of the dtype's policy."""
    p = np.asarray(p)
    if p.dtype == np.float64:
        zero = np.zeros(p.shape[:-1])
        S = []
        for n in range(8):
            s = zero + p[..., 4 * n]
            for k in range(1, 4):
                s = s + p[..., 4 * n + k]
            S.append(s)
        T = [S[2 * j] + S[2 * j + 1] for j in range(4)]
        r = zero + T[0]
        for j in range(1, 4):
            r = r + T[j]
        return r
    p = p.copy()
    for off in (16, 8, 4, 2, 1):
        p = p + p[..., np.arange(32) ^ off]
    return p[..., 0]


def warp_sum(t):
    return cross_lane_sum(lane_partials(t))


@_quiet
def stages(p):
    """fp64: the intermediate values S_n, T_j and the partial sums of the second chain (all finite = no overflow)."""
    p = np.asarray(p, np.float64)
    S = [(((0.0 + p[4 * n]) + p[4 * n + 1]) + p[4 * n + 2]) + p[4 * n + 3] for n in range(8)]
    T = [S[2 * j] + S[2 * j + 1] for j in range(4)]
    R = [0.0 + T[0]]
    for j in range(1, 4):
        R.append(R[-1] + T[j])
    return np.array(list(p) + S + T + R)


# ---- the functors of csrc/cno_functors.cuh in that order ----------------------------------------------------------------
@_quiet
def model_rosenbrock(x):
    x = np.asarray(x)
    T = x.dtype.type
    xi, xn = x[..., :-1], x[..., 1:]
    t1 = T(1) - xi
    t2 = xn - xi * xi
    term = np.zeros_like(x)
    term[..., :-1] = t1 * t1 + T(100) * t2 * t2
    A = T(-2) * (T(1) - xi) + T(200) * (xn - xi * xi) * (T(-2) * xi)
    Bv = T(200) * (xn - xi * xi)
    g = np.zeros_like(x)
    g[..., 0] = A[..., 0]
    g[..., 1:-1] = Bv[..., :-1] + A[..., 1:]
    g[..., -1] = Bv[..., -1]
    return warp_sum(term), g


@_quiet
def model_half_squared_norm(x):
    x = np.asarray(x)
    return x.dtype.type(0.5) * warp_sum(x * x), x.copy()


@_quiet
def model_diag_quadratic(x):
    x = np.asarray(x)
    T = x.dtype.type
    f = T(5) * x[..., 0] * x[..., 0] + T(100) * x[..., 1] * x[..., 1] + T(5)
    return f, np.stack([T(10) * x[..., 0], T(200) * x[..., 1]], -1)


@_quiet
def model_dense_quadratic(x, data):
    """data: [B, >= d*d + d] = [A column-major | b]; (Ax)_i = sum_j A_ij x_j, j ascending from the first product."""
    x = np.asarray(x)
    d = x.shape[-1]
    A = data[:, :d * d].reshape(-1, d, d)  # A[b, j, i] = A_ij
    b = data[:, d * d:d * d + d]
    Ax = A[:, 0, :] * x[:, :1]
    for j in range(1, d):
        Ax = Ax + A[:, j, :] * x[:, j:j + 1]
    p1, p2 = warp_sum(x * Ax), warp_sum(b * x)
    return x.dtype.type(0.5) * p1 - p2, Ax - b


# ---- exact references ---------------------------------------------------------------------------------------------------
def _fr(v):
    return Fraction(float(v))


def exact_rosenbrock(x, dtype):
    """(value, abs, k), [(g_i, abs_i)], k_g for one instance.  term: t1 t1 (3) + (100 t2) t2 (6) -> 7;
    A_i = -2 (1 - x_i) (2) + (200 t2)(-2 x_i) (5) -> 6, B_i = 200 t2 (3), g_i = B_{i-1} + A_i -> 7."""
    X = [_fr(v) for v in x]
    a = [abs(v) for v in X]
    d = len(X)
    val = vabs = Fraction(0)
    A, Aa, Bv, Ba = [], [], [], []
    for i in range(d - 1):
        t1, t1a = 1 - X[i], 1 + a[i]
        t2, t2a = X[i + 1] - X[i] * X[i], a[i + 1] + a[i] * a[i]
        val += t1 * t1 + 100 * t2 * t2
        vabs += t1a * t1a + 100 * t2a * t2a
        A.append(-2 * t1 + 200 * t2 * (-2 * X[i]))
        Aa.append(2 * t1a + 200 * t2a * 2 * a[i])
        Bv.append(200 * t2)
        Ba.append(200 * t2a)
    g = [(A[0], Aa[0])] + [(Bv[i - 1] + A[i], Ba[i - 1] + Aa[i]) for i in range(1, d - 1)] + [(Bv[-1], Ba[-1])]
    return (val, vabs, 7 + lane_depth(d) + cross_depth(dtype)), g, 7


def exact_half_squared_norm(x, dtype):
    """0.5 * sum x_i x_i: one product per term, the tree, the final scaling; the gradient is x itself (k = 0)."""
    X = [_fr(v) for v in x]
    s = sum(v * v for v in X) / 2
    return (s, s, 1 + lane_depth(len(X)) + cross_depth(dtype) + 1), [(v, abs(v)) for v in X], 0


def exact_diag_quadratic(x, dtype):
    """((5 x0) x0 + (100 x1) x1) + 5: depth 4; gradient 10 x0, 200 x1: depth 1 (no warp sum)."""
    x0, x1 = _fr(x[0]), _fr(x[1])
    v = 5 * x0 * x0 + 100 * x1 * x1 + 5
    return (v, abs(v), 4), [(10 * x0, abs(10 * x0)), (200 * x1, abs(200 * x1))], 1


def exact_dense_quadratic(x, row, dtype):
    """(Ax)_i is a chain of d products (depth d), x_i (Ax)_i adds one, then the tree, 0.5 * p1 one more, and the
    final subtraction one: k = d + 1 + tree + 1 + 1 (the b'x side is shallower).  g_i = (Ax)_i - b_i: d + 1."""
    d = len(x)
    X = [_fr(v) for v in x]
    Aij = lambda i, j: _fr(row[i + j * d])  # noqa: E731  (column-major)
    Ax, Axa = [], []
    for i in range(d):
        Ax.append(sum(Aij(i, j) * X[j] for j in range(d)))
        Axa.append(sum(abs(Aij(i, j) * X[j]) for j in range(d)))
    b = [_fr(row[d * d + i]) for i in range(d)]
    v = sum(X[i] * Ax[i] for i in range(d)) / 2 - sum(b[i] * X[i] for i in range(d))
    va = sum(abs(X[i]) * Axa[i] for i in range(d)) / 2 + sum(abs(b[i] * X[i]) for i in range(d))
    k = d + 1 + lane_depth(d) + cross_depth(dtype) + 2
    return (v, va, k), [(Ax[i] - b[i], Axa[i] + abs(b[i])) for i in range(d)], d + 1


def within(computed, exact, absval, k, dtype, slack=0):
    """|computed - exact| <= gamma_k * abs + slack * eta, for a finite computed value."""
    c = float(computed)
    if not np.isfinite(c):
        return False
    return abs(Fraction(c) - exact) <= gamma(k, dtype) * absval + slack * ETA[dtype]


# ---- fp64 edge vectors of the cross-lane sum: 32 lane partials each ------------------------------------------------------
def edge_partials():
    """name -> p[0..31].  Subnormal partials, normals cancelling to a subnormal, DBL_MAX placed so that the
    overflow happens in the first MMA chain, in T_j or in the second chain, absorption of 1 between +-1e300,
    +Inf, +Inf with -Inf, a NaN in each lane position, and all -0.0."""
    rng = np.random.default_rng(2024)
    normals = lambda: rng.uniform(-4, 4, 32)  # noqa: E731
    M = F64_MAX
    v = {"min_subnormal": np.full(32, SUB64)}
    k = rng.integers(-40, 41, 32).astype(np.float64)
    k[0] = 3.0 - (k.sum() - k[0])  # exact sum 3 * 2^-1074
    v["mixed_subnormals"] = k * SUB64
    p = np.zeros(32)
    a = 1.75 * 2.0 ** -1020
    p[0], p[31] = a, -(a - 5 * 2.0 ** -1072)  # Sterbenz: a - (a - 5 ulp) = 5 * 2^-1072, subnormal
    p[8], p[9] = 1e-300, -1e-300
    v["normals_cancel_to_subnormal"] = p
    p = np.zeros(32)
    p[0], p[1], p[2], p[3] = M, M, -M, -M  # S_0 = M + M - M - M: Inf, not 0
    v["overflow_first_mma"] = p
    p = np.zeros(32)
    p[0], p[4], p[8] = M, M, -M  # S_0 = S_1 = M: T_0 = Inf
    v["overflow_in_T"] = p
    p = np.zeros(32)
    p[0], p[8], p[16], p[24] = M, M, -M, -M  # T_0 .. T_3 = M, M, -M, -M: the second chain overflows
    v["overflow_second_mma"] = p
    p = np.zeros(32)
    p[0], p[1], p[2] = 1e300, 1.0, -1e300
    v["absorb_one_first_mma"] = p
    p = np.zeros(32)
    p[0], p[16], p[31] = 1e300, 1.0, -1e300
    v["absorb_one_second_mma"] = p
    p = normals()
    p[13] = np.inf
    v["plus_inf"] = p
    p = normals()
    p[2], p[27] = np.inf, -np.inf
    v["inf_minus_inf"] = p
    for lane in range(32):
        p = normals()
        p[lane] = np.nan
        v["nan_lane_%02d" % lane] = p
    v["negative_zero"] = np.full(32, -0.0)
    return v


def neg_sum_probe(p):
    """DenseQuadratic d = 64 with A = 0, x = 1 and b = (p_0, -0, p_1, -0, ...): lane l's partial of b'x is
    p_l + (-0) = p_l, so the value is 0.5 * 0 - sum(p) and the gradient 0 - b.  Drives sum `b` of warp_sum_pair."""
    B = len(p)
    b = np.full((B, 64), -0.0)
    b[:, 0::2] = p
    data = np.concatenate([np.zeros((B, 64 * 64)), b], 1)
    return np.ones((B, 64)), data


def diag_probe(p):
    """DenseQuadratic d = 64 with A = diag(p_0, -0, p_1, -0, ...) and -0.0 off the diagonal, b = 0, x = 1: every
    (Ax)_i is exactly its diagonal entry (also -0.0), lane l's partial of x'Ax is p_l, the value 0.5 * sum(p)
    and the gradient Ax.  Drives sum `a` of warp_sum_pair."""
    B = len(p)
    diag = np.full((B, 64), -0.0)
    diag[:, 0::2] = p
    A = np.full((B, 64, 64), -0.0)
    A[:, np.arange(64), np.arange(64)] = diag
    data = np.concatenate([A.transpose(0, 2, 1).reshape(B, -1), np.zeros((B, 64))], 1)
    return np.ones((B, 64)), data


def half_norm_points():
    """HalfSquaredNorm d = 50 (E = 2, lanes 0..24 hold data): name -> x, for non-negative partials through
    warp_sum.  Squares that are exact subnormals (k 2^-537 squared), DBL_MAX-sized squares overflowing in each
    stage, absorption, +Inf, a NaN in each data lane, -0.0."""
    rng = np.random.default_rng(50)
    v = {"min_subnormal": np.full(50, 2.0 ** -537)}
    v["subnormal_squares"] = rng.integers(0, 7, 50) * 2.0 ** -537
    for name, slots in (("overflow_first_mma", (0, 2)), ("overflow_in_T", (0, 8)), ("overflow_second_mma", (0, 16))):
        x = np.zeros(50)
        x[list(slots)] = 1e154  # squares 1e308: lanes 0 and 1 / 0 and 4 / 0 and 8
        v[name] = x
    x = np.zeros(50)
    x[0], x[1] = 1e150, 1.0
    v["absorb_one"] = x
    x = rng.uniform(-2, 2, 50)
    x[13] = np.inf
    v["plus_inf"] = x
    for lane in range(25):
        x = rng.uniform(-2, 2, 50)
        x[2 * lane + (lane & 1)] = np.nan
        v["nan_lane_%02d" % lane] = x
    v["negative_zero"] = np.full(50, -0.0)
    return v


# ---- fp32 Rosenbrock edges --------------------------------------------------------------------------------------------
SUBNORMAL_G = np.float32(-200.0 * 2.0 ** -140)  # g[d-1] = 200 (0 - (2^-70)^2) = -1.43493e-40, an fp32 subnormal


def rosenbrock_f32_points(d):
    """name -> x (float32).  x[d-2] = 2^-70, x[d-1] = 0 gives the subnormal g[d-1] above; x = 1e10 overflows the
    value (100 t2^2 ~ 1e42) while the gradient stays finite (~ 4e32); NaN starts."""
    rng = np.random.default_rng(d)
    v = {}
    x = rng.uniform(-2, 2, d).astype(np.float32)
    x[d - 2], x[d - 1] = np.float32(2.0 ** -70), np.float32(0.0)
    v["subnormal_gradient"] = x
    v["huge"] = np.full(d, 1e10, np.float32)
    for i in (0, d // 2, d - 1):
        x = rng.uniform(-2, 2, d).astype(np.float32)
        x[i] = np.nan
        v["nan_at_%d" % i] = x
    return v


ROSENBROCK, HALF_SQUARED_NORM, DENSE_QUADRATIC = 0, 2, 4  # cno_function_t


def probe_cases():
    """(name, family, x, data, vector names, (model value, model gradient)) of every edge vector above, per probe."""
    cases = []
    p = edge_partials()
    P = np.stack(list(p.values()))
    for probe, build in (("neg_sum", neg_sum_probe), ("diag", diag_probe)):
        x, data = build(P)
        cases.append((probe, DENSE_QUADRATIC, x, data, list(p), model_dense_quadratic(x, data)))
    h = half_norm_points()
    x = np.stack(list(h.values()))
    cases.append(("half_norm", HALF_SQUARED_NORM, x, None, list(h), model_half_squared_norm(x)))
    for d in (32, 37, 128):
        r = rosenbrock_f32_points(d)
        x = np.stack(list(r.values()))
        cases.append(("rosenbrock_f32_d%d" % d, ROSENBROCK, x, None, list(r), model_rosenbrock(x)))
    return cases


@_quiet
def chain_finite(family, x, data=None):
    """Per instance: every input and every intermediate of the model's sums is finite (where the exact-sum bound
    applies).  fp64 sums: the lane partials, S_n, T_j and the second chain; fp32: the inputs and the results."""
    x = np.asarray(x)
    ok = np.isfinite(x).all(-1)
    if family == ROSENBROCK:
        f, g = model_rosenbrock(x)
        return ok & np.isfinite(f) & np.isfinite(g).all(-1)
    if family == HALF_SQUARED_NORM:
        parts = [x * x]
    else:
        d = x.shape[-1]
        ok &= np.isfinite(data).all(-1)
        A = data[:, :d * d].reshape(-1, d, d)
        Ax = A[:, 0, :] * x[:, :1]
        for j in range(1, d):
            Ax = Ax + A[:, j, :] * x[:, j:j + 1]
        parts = [x * Ax, data[:, d * d:d * d + d] * x]
    for t in parts:
        ok &= np.array([np.isfinite(stages(p)).all() for p in lane_partials(t)])
    return ok


def exact(family, x, row, dtype):
    """(value, abs, k), [(g_i, abs_i)], k_g and the value's underflow slack (in eta) for one instance."""
    if family == ROSENBROCK:
        return (*exact_rosenbrock(x, dtype), 0)
    if family == HALF_SQUARED_NORM:
        return (*exact_half_squared_norm(x, dtype), 1)  # 0.5 * sum may round a subnormal
    if family == DENSE_QUADRATIC:
        return (*exact_dense_quadratic(x, row, dtype), 1)
    return (*exact_diag_quadratic(x, dtype), 0)


def check_exact(family, x, data, f, g, dtype):
    """Asserts the exact-sum bound on every instance's value and gradient components."""
    for i in range(x.shape[0]):
        (v, va, k), comps, kg, slack = exact(family, x[i], None if data is None else data[i], dtype)
        assert within(f[i], v, va, k, dtype, slack), (i, float(f[i]), float(v), k)
        for j, (gv, ga) in enumerate(comps):
            assert within(g[i, j], gv, ga, kg, dtype), (i, j, float(g[i, j]), float(gv), kg)


def same_bits(a, b):
    """Bit-for-bit equality, except that a NaN only has to be a NaN (its sign and payload are not specified)."""
    a, b = np.atleast_1d(a), np.atleast_1d(b)
    if a.dtype != b.dtype:
        return False
    if a.dtype.kind == "f":
        nan = np.isnan(a)
        if not np.array_equal(nan, np.isnan(b)):
            return False
        a, b = np.where(nan, 0, a), np.where(nan, 0, b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
