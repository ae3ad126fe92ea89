"""The rare branches of the two Bfgs kernels (csrc/cno_bfgs.cuh): the reset of H to the identity (bfgs.h:88-92, phi > 0
or phi NaN; in bfgs_smem_minimize_kernel this is set_identity(), which rewrites the warp's whole shared-memory slice),
the refused update (bfgs.h:125: H kept, `fresh` kept, the curvature decided by curvature_above_eps's square-root-free
bound or by its fallback to the specification's expression) and non-finite line-search results.  Ordinary starts reach
none of them.  Each case first shows, from the oracle's path counts (oracle_binding.bfgs_paths) under the stop it runs
with, that it reaches the branches it claims; then the reference's own bfgs.h (oracle/_ref), the device source under the
CPU warp emulation (tests/emu/emu_bfgs.cc) and, on the GPU, every Bfgs Rosenbrock kernel of cno_api.cu's dispatch table,
with the case mixed into a full batch of ordinary starts, must equal the oracle on every output.

Every branch is reached on every kernel, HagerZhang included: its phi > 0 resets come from 10^6 spikes, its curvature
fallback from 10^39 spikes, and its NaN resets and non-finite line searches from the NaN-start case.  The fp32 phi > 0
reset needs small spikes (10^2 at every 4th or every 128th coordinate); larger fp32 spikes overflow into NaN resets.

Outputs compare bit for bit, except that a NaN only has to be a NaN in both: its sign and payload are not part of the
contract (x86 propagates an operand's NaN, the GPU writes the canonical quiet NaN), and the runs that go NaN here flip
that sign with every negation of the gradient, so even the oracle, the reference and the emulation, all on the CPU,
disagree on it where they order the operands of one operation differently."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_binding as ob

HERE = os.path.dirname(__file__)
EMU_DIR = os.path.join(HERE, "emu")
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
MT, HZ = ob.LS_MORE_THUENTE, ob.LS_HAGER_ZHANG

# name -> (d, dtype, line search, warps per CTA) of every Bfgs Rosenbrock entry of cno_api.cu's kTable.  The warps are
# BfgsSmem<T, d>::kWarps (d <= 32, H in registers) or BfgsBigSmem<T, d>::kWarps (d > 32, H in shared memory).
KERNELS = {
    "d2": (2, np.float64, MT, 12),
    "d8": (8, np.float64, MT, 12),
    "d32": (32, np.float64, MT, 10),
    "d37": (37, np.float64, MT, 8),
    "d64": (64, np.float64, MT, 6),
    "d128": (128, np.float64, MT, 1),
    "f32_d32": (32, np.float32, MT, 12),
    "f32_d128": (128, np.float32, MT, 3),
    "hz_d8": (8, np.float64, HZ, 12),
    "hz_d32": (32, np.float64, HZ, 10),
    "hz_d64": (64, np.float64, HZ, 6),
}

# kernel -> (row, iterations) of the near-minimiser start: the shortest run that refuses at least three updates after H
# was updated (the first iterations still converge; at d >= 64 that takes longer).
NEAR = {"d2": (0, 10), "d8": (0, 14), "d32": (0, 14), "d37": (0, 14), "d64": (0, 34), "d128": (1, 22),
        "f32_d32": (0, 10), "f32_d128": (1, 14), "hz_d8": (0, 14), "hz_d32": (0, 44), "hz_d64": (1, 98)}

# kernel -> (exponent, stride, seed, row) of the spiked starts: row `row` of fill_uniform((8, d), 0, seed, -2, 2) with
# every stride-th coordinate times 10^exponent.  The rows are picked so that together they reach every claim of the
# kernel's spike case within 8 iterations; the 10^11.5 rows of the MoreThuente fp64 kernels add the middle scale.
SPIKES = {
    "d2": [(10.0, 4, 21, 4), (11.5, 4, 21, 0), (17.5, 4, 21, 0)],
    "d8": [(10.0, 4, 21, 4), (11.5, 4, 21, 0), (17.5, 4, 21, 1)],
    "d32": [(10.0, 4, 21, 1), (11.5, 4, 21, 0), (17.5, 4, 21, 2)],
    "d37": [(10.0, 4, 21, 4), (11.5, 4, 21, 0), (17.5, 4, 21, 3)],
    "d64": [(10.0, 4, 21, 3), (11.5, 4, 21, 0), (17.5, 4, 21, 0)],
    "d128": [(10.0, 4, 21, 5), (11.5, 4, 21, 0), (17.5, 4, 21, 1)],
    "f32_d32": [(2.0, 4, 21, 0), (5.0, 4, 21, 0), (7.0, 4, 21, 0)],
    "f32_d128": [(2.0, 128, 21, 0), (5.0, 4, 21, 0), (7.0, 4, 21, 0)],
    "hz_d8": [(6.0, 3, 22, 7), (40.0, 4, 21, 1)],
    "hz_d32": [(6.0, 8, 21, 2), (39.0, 1, 21, 0)],
    "hz_d64": [(6.5, 64, 21, 0), (39.0, 1, 21, 0)],
}
SPIKE_CAP, NONFINITE_CAP = 8, 4

# Claims (ob.BFGS_PATHS, summed over the case's rows).
CLAIMS = {
    "near": ("refused_updated",),
    "spikes": ("reset_positive", "reset_nan", "refused_fresh", "curvature_fallback_true", "nonfinite"),
    "spikes_hz": ("reset_positive", "curvature_fallback_true"),
    "minimiser": ("refused_fresh", "curvature_fallback_false", "small_direction"),
    "nonfinite": ("reset_nan", "refused_fresh", "nonfinite", "small_direction"),
}
KINDS = ("near", "spikes", "minimiser", "nonfinite")
CASES = [(k, kind) for k in KERNELS for kind in KINDS]
CASE_IDS = [f"{k}-{kind}" for k, kind in CASES]


def capped_stop(iterations):
    s = ob.default_stop()
    s.num_iterations = iterations
    return s


def zero_tolerance_stop(iterations):
    s = capped_stop(iterations)
    s.x_delta = s.f_delta = s.gradient_norm = 0.0
    s.past = 0
    return s


def nonfinite_starts(d, dtype):
    """[-2, 2] starts with one NaN, +Inf or -Inf coordinate, with a -0.0 coordinate, and with one coordinate whose fourth
    power overflows (f = +Inf at a finite x)."""
    x = ob.fill_uniform((5, d), 0, 5, -2.0, 2.0).astype(dtype)
    x[0, d // 3] = np.nan
    x[1, d // 2] = np.inf
    x[2, d - 1] = -np.inf
    x[3, 1] = -0.0
    x[4, 0] = 1e100 if dtype == np.float64 else 1e12
    return x


def case(kernel, kind):
    """(x0, stop, claims) of one case of a kernel."""
    d, dt, ls, _ = KERNELS[kernel]
    if kind == "near":  # x* + 1e-12 noise (1e-5 in fp32), zero tolerances: the steps shrink until s.y fails the test
        row, iterations = NEAR[kernel]
        scale = 1e-5 if dt == np.float32 else 1e-12
        x = (1.0 + scale * ob.fill_uniform((2, d), 0, 24, -1.0, 1.0)).astype(dt)[[row]]
        return x, zero_tolerance_stop(iterations), CLAIMS["near"]
    if kind == "spikes":
        rows = []
        for e, stride, seed, row in SPIKES[kernel]:
            x = ob.fill_uniform((8, d), 0, seed, -2.0, 2.0)
            x[:, ::stride] *= 10.0 ** e
            rows.append(x[row])
        return np.array(rows).astype(dt), capped_stop(SPIKE_CAP), CLAIMS["spikes_hz" if ls == HZ else "spikes"]
    if kind == "minimiser":  # x = x* exactly: g = 0, d = 0, s = y = 0 with H still the identity
        return np.ones((1, d), dt), ob.default_stop(), CLAIMS["minimiser"]
    return nonfinite_starts(d, dt), capped_stop(NONFINITE_CAP), CLAIMS["nonfinite"]


def assert_reached(paths, claims):
    for c in claims:
        assert paths[c].sum() > 0, (c, {k: int(v.sum()) for k, v in paths.items()})


def assert_equal(a, b):
    """Every output bit for bit; a NaN must be a NaN in both, of any sign and payload."""
    for k in KEYS:
        u, v = np.asarray(a[k]), np.asarray(b[k])
        if u.dtype.kind == "f":
            nan = np.isnan(u)
            assert np.array_equal(nan, np.isnan(v)), f"{k}: NaN pattern differs"
            u, v = np.where(nan, 0, u), np.where(nan, 0, v)
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8)), k


def oracle_paths(kernel, x0, stop):
    return ob.bfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop, linesearch=KERNELS[kernel][2])


# ---------------------------------------------------------------- proof of reach (CPU) ----

@pytest.mark.parametrize("kernel,kind", CASES, ids=CASE_IDS)
def test_case_reaches_its_paths(kernel, kind):
    x0, stop, claims = case(kernel, kind)
    _, paths = oracle_paths(kernel, x0, stop)
    assert_reached(paths, claims)


def test_path_counts_leave_the_arithmetic_alone():
    """bfgs_paths returns what minimize returns, on the rare starts of every kind."""
    for kernel in ("d8", "d37", "f32_d32", "hz_d32"):
        for kind in KINDS:
            x0, stop, _ = case(kernel, kind)
            o, _ = oracle_paths(kernel, x0, stop)
            plain = ob.minimize(ob.BFGS, ob.FN_ROSENBROCK, x0, stop=stop, linesearch=KERNELS[kernel][2])
            for k in KEYS:
                assert np.array_equal(np.asarray(o[k]).view(np.uint8), np.asarray(plain[k]).view(np.uint8)), k


# ---------------------------------------------------------------- the oracle against the reference (CPU) ----

@pytest.mark.parametrize("kernel,kind", CASES, ids=CASE_IDS)
def test_oracle_equals_reference_bfgs(kernel, kind):
    """The oracle's reset, refusal and non-finite semantics against the reference's own bfgs.h and line searches on the
    Eigen-API shim: every output."""
    if not ob.ref_available():
        pytest.skip("oracle/_ref not built")
    x0, stop, claims = case(kernel, kind)
    o, paths = oracle_paths(kernel, x0, stop)
    assert_reached(paths, claims)
    assert_equal(ob.minimize(ob.BFGS, ob.FN_ROSENBROCK, x0, stop=stop, linesearch=KERNELS[kernel][2], impl="ref"), o)


# ---------------------------------------------------------------- emulation (CPU) ----

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/emu/emu_bfgs.cc compiled with the flags of tests/emu/Makefile into a temporary directory."""
    out = str(tmp_path_factory.mktemp("emu_bfgs") / "libcno_emu_bfgs.so")
    root = os.path.join(HERE, "..")
    subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-pthread",
                    "-DCNO_WARP_EMULATION", "-Wno-unknown-pragmas", "-Wno-attributes", "-shared", "-I", EMU_DIR,
                    "-I", os.path.join(root, "cppnumericalsolvers_b200", "csrc"), "-I", os.path.join(root, "include"),
                    os.path.join(EMU_DIR, "emu_bfgs.cc"), "-o", out], check=True)
    return C.CDLL(out)


def _emulated(emu, x0, stop, ls):
    B, d = x0.shape
    prob = ob.Problem(ob.FN_ROSENBROCK, ob._np_dtype(x0), d, 0, 0.0, None, 0, ob.device_policy(x0.dtype), 0, 0)
    r, out = ob._batch_out(x0)
    assert emu.emu_bfgs(int(ls == HZ), C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                        C.byref(out)) == 0
    return r


@pytest.mark.parametrize("kernel,kind", CASES, ids=CASE_IDS)
def test_emulated_kernel_equals_oracle(emu, kernel, kind):
    """bfgs_minimize_kernel (d <= 32) or bfgs_smem_minimize_kernel (d > 32) under the warp emulation, one warp draining
    the case's rows in order: every output against the oracle."""
    x0, stop, claims = case(kernel, kind)
    o, paths = oracle_paths(kernel, x0, stop)
    assert_reached(paths, claims)
    assert_equal(_emulated(emu, x0, stop, KERNELS[kernel][2]), o)


def test_emulated_warp_inherits_nothing_from_a_reset_instance(emu):
    """d = 37, H in shared memory: one warp drains a spiked start that resets H, then an ordinary start, then the NaN
    start, then x*: each later instance must equal its own solve, whatever the slice held before it."""
    spikes, _, _ = case("d37", "spikes")
    x0 = np.concatenate([spikes[:1], ob.fill_uniform((1, 37), 0, 3, -2.0, 2.0), nonfinite_starts(37, np.float64)[:1],
                         np.ones((1, 37))])
    stop = capped_stop(SPIKE_CAP)
    o, paths = oracle_paths("d37", x0, stop)
    assert paths["reset_positive"][0] > 0 and paths["reset_nan"][2] > 0
    assert_equal(_emulated(emu, x0, stop, MT), o)


def test_emulation_rejects_an_uncompiled_shape(emu):
    x0 = ob.fill_uniform((1, 16), 0, 1, -2.0, 2.0)
    prob = ob.Problem(ob.FN_ROSENBROCK, 0, 16, 0, 0.0, None, 0, ob.device_policy(x0.dtype), 0, 0)
    _, out = ob._batch_out(x0)
    stop = ob.default_stop()
    assert emu.emu_bfgs(0, C.byref(prob), C.c_longlong(1), C.c_void_p(x0.ctypes.data), C.byref(stop),
                        C.byref(out)) != 0


# ---------------------------------------------------------------- the GPU ----

def _gpu(x0, stop, ls, family=ob.FN_ROSENBROCK):
    import torch

    import cppnumericalsolvers_b200 as cn
    solver = cn.Bfgs(cn.Progress.from_c(stop), linesearch=cn.HagerZhang if ls == HZ else cn.MoreThuente)
    tdt = torch.float64 if x0.dtype == np.float64 else torch.float32
    d = x0.shape[1]
    fn = {ob.FN_ROSENBROCK: lambda: cn.Rosenbrock(d, tdt), ob.FN_DIAG_QUADRATIC: lambda: cn.DiagQuadratic(tdt),
          ob.FN_HALF_SQUARED_NORM: lambda: cn.HalfSquaredNorm(d, tdt)}[family]()
    st, pr = solver.Minimize(fn, cn.BatchedFunctionState(torch.from_numpy(x0).to("cuda:0")), timed=True)
    torch.cuda.synchronize()
    g = dict(x=st.x.cpu().numpy(), value=st.value.cpu().numpy(), gradient=st.gradient.cpu().numpy(),
             num_iterations=pr.num_iterations.cpu().numpy().astype(np.uint32), status=pr.status.cpu().numpy(),
             nfev=pr.nfev.cpu().numpy().astype(np.uint32), x_delta=pr.x_delta.cpu().numpy(),
             f_delta=pr.f_delta.cpu().numpy(), gradient_norm=pr.gradient_norm.cpu().numpy())
    return g, pr.launch


def _mixed(d, dtype, warps, rare, seed):
    """2 * SMs * warps + 3 ordinary [-2, 2] starts (more than one wave of resident warps) with the rare rows at seeded
    random positions, so that resetting and NaN instances share CTAs, and their shared memory, with ordinary ones."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 2 * sms * warps + 3
    x0 = ob.fill_uniform((B, d), 0, seed, -2.0, 2.0).astype(dtype)
    rows = np.random.default_rng(seed).choice(B, size=len(rare), replace=False)
    x0[rows] = rare
    return x0, rows


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,kind", CASES, ids=CASE_IDS)
def test_gpu_equals_oracle_on_rare_starts(kernel, kind):
    """Each Bfgs Rosenbrock kernel on each case mixed into a full batch: every row against the oracle."""
    d, dt, ls, warps = KERNELS[kernel]
    rare, stop, claims = case(kernel, kind)
    x0, rows = _mixed(d, dt, warps, rare, 9000 + d + 17 * KINDS.index(kind) + 101 * ls)
    o, paths = oracle_paths(kernel, x0, stop)
    assert_reached({k: v[rows] for k, v in paths.items()}, claims)
    g, launch = _gpu(x0, stop, ls)
    assert launch.warps_per_cta == warps
    assert_equal(g, o)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_gpu_small_batches(kernel):
    """B = 1 (the first spiked row, which resets H) and B = warps + 1 rare rows (a CTA only partly filled, not a multiple
    of the warps per CTA unless the kernel runs one warp): every row against the oracle."""
    d, dt, ls, warps = KERNELS[kernel]
    spikes, stop, _ = case(kernel, "spikes")
    g, _ = _gpu(spikes[:1].copy(), stop, ls)
    assert_equal(g, oracle_paths(kernel, spikes[:1].copy(), stop)[0])
    pool = np.concatenate([spikes, nonfinite_starts(d, dt), np.ones((1, d), dt)])
    x0 = pool[np.arange(warps + 1) % len(pool)]
    g, _ = _gpu(x0, stop, ls)
    assert_equal(g, oracle_paths(kernel, x0, stop)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("family", [ob.FN_DIAG_QUADRATIC, ob.FN_HALF_SQUARED_NORM], ids=["diag_quadratic", "half_sq_norm"])
def test_gpu_d2_functions_at_the_minimiser_and_nan(family):
    """The d = 2 DiagQuadratic and HalfSquaredNorm kernels: x* = 0 (refused while fresh, ||d|| <= eps) and a NaN start
    (NaN resets, non-finite line searches) in a full batch of ordinary starts."""
    rare = np.array([[0.0, 0.0], [np.nan, 0.5]])
    stop = capped_stop(NONFINITE_CAP * 5)
    x0, rows = _mixed(2, np.float64, 12, rare, 9500 + family)
    o, paths = ob.bfgs_paths(family, x0, stop=stop)
    assert_reached({k: v[rows] for k, v in paths.items()}, ("refused_fresh", "small_direction", "reset_nan", "nonfinite"))
    g, launch = _gpu(x0, stop, MT, family)
    assert launch.warps_per_cta == 12
    assert_equal(g, o)
