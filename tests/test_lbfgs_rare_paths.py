"""The rare branches of the plain L-BFGS kernel where it keeps its newest (s, y) pairs in registers (csrc/cno_lbfgs.cuh:
LbfgsPlan).  Ordinary starts never skip a pair (|s.y| < eps), never refuse one (curvature test) and never fall back to
-g with a non-empty history, so the warm-up branch of the two-loop recursion -- which runs whenever a pair is
unusable -- and the reset of the register slots are only reached from the starts below.  Each case first shows, from
the oracle's path counts (oracle_binding.lbfgs_paths), that it reaches the branches it claims, then compares every
output bit for bit: the device source under the CPU warp emulation, the reference's own lbfgs.h (oracle/_ref) and
the GPU against the oracle."""
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
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")

FAST, EIGEN = ob.POLICY_DMMA_TREE, ob.POLICY_EIGEN_SSE2
# name -> (d, m, reduction policy, launcher of cno_api.cu's kTable, register pairs R, warps per CTA) of every fp64
# Rosenbrock kernel whose LbfgsPlan keeps pairs in registers, and of the m = 5 kernels of the same d (no register
# pairs), which serve as controls on the GPU.
REGISTER_KERNELS = {
    "d128_m10": (128, 10, FAST, ("lbfgs_rosenbrock", "double, 128"), 1, 12),
    "d37_m20": (37, 20, FAST, ("lbfgs_rosenbrock_m", "double, 37, 20"), 2, 12),
    "d128_m20": (128, 20, FAST, ("lbfgs_rosenbrock_m", "double, 128, 20"), 2, 6),
    "d128_m10_eigen": (128, 10, EIGEN, ("lbfgs_rosenbrock_d128_eigen", ""), 2, 12),
}
CONTROL_KERNELS = {
    "d37_m5": (37, 5, FAST, ("lbfgs_rosenbrock_m", "double, 37, 5"), 0, 16),
    "d128_m5": (128, 5, FAST, ("lbfgs_rosenbrock_m", "double, 128, 5"), 0, 20),
}


def zero_tolerance_stop(iterations):
    s = ob.default_stop()
    s.num_iterations = iterations
    s.x_delta = s.f_delta = s.gradient_norm = 0.0
    s.past = 0
    return s


def near_minimiser(d, rows, scale=1e-12):
    """x* + 1e-12 noise: the steps shrink to the rounding level, so s.y falls below eps (skipped pairs, at k < m and
    at k = m, in every position) and the curvature test refuses pairs while the history is full.  With 1e-6 noise
    the first pairs are usable and the later ones are not, so the history holds both kinds at once."""
    return (1.0 + scale * ob.fill_uniform((2, d), 0, 24, -1.0, 1.0))[rows]


def spikes(d, picks):
    """[-2, 2] starts with every `stride`-th coordinate scaled by 10^e: the first step is accepted, and the second
    fails the descent test, so the fallback empties a history that holds one pair, in a register slot."""
    rows = []
    for e, stride, row in picks:
        x = ob.fill_uniform((8, d), 0, 21, -2.0, 2.0)
        x[:, ::stride] *= 10.0 ** e
        rows.append(x[row])
    return np.array(rows)


SPIKES = {37: [(11.5, 4, 0), (12.0, 1, 6), (17.5, 37, 2)], 128: [(11.5, 16, 5), (13.5, 16, 0)]}

# (kernel, kind) -> (x0, stop, claims).  Claims: "skip_warmup" / "skip_full" = skipped pairs at k < m / k = m in each
# position from the newest pair (0, 1, >= 2); "rejected" = refused pairs with a non-empty history; "fallback_reg" =
# a fallback while every pair of the history was in registers (1 <= k <= R; k = 1 when R = 0); "fallback_0" /
# "nonfinite_0" = a fallback / a non-finite trial value with an empty history (k = 0).
NEAR = ("skip_warmup", "skip_full", "rejected")
NEAR_ROWS = {"d128_m10": ([1], 150), "d37_m20": ([0], 120), "d128_m20": ([1], 120), "d128_m10_eigen": ([1], 150)}


def case(kernel, kind):
    """(x0, stop, claims) of the near-minimiser or spike starts of a kernel's d (rows and lengths chosen for the
    kernels with register pairs; the controls reuse those of the same d)."""
    d = (REGISTER_KERNELS | CONTROL_KERNELS)[kernel][0]
    if kind == "near":
        rows, iterations = NEAR_ROWS.get(kernel, NEAR_ROWS["d128_m10" if d == 128 else "d37_m20"])
        return near_minimiser(d, rows), zero_tolerance_stop(iterations), NEAR
    if kind == "mixed":
        return near_minimiser(d, [0], 1e-6), zero_tolerance_stop(60), ("skip_full",)
    return spikes(d, SPIKES[d]), ob.default_stop(), ("fallback_reg",)


KINDS = ("near", "mixed", "spikes")
CASES = [(k, kind) for k in REGISTER_KERNELS for kind in KINDS]
CASE_IDS = [f"{k}-{kind}" for k, kind in CASES]


def assert_reached(paths, regs, claims):
    """Every claim holds for the batch as a whole (the counts of all rows added up); regs = the kernel's register
    pairs R."""
    sk = paths["skipped"].sum(0)
    for c in claims:
        if c == "skip_warmup":
            assert (sk[0] > 0).all(), ("skipped pairs at k < m by position", sk[0])
        elif c == "skip_full":
            assert (sk[1] > 0).all(), ("skipped pairs at k = m by position", sk[1])
        elif c == "rejected":
            assert paths["rejected"].sum() > 0, "no pair refused with a non-empty history"
        elif c == "fallback_reg":
            fb = paths["fallback"].sum(0)
            assert fb[1:max(regs, 1) + 1].sum() > 0, ("fallbacks by mem_count", fb)
        elif c == "fallback_0":
            assert paths["fallback"].sum(0)[0] > 0, ("fallbacks by mem_count", paths["fallback"].sum(0))
        elif c == "nonfinite_0":
            assert paths["nonfinite"].sum(0)[0] > 0, ("non-finite trials by mem_count", paths["nonfinite"].sum(0))
        else:
            raise AssertionError(c)


def bitwise_equal(a, b):
    for k in KEYS:
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


# ---------------------------------------------------------------- the plan table (CPU) ----

PLAN_OF = {  # launcher template of cno_api.cu's kTable -> the LbfgsPlan of the kernel it launches
    "lbfgs_rosenbrock": "LbfgsPlan<RosenbrockFn<{0}, {1}>, CNO_LBFGS_M>",
    "lbfgs_rosenbrock_m": "LbfgsPlan<RosenbrockFn<{0}, {1}>, {2}>",
    "lbfgs_rosenbrock_second": "LbfgsPlan<SecondMode<RosenbrockFn<{0}, {1}>>, CNO_LBFGS_M>",
    "lbfgs_rosenbrock_steps": "LbfgsPlan<RosenbrockFn<{0}, {1}>, CNO_LBFGS_M, true>",
    "lbfgs_rosenbrock_hz": "LbfgsPlan<RosenbrockFn<{0}, {1}>, CNO_LBFGS_M, false, LsHagerZhang>",
    "lbfgs_rosenbrock_d128_eigen": "LbfgsPlan<RosenbrockFn<double, 128, PolicyEigenSSE2>, CNO_LBFGS_M>",
}


@pytest.fixture(scope="module")
def plan_table(tmp_path_factory):
    """(launcher, template arguments) -> (kRegPairs, SM::kWarps, m) for every L-BFGS Rosenbrock launcher of the
    dispatch table, from a host-only program compiled against the kernel headers."""
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    src = open(os.path.join(CSRC, "cno_api.cu")).read()
    table = src[src.index("const Entry kTable[] = {"):]
    table = table[:table.index("\n};")]
    launchers = sorted(set(re.findall(r"\b(lbfgs_rosenbrock\w*)(?:<([^>]*)>)?", table)))
    assert len(launchers) > 10
    lines = []
    for name, args in launchers:
        assert name in PLAN_OF, f"an L-BFGS launcher this test does not know: {name}"
        a = [s.strip() for s in args.split(",")] if args else []
        plan = PLAN_OF[name].format(*a)
        m = a[2] if name == "lbfgs_rosenbrock_m" else "CNO_LBFGS_M"
        lines.append(f'  printf("%s|%s|%d|%d|%d\\n", "{name}", "{args}", {plan}::kRegPairs, {plan}::SM::kWarps, {m});')
    tmp = tmp_path_factory.mktemp("plan")
    prog = tmp / "plan.cu"
    prog.write_text('#include <cstdio>\n#include "cno_functors.cuh"\n#include "cno_lbfgs.cuh"\nusing namespace cno;\n'
                    "int main() {\n" + "\n".join(lines) + "\n}\n")
    exe = tmp / "plan"
    subprocess.run([NVCC, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC,
                    "-I", os.path.join(HERE, "..", "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    rows = {}
    for line in out.splitlines():
        name, args, r, w, m = line.split("|")
        rows[(name, args)] = (int(r), int(w), int(m))
    return rows


def test_register_pairs_only_in_the_kernels_this_file_covers(plan_table):
    """The plans with register pairs are exactly those of REGISTER_KERNELS, at their warp counts, and each has a
    near-minimiser and a spike case here: a plan change that moves a register pair into another kernel fails."""
    with_pairs = {launcher: (r, w) for launcher, (r, w, _) in plan_table.items() if r > 0}
    assert with_pairs == {k[3]: (k[4], k[5]) for k in REGISTER_KERNELS.values()}
    assert {k for k, _ in CASES} == set(REGISTER_KERNELS)
    for d, m, _, launcher, r, w in (REGISTER_KERNELS | CONTROL_KERNELS).values():
        assert plan_table[launcher] == (r, w, m), launcher


# ---------------------------------------------------------------- proof of reach (CPU) ----

@pytest.mark.parametrize("kernel,kind", CASES, ids=CASE_IDS)
def test_case_reaches_its_paths(kernel, kind):
    d, m, policy, _, regs, _ = REGISTER_KERNELS[kernel]
    x0, stop, claims = case(kernel, kind)
    _, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop, lbfgs_m=m, policy=policy)
    assert_reached(paths, regs, claims)


# ---------------------------------------------------------------- emulation (CPU) ----

@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    return C.CDLL(os.path.join(EMU_DIR, "libcno_emu.so"))


def _emulated(emu, x0, stop, m, policy):
    B, d = x0.shape
    prob = ob.Problem(ob.FN_ROSENBROCK, ob._np_dtype(x0), d, 0, 0.0, None, 0, policy, 0, m)
    r, out = ob._batch_out(x0)
    assert emu.emu_minimize(ob.LBFGS, 0, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                            C.byref(out)) == 0
    return r


@pytest.mark.parametrize("kernel,kind", CASES, ids=CASE_IDS)
def test_emulated_kernel_equals_oracle(emu, kernel, kind):
    """lbfgs_minimize_kernel<RosenbrockFn<double, d, policy>, m> under the warp emulation: every output bit for
    bit."""
    d, m, policy, _, regs, _ = REGISTER_KERNELS[kernel]
    x0, stop, claims = case(kernel, kind)
    o, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop, lbfgs_m=m, policy=policy)
    assert_reached(paths, regs, claims)
    bitwise_equal(_emulated(emu, x0, stop, m if m != 10 else 0, policy), o)


def test_emulation_rejects_an_uncompiled_m(emu):
    x0 = ob.fill_uniform((1, 37), 0, 1, -2.0, 2.0)
    prob = ob.Problem(ob.FN_ROSENBROCK, 0, 37, 0, 0.0, None, 0, FAST, 0, 7)
    _, out = ob._batch_out(x0)
    stop = ob.default_stop()
    assert emu.emu_minimize(ob.LBFGS, 0, C.byref(prob), C.c_longlong(1), C.c_void_p(x0.ctypes.data), C.byref(stop),
                            C.byref(out)) != 0


# ---------------------------------------------------------------- the oracle against the reference (CPU) ----

@pytest.mark.parametrize("kernel,kind", CASES, ids=CASE_IDS)
def test_oracle_equals_reference_lbfgs(kernel, kind):
    """The oracle's skip, refusal and fallback semantics against the reference's own lbfgs.h on the Eigen-API
    shim."""
    if not ob.ref_available():
        pytest.skip("oracle/_ref not built")
    _, m, policy, *_ = REGISTER_KERNELS[kernel]
    x0, stop, _ = case(kernel, kind)
    bitwise_equal(ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop, lbfgs_m=m, policy=policy, impl="ref"),
                  ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop, lbfgs_m=m, policy=policy))


# ---------------------------------------------------------------- the GPU ----

def _interleaved(d, warps, rare, seed):
    """3 * SMs * warps + 5 rows: every 7th row a rare start, the others ordinary [-2, 2] starts, so that rare
    instances share CTAs with ordinary ones and every warp drains several instances."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 3 * sms * warps + 5
    x0 = ob.fill_uniform((B, d), 0, seed, -2.0, 2.0)
    rows = np.arange(3, B, 7)
    x0[rows] = rare[np.arange(len(rows)) % len(rare)]
    return x0, rows


def _gpu(x0, stop, m, policy=FAST, every=0):
    import torch

    import cppnumericalsolvers_b200 as cn
    solver = cn.Lbfgs(cn.Progress.from_c(stop), m=m)
    if every:
        solver.SetCallback(lambda *_: None, every=every)
    fn = cn.Rosenbrock(x0.shape[1])
    fn.policy = policy
    st, pr = solver.Minimize(fn, cn.BatchedFunctionState(torch.from_numpy(x0).to("cuda:0")), timed=not every)
    torch.cuda.synchronize()
    g = dict(x=st.x.cpu().numpy(), value=st.value.cpu().numpy(), gradient=st.gradient.cpu().numpy(),
             num_iterations=pr.num_iterations.cpu().numpy().astype(np.uint32), status=pr.status.cpu().numpy(),
             nfev=pr.nfev.cpu().numpy().astype(np.uint32), x_delta=pr.x_delta.cpu().numpy(),
             f_delta=pr.f_delta.cpu().numpy(), gradient_norm=pr.gradient_norm.cpu().numpy())
    return g, pr.launch


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("kernel", list(REGISTER_KERNELS | CONTROL_KERNELS))
def test_gpu_equals_oracle_on_rare_path_starts(kernel, kind):
    """Each kernel with register pairs, and the m = 5 kernel of the same d, on the rare-path starts of its d mixed
    into a full batch: every output bit for bit against the oracle."""
    d, m, policy, _, regs, warps = (REGISTER_KERNELS | CONTROL_KERNELS)[kernel]
    rare, stop, claims = case(kernel, kind)
    x0, rows = _interleaved(d, warps, rare, 7000 + d + m)
    o, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop, lbfgs_m=m, policy=policy)
    assert_reached({k: v[rows] for k, v in paths.items()}, regs, claims)
    g, launch = _gpu(x0, stop, m, policy)
    assert launch.warps_per_cta == warps
    bitwise_equal(g, o)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_stepwise_kernel_equals_register_pair_kernel(kind):
    """d = 128, m = 10: cno_minimize_steps (whole history in shared memory) against the one-shot kernel (one pair in
    registers), device against device, on the same starts."""
    rare, stop, _ = case("d128_m10", kind)
    x0, _ = _interleaved(128, 12, rare, 7100)
    one_shot, launch = _gpu(x0, stop, 10)
    assert launch.warps_per_cta == 12
    stepwise, _ = _gpu(x0, stop, 10, every=40)
    bitwise_equal(stepwise, one_shot)
