"""The rare branches of the group L-BFGS kernel (csrc/cno_lbfgs_group.cuh, d = 256 .. 1024), the only solver at d = 512
and 1024: the `valid` mask that skips a pair (|s.y| < eps) in both loops of the two-loop recursion and its shift once
the history is full, pairs refused by the curvature test, the -g fallback that empties the history, the untouched
state of a search along a direction with dginit >= 0, and the non-finite trial value.  Ordinary starts reach none of
them.  Each case below first shows from the oracle's path counts (oracle_binding.lbfgs_paths) that it reaches the
branches it claims; then the oracle must equal the reference's own lbfgs.h (oracle/_ref), the device source under the
CPU warp emulation must equal the oracle, and on the GPU every case is mixed into a full batch of ordinary starts, so a
group on a rare path shares its CTA (two groups per CTA at d = 512) with groups that are not, and must equal the oracle
and the one-warp kernel (tests/cpp/one_warp_rosenbrock.cu) bit for bit.  Random Progress settings run through the same
kernel, whose W warps each keep their own copy of the past-f ring.

Not covered: a fallback with two or more stored pairs, and a non-finite trial value with pairs stored.  No start found
reaches either at d = 512 or 1024 (spikes of 10^11 .. 10^150 at strides 1 .. d / 2, and starts 1e-14 .. 1e-4 off the
minimiser, up to 1500 iterations).

The CPU part costs about four minutes serial, most of it in the emulated near-minimiser runs, the queue of rare
starts and the Progress sweep."""
import numpy as np
import pytest

from oracle import oracle_binding as ob
from test_lbfgs_group import _emulated, bitwise_equal, build_emu_group
from test_lbfgs_rare_paths import assert_reached, near_minimiser, spikes, zero_tolerance_stop

DS = (256, 512, 1024)
GPU_DS = (512, 1024)
GROUPS = {512: 2, 1024: 1}  # groups (resident instances) per CTA
MAX_PAST = 8                # CNO_MAX_PAST: the past-f ring of each warp

# kind -> {d: (e, stride, row)} of test_lbfgs_rare_paths.spikes: [-2, 2] starts with every stride-th coordinate scaled
# by 10^e.  "fallback_1": the first step is accepted and the second fails the descent test, so the fallback empties a
# history of one pair; "fallback_0": the first direction already fails it; "nonfinite_0": the first trial value
# overflows to inf.
SPIKES = {
    "fallback_1": {256: (12.0, 1, 6), 512: (11.5, 1, 5), 1024: (11.5, 64, 2)},
    "fallback_0": {256: (60.0, 1, 0), 512: (30.0, 256, 7), 1024: (60.0, 1, 0)},
    "nonfinite_0": {256: (30.0, 1, 0), 512: (30.0, 1, 0), 1024: (30.0, 1, 0)},
}
NEAR = ("skip_warmup", "skip_full", "rejected")
KINDS = ("near", "mixed", "fallback_1", "fallback_0", "nonfinite_0", "nan", "minimiser")
# claims as in test_lbfgs_rare_paths.assert_reached, called with no register pairs (R = 0), so "fallback_reg" is a
# fallback with exactly one stored pair
CLAIMS = {"near": NEAR, "mixed": ("skip_full",), "fallback_1": ("fallback_reg",), "fallback_0": ("fallback_0",),
          "nonfinite_0": ("nonfinite_0",), "nan": ("fallback_0", "nonfinite_0"), "minimiser": ("fallback_0",)}


def case(d, kind):
    """(x0, stop, claims) of a rare-path start at d.  "near": two rows 1e-12 off x* under a stop that only ends at 150
    iterations (skipped pairs at k < m and k = m in every position, refused pairs); "mixed": 1e-6 off x*, 60
    iterations (usable and skipped pairs in one full history); "nan": a NaN coordinate, 5 iterations; "minimiser":
    x = 1, where g = 0, the fallback's +g search has dginit = 0 and the state stays untouched."""
    if kind == "near":
        return near_minimiser(d, [0, 1]), zero_tolerance_stop(150), NEAR
    if kind == "mixed":
        return near_minimiser(d, [0], 1e-6), zero_tolerance_stop(60), CLAIMS[kind]
    if kind in SPIKES:
        return spikes(d, [SPIKES[kind][d]]), ob.default_stop(), CLAIMS[kind]
    if kind == "nan":
        x = ob.fill_uniform((1, d), 0, 4, -2.0, 2.0)
        x[0, d // 3] = np.nan
        stop = ob.default_stop()
        stop.num_iterations = 5
        return x, stop, CLAIMS[kind]
    if kind == "minimiser":
        return np.ones((1, d)), ob.default_stop(), CLAIMS[kind]
    raise AssertionError(kind)


def assert_case_reached(kind, o, paths):
    """The claims of `kind` from the path counts of its rows (o, paths: lbfgs_paths of those rows only)."""
    assert_reached(paths, 0, CLAIMS[kind])
    if kind == "minimiser":  # no trial at all: the search along +g returned the state untouched
        assert (o["nfev"] == 1).all() and (o["num_iterations"] == 1).all(), (o["nfev"], o["num_iterations"])


CASES = [(d, kind) for d in DS for kind in KINDS]


def _ids(cases):
    return [f"d{d}-{kind}" for d, kind in cases]


# ---------------------------------------------------------------- proof of reach (CPU) ----

@pytest.mark.parametrize("d,kind", CASES, ids=_ids(CASES))
def test_case_reaches_its_paths(d, kind):
    x0, stop, _ = case(d, kind)
    o, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop)
    assert_case_reached(kind, o, paths)


# ---------------------------------------------------------------- the oracle against the reference (CPU) ----

REF_CASES = [(d, kind) for d in GPU_DS for kind in KINDS]


@pytest.mark.parametrize("d,kind", REF_CASES, ids=_ids(REF_CASES))
def test_oracle_equals_reference_lbfgs(d, kind):
    """The oracle's skip, refusal, fallback and non-finite semantics against the reference's own lbfgs.h /
    more_thuente.h on the Eigen-API shim."""
    if not ob.ref_available():
        pytest.skip("oracle/_ref not built")
    x0, stop, _ = case(d, kind)
    bitwise_equal(ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop, impl="ref"),
                  ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop))


# ---------------------------------------------------------------- emulation (CPU) ----

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emu_group(tmp_path_factory.mktemp("emu_group_rare"))


# d -> (rows, iterations, claims) of the near case under the emulation, which costs about 0.1 s per iteration and row
# at d = 256 and 0.7 s at d = 1024: the rows that refuse a pair at d = 256 and 512; at d = 1024 one row for 40
# iterations (skipped pairs in every position, no refusal; refusals are left to the GPU and reference tests).
EMU_NEAR = {256: ([0], 150, NEAR), 512: ([1], 150, NEAR), 1024: ([0], 40, ("skip_warmup", "skip_full"))}
EMU_CASES = [(d, kind) for d in DS for kind in KINDS if kind != "mixed" or d != 1024]


@pytest.mark.parametrize("d,kind", EMU_CASES, ids=_ids(EMU_CASES))
def test_emulated_group_kernel_equals_oracle(emu, d, kind):
    """lbfgs_group_minimize_kernel<GroupRosenbrockFn<double, d>, 10> under the warp emulation (one group of d / 128
    warps): every output bit for bit."""
    x0, stop, claims = case(d, kind)
    if kind == "near":
        rows, iterations, claims = EMU_NEAR[d]
        x0, stop = x0[rows], zero_tolerance_stop(iterations)
    x0 = np.ascontiguousarray(x0)
    o, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop)
    assert_reached(paths, 0, claims)
    bitwise_equal(_emulated(emu, x0, stop), o)


def queue_stop():
    """Zero tolerances and 25 iterations, except that a step of exactly zero ends the run: the rows that sit still
    after a fallback or a refused step stop at once, while the near row keeps storing pairs for 26 iterations, so its
    history is full and has wrapped round when it ends."""
    s = zero_tolerance_stop(25)
    s.x_delta = 5e-324
    return s


def _queue(d):
    """The near row, then fallback with one pair, non-finite trial, NaN coordinate, x = 1 and an ordinary start."""
    return np.concatenate([case(d, "near")[0][1:], *[case(d, k)[0] for k in
                                                      ("fallback_1", "nonfinite_0", "nan", "minimiser")],
                           ob.fill_uniform((1, d), 0, 1, -2.0, 2.0)])


@pytest.mark.parametrize("order", ("forward", "reversed"))
def test_one_group_drains_a_queue_of_rare_starts(emu, order):
    """d = 512: one group solves the rare starts one after another, so each instance finds the S, Y, rho, alpha,
    past-f ring and exchange block of the one before it in the group's shared memory; every row must equal the oracle,
    which starts each instance afresh."""
    x0 = _queue(512)
    if order == "reversed":
        x0 = x0[::-1]
    x0 = np.ascontiguousarray(x0)
    stop = queue_stop()
    o, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0, stop=stop)
    near = 0 if order == "forward" else len(x0) - 1
    assert_reached({k: v[near:near + 1] for k, v in paths.items()}, 0, ("skip_full",))
    assert o["num_iterations"][near] == 26 and paths["rejected"][near] == 0
    assert_reached(paths, 0, ("fallback_reg", "nonfinite_0", "fallback_0"))
    bitwise_equal(_emulated(emu, x0, stop), o)


def random_stops(rng, n):
    """n Progress settings drawn like test_oracle_pins._random_stop, iteration limits capped at 40 so that the oracle
    can check every row of a full batch; the first has past = CNO_MAX_PAST, so each warp's ring fills its slot."""
    stops = []
    for k in range(n):
        s = ob.default_stop()
        s.num_iterations = int(rng.choice([3, 7, 25, 40]))
        s.x_delta = float(rng.choice([0.0, 1e-9, 1e-4, 1e-2]))
        s.x_delta_violations = int(rng.integers(1, 4))
        s.f_delta = float(rng.choice([0.0, 0.0, 1e-8, 1e-3, 1e-1]))
        s.f_delta_violations = int(rng.integers(1, 4))
        s.f_delta_relative = int(rng.integers(0, 2))
        s.gradient_norm = float(rng.choice([0.0, 1e-5, 1e-2, 1.0]))
        s.gradient_norm_relative = int(rng.integers(0, 2))
        s.past = MAX_PAST if k == 0 else int(rng.integers(0, MAX_PAST + 1))
        s.past_delta = float(rng.choice([1e-10, 1e-6, 1e-2]))
        stops.append(s)
    return stops


def test_emulated_group_kernel_follows_progress_update_under_random_settings(emu):
    """d = 512: progress_update with the group's W per-warp rings, six random settings of two rows each: every output
    bit for bit against the oracle, and the sweep ends in at least three different statuses."""
    seen = set()
    for k, stop in enumerate(random_stops(np.random.default_rng(512), 6)):
        x0 = ob.fill_uniform((2, 512), 31 * k, 808, -2.0, 2.0)
        o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop)
        bitwise_equal(_emulated(emu, x0, stop), o)
        seen.update(o["status"].tolist())
    assert len(seen) >= 3, seen


# ---------------------------------------------------------------- the GPU ----

def _interleaved(d, rare, seed):
    """3 * SMs * groups + 5 rows: every 7th row a rare start, the others ordinary [-2, 2] starts."""
    import test_lbfgs_group_gpu as gg
    B = 3 * gg.sms() * GROUPS[d] + 5
    x0 = ob.fill_uniform((B, d), 0, seed, -2.0, 2.0)
    rows = np.arange(3, B, 7)
    x0[rows] = rare[np.arange(len(rows)) % len(rare)]
    return x0, rows


@pytest.fixture(scope="module")
def one_warp(tmp_path_factory):
    import test_lbfgs_group_gpu as gg
    return gg.build_one_warp(tmp_path_factory.mktemp("one_warp_rare"))


GPU_CASES = [(d, kind) for d in GPU_DS for kind in KINDS]


@pytest.mark.gpu
@pytest.mark.parametrize("d,kind", GPU_CASES, ids=_ids(GPU_CASES))
def test_gpu_mixed_batch_equals_oracle_and_one_warp_kernel(one_warp, d, kind):
    """A rare-path case mixed into a full batch: the rare rows reach their claims; the group kernel equals the oracle
    on every row when the stop caps the iterations (near, mixed, nan) and otherwise on the rare rows and a strided
    sample of the others; and it equals the one-warp kernel on every row."""
    import test_lbfgs_group_gpu as gg
    rare, stop, _ = case(d, kind)
    x0, rows = _interleaved(d, rare, 7300 + d + KINDS.index(kind))
    g, info = gg.minimize_c(x0, stop)
    assert info.warps_per_cta == GROUPS[d]
    check = np.arange(len(x0)) if stop.num_iterations <= 150 else np.union1d(rows, gg.sample(len(x0)))
    o, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0[check], stop=stop)
    is_rare = np.isin(check, rows)
    assert_case_reached(kind, {k: v[is_rare] for k, v in o.items() if k != "seconds"},
                        {k: v[is_rare] for k, v in paths.items()})
    gg.bitwise_equal({k: v[check] for k, v in g.items()}, o)
    gg.bitwise_equal(gg.minimize_one_warp(one_warp, x0, stop), g)


@pytest.mark.gpu
@pytest.mark.parametrize("d", GPU_DS)
def test_gpu_follows_progress_update_under_random_settings(d):
    """Twelve random Progress settings on full batches of ordinary starts with the fallback, non-finite, NaN and x = 1
    starts mixed in: every row bit for bit against the oracle, and the sweep ends in at least three statuses."""
    import test_lbfgs_group_gpu as gg
    rare = np.concatenate([case(d, k)[0] for k in ("fallback_1", "fallback_0", "nonfinite_0", "nan", "minimiser")])
    seen = set()
    for k, stop in enumerate(random_stops(np.random.default_rng(d), 12)):
        x0, _ = _interleaved(d, rare, 7400 + 31 * k)
        g, info = gg.minimize_c(x0, stop)
        assert info.warps_per_cta == GROUPS[d]
        o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop)
        gg.bitwise_equal(g, o)
        seen.update(o["status"].tolist())
    assert len(seen) >= 3, seen
