"""Lbfgs on Rosenbrock fp64 at d = 512 and 1024 on the GPU (csrc/cno_lbfgs_group.cuh: one group of d / 128 warps per
instance): every output bit for bit against the CPU oracle, the committed fixtures, per-group isolation in a full
batch, the stop and sentinel behaviour of the C ABI, the launch shape, the Python / MinimizeHost / C++ mirror paths,
and the one-warp kernel on the same objective as a user functor."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import cppnumericalsolvers_b200 as cn
from cppnumericalsolvers_b200 import _lib
from oracle import oracle_binding as ob

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
DEV = "cuda:0"
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
DS = (512, 1024)
GROUPS = {512: 2, 1024: 1}           # resident instances (groups) per CTA
THREADS = {512: 256, 1024: 256}      # block
SMEM = {512: 186144, 1024: 186128}   # dynamic shared memory per CTA
SENTINEL = 0x5A


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _outputs(B, d, rows=None):
    """Device output arrays of `rows` (>= B) rows filled with the sentinel byte."""
    rows = B if rows is None else rows
    t = dict(x=torch.empty(rows, d, dtype=torch.float64, device=DEV), value=torch.empty(rows, dtype=torch.float64, device=DEV),
             gradient=torch.empty(rows, d, dtype=torch.float64, device=DEV),
             num_iterations=torch.empty(rows, dtype=torch.int32, device=DEV),
             status=torch.empty(rows, dtype=torch.int8, device=DEV), nfev=torch.empty(rows, dtype=torch.int32, device=DEV),
             x_delta=torch.empty(rows, dtype=torch.float64, device=DEV),
             f_delta=torch.empty(rows, dtype=torch.float64, device=DEV),
             gradient_norm=torch.empty(rows, dtype=torch.float64, device=DEV))
    for v in t.values():
        v.view(torch.uint8).fill_(SENTINEL)
    return t


def _host(t):
    r = {k: v.cpu().numpy() for k, v in t.items()}
    r["num_iterations"] = r["num_iterations"].astype(np.uint32)
    r["nfev"] = r["nfev"].astype(np.uint32)
    return r


def minimize_c(x0, stop=None, skip=(), rows=None):
    """cno_minimize on the built-in family; outputs named in `skip` are not requested (NULL)."""
    B, d = x0.shape
    xd = torch.from_numpy(np.ascontiguousarray(x0)).to(DEV)
    t = _outputs(B, d, rows)
    out = _lib.BatchOut(*[0 if k in skip else t[k].data_ptr() for k in
                          ("x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta",
                           "gradient_norm")])
    prob = _lib.Problem(family=0, dtype=_lib.F64, d=d, policy=_lib.POLICY_DMMA_TREE)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    info = _lib.LaunchInfo()
    s = (stop if stop is not None else ob.default_stop())
    sp = C.cast(C.pointer(s), C.POINTER(_lib.Stop))
    _lib.check(_lib.lib().cno_minimize(_lib.LBFGS, C.byref(prob), B, xd.data_ptr(), sp, C.byref(out), ws.data_ptr(),
                                       ws.numel(), torch.cuda.current_stream().cuda_stream, C.byref(info)),
               "cno_minimize")
    torch.cuda.synchronize()
    return _host(t), info


def bitwise_equal(a, b, rows=slice(None)):
    for k in KEYS:
        assert np.array_equal(np.asarray(a[k])[rows].view(np.uint8), np.asarray(b[k])[rows].view(np.uint8)), k


def sample(B):
    """A strided sample of at most 64 rows (the oracle costs up to a second per instance at d = 1024)."""
    return np.unique(np.linspace(0, B - 1, min(B, 64)).astype(int))


@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("which", ("1", "7", "full"))
def test_gpu_equals_oracle(d, which):
    B = {"1": 1, "7": 7, "full": 3 * sms() * GROUPS[d] + 5}[which]
    x0 = ob.fill_uniform((B, d), 0, 100 + d, -2.0, 2.0)
    g, _ = minimize_c(x0)
    rows = sample(B)
    bitwise_equal({k: v[rows] for k, v in g.items()}, ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0[rows]))


@pytest.mark.parametrize("d", DS)
def test_gpu_reproduces_fixture(d):
    z = np.load(os.path.join(GOLDEN, f"lbfgs_rosenbrock_d{d}_f64.npz"))
    g, _ = minimize_c(z["x0"])
    bitwise_equal(g, {k: z[k] for k in KEYS})


@pytest.mark.parametrize("d", DS)
def test_groups_are_isolated(d):
    """Each rare-path case of test_lbfgs_group_rare_paths (skipped and refused pairs; usable and skipped pairs in one
    history; the fallback with one pair and with none; a non-finite trial; a NaN coordinate; x = 1), which first
    proves from the oracle's path counts that it reaches its branches, mixed into a batch of 3 * SMs * groups + 5
    ordinary rows under the case's own stop: the rare rows equal the same starts solved alone, and the oracle."""
    from test_lbfgs_group_rare_paths import KINDS, assert_case_reached, case
    for kind in KINDS:
        rare, stop, _ = case(d, kind)
        B = 3 * sms() * GROUPS[d] + 5
        x0 = ob.fill_uniform((B, d), 0, 300 + d, -2.0, 2.0)
        rows = np.arange(2, B, 11)
        x0[rows] = rare[np.arange(len(rows)) % len(rare)]
        g, _ = minimize_c(x0, stop)
        for r in rows[:2 * len(rare)]:
            alone, _ = minimize_c(x0[r:r + 1], stop)
            bitwise_equal({k: v[r:r + 1] for k, v in g.items()}, alone)
        o, paths = ob.lbfgs_paths(ob.FN_ROSENBROCK, x0[rows[:len(rare)]], stop=stop)
        assert_case_reached(kind, o, paths)
        bitwise_equal({k: v[rows[:len(rare)]] for k, v in g.items()}, o)


@pytest.mark.parametrize("d", DS)
def test_iteration_limit(d):
    stop = ob.default_stop()
    stop.num_iterations = 5
    x0 = ob.fill_uniform((9, d), 0, 7, -2.0, 2.0)
    g, _ = minimize_c(x0, stop)
    assert (g["status"] == 1).all() and (g["num_iterations"] == 6).all()  # CNO_STATUS_ITERATION_LIMIT
    bitwise_equal(g, ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop))


@pytest.mark.parametrize("d", DS)
def test_rows_past_batch_and_unrequested_outputs_keep_their_sentinel(d):
    B = 5
    x0 = ob.fill_uniform((B, d), 0, 8, -2.0, 2.0)
    skip = ("gradient", "nfev", "f_delta")
    g, _ = minimize_c(x0, skip=skip, rows=B + 3)
    for k, v in g.items():
        raw = np.asarray(v).view(np.uint8).reshape(B + 3, -1)
        assert (raw[B:] == SENTINEL).all(), k
        if k in skip:
            assert (raw == SENTINEL).all(), k
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0)
    for k in KEYS:
        if k not in skip:
            assert np.array_equal(np.asarray(g[k])[:B].view(np.uint8), np.asarray(o[k]).view(np.uint8)), k


@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("B", (1, 37, 4096))
def test_launch_shape(d, B):
    stop = ob.default_stop()
    stop.num_iterations = 3
    _, info = minimize_c(ob.fill_uniform((B, d), 0, 9, -2.0, 2.0), stop)
    assert info.kernel_launches == 1
    assert (info.block, info.warps_per_cta, info.dynamic_smem) == (THREADS[d], GROUPS[d], SMEM[d])
    assert info.grid == min(-(-B // GROUPS[d]), sms())


@pytest.mark.parametrize("d", DS)
def test_python_and_host_paths(d):
    x0 = ob.fill_uniform((6, d), 0, 10, -2.0, 2.0)
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0)
    solver = cn.Lbfgs()
    st, pr = solver.Minimize(cn.Rosenbrock(d), cn.BatchedFunctionState(torch.from_numpy(x0).to(DEV)))
    torch.cuda.synchronize()
    assert np.array_equal(st.x.cpu().numpy().view(np.uint64), o["x"].view(np.uint64))
    assert np.array_equal(pr.num_iterations.cpu().numpy().astype(np.uint32), o["num_iterations"])
    hs, hp = cn.Lbfgs().MinimizeHost(cn.Rosenbrock(d), torch.from_numpy(x0))
    assert np.array_equal(hs.x.numpy().view(np.uint64), o["x"].view(np.uint64))
    assert np.array_equal(hs.value.numpy().view(np.uint64), o["value"].view(np.uint64))
    assert np.array_equal(hp.nfev.numpy().astype(np.uint32), o["nfev"])
    cb = cn.Lbfgs()
    cb.SetCallback(lambda *_: None, every=5)
    with pytest.raises(_lib.CnoError):
        cb.Minimize(cn.Rosenbrock(d), cn.BatchedFunctionState(torch.from_numpy(x0).to(DEV)))


def test_cpp_mirror_at_d1024(tmp_path):
    """cppoptlib::solver::Lbfgs<cppoptlib::function::Rosenbrock<double, 1024>> from a plain g++ translation unit."""
    src = tmp_path / "mirror.cc"
    src.write_text(r'''
#include <cstdio>
#include <vector>
#include "cppoptlib_b200/cppoptlib.h"
int main() {
  using F = cppoptlib::function::Rosenbrock<double, 1024>;
  cppoptlib::solver::Lbfgs<F> solver;
  const int B = 3;
  std::vector<double> x0(B * 1024);
  for (size_t i = 0; i < x0.size(); ++i) x0[i] = (i % 7) * 0.25 - 0.75;
  auto [state, progress] = solver.Minimize(F{}, cppoptlib::function::BatchedFunctionState<double, 1024>::FromHost(x0, B));
  const std::vector<int8_t> st = progress.status.ToHost();
  const std::vector<uint32_t> it = progress.num_iterations.ToHost();
  const std::vector<double> f = state.value.ToHost();
  for (int b = 0; b < B; ++b) std::printf("%d %d %.17g\n", (int)st[b], (int)it[b], f[b]);
  return 0;
}
''')
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib = os.path.join(ROOT, "cppnumericalsolvers_b200")
    exe = tmp_path / "mirror"
    r = subprocess.run(["g++", "-std=c++17", "-O2", str(src), "-I" + os.path.join(ROOT, "include"), f"-I{cuda}/include",
                        "-o", str(exe), f"-L{lib}", "-lcno", f"-L{cuda}/lib64", "-lcudart", f"-Wl,-rpath,{lib}",
                        f"-Wl,-rpath,{cuda}/lib64"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail(r.stderr[-3000:])
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300, check=True)
    x0 = np.array([(i % 7) * 0.25 - 0.75 for i in range(3 * 1024)]).reshape(3, 1024)
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0)
    got = [line.split() for line in run.stdout.splitlines()]
    assert [(int(s), int(i)) for s, i, _ in got] == list(zip(o["status"].tolist(), o["num_iterations"].tolist()))
    assert [float(v) for _, _, v in got] == o["value"].tolist()


def build_one_warp(out_dir):
    """tests/cpp/one_warp_rosenbrock.cu compiled into `out_dir`: the one-warp kernel on the same objective as a user
    functor."""
    out = os.path.join(str(out_dir), "libcno_one_warp.so")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib = os.path.join(ROOT, "cppnumericalsolvers_b200")
    subprocess.run([os.environ.get("NVCC", f"{cuda}/bin/nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3",
                    "-std=c++17", "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false", "-shared",
                    "-Xcompiler", "-fPIC", os.path.join(HERE, "cpp", "one_warp_rosenbrock.cu"),
                    "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(lib, "csrc"), "-o", out,
                    f"-L{lib}", "-lcno", "-Xlinker", f"-rpath={lib}"], check=True)
    _lib.lib()
    return C.CDLL(out)


@pytest.fixture(scope="module")
def one_warp(tmp_path_factory):
    return build_one_warp(tmp_path_factory.mktemp("one_warp"))


def minimize_one_warp(one_warp, x0, stop=None):
    """cno_one_warp_rosenbrock_minimize on x0 -> host outputs."""
    B, d = x0.shape
    xd = torch.from_numpy(np.ascontiguousarray(x0)).to(DEV)
    t = _outputs(B, d)
    out = _lib.BatchOut(*[t[k].data_ptr() for k in ("x", "value", "gradient", "num_iterations", "status", "nfev",
                                                     "x_delta", "f_delta", "gradient_norm")])
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    stop = stop if stop is not None else ob.default_stop()
    rc = one_warp.cno_one_warp_rosenbrock_minimize(d, C.c_int64(B), C.c_void_p(xd.data_ptr()), C.byref(stop),
                                                   C.byref(out), C.c_void_p(ws.data_ptr()), C.c_size_t(256),
                                                   C.c_void_p(torch.cuda.current_stream().cuda_stream), None)
    assert rc == 0
    torch.cuda.synchronize()
    return _host(t)


@pytest.mark.parametrize("d", DS)
def test_one_warp_user_functor_is_bit_identical(one_warp, d):
    B = 2 * sms() + 3
    x0 = ob.fill_uniform((B, d), 0, 11, -2.0, 2.0)
    group, _ = minimize_c(x0)
    bitwise_equal(minimize_one_warp(one_warp, x0), group)
