"""Lbfgsb<Rosenbrock, 5> fp64 at d = 256, 512 and 1024 on the GPU (csrc/cno_lbfgsb_group.cuh: one group of d / 128
warps per instance): every output bit for bit against the reference's own lbfgsb.h (oracle/_ref) on mixed batches,
exact ties against the kernel's device source under the CPU warp emulation, sentinels, the launch shape, the Python
and C++ mirror paths, and which keys cno_lbfgsb_supported accepts."""
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
needs_ref = pytest.mark.skipif(not ob.ref_available(), reason="oracle/_ref not built")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda:0"
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
DS = (256, 512, 1024)
GROUPS = {256: 4, 512: 2, 1024: 1}                      # resident instances (groups) per CTA
SMEM = {256: 131904, 512: 131872, 1024: 131856}          # dynamic shared memory per CTA
SENTINEL = 0x5A
DMAX = np.finfo(np.float64).max


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bitwise_equal(a, b, rows=slice(None)):
    for k in KEYS:
        assert np.array_equal(np.asarray(a[k])[rows].view(np.uint8), np.asarray(b[k])[rows].view(np.uint8)), k


def minimize_c(x0, lo, hi, stop=None, skip=(), rows=None):
    """cno_lbfgsb_minimize on Rosenbrock; lo / hi: [d], [B, d] or None; outputs named in `skip` are not requested."""
    B, d = x0.shape
    rows = B if rows is None else rows
    t = dict(x=torch.empty(rows, d, dtype=torch.float64, device=DEV),
             value=torch.empty(rows, dtype=torch.float64, device=DEV),
             gradient=torch.empty(rows, d, dtype=torch.float64, device=DEV),
             num_iterations=torch.empty(rows, dtype=torch.int32, device=DEV),
             status=torch.empty(rows, dtype=torch.int8, device=DEV), nfev=torch.empty(rows, dtype=torch.int32, device=DEV),
             x_delta=torch.empty(rows, dtype=torch.float64, device=DEV),
             f_delta=torch.empty(rows, dtype=torch.float64, device=DEV),
             gradient_norm=torch.empty(rows, dtype=torch.float64, device=DEV))
    for v in t.values():
        v.view(torch.uint8).fill_(SENTINEL)
    out = _lib.BatchOut(*[0 if k in skip else t[k].data_ptr() for k in
                          ("x", "value", "gradient", "num_iterations", "status", "nfev", "x_delta", "f_delta",
                           "gradient_norm")])
    xd = torch.from_numpy(np.ascontiguousarray(x0)).to(DEV)
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(DEV)  # noqa: E731
    lod, hid = dev(lo), dev(hi)
    stride = d if any(a is not None and a.dim() == 2 for a in (lod, hid)) else 0
    bounds = _lib.Bounds(None if lod is None else lod.data_ptr(), None if hid is None else hid.data_ptr(), stride)
    prob = _lib.Problem(family=0, dtype=_lib.F64, d=d, policy=_lib.POLICY_DMMA_TREE)
    ws = torch.zeros(256, dtype=torch.uint8, device=DEV)
    info = _lib.LaunchInfo()
    s = stop if stop is not None else ob.lbfgsb_stop()
    sp = C.cast(C.pointer(s), C.POINTER(_lib.Stop))
    _lib.check(_lib.lib().cno_lbfgsb_minimize(C.byref(prob), C.byref(bounds), B, xd.data_ptr(), sp, C.byref(out),
                                              ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream,
                                              C.byref(info)), "cno_lbfgsb_minimize")
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy() for k, v in t.items()}
    r["num_iterations"] = r["num_iterations"].astype(np.uint32)
    r["nfev"] = r["nfev"].astype(np.uint32)
    return r, info


def mixed_batch(d, B, seed):
    """Per-instance boxes on every row: random boxes (starts in U(-2.5, 2.5), mostly outside them), and every fifth
    row unbounded (the reference's default bounds, -+DBL_MAX)."""
    rng = np.random.default_rng(seed)
    x0 = ob.fill_uniform((B, d), 0, seed, -2.5, 2.5)
    lo = rng.uniform(-1.5, -0.2, (B, d))
    hi = lo + rng.uniform(0.3, 2.0, (B, d))
    lo[::5], hi[::5] = -DMAX, DMAX
    return x0, lo, hi


@needs_ref
@pytest.mark.parametrize("d", DS)
def test_mixed_batch_equals_reference(d):
    """B = 2 SMs + 3 rows of boxed, infeasible and unbounded starts under one stop (the unbounded rows reach its
    iteration cap, the boxed ones converge first): every row equals the reference's own solve of that row."""
    B = 2 * sms() + 3
    x0, lo, hi = mixed_batch(d, B, 500 + d)
    stop = ob.lbfgsb_stop()
    stop.num_iterations = 60
    g, _ = minimize_c(x0, lo, hi, stop)
    o = ob.ref_lbfgsb_minimize(ob.FN_ROSENBROCK, x0, lo, hi, stop=stop)
    bitwise_equal(g, o)
    assert (g["x"] >= lo).all() and (g["x"] <= hi).all()
    assert (g["num_iterations"] == 61).any() and (g["num_iterations"] < 40).any()
    # one shared box
    g, _ = minimize_c(x0[:9], np.full(d, -0.5), np.full(d, 0.8))
    bitwise_equal(g, ob.ref_lbfgsb_minimize(ob.FN_ROSENBROCK, x0[:9], np.full(d, -0.5), np.full(d, 0.8)))


def build_emu(out_dir):
    from test_lbfgsb_group import build_emu as build
    return build(out_dir)


@pytest.mark.parametrize("d", (256,))
def test_exact_ties_equal_emulation(tmp_path, d):
    """x0 = 0.3 in the shared box [-0.5, 0.8]: every interior coordinate has the same breakpoint, so crossed
    breakpoints tie exactly.  The reference's std::sort orders such ties arbitrarily; the kernel visits them by
    ascending index, on the GPU as in its device source under the emulation."""
    from test_lbfgsb_group import emulated
    emu = build_emu(tmp_path)
    x0 = np.full((2, d), 0.3)
    x0[1, ::2] = 0.6
    lo, hi = np.full(d, -0.5), np.full(d, 0.8)
    stop = ob.lbfgsb_stop()
    stop.num_iterations = 10
    g, _ = minimize_c(x0, lo, hi, stop)
    bitwise_equal(g, emulated(emu, x0, lo, hi, stop))
    assert (g["x"] >= lo).all() and (g["x"] <= hi).all()


@pytest.mark.parametrize("d", DS)
def test_rows_past_batch_and_unrequested_outputs_keep_their_sentinel(d):
    B = 5
    x0 = ob.fill_uniform((B, d), 0, 8, -2.5, 2.5)
    lo, hi = np.full(d, -0.5), np.full(d, 0.8)
    skip = ("gradient", "nfev", "f_delta")
    g, _ = minimize_c(x0, lo, hi, skip=skip, rows=B + 3)
    full, _ = minimize_c(x0, lo, hi)
    for k, v in g.items():
        raw = np.asarray(v).view(np.uint8).reshape(B + 3, -1)
        assert (raw[B:] == SENTINEL).all(), k
        if k in skip:
            assert (raw == SENTINEL).all(), k
        else:
            assert np.array_equal(np.asarray(v)[:B].view(np.uint8), np.asarray(full[k]).view(np.uint8)), k


@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("B", (1, 37, 4096))
def test_launch_shape(d, B):
    stop = ob.lbfgsb_stop()
    stop.num_iterations = 2
    _, info = minimize_c(ob.fill_uniform((B, d), 0, 9, -2.5, 2.5), np.full(d, -0.5), np.full(d, 0.8), stop)
    assert info.kernel_launches == 1
    assert (info.block, info.warps_per_cta, info.dynamic_smem) == (256, GROUPS[d], SMEM[d])
    assert info.grid == min(-(-B // GROUPS[d]), sms())


@pytest.mark.parametrize("d", DS)
def test_python_path_equals_c_abi(d):
    x0, lo, hi = mixed_batch(d, 6, 700 + d)
    c, _ = minimize_c(x0, lo, hi)
    solver = cn.Lbfgsb()
    solver.SetBounds(torch.from_numpy(lo).to(DEV), torch.from_numpy(hi).to(DEV))
    assert solver.supported(cn.Rosenbrock(d))
    st, pr = solver.Minimize(cn.Rosenbrock(d), cn.BatchedFunctionState(torch.from_numpy(x0).to(DEV)))
    torch.cuda.synchronize()
    p = dict(x=st.x.cpu().numpy(), value=st.value.cpu().numpy(), gradient=st.gradient.cpu().numpy(),
             num_iterations=pr.num_iterations.cpu().numpy().astype(np.uint32), status=pr.status.cpu().numpy(),
             nfev=pr.nfev.cpu().numpy().astype(np.uint32), x_delta=pr.x_delta.cpu().numpy(),
             f_delta=pr.f_delta.cpu().numpy(), gradient_norm=pr.gradient_norm.cpu().numpy())
    bitwise_equal(p, c)
    assert (p["x"] >= lo).all() and (p["x"] <= hi).all()
    assert not cn.Lbfgsb(m=10).supported(cn.Rosenbrock(d))


def test_cpp_mirror_at_d1024(tmp_path):
    """cppoptlib::solver::Lbfgsb<cppoptlib::function::Rosenbrock<double, 1024>> with SetBounds, from host buffers in
    a plain g++ translation unit: the same bits as cno_lbfgsb_minimize."""
    src = tmp_path / "mirror.cc"
    src.write_text(r'''
#include <cstdio>
#include <cstring>
#include <vector>
#include "cppoptlib_b200/cppoptlib.h"
int main() {
  using F = cppoptlib::function::Rosenbrock<double, 1024>;
  cppoptlib::solver::Lbfgsb<F> solver;
  const int B = 3;
  std::vector<double> x0(B * 1024), lo(1024, -0.5), hi(1024, 0.8);
  for (size_t i = 0; i < x0.size(); ++i) x0[i] = (i % 7) * 0.5 - 1.5;
  solver.SetBounds(lo, hi);
  auto [state, progress] = solver.Minimize(F{}, cppoptlib::function::BatchedFunctionState<double, 1024>::FromHost(x0, B));
  const std::vector<int8_t> st = progress.status.ToHost();
  const std::vector<uint32_t> it = progress.num_iterations.ToHost();
  const std::vector<double> f = state.value.ToHost();
  const std::vector<double> x = state.x.ToHost();
  for (int b = 0; b < B; ++b) {
    unsigned long long h = 1469598103934665603ull;  // FNV-1a of x's bytes
    for (int i = 0; i < 1024; ++i) {
      unsigned long long u;
      std::memcpy(&u, &x[b * 1024 + i], 8);
      for (int k = 0; k < 8; ++k) { h ^= (u >> (8 * k)) & 0xff; h *= 1099511628211ull; }
    }
    std::printf("%d %d %.17g %llu\n", (int)st[b], (int)it[b], f[b], h);
  }
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
    x0 = np.array([(i % 7) * 0.5 - 1.5 for i in range(3 * 1024)]).reshape(3, 1024)
    c, _ = minimize_c(x0, np.full(1024, -0.5), np.full(1024, 0.8))
    assert (c["x"] >= -0.5).all() and (c["x"] <= 0.8).all()

    def fnv(row):
        h = 1469598103934665603
        for byte in row.tobytes():
            h = ((h ^ byte) * 1099511628211) % (1 << 64)
        return h
    got = [line.split() for line in run.stdout.splitlines()]
    want = [[str(int(c["status"][b])), str(int(c["num_iterations"][b])), repr(float(c["value"][b])), str(fnv(c["x"][b]))]
            for b in range(3)]
    assert [[s, i, repr(float(v)), h] for s, i, v, h in got] == want


def test_supported_keys():
    """cno_lbfgsb_supported is true for Rosenbrock fp64 m = 5 at d = 256, 512, 1024 and false at nearby keys."""
    def ok(d, dtype=_lib.F64, m=0, family=0):
        p = _lib.Problem(family=family, dtype=dtype, d=d,
                         policy=_lib.POLICY_DMMA_TREE if dtype == _lib.F64 else _lib.POLICY_WARP_TREE)
        p.lbfgs_m = m
        return _lib.lib().cno_lbfgsb_supported(C.byref(p)) == _lib.OK
    for d in DS:
        assert ok(d) and ok(d, m=5)
        assert not ok(d, m=10) and not ok(d, dtype=_lib.F32)
        for family in (1, 2, 3):
            assert not ok(d, family=family)
    for d in (192, 384, 768, 2048):
        assert not ok(d)
