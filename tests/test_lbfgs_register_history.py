"""The plain L-BFGS kernel at d = 128 fp64, m = 10 keeps its newest (s, y) pair in registers and the older nine in
shared memory (csrc/cno_lbfgs.cuh: LbfgsPlan), which fits 12 instances per SM instead of 11.  Only where the vectors
are stored changes, so results stay bit-identical to the oracle: checked on the device source under the CPU warp
emulation, in the SASS, and on the GPU."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from cppnumericalsolvers_b200 import _lib
from oracle import oracle_binding as ob

EMU_DIR = os.path.join(os.path.dirname(__file__), "emu")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
HEADLINE = "_ZN3cno21lbfgs_minimize_kernelINS_12RosenbrockFnIdLi128ENS_10PolicyFastEEELi10ELb0ENS_13LsMoreThuente"


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    return C.CDLL(os.path.join(EMU_DIR, "libcno_emu.so"))


def _emulated(emu, x0, stop):
    B, d = x0.shape
    prob = ob.Problem(ob.FN_ROSENBROCK, ob._np_dtype(x0), d, 0, 0.0, None, 0, ob.device_policy(x0.dtype), 0)
    r = dict(x=np.zeros_like(x0), value=np.zeros(B), gradient=np.zeros_like(x0),
             num_iterations=np.zeros(B, np.uint32), status=np.zeros(B, np.int8), nfev=np.zeros(B, np.uint32),
             x_delta=np.zeros(B), f_delta=np.zeros(B), gradient_norm=np.zeros(B))
    out = ob.BatchOut(*[r[n].ctypes.data for n, _ in ob.BatchOut._fields_])
    assert emu.emu_minimize(ob.LBFGS, 0, C.byref(prob), C.c_longlong(B), C.c_void_p(x0.ctypes.data), C.byref(stop),
                            C.byref(out)) == 0
    return r


@pytest.mark.parametrize("seed,limit", [(1, 300), (2, 0)])
def test_register_pair_history_equals_oracle_under_emulation(emu, seed, limit):
    """Long Rosenbrock runs of the headline kernel: the shared ring wraps many times, so every pair passes through
    the register slot, is moved into the ring and leaves it.  Every output bit for bit."""
    x0 = ob.fill_uniform((2, 128), 0, 4000 + seed, -2.0, 2.0, np.float64)
    stop = ob.default_stop()
    stop.num_iterations = limit
    r = _emulated(emu, x0, stop)
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, stop=stop)
    assert int(o["num_iterations"].min()) > 3 * 10
    for k in KEYS:
        assert np.array_equal(r[k].view(np.uint8), o[k].view(np.uint8)), k


@pytest.fixture(scope="module")
def resources():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([CUOBJDUMP, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    return dict(re.findall(r"Function (\S+):\s*\n\s*(REG:\d+ STACK:\d+[^\n]*)", txt))


def test_headline_kernel_holds_a_register_pair_without_spilling(resources):
    """12 warps per SM leave 168 registers per thread (16384 per sub-partition over 3 warps): the headline kernel
    with one pair in registers fits in them with no stack and no local-memory traffic."""
    hits = [v for k, v in resources.items() if k.startswith(HEADLINE)]
    assert len(hits) == 1, hits
    regs = int(re.search(r"REG:(\d+)", hits[0]).group(1))
    assert "STACK:0" in hits[0]
    assert regs <= 168
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", [k for k in resources if k.startswith(HEADLINE)][0],
                           _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert not re.search(r"\b(LDL|STL)\b", sass)


@pytest.mark.gpu
def test_headline_plan_and_parity_on_the_gpu():
    import torch

    import cppnumericalsolvers_b200 as cn
    B = 1 << 14
    x0 = torch.empty(B, 128, dtype=torch.float64, device="cuda")
    cn.fill_uniform(x0, 0, 2024, -2.0, 2.0)
    state, prog = cn.Lbfgs().Minimize(cn.Rosenbrock(128), cn.BatchedFunctionState(x0), timed=True)
    torch.cuda.synchronize()
    assert prog.launch.warps_per_cta == 12
    o = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0.cpu().numpy())
    g = dict(x=state.x.cpu().numpy(), value=state.value.cpu().numpy(), gradient=state.gradient.cpu().numpy(),
             num_iterations=prog.num_iterations.cpu().numpy().astype(np.uint32), status=prog.status.cpu().numpy(),
             nfev=prog.nfev.cpu().numpy().astype(np.uint32), x_delta=prog.x_delta.cpu().numpy(),
             f_delta=prog.f_delta.cpu().numpy(), gradient_norm=prog.gradient_norm.cpu().numpy())
    for k in KEYS:
        assert np.array_equal(g[k].view(np.uint8), o[k].view(np.uint8)), k
