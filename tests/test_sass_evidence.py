"""Static evidence that libcno.so is Hopper-native code for this path (no GPU
needed: cuobjdump reads the cubin): FP64 tensor-core MMAs for the reductions,
TMA bulk copies for the staged per-instance blocks, warp votes instead of
divergence slow paths, and no FMA contraction in the arithmetic (the spec
forbids it)."""
import os
import re
import shutil
import subprocess

import pytest

from cppnumericalsolvers_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", txt)[1:]:
        out[f.split("\n")[0]] = f
    return out


def _find(kernels, *needles):
    hits = [v for k, v in kernels.items() if all(n in k for n in needles)]
    assert hits, needles
    return hits[0]


def test_compiled_for_sm_90a():
    txt = subprocess.run([CUOBJDUMP, "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in txt


def test_lbfgs_d128_uses_tensor_core_reductions(kernels):
    k = _find(kernels, "lbfgs_minimize_kernel", "RosenbrockFnIdLi128")
    assert k.count("DMMA") >= 20          # fp64 reductions on the FP64 tensor core
    assert "VOTE" in k and "BRA.DIV" not in k   # provably converged warps
    assert "REDUX" in k                   # lpNorm<Infinity> via REDUX.MAX


def test_newton_and_logistic_stage_with_tma(kernels):
    for k in (_find(kernels, "newton_minimize_kernel", "DenseQuadraticFnIdLi64"),
              _find(kernels, "lbfgs_minimize_kernel", "LogisticFn")):
        assert "UBLKCP" in k and "SYNCS" in k   # cp.async.bulk + mbarrier


def test_logistic_kernel_runs_two_warps_per_instance(kernels):
    """LogisticFn declares a helper warp per instance (csrc/cno_logistic.cuh): the kernel meets it at named barriers
    (BAR.SYNC with a register barrier id and 64 threads), the instance's block arrives by a TMA bulk copy, and exp's
    scaling is a multiplication (no libdevice ldexpf call left: the kernel's only subroutines are the division /
    square-root slow paths)."""
    k = _find(kernels, "lbfgs_minimize_kernel", "LogisticFn")
    assert len(re.findall(r"BAR\.SYNC\.DEFER_BLOCKING R\d+, 0x40", k)) >= 6
    assert "UBLKCP" in k
    n_instr = len(re.findall(r"^\s+/\*[0-9a-f]{4,6}\*/", k, flags=re.M))
    assert n_instr < 4500, n_instr   # code size is a performance property here (DESIGN.md 2.4: L0 instruction cache)


def test_newton_tensor_core_kernel_factors_on_the_fp64_tensor_core(kernels):
    """newton_dmma_minimize_kernel (CNO_POLICY_DMMA_LU): the trailing update of the blocked elimination is DMMA.8x8x4
    (many more than the 12 a kernel has for its reductions alone), the shared divisions start from MUFU.RCP64H, the
    next block is prefetched into L2."""
    k = _find(kernels, "newton_dmma_minimize_kernel")
    assert len(re.findall(r"\bDMMA\b", k)) >= 60
    assert "MUFU.RCP64H" in k
    assert "CCTL" in k or "PREFETCH" in k.upper() or "LDG.E.LTC" in k or "CCTL.E.PF2" in k or "PF" in k
    assert "BRA.DIV" not in k
    # ... while the default-policy kernel stays free of tensor-core factorisation work (its DMMAs are the reductions)
    k0 = _find(kernels, "newton_minimize_kernel", "DenseQuadraticFnIdLi64")
    assert len(re.findall(r"\bDMMA\b", k0)) < 40


def test_no_fma_contraction_in_fp32_kernels(kernels):
    """fp32 arithmetic must be FMUL/FADD (spec: products rounded before they are added);
    FFMA may only appear inside division / sqrt sequences, which are rare."""
    k = _find(kernels, "lbfgs_minimize_kernel", "RosenbrockFnIfLi128")
    ffma = len(re.findall(r"\bFFMA\b", k))
    fmul = len(re.findall(r"\bFMUL\b", k))
    fadd = len(re.findall(r"\bFADD\b", k))
    assert fmul > 100 and fadd > 100 and ffma < (fmul + fadd) // 2
