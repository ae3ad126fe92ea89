"""Builds libcno.so (hand-written sm_90a CUDA + the extern "C" layer) in-tree.

nvcc cross-compiles without a GPU; the .so is a build product (git-ignored).  -fmad=false is part of the arithmetic
specification (no FMA contraction, like the reference's canonical build).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcno.so")
USER_GROUP_PARTS = 5  # translation units of tests/cpp/user_group_functions.cu (CNO_USER_GROUP_PART)

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-shared", "-Xcompiler", "-fPIC",
]


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "include", "cno.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, *NVCC_FLAGS, "-o", LIB, *sources(), "-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True)
    return LIB


def build_cpp_tests(verbose: bool = False) -> list:
    """Compiles the C++ host-API programs under tests/cpp (g++ and nvcc translation
    units) into tests/cpp/build/ (git-ignored).  A program newer than its source and every header it can include
    is left alone, so the tests that call this can run from a tree they may only read once it has been built."""
    root = os.path.dirname(HERE)
    src = os.path.join(root, "tests", "cpp")
    out = os.path.join(src, "build")
    inc_dir = os.path.join(root, "include")
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(inc_dir, f) for f in os.listdir(inc_dir) if f.endswith(".h")] + \
           [os.path.join(inc_dir, "cppoptlib_b200", f) for f in os.listdir(os.path.join(inc_dir, "cppoptlib_b200"))]

    def current(source, target):
        return os.path.exists(target) and all(os.path.getmtime(d) <= os.path.getmtime(target) for d in deps + [source])

    os.makedirs(out, exist_ok=True)
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    inc = ["-I" + inc_dir, "-I" + CSRC, f"-I{cuda}/include"]
    link = [f"-L{HERE}", "-lcno", f"-L{cuda}/lib64", "-lcudart", f"-Wl,-rpath,{HERE}", f"-Wl,-rpath,{cuda}/lib64"]
    exes = []
    # verify_host; the constrained C++ mirror (run by tests/test_al_gpu.py); the multi-GPU path below Python:
    # MinimizeSharded + cno_allgather_done (NCCL resolved with dlopen)
    for name, extra, extra_link, listed in (("verify_host", [], [], True), ("al_host", [], [], False),
                                            ("sharded_nccl", ["-pthread"], ["-ldl"], True)):
        source, target = os.path.join(src, name + ".cc"), os.path.join(out, name)
        if not current(source, target):
            cmd = ["g++", "-std=c++17", "-O2", "-Wall", *extra, source, *inc, "-o", target, *link, *extra_link]
            subprocess.run(cmd, check=True)
        if listed:
            exes.append(target)
    nvcc = os.environ.get("NVCC", f"{cuda}/bin/nvcc")
    xlink = ["-Xlinker", f"-rpath={HERE}"]
    dev_flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
                 "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false"]
    jobs = [(os.path.join(src, "user_functor.cu"), os.path.join(out, "user_functor"), []),
            # user functors + composites as a shared library for the Python parity tests (tests/usertest_binding.py)
            (os.path.join(src, "user_functions.cu"), os.path.join(out, "libcno_usertest.so"),
             ["-shared", "-Xcompiler", "-fPIC"])]
    procs = []
    for source, target, extra in jobs:
        if current(source, target):
            continue
        procs.append(subprocess.Popen([nvcc, *dev_flags, *extra, source, *inc, "-o", target, f"-L{HERE}", "-lcno", *xlink]))
    # user functors and composites at d = 512 / 1024 (tests/test_user_group_gpu.py): compiled in parts, in parallel
    group_src, group_lib = os.path.join(src, "user_group_functions.cu"), os.path.join(out, "libcno_usergroup.so")
    group_objs = [os.path.join(out, f"user_group_functions.{k}.o") for k in range(USER_GROUP_PARTS)]
    if not current(group_src, group_lib):
        procs += [subprocess.Popen([nvcc, *dev_flags, "-c", "-Xcompiler", "-fPIC", f"-DCNO_USER_GROUP_PART={k}",
                                    group_src, *inc, "-o", obj]) for k, obj in enumerate(group_objs)]
    for p in procs:
        if p.wait() != 0:
            raise subprocess.CalledProcessError(p.returncode, p.args)
    if not current(group_src, group_lib):
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", *group_objs, "-o", group_lib,
                        f"-L{HERE}", "-lcno", *xlink], check=True)
    exes.append(os.path.join(out, "user_functor"))
    return exes


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
