"""Generates tests/golden/lbfgs_rosenbrock_d{512,1024}_f64.npz from oracle/_ref = the REFERENCE'S OWN headers
(compiled against oracle/ref_shim): Lbfgs<Rosenbrock, 10> with MoreThuente, the default stopping preset, from the
seeded U(-2, 2) starts of cno_fill_uniform.  At these d the kernel is csrc/cno_lbfgs_group.cuh.  The reference tree
is not on the GPU machines, so the vectors are committed; rerun this script where oracle/_ref is built:

    python tests/golden/make_golden_large_d.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle_binding as ob  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
SEED = 12345
CASES = [(512, 6), (1024, 4)]  # d, instances


def main():
    assert ob.ref_available(), "oracle/_ref is not built (needs the reference tree)"
    for d, B in CASES:
        name = f"lbfgs_rosenbrock_d{d}_f64"
        x0 = ob.fill_uniform((B, d), 0, SEED, -2.0, 2.0)
        r = ob.minimize(ob.LBFGS, ob.FN_ROSENBROCK, x0, impl="ref")
        np.savez_compressed(os.path.join(HERE, name + ".npz"), x0=x0,
                            **{k: r[k] for k in ("x", "value", "gradient", "num_iterations", "status", "nfev",
                                                 "x_delta", "f_delta", "gradient_norm")},
                            solver=ob.LBFGS, family=ob.FN_ROSENBROCK, policy=ob.POLICY_DMMA_TREE)
        print(name, "iterations", r["num_iterations"], "seconds", round(r["seconds"], 2))


if __name__ == "__main__":
    main()
