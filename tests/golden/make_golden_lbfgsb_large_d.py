"""Generates tests/golden/lbfgsb_rosenbrock_d{512,1024}_*.npz from oracle/_ref: the reference's own solver/lbfgsb.h
(compiled from a checkout of the reference against the Eigen-API shim), Lbfgsb<F, 5> with SetBounds, at the sizes the
group kernel runs (csrc/cno_lbfgsb_group.cuh).  A shared box and per-instance random boxes per d, B = 4, seeded starts
in U(-2, 2).  Run where the reference checkout exists (oracle/_ref built)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle_binding as ob  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("num_iterations", "status", "nfev", "x", "value", "gradient", "x_delta", "f_delta", "gradient_norm")
rng = np.random.default_rng(2026)
CASES = [  # name, d, B, lower, upper
    ("rosenbrock_d512_box", 512, 4, np.full(512, -0.5), np.full(512, 0.8)),
    ("rosenbrock_d512_per_instance_boxes", 512, 4, "rand", "rand"),
    ("rosenbrock_d1024_box", 1024, 4, np.full(1024, -0.5), np.full(1024, 0.8)),
    ("rosenbrock_d1024_per_instance_boxes", 1024, 4, "rand", "rand"),
]
for name, d, B, lo, hi in CASES:
    x0 = ob.fill_uniform((B, d), 0, 99 + d, -2.0, 2.0)
    if isinstance(lo, str):
        lo = rng.uniform(-1.5, -0.2, (B, d))
        hi = lo + rng.uniform(0.3, 2.0, (B, d))
    r = ob.ref_lbfgsb_minimize(ob.FN_ROSENBROCK, x0, lo, hi)
    np.savez_compressed(os.path.join(HERE, f"lbfgsb_{name}.npz"), x0=x0, lower=lo, upper=hi, **{k: r[k] for k in KEYS})
    print(name, r["num_iterations"], r["status"], r["value"][:3])
