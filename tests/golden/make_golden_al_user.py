"""Generates tests/golden/user_al_*.npz from oracle/_ref = the REFERENCE'S OWN augmented_lagrangian.h /
function_problem.h / function_expressions.h / lbfgs.h on FunctionCRTP functors and composites
(oracle/ref_al_user.cc: cno_ref_al_minimize_expr; device twins tests/cpp/al_user_problems.cuh):

    python tests/golden/make_golden_al_user.py

(named user_al_* so that the row-constraint fixtures al_*.npz keep their own glob)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import al_user_ref as ar  # noqa: E402
from oracle import oracle_binding as ob  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def case(name, problem, x0, penalty0, outer_limit):
    n_eq, n_ineq = ar.COUNTS[problem]
    stop = ob.al_default_stop()
    stop.num_iterations = outer_limit
    r = ar.minimize(problem, x0, penalty0=penalty0, outer_stop=stop)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), problem=problem, x0=x0, n_eq=n_eq, n_ineq=n_ineq,
                        penalty0=penalty0, outer_limit=outer_limit, **{k: r[k] for k in ar.OUT_KEYS})
    print(name, "outer iterations", r["num_iterations"], "status", r["status"], "max violation",
          r["max_violation"].max())


def main():
    assert ar.available(), "oracle/_ref/libcno_ref_al_user.so is not built (needs the reference tree)"
    # augmented_lagrangian_test.cc:1106-1154 from (1, 1) and 15 more starts inside the ellipse
    x0 = np.concatenate([[[1.0, 1.0]], ob.fill_uniform((15, 2), 0, 29, -3.0, 3.0)])
    case("user_al_hs029_d2_f64", ar.AL_P_HS029, x0, 0.0, 10000)
    case("user_al_composites_d8_f64", ar.AL_P_COMPOSITES, ob.fill_uniform((8, 8), 0, 41, -1.5, 1.5), 0.0, 15)


if __name__ == "__main__":
    main()
