"""tools/sanitize_newton_dmma.py -- tiny runs of the tensor-core NewtonDescent kernel with row exchanges forced, and of the
condition-number kernel, for compute-sanitizer.  Usage:  compute-sanitizer --tool racecheck python tools/sanitize_newton_dmma.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cppnumericalsolvers_b200 as cn  # noqa: E402
from cppnumericalsolvers_b200 import _lib  # noqa: E402

dev = "cuda"
rng = np.random.default_rng(0)
d, B = 64, 30
M = rng.uniform(-1, 1, (B, d, d))
A = np.einsum("bki,bkj->bij", M, M) / d + np.eye(d)
A = (A + A.transpose(0, 2, 1)) / 2
A[::3] = (M[::3] + M[::3].transpose(0, 2, 1)) / 2  # indefinite: pivots move, rows are exchanged
data = torch.from_numpy(np.concatenate([A.transpose(0, 2, 1).reshape(B, -1), rng.uniform(-1, 1, (B, d))], 1)).to(dev)
p = cn.Progress(num_iterations=3, gradient_norm=1e-5, x_delta=1e-9, x_delta_violations=1, past=3, past_delta=1e-6)
x0 = torch.empty(B, d, dtype=torch.float64, device=dev)
cn.fill_uniform(x0, 0, 1, -2.0, 2.0)
cn.NewtonDescent(p).Minimize(cn.DenseQuadratic(data, d, policy=_lib.POLICY_DMMA_LU), cn.BatchedFunctionState(x0))
cn.ConditionHessian(cn.DenseQuadratic(data, d), x0)
cn.ConditionHessian(cn.RosenbrockFull(8), x0[:, :8].contiguous())
torch.cuda.synchronize()
print("done")
