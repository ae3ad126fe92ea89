"""tools/sanitize_logistic.py -- tiny run of the two-warps-per-instance logistic kernel (csrc/cno_logistic.cuh: named
barriers, exchange buffers in shared memory, TMA-staged block), for compute-sanitizer.
   compute-sanitizer --tool racecheck python tools/sanitize_logistic.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cppnumericalsolvers_b200 as cn  # noqa: E402

dev = "cuda"
p = cn.Progress(num_iterations=10, gradient_norm=1e-5, x_delta=1e-9, x_delta_violations=1, past=3, past_delta=1e-6)
rng = np.random.default_rng(0)
B, n, d = 23, 256, 64   # 23 instances: CTAs whose solver warps take a different number of instances (incl. none)
X = rng.uniform(-1, 1, (B, n, d)).astype(np.float32)
y = np.sign(rng.normal(size=(B, n))).astype(np.float32)
data = np.ascontiguousarray(np.concatenate([X.transpose(0, 2, 1).reshape(B, -1), y], 1))
st = cn.Lbfgs(p).Minimize(cn.Logistic(torch.from_numpy(data).to(dev), n, d, 1e-2),
                          cn.BatchedFunctionState(torch.zeros(B, d, device=dev)))
torch.cuda.synchronize()
print("sanitize_logistic done")
