"""cppnumericalsolvers_b200 -- H100-native batched unconstrained minimisation.

Host-side mirror of cppoptlib's solver::{Lbfgs,Lbfgsb,Bfgs,NewtonDescent,GradientDescent,
ConjugatedGradientDescent}::Minimize
with a batch axis; the compute is hand-written sm_90a CUDA in libcno.so behind
the C ABI of include/cno.h.  No CPU fallback.
"""
from . import _lib  # noqa: F401
from .constrained import (AugmentedLagrangeState, AugmentedLagrangian,  # noqa: F401
                          AugmentedLagrangianConfig, ConstrainedOptimizationProblem, ConstrainedStop)
from .function import (BatchedFunctionState, DenseQuadratic, DenseQuadraticFirst, DiagQuadratic,  # noqa: F401
                       DifferentiabilityMode, Function, HalfSquaredNorm, Logistic, Rosenbrock,
                       RosenbrockFull)
from .solver import (BatchedProgress, Bfgs, ConditionHessian, ConjugatedGradientDescent,  # noqa: F401
                     ConservativeStoppingSolverProgress, DefaultStoppingSolverProgress,
                     GradientDescent, HagerZhang, Lbfgs, Lbfgsb, MoreThuente, NewtonDescent, PrintProgressCallback,
                     Progress, Solver,
                     Status, fill_uniform)

__all__ = [
    "AugmentedLagrangeState", "AugmentedLagrangian", "AugmentedLagrangianConfig",
    "ConstrainedOptimizationProblem", "ConstrainedStop",
    "BatchedFunctionState", "BatchedProgress", "Bfgs", "ConditionHessian", "ConjugatedGradientDescent",
    "ConservativeStoppingSolverProgress", "GradientDescent", "HagerZhang", "MoreThuente",
    "DefaultStoppingSolverProgress", "DenseQuadratic", "DenseQuadraticFirst", "DiagQuadratic", "DifferentiabilityMode",
    "Function", "HalfSquaredNorm", "Lbfgs", "Lbfgsb", "Logistic", "NewtonDescent", "PrintProgressCallback", "Progress",
    "Rosenbrock", "RosenbrockFull", "Solver", "Status", "fill_uniform",
]
