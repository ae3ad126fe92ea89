// tests/cpp/al_user_host.cu -- the C++ mirror of AugmentedLagrangian on user functors, written like
// src/test/augmented_lagrangian_test.cc:1106-1154 (AugmentedLagrangianNonConvex.Hs029EllipseEscapesOrigin): objective
// -x0 x1, inequality 48 - x0^2 - 2 x1^2 >= 0, from (1, 1).  One nvcc translation unit both instantiates the problem for
// the device and drives it through cppoptlib::solver::AugmentedLagrangian.  Run by tests/test_al_user_gpu.py.
#include <cmath>
#include <cstdio>
#include <vector>

#include "cppoptlib_b200/device.cuh"

template <class F>
using Function2d = cppoptlib::function::FunctionCRTP<F, double, cppoptlib::function::DifferentiabilityMode::First, 2>;
using FunctionExpr2d = cppoptlib::function::FunctionExpr<double, cppoptlib::function::DifferentiabilityMode::First, 2>;

// f(x) = -x0 x1 (augmented_lagrangian_test.cc: ProductObjective3D); lane 0 holds x0, lane 1 holds x1
struct NegProduct : Function2d<NegProduct> {
  __device__ double operator()(const cno::EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    const double x0 = __shfl_sync(cno::kFullMask, x[0], 0), x1 = __shfl_sync(cno::kFullMask, x[0], 1);
    if (grad) (*grad)[0] = (c.lane == 0) ? -x1 : ((c.lane == 1) ? -x0 : 0.0);
    return -x0 * x1;
  }
};
// c(x) = 48 - x0^2 - 2 x1^2 >= 0 (Hs029Ellipse)
struct Ellipse : Function2d<Ellipse> {
  __device__ double operator()(const cno::EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    const double x0 = __shfl_sync(cno::kFullMask, x[0], 0), x1 = __shfl_sync(cno::kFullMask, x[0], 1);
    if (grad) (*grad)[0] = (c.lane == 0) ? -2.0 * x0 : ((c.lane == 1) ? -4.0 * x1 : 0.0);
    return 48.0 - x0 * x0 - 2.0 * x1 * x1;
  }
};

using cppoptlib::function::Equalities;
using cppoptlib::function::Inequalities;
using P = cppoptlib::function::ConstrainedOptimizationProblem<NegProduct, Equalities<>, Inequalities<Ellipse>>;
CNO_DECLARE_CONSTRAINED(hs029, P)
CNO_INSTANTIATE_CONSTRAINED(hs029, P)

int main() {
  using namespace cppoptlib;
  solver::Lbfgs<FunctionExpr2d> inner_solver;
  solver::AugmentedLagrangian<P, decltype(inner_solver)> solver(P{NegProduct{}, {}, {Ellipse{}}}, inner_solver);
  // (1, 1) as in the reference's test, and a second start inside the ellipse
  const int64_t B = 2;
  auto state = solver::BatchedAugmentedLagrangeState<double, 2>::FromHost({1.0, 1.0, 2.0, -0.5}, B, 0, 1, 0.0);
  auto [solution, progress] = solver.Minimize(state);
  const std::vector<double> x = solution.x.ToHost();
  const double x0_star = 2.0 * std::sqrt(6.0), x1_star = 2.0 * std::sqrt(3.0), f_star = -12.0 * std::sqrt(2.0);
  int bad = 0;
  for (int b = 0; b < B; ++b) {
    const double f = -x[2 * b] * x[2 * b + 1];
    // the optimum is (+-x0*, +-x1*) with equal signs
    bad += !(std::fabs(std::fabs(x[2 * b]) - x0_star) <= 2e-1 && std::fabs(std::fabs(x[2 * b + 1]) - x1_star) <= 2e-1);
    bad += !(std::fabs(f - f_star) <= 5e-1);
  }
  bad += !(std::fabs(x[0] - x0_star) <= 2e-1 && std::fabs(x[1] - x1_star) <= 2e-1);
  std::printf("x = (%g, %g), f = %g, outer iterations = %u, kernel launches = %d%s\n", x[0], x[1], -x[0] * x[1],
              progress.num_iterations.ToHost()[0], progress.launch.kernel_launches, bad ? "  FAIL" : "");
  if (!bad) std::printf("PASS\n");
  return bad;
}
