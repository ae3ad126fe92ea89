// oracle/ref_al_user.cc -- the reference twins of the functor-constrained AugmentedLagrangian test problems
// (tests/cpp/al_user_problems.cuh): each problem built from FunctionCRTP functors and the REFERENCE'S OWN operators
// (function_expressions.h:403-518, compiled from the reference tree, unmodified) and solved by its own
// AugmentedLagrangian<ConstrainedOptimizationProblem<T, First, Dynamic>, Lbfgs<FunctionExpr>>.  TEST INFRASTRUCTURE ONLY.
// Built by oracle/ref_al_user.mk into _ref/libcno_ref_al_user.so; linear algebra from oracle/ref_shim, as for ref_driver.cc.
#include <cstdint>
#include <type_traits>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "cno_al_oracle.h"
#include "cno_oracle.h"
#include "cppoptlib/function.h"
#include "cppoptlib/function_expressions.h"
#include "cppoptlib/solver/augmented_lagrangian.h"
#include "cppoptlib/solver/lbfgs.h"

namespace {

using cppoptlib::function::DifferentiabilityMode;
using cppoptlib::function::FunctionCRTP;

// The objective families of ref_driver.cc with the same arithmetic (evaluations are counted by CountedObjective below).
// Chained Rosenbrock.
template <class T, DifferentiabilityMode Mode>
struct Rosenbrock : FunctionCRTP<Rosenbrock<T, Mode>, T, Mode> {
  using Base = FunctionCRTP<Rosenbrock<T, Mode>, T, Mode>;
  using typename Base::VectorType;
  T operator()(const VectorType& x, VectorType* gradient = nullptr) const {
    const int d = static_cast<int>(x.size());
    VectorType term = VectorType::Zero(d);
    if (gradient) *gradient = VectorType::Zero(d);
    for (int i = 0; i + 1 < d; ++i) {
      const T t1 = (1 - x[i]);
      const T t2 = (x[i + 1] - x[i] * x[i]);
      term[i] = t1 * t1 + 100 * t2 * t2;
      if (gradient) {
        const T a = -2 * (1 - x[i]) + 200 * (x[i + 1] - x[i] * x[i]) * (-2 * x[i]);
        const T b = 200 * (x[i + 1] - x[i] * x[i]);
        (*gradient)[i] = (i == 0) ? a : ((*gradient)[i] + a);
        (*gradient)[i + 1] = b;
      }
    }
    return term.sum();
  }
};
// src/test/augmented_lagrangian_test.cc:123-130
template <class T, DifferentiabilityMode Mode>
struct HalfSquaredNorm : FunctionCRTP<HalfSquaredNorm<T, Mode>, T, Mode> {
  using Base = FunctionCRTP<HalfSquaredNorm<T, Mode>, T, Mode>;
  using typename Base::VectorType;
  T operator()(const VectorType& x, VectorType* grad = nullptr) const {
    if (grad) *grad = x;
    return T(0.5) * x.squaredNorm();
  }
};
// f(x) = sum_i a_i (x_i - c)^2, a_i = 1 + i/8
template <class T, DifferentiabilityMode Mode>
struct Bowl : FunctionCRTP<Bowl<T, Mode>, T, Mode> {
  using Base = FunctionCRTP<Bowl<T, Mode>, T, Mode>;
  using typename Base::VectorType;
  T c = T(0);
  T operator()(const VectorType& x, VectorType* grad = nullptr) const {
    const int d = static_cast<int>(x.size());
    VectorType t(d);
    if (grad) *grad = VectorType::Zero(d);
    for (int i = 0; i < d; ++i) {
      const T a = T(1.0) + T(0.125) * i;
      const T r = x[i] - c;
      t[i] = a * r * r;
      if (grad) (*grad)[i] = T(2.0) * a * r;
    }
    return t.sum();
  }
};
// src/test/augmented_lagrangian_test.cc: DiagonalQuadratic2dSecond, f = 2 x0^2 + x1^2
template <class T, DifferentiabilityMode Mode>
struct DiagonalQuadratic2d : FunctionCRTP<DiagonalQuadratic2d<T, Mode>, T, Mode> {
  using Base = FunctionCRTP<DiagonalQuadratic2d<T, Mode>, T, Mode>;
  using typename Base::MatrixType;
  using typename Base::VectorType;
  T operator()(const VectorType& x, VectorType* grad = nullptr, MatrixType* hess = nullptr) const {
    if (grad) {
      *grad = VectorType::Zero(2);
      (*grad)[0] = 4 * x[0];
      (*grad)[1] = 2 * x[1];
    }
    if (hess) {
      *hess = MatrixType::Zero(2, 2);
      (*hess)(0, 0) = 4;
      (*hess)(1, 1) = 2;
    }
    return 2 * x[0] * x[0] + x[1] * x[1];
  }
};

}  // namespace

// ---- AugmentedLagrangian on functor constraints: the twins of the device problems of tests/cpp/al_user_problems.cuh,
// built from FunctionCRTP functors and the reference's own operators (function_expressions.h:403-518), solved by its
// AugmentedLagrangian<ConstrainedOptimizationProblem<T, First, Dynamic>, Lbfgs<FunctionExpr>> ----------------------
namespace {

enum {  // keep in step with tests/cpp/al_user_problems.cuh and tests/al_user_ref.py AL_P_*
  AL_P_HS029 = 0,           // -x0 x1 s.t. 48 - x0^2 - 2 x1^2 >= 0 (augmented_lagrangian_test.cc:1106-1154)
  AL_P_SIMPLE = 1,          // src/examples/constrained_simple.cc
  AL_P_COMPOSITE_CONS = 2,  // 0.5 |x|^2, eq X0MinusTarget(1) - 0.5, ineq 0.5 - X0MinusTarget(1) (:842-880)
  AL_P_COMPOSITES = 3,      // Rosenbrock + 0.5 HalfSquaredNorm, eq HalfSquaredNorm - 2, ineq 3 - Bowl(0.25)
  AL_P_BALL_OF_INSTANCE = 4,  // Rosenbrock, ineq r_b^2 - x.x >= 0, r_b = data[b]
  AL_P_BOWL = 6,            // Bowl(0.5), no constraints (:661-692)
  AL_P_DOWNGRADE = 7        // DiagonalQuadratic2dSecond through FunctionExpr<First>, eq X0MinusTarget(1) (:882-896)
};

template <class T>
using AlExpr = cppoptlib::function::FunctionExpr<T, DifferentiabilityMode::First, Eigen::Dynamic>;

// augmented_lagrangian_test.cc:1081-1104
struct ProductObjective : FunctionCRTP<ProductObjective, double, DifferentiabilityMode::First> {
  double operator()(const VectorType& x, VectorType* grad = nullptr) const {
    if (grad) {
      *grad = VectorType::Zero(2);
      (*grad)[0] = -x[1];
      (*grad)[1] = -x[0];
    }
    return -x[0] * x[1];
  }
};
struct Hs029Ellipse : FunctionCRTP<Hs029Ellipse, double, DifferentiabilityMode::First> {
  double operator()(const VectorType& x, VectorType* grad = nullptr) const {
    if (grad) {
      *grad = VectorType::Zero(2);
      (*grad)[0] = -2.0 * x[0];
      (*grad)[1] = -4.0 * x[1];
    }
    return 48.0 - x[0] * x[0] - 2.0 * x[1] * x[1];
  }
};
// src/examples/constrained_simple.cc
struct QuadraticObjective2 : FunctionCRTP<QuadraticObjective2, double, DifferentiabilityMode::First> {
  double operator()(const VectorType& x, VectorType* gradient = nullptr) const {
    if (gradient) {
      VectorType ref(2);
      ref[0] = 1;
      ref[1] = 2;
      *gradient = 2 * (x - ref);
    }
    return (x(0) - 1) * (x(0) - 1) + (x(1) - 2) * (x(1) - 2);
  }
};
struct InequalityConstraint3 : FunctionCRTP<InequalityConstraint3, double, DifferentiabilityMode::First> {
  double operator()(const VectorType& x, VectorType* gradient = nullptr) const {
    if (gradient) {
      *gradient = VectorType(2);
      (*gradient)[0] = -1;
      (*gradient)[1] = -1;
    }
    return 2 - (x(0) + x(1));
  }
};
// augmented_lagrangian_test.cc:158-172 (constrained_simple.cc's EqualityConstraint2 is target 0.5)
struct X0MinusTarget : FunctionCRTP<X0MinusTarget, double, DifferentiabilityMode::First> {
  double target = 0;
  double operator()(const VectorType& x, VectorType* grad = nullptr) const {
    if (grad) {
      *grad = VectorType::Zero(2);
      (*grad)[0] = 1.0;
    }
    return x[0] - target;
  }
};
// r_b^2 - x.x >= 0 with the radius of instance b
template <class T>
struct BallOfInstance : FunctionCRTP<BallOfInstance<T>, T, DifferentiabilityMode::First> {
  using Base = FunctionCRTP<BallOfInstance<T>, T, DifferentiabilityMode::First>;
  using typename Base::VectorType;
  T radius = T(0);
  T operator()(const VectorType& x, VectorType* grad = nullptr) const {
    if (grad) *grad = T(-2) * x;
    return radius * radius - x.squaredNorm();
  }
};
// Counts evaluations of the whole objective (a composite's leaves would count once each), as the device counts them.
template <class T, class F>
struct CountedObjective : FunctionCRTP<CountedObjective<T, F>, T, DifferentiabilityMode::First> {
  using Base = FunctionCRTP<CountedObjective<T, F>, T, DifferentiabilityMode::First>;
  using typename Base::VectorType;
  const F* f = nullptr;
  uint32_t* counter = nullptr;
  T operator()(const VectorType& x, VectorType* grad = nullptr) const {
    ++*counter;
    return (*f)(x, grad);
  }
};

struct AlExprJob {
  int d;
  int64_t b;
  const void* x0;
  const void* eq0;
  const void* ineq0;
  const void* penalty0;
  const cno_stop_t* inner_stop;
  const cno_al_stop_t* ostop;
  const cno_al_config_t* cfg;
  const cno_al_out_t* out;
};

// The solve and the outputs of al_run_one for a problem built from FunctionExprs.
template <class T, class Obj>
void al_expr_solve(const Obj& objective, const std::vector<AlExpr<T>>& eqs, const std::vector<AlExpr<T>>& ineqs,
                   const AlExprJob& j) {
  using Problem = cppoptlib::function::ConstrainedOptimizationProblem<T, DifferentiabilityMode::First, Eigen::Dynamic>;
  using Inner = cppoptlib::solver::Lbfgs<AlExpr<T>>;
  using State = cppoptlib::solver::AugmentedLagrangeState<T, Eigen::Dynamic>;
  const int d = j.d, ne = static_cast<int>(eqs.size()), ni = static_cast<int>(ineqs.size());
  const int64_t b = j.b;
  uint32_t counter = 0;
  CountedObjective<T, Obj> counted;
  counted.f = &objective;
  counted.counter = &counter;
  Problem problem(AlExpr<T>(counted), eqs, ineqs);

  Inner inner;  // DefaultStoppingSolverProgress (progress.h:353)
  if (const cno_stop_t* s = j.inner_stop) {
    auto& p = inner.stopping_progress;
    p.num_iterations = s->num_iterations;
    p.x_delta = static_cast<T>(s->x_delta);
    p.x_delta_violations = s->x_delta_violations;
    p.f_delta = static_cast<T>(s->f_delta);
    p.f_delta_violations = s->f_delta_violations;
    p.f_delta_relative = s->f_delta_relative != 0;
    p.gradient_norm = static_cast<T>(s->gradient_norm);
    p.gradient_norm_relative = s->gradient_norm_relative != 0;
    p.condition_hessian = static_cast<T>(s->condition_hessian);
    p.past = s->past;
    p.past_delta = static_cast<T>(s->past_delta);
  }
  const cno_al_config_t* cfg = j.cfg;
  cppoptlib::solver::AugmentedLagrangianConfig<T> config;
  config.penalty_growth_factor = static_cast<T>(cfg->penalty_growth_factor);
  config.violation_shrink_ratio = static_cast<T>(cfg->violation_shrink_ratio);
  config.auto_scale_initial_penalty = cfg->auto_scale_initial_penalty != 0;
  config.penalty_auto_objective_scale = static_cast<T>(cfg->penalty_auto_objective_scale);
  config.penalty_auto_min = static_cast<T>(cfg->penalty_auto_min);
  config.penalty_auto_max = static_cast<T>(cfg->penalty_auto_max);
  config.warmup_max_inner_iterations = cfg->warmup_max_inner_iterations;
  config.warmup_inner_gradient_tolerance = static_cast<T>(cfg->warmup_inner_gradient_tolerance);
  config.multiplier_max = static_cast<T>(cfg->multiplier_max);
  config.kkt_gradient_tolerance = static_cast<T>(cfg->kkt_gradient_tolerance);
  cppoptlib::solver::AugmentedLagrangian<Problem, Inner> solver(problem, inner, config);
  solver.stopping_progress.num_iterations = j.ostop->num_iterations;
  solver.stopping_progress.constraint_threshold = static_cast<T>(j.ostop->constraint_threshold);
  solver.stopping_progress.kkt_stationarity_threshold = static_cast<T>(j.ostop->kkt_stationarity_threshold);

  typename AlExpr<T>::VectorType x(d);
  for (int i = 0; i < d; ++i) x[i] = static_cast<const T*>(j.x0)[b * d + i];
  const T penalty0 = j.penalty0 ? static_cast<const T*>(j.penalty0)[b] : T(0);
  State state(x, static_cast<size_t>(ne), static_cast<size_t>(ni), penalty0);
  for (int i = 0; i < ne; ++i)
    state.multiplier_state.equality_multipliers[i] = j.eq0 ? static_cast<const T*>(j.eq0)[b * ne + i] : T(0);
  for (int i = 0; i < ni; ++i)
    state.multiplier_state.inequality_multipliers[i] = j.ineq0 ? static_cast<const T*>(j.ineq0)[b * ni + i] : T(0);
  auto [sol, prog] = solver.Minimize(problem, state);

  const cno_al_out_t* out = j.out;
  if (out->x) for (int i = 0; i < d; ++i) static_cast<T*>(out->x)[b * d + i] = sol.x[i];
  if (out->equality_multipliers)
    for (int i = 0; i < ne; ++i)
      static_cast<T*>(out->equality_multipliers)[b * ne + i] = sol.multiplier_state.equality_multipliers[i];
  if (out->inequality_multipliers)
    for (int i = 0; i < ni; ++i)
      static_cast<T*>(out->inequality_multipliers)[b * ni + i] = sol.multiplier_state.inequality_multipliers[i];
  if (out->penalty) static_cast<T*>(out->penalty)[b] = sol.penalty_state.penalty;
  if (out->max_violation) static_cast<T*>(out->max_violation)[b] = sol.max_violation;
  if (out->max_lagrangian_gradient) static_cast<T*>(out->max_lagrangian_gradient)[b] = sol.max_lagrangian_gradient;
  if (out->num_iterations) out->num_iterations[b] = static_cast<uint32_t>(prog.num_iterations);
  if (out->status) out->status[b] = static_cast<int8_t>(prog.status);
  if (out->nfev) out->nfev[b] = counter;
  if (out->x_delta) static_cast<T*>(out->x_delta)[b] = prog.x_delta;
  if (out->f_delta) static_cast<T*>(out->f_delta)[b] = prog.f_delta;
  if (out->gradient_norm) static_cast<T*>(out->gradient_norm)[b] = prog.gradient_norm;
}

template <class T>
int al_expr_dispatch(int problem, const void* data, const AlExprJob& j) {
  constexpr auto First = DifferentiabilityMode::First;
  constexpr auto Second = DifferentiabilityMode::Second;
  using V = std::vector<AlExpr<T>>;
  if constexpr (std::is_same_v<T, double>) {
    switch (problem) {
      case AL_P_HS029:
        al_expr_solve<T>(ProductObjective{}, V{}, V{AlExpr<T>(Hs029Ellipse{})}, j);
        return 0;
      case AL_P_SIMPLE: {
        X0MinusTarget eq;
        eq.target = 0.5;
        al_expr_solve<T>(QuadraticObjective2{}, V{AlExpr<T>(eq)}, V{AlExpr<T>(InequalityConstraint3{})}, j);
        return 0;
      }
      case AL_P_COMPOSITE_CONS: {
        HalfSquaredNorm<T, First> h;
        X0MinusTarget t;
        t.target = 1.0;
        const AlExpr<T> target_one = t;
        al_expr_solve<T>(h, V{target_one - 0.5}, V{0.5 - target_one}, j);
        return 0;
      }
      case AL_P_BOWL: {
        Bowl<T, First> bowl;
        bowl.c = 0.5;
        al_expr_solve<T>(bowl, V{}, V{}, j);
        return 0;
      }
      case AL_P_DOWNGRADE: {
        DiagonalQuadratic2d<T, Second> q;
        const AlExpr<T> wrapped = q;  // function_base.h:210-230
        X0MinusTarget eq;
        eq.target = 1.0;
        al_expr_solve<T>(wrapped, V{AlExpr<T>(eq)}, V{}, j);
        return 0;
      }
    }
  }
  switch (problem) {
    case AL_P_COMPOSITES: {
      Rosenbrock<T, First> r;
      HalfSquaredNorm<T, First> h;
      Bowl<T, First> bowl;
      bowl.c = T(0.25);
      const auto objective = r + T(0.5) * h;
      al_expr_solve<T>(objective, V{h - T(2)}, V{T(3) - bowl}, j);
      return 0;
    }
    case AL_P_BALL_OF_INSTANCE: {
      Rosenbrock<T, First> r;
      BallOfInstance<T> ball;
      ball.radius = static_cast<const T*>(data)[j.b];
      al_expr_solve<T>(r, V{}, V{AlExpr<T>(ball)}, j);
      return 0;
    }
  }
  return CNO_ERR_UNSUPPORTED;
}

}  // namespace

// AugmentedLagrangian<ConstrainedOptimizationProblem, Lbfgs<FunctionExpr>>::Minimize per instance on test problem
// `problem` (AL_P_*) at (dtype, d); data = the radii [B] of AL_P_BALL_OF_INSTANCE.  Same outputs as
// cno_ref_al_minimize; nfev counts evaluations of the objective as a whole.
extern "C" int cno_ref_al_minimize_expr(int problem, int dtype, int d, const void* data, int64_t batch, const void* x0,
                                        const void* eq0, const void* ineq0, const void* penalty0,
                                        const cno_stop_t* inner_stop, const cno_al_stop_t* outer_stop,
                                        const cno_al_config_t* config, const cno_al_out_t* out, int threads) {
  if (!x0 || !out || d <= 0) return CNO_ERR_INVALID_ARGUMENT;
  cno_al_stop_t odflt;
  if (!outer_stop) { cno_al_oracle_default_stop(&odflt); outer_stop = &odflt; }
  cno_al_config_t cdflt;
  if (!config) { cno_al_oracle_default_config(&cdflt); config = &cdflt; }
  Eigen::cno_policy_ref() = dtype == CNO_F64 ? CNO_POLICY_DMMA_TREE : CNO_POLICY_WARP_TREE;
  int rc = 0;
#ifdef _OPENMP
  if (threads <= 0) threads = omp_get_max_threads();
#else
  threads = 1;
#endif
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int64_t b = 0; b < batch; ++b) {
    const AlExprJob j{d, b, x0, eq0, ineq0, penalty0, inner_stop, outer_stop, config, out};
    const int r = dtype == CNO_F64 ? al_expr_dispatch<double>(problem, data, j) : al_expr_dispatch<float>(problem, data, j);
    if (r) rc = r;
  }
  return rc;
}
