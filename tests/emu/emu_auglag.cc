// tests/emu/emu_auglag.cc -- runs the DEVICE SOURCE of the AugmentedLagrangian path
// (csrc/cno_auglag.cuh: AugLagFn, al_autoscale_kernel, al_outer_step_kernel,
// al_finalize_kernel, on top of csrc/cno_functors.cuh) on the CPU under the warp
// emulation of warp_emu.h.  TEST INFRASTRUCTURE ONLY: the first GPU run of this path is
// still pending, so this is how its logic is checked against the oracle meanwhile
// (tests/test_device_emulated.py).  Built by tests/emu/Makefile into libcno_emu.so.
#include "cno_functors.cuh"
#include "cno_auglag.cuh"
#include "cno_auglag_host.h"
#include "cno_lbfgs.cuh"
#include "cno_bfgs.cuh"
#include "cno_descent.cuh"
#include "cno_newton.cuh"
#include "cno_newton_dmma.cuh"
#include "cno_lbfgsb.cuh"
#include "cno_logistic.cuh"
#include "cno_evaluate.cuh"

#define CNO_EMU_COMMA ,

namespace {

template <class F>
void launch(long long batch, F&& body) {  // grid of ceil(batch / kAlWarps) blocks x kAlWarps warps
  const int blocks = (int)((batch + cno::kAlWarps - 1) / cno::kAlWarps);
  for (int blk = 0; blk < blocks; ++blk)
    for (int w = 0; w < cno::kAlWarps; ++w)
      emu::run_warp([&](int lane) {
        blockIdx.x = (unsigned)blk;
        threadIdx.x = (unsigned)(w * 32 + lane);
        body();
      });
}

struct EmuArrays {  // mirrors cno::AlArrays<T> with untyped pointers
  void *x, *x_work, *lambda, *mu, *penalty, *prev_penalty, *max_violation, *max_lagrangian_gradient;
  uint32_t* num_iterations;
  int8_t* status;
  uint32_t* nfev;
  const uint32_t* inner_nfev;
  void *x_delta, *f_delta, *gradient_norm;
  int8_t* best_recorded;
  void *best_x, *best_lambda, *best_mu, *best_penalty, *best_objective, *best_violation, *best_kkt;
  int* remaining;
};

template <class T>
cno::AlArrays<T> arrays(const EmuArrays& e) {
  cno::AlArrays<T> a{};
  a.x = (T*)e.x; a.x_work = (T*)e.x_work; a.lambda = (T*)e.lambda; a.mu = (T*)e.mu;
  a.penalty = (T*)e.penalty; a.prev_penalty = (T*)e.prev_penalty; a.max_violation = (T*)e.max_violation;
  a.max_lagrangian_gradient = (T*)e.max_lagrangian_gradient; a.num_iterations = e.num_iterations;
  a.status = e.status; a.nfev = e.nfev; a.inner_nfev = e.inner_nfev; a.x_delta = (T*)e.x_delta;
  a.f_delta = (T*)e.f_delta; a.gradient_norm = (T*)e.gradient_norm; a.best_recorded = e.best_recorded;
  a.best_x = (T*)e.best_x; a.best_lambda = (T*)e.best_lambda; a.best_mu = (T*)e.best_mu;
  a.best_penalty = (T*)e.best_penalty; a.best_objective = (T*)e.best_objective;
  a.best_violation = (T*)e.best_violation; a.best_kkt = (T*)e.best_kkt; a.remaining = e.remaining;
  return a;
}

template <class T>
cno::AlView<T> view(const cno_constraints_t* k, const EmuArrays& e) {
  cno::AlView<T> v{};
  v.rows = (const T*)k->data;
  v.row_stride = (long long)k->data_stride;
  v.kinds = (const int*)k->kinds;
  v.n_eq = k->n_eq;
  v.n_ineq = k->n_ineq;
  v.lambda = (const T*)e.lambda;
  v.mu = (const T*)e.mu;
  v.penalty = (const T*)e.penalty;
  v.status = e.status;
  return v;
}

template <class T>
cno::AlParams<T> params(const cno_al_config_t* c, const cno_al_stop_t* s) {  // as al_run (csrc/cno_api.cu)
  cno::AlParams<T> p{};
  p.penalty_growth_factor = (T)c->penalty_growth_factor;
  p.violation_shrink_ratio = (T)c->violation_shrink_ratio;
  p.auto_scale_initial_penalty = c->auto_scale_initial_penalty;
  p.penalty_auto_objective_scale = (T)c->penalty_auto_objective_scale;
  p.penalty_auto_min = (T)c->penalty_auto_min;
  p.penalty_auto_max = (T)c->penalty_auto_max;
  p.multiplier_max = (T)c->multiplier_max;
  p.num_iterations = s->num_iterations;
  p.constraint_threshold = (T)s->constraint_threshold;
  p.kkt_stationarity_threshold = s->kkt_stationarity_threshold;
  return p;
}

enum Op { kComposite = 0, kAutoscale = 1, kOuterStep = 2, kFinalize = 3, kInner = 4 };

template <class Obj>
int run(const Obj& obj, int op, const cno_constraints_t* k, long long B, const EmuArrays& e, const cno_al_config_t* cfg,
        const cno_al_stop_t* stop, const void* x_in, void* value_out, void* grad_out) {
  using T = typename Obj::Scalar;
  constexpr int D = Obj::Dim;
  constexpr int E = cno::Shape<D>::E;
  const cno::AlView<T> v = view<T>(k, e);
  if (op == kComposite) {  // AugLagFn::operator() at x_in under (lambda, mu, penalty)
    const cno::AugLagFn<Obj> fn{obj, v};
    for (long long b = 0; b < B; ++b)
      emu::run_warp([&](int lane) {
        const cno::EvalCtx ctx{lane, b, nullptr};
        T x[E], g[E];
        cno::al_load<T, D>((const T*)x_in + b * D, lane, x);
        const T f = fn(ctx, x, &g);
        cno::al_store<T, D>((T*)grad_out + b * D, lane, g);
        if (lane == 0) ((T*)value_out)[b] = f;
      });
    return 0;
  }
  const cno::AlArrays<T> a = arrays<T>(e);
  if (op == kInner) {
    // the fused inner solve: lbfgs_minimize_kernel<AugLagFn<Obj>> exactly as al_run launches it
    // (x0 = state x, out.x = x_work, out.nfev = inner_nfev), one emulated warp draining the queue.
    {
      const cno::AugLagFn<Obj> fn{obj, v};
      const cno_stop_t* inner = static_cast<const cno_stop_t*>(x_in);
      cno_batch_out_t o{};
      o.x = a.x_work;
      o.nfev = const_cast<uint32_t*>(a.inner_nfev);
      unsigned long long queue = 0;
      emu::run_warp([&](int lane) {
        blockIdx.x = 0;
        threadIdx.x = (unsigned)lane;
        cno::lbfgs_minimize_kernel<cno::AugLagFn<Obj>, CNO_LBFGS_M>(fn, a.x, B, cno::make_stop<T>(*inner),
                                                                   cno::make_out<T>(o), &queue,
                                                                   cno::ResumeArgs{nullptr, 0, 0, 0});
      });
      return 0;
    }
  }
  const cno::AlParams<T> p = params<T>(cfg, stop);
  if (op == kAutoscale) launch(B, [&] { cno::al_autoscale_kernel<Obj>(obj, v, B, p, a); });
  else if (op == kOuterStep) launch(B, [&] { cno::al_outer_step_kernel<Obj>(obj, v, B, p, a); });
  else launch(B, [&] { cno::al_finalize_kernel<T, D>(B, k->n_eq, k->n_ineq, a); });
  return 0;
}

}  // namespace

// ---- the unconstrained solver kernels under emulation (one warp draining the queue) ----
template <class Fn, class LS, int M = CNO_LBFGS_M>
int run_solver(int solver, long long B, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out,
               const Fn fn = Fn{}) {
  using T = typename Fn::Scalar;
  unsigned long long queue = 0;
  int rc = 0;
  emu::run_warp([&](int lane) {
    blockIdx.x = 0;
    threadIdx.x = (unsigned)lane;
    const auto sp = cno::make_stop<T>(*stop);
    const auto bo = cno::make_out<T>(*out);
    if (solver == CNO_LBFGS) {
      cno::lbfgs_minimize_kernel<Fn, M, false, LS>(fn, (const T*)x0, B, sp, bo, &queue, cno::ResumeArgs{nullptr, 0, 0, 0});
    } else if (solver == CNO_BFGS) {
      if constexpr (Fn::Dim <= 32) cno::bfgs_minimize_kernel<Fn, LS>(fn, (const T*)x0, B, sp, bo, &queue);
      else cno::bfgs_smem_minimize_kernel<Fn, LS>(fn, (const T*)x0, B, sp, bo, &queue);  // H in shared memory
    } else if (solver == CNO_GRADIENT_DESCENT) {
      cno::descent_minimize_kernel<Fn, false, LS>(fn, (const T*)x0, B, sp, bo, &queue);
    } else if (solver == CNO_CONJUGATED_GRADIENT_DESCENT) {
      cno::descent_minimize_kernel<Fn, true, LS>(fn, (const T*)x0, B, sp, bo, &queue);
    } else {
      rc = CNO_ERR_UNSUPPORTED;
    }
  });
  return rc;
}

// solver: CNO_LBFGS / CNO_BFGS / CNO_GRADIENT_DESCENT / CNO_CONJUGATED_GRADIENT_DESCENT; hager_zhang selects
// the LineSearch policy; p->lbfgs_m selects Lbfgs<F, m> (0 = the default m).  Host pointers.
extern "C" int emu_minimize(int solver, int hager_zhang, const cno_problem_t* p, long long batch, const void* x0,
                            const cno_stop_t* stop, const cno_batch_out_t* out) {
  // Lbfgs<F, m> for the other compiled m (lbfgs.h:40-41): at m = 20 the plan keeps two pairs in registers, at m = 5 none
  if (solver == CNO_LBFGS && p->lbfgs_m != 0 && p->lbfgs_m != CNO_LBFGS_M) {
    if (hager_zhang || p->family != CNO_FN_ROSENBROCK || p->dtype != CNO_F64 || p->mode == 2 ||
        p->policy == CNO_POLICY_EIGEN_SSE2)
      return CNO_ERR_UNSUPPORTED;
#define LBFGS_M_CASE(DIM, M) \
  if (p->d == DIM && p->lbfgs_m == M) \
    return run_solver<cno::RosenbrockFn<double, DIM>, cno::LsMoreThuente, M>(solver, batch, x0, stop, out);
    LBFGS_M_CASE(37, 5)
    LBFGS_M_CASE(37, 20)
    LBFGS_M_CASE(128, 5)
    LBFGS_M_CASE(128, 20)
#undef LBFGS_M_CASE
    return CNO_ERR_UNSUPPORTED;
  }
  if (solver == CNO_LBFGS && !hager_zhang && p->family == CNO_FN_DENSE_QUADRATIC && p->dtype == CNO_F64 && p->mode != 2) {
    const double* data = (const double*)p->data;
    const long long stride = (long long)p->data_stride;
    if (p->d == 8)
      return run_solver<cno::DenseQuadraticGlobalFn<double, 8>, cno::LsMoreThuente>(solver, batch, x0, stop, out, {data, stride});
    if (p->d == 64)
      return run_solver<cno::DenseQuadraticGlobalFn<double, 64>, cno::LsMoreThuente>(solver, batch, x0, stop, out, {data, stride});
  }
  // Lbfgs on a Second-mode function (diagonal preconditioner, lbfgs.h:116-139) and the Eigen-SSE2 parity policy
  if (solver == CNO_LBFGS && !hager_zhang && p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64) {
    if (p->mode == 2 && p->d == 37)
      return run_solver<cno::SecondMode<cno::RosenbrockFn<double, 37>>, cno::LsMoreThuente>(solver, batch, x0, stop, out);
    if (p->mode == 2 && p->d == 128)
      return run_solver<cno::SecondMode<cno::RosenbrockFn<double, 128>>, cno::LsMoreThuente>(solver, batch, x0, stop, out);
    if (p->policy == CNO_POLICY_EIGEN_SSE2 && p->d == 128)
      return run_solver<cno::RosenbrockFn<double, 128, cno::PolicyEigenSSE2>, cno::LsMoreThuente>(solver, batch, x0, stop, out);
  }
#define SOLVER_CASE(DT, TY, DIM)                                                                         \
  if (p->family == CNO_FN_ROSENBROCK && p->dtype == DT && p->d == DIM)                                   \
    return hager_zhang ? run_solver<cno::RosenbrockFn<TY, DIM>, cno::LsHagerZhang>(solver, batch, x0, stop, out) \
                       : run_solver<cno::RosenbrockFn<TY, DIM>, cno::LsMoreThuente>(solver, batch, x0, stop, out);
  SOLVER_CASE(CNO_F64, double, 2)
  SOLVER_CASE(CNO_F64, double, 8)
  SOLVER_CASE(CNO_F64, double, 37)
  SOLVER_CASE(CNO_F64, double, 128)
  SOLVER_CASE(CNO_F32, float, 37)
#undef SOLVER_CASE
  return CNO_ERR_UNSUPPORTED;
}

// NewtonDescent (csrc/cno_newton.cuh) under emulation: the TMA bulk copy is a memcpy.
template <class Fn>
int run_newton(const Fn& fn, long long B, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out) {
  using T = typename Fn::Scalar;
  unsigned long long queue = 0;
  emu::run_warp([&](int lane) {
    blockIdx.x = 0;
    threadIdx.x = (unsigned)lane;
    cno::newton_minimize_kernel<Fn>(fn, (const T*)x0, B, cno::make_stop<T>(*stop), cno::make_out<T>(*out), &queue);
  });
  return 0;
}

extern "C" int emu_newton(const cno_problem_t* p, long long batch, const void* x0, const cno_stop_t* stop,
                          const cno_batch_out_t* out) {
  if (p->policy == CNO_POLICY_DMMA_LU) {  // csrc/cno_newton_dmma.cuh: blocked LU, trailing update as DMMA.8x8x4
    if (!(p->family == CNO_FN_DENSE_QUADRATIC && p->dtype == CNO_F64 && p->d == 64)) return CNO_ERR_UNSUPPORTED;
    cno::DenseQuadraticDmmaFn fn;
    fn.data = static_cast<const double*>(p->data);
    fn.stride = (long long)p->data_stride;
    unsigned long long queue = 0;
    emu::run_warp([&](int lane) {
      blockIdx.x = 0;
      threadIdx.x = (unsigned)lane;
      cno::newton_dmma_minimize_kernel<cno::DenseQuadraticDmmaFn>(fn, (const double*)x0, batch, cno::make_stop<double>(*stop),
                                                                  cno::make_out<double>(*out), &queue);
    });
    return 0;
  }
  if (p->family == CNO_FN_DENSE_QUADRATIC) {
#define NEWTON_CASE(DT, TY, DIM)                                                                   \
  if (p->dtype == DT && p->d == DIM)                                                               \
    return run_newton(cno::DenseQuadraticFn<TY, DIM>{static_cast<const TY*>(p->data), (long long)p->data_stride}, \
                      batch, x0, stop, out);
    NEWTON_CASE(CNO_F64, double, 64)
    NEWTON_CASE(CNO_F64, double, 12)
    NEWTON_CASE(CNO_F32, float, 64)
#undef NEWTON_CASE
  }
  if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 2)
    return run_newton(cno::RosenbrockFullFn<double, 2>{}, batch, x0, stop, out);
  if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 8)
    return run_newton(cno::RosenbrockFullFn<double, 8>{}, batch, x0, stop, out);
  return CNO_ERR_UNSUPPORTED;
}

// Progress::condition_hessian on request (csrc/cno_newton.cuh: condition_hessian_kernel) under emulation.
template <class Fn>
int run_condition(const Fn& fn, long long B, const void* x, void* out) {
  using T = typename Fn::Scalar;
  unsigned long long queue = 0;
  emu::run_warp([&](int lane) {
    blockIdx.x = 0;
    threadIdx.x = (unsigned)lane;
    cno::condition_hessian_kernel<Fn>(fn, (const T*)x, B, (T*)out, &queue);
  });
  return 0;
}
extern "C" int emu_condition_hessian(const cno_problem_t* p, long long batch, const void* x, void* out) {
  if (p->family == CNO_FN_DENSE_QUADRATIC) {
#define COND_CASE(DT, TY, DIM)                                                                                       \
  if (p->dtype == DT && p->d == DIM)                                                                                 \
    return run_condition(cno::DenseQuadraticFn<TY, DIM>{static_cast<const TY*>(p->data), (long long)p->data_stride}, \
                         batch, x, out);
    COND_CASE(CNO_F64, double, 64)
    COND_CASE(CNO_F64, double, 12)
    COND_CASE(CNO_F32, float, 64)
#undef COND_CASE
  }
  if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 2)
    return run_condition(cno::RosenbrockFullFn<double, 2>{}, batch, x, out);
  if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 8)
    return run_condition(cno::RosenbrockFullFn<double, 8>{}, batch, x, out);
  return CNO_ERR_UNSUPPORTED;
}

// L-BFGS on the logistic-regression functor (csrc/cno_logistic.cuh: per-instance data staged by TMA into shared
// memory) under emulation.
extern "C" int emu_logistic(const cno_problem_t* p, long long batch, const void* x0, const cno_stop_t* stop,
                            const cno_batch_out_t* out) {
  if (!(p->family == CNO_FN_LOGISTIC && p->dtype == CNO_F32 && p->d == 64 && p->n == 256)) return CNO_ERR_UNSUPPORTED;
  using Fn = cno::LogisticFn<float, 64, 256>;
  const Fn fn{static_cast<const float*>(p->data), (long long)p->data_stride, (float)p->param};
  unsigned long long queue = 0;
  // one team of the kernel's CTA: solver warp 0 and its helper warp (the functor declares kHelperWarps)
  using SM = cno::LbfgsPlan<Fn, CNO_LBFGS_M>::SM;
  emu::run_team([&](int lane, int w) {
    blockIdx.x = 0;
    threadIdx.x = (unsigned)(32 * (w ? SM::kHelperBase : 0) + lane);
    cno::lbfgs_minimize_kernel<Fn, CNO_LBFGS_M>(fn, (const float*)x0, batch, cno::make_stop<float>(*stop),
                                                cno::make_out<float>(*out), &queue, cno::ResumeArgs{nullptr, 0, 0, 0});
  });
  return 0;
}

// The logistic functor alone, evaluated by a team at given points: value only (g == nullptr: the helper gets the
// value-only command) or value + gradient.  One team, the instances one after the other (staging included).
extern "C" int emu_logistic_evaluate(const cno_problem_t* p, long long batch, const float* x, float* f, float* g) {
  if (!(p->family == CNO_FN_LOGISTIC && p->dtype == CNO_F32 && p->d == 64 && p->n == 256)) return CNO_ERR_UNSUPPORTED;
  using Fn = cno::LogisticFn<float, 64, 256>;
  constexpr int E = Fn::E;
  const Fn fn{static_cast<const float*>(p->data), (long long)p->data_stride, (float)p->param};
  alignas(16) static float stage[Fn::kStageElems];
  emu::run_team([&](int lane, int w) {
    cno::EvalCtx ctx{lane, 0, stage, 0};
    if (w == 1) { fn.helper(ctx); return; }
    uint32_t parity = 0;
    fn.init_stage(ctx);
    for (long long b = 0; b < batch; ++b) {
      ctx.instance = b;
      fn.stage(ctx, parity);
      float xv[E], gv[E];
      for (int e = 0; e < E; ++e) xv[e] = x[b * 64 + lane * E + e];
      const float v = g ? fn(ctx, xv, &gv) : fn(ctx, xv, nullptr);
      if (lane == 0) f[b] = v;
      if (g) for (int e = 0; e < E; ++e) g[b * 64 + lane * E + e] = gv[e];
    }
    fn.release_helper(ctx);
  });
  return 0;
}

// cno_evaluate under emulation: evaluate_kernel (csrc/cno_evaluate.cuh) as one CTA of kEvalWarps warps, run one
// after the other, on the functors of kEvalTable (csrc/cno_api.cu).  value or gradient may be null, as at the C ABI.
template <class Fn>
int run_evaluate(const Fn& fn, long long B, const void* x, void* value, void* gradient) {
  using T = typename Fn::Scalar;
  for (int w = 0; w < cno::kEvalWarps; ++w)
    emu::run_warp([&](int lane) {
      gridDim.x = 1;
      blockIdx.x = 0;
      threadIdx.x = (unsigned)(32 * w + lane);
      cno::evaluate_kernel<Fn>(fn, (const T*)x, B, (T*)value, (T*)gradient);
    });
  return 0;
}

extern "C" int emu_evaluate(const cno_problem_t* p, long long batch, const void* x, void* value, void* gradient) {
#define EVAL_CASE(FAM, DT, TY, DIM, FN)                               \
  if (p->family == FAM && p->dtype == DT && p->d == DIM) return run_evaluate(cno::FN, batch, x, value, gradient);
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 2, RosenbrockFn<double CNO_EMU_COMMA 2>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 3, RosenbrockFn<double CNO_EMU_COMMA 3>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 8, RosenbrockFn<double CNO_EMU_COMMA 8>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 32, RosenbrockFn<double CNO_EMU_COMMA 32>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 37, RosenbrockFn<double CNO_EMU_COMMA 37>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 64, RosenbrockFn<double CNO_EMU_COMMA 64>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 128, RosenbrockFn<double CNO_EMU_COMMA 128>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F32, float, 2, RosenbrockFn<float CNO_EMU_COMMA 2>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F32, float, 32, RosenbrockFn<float CNO_EMU_COMMA 32>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F32, float, 37, RosenbrockFn<float CNO_EMU_COMMA 37>{})
  EVAL_CASE(CNO_FN_ROSENBROCK, CNO_F32, float, 128, RosenbrockFn<float CNO_EMU_COMMA 128>{})
  EVAL_CASE(CNO_FN_DIAG_QUADRATIC, CNO_F64, double, 2, DiagQuadraticFn<double>{})
  EVAL_CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, double, 2, HalfSquaredNormFn<double CNO_EMU_COMMA 2>{})
  EVAL_CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, double, 8, HalfSquaredNormFn<double CNO_EMU_COMMA 8>{})
  EVAL_CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, double, 50, HalfSquaredNormFn<double CNO_EMU_COMMA 50>{})
  const double* data = (const double*)p->data;
  const long long stride = (long long)p->data_stride;
  EVAL_CASE(CNO_FN_DENSE_QUADRATIC, CNO_F64, double, 2, DenseQuadraticGlobalFn<double CNO_EMU_COMMA 2>{data CNO_EMU_COMMA stride})
  EVAL_CASE(CNO_FN_DENSE_QUADRATIC, CNO_F64, double, 8, DenseQuadraticGlobalFn<double CNO_EMU_COMMA 8>{data CNO_EMU_COMMA stride})
  EVAL_CASE(CNO_FN_DENSE_QUADRATIC, CNO_F64, double, 64, DenseQuadraticGlobalFn<double CNO_EMU_COMMA 64>{data CNO_EMU_COMMA stride})
#undef EVAL_CASE
  return CNO_ERR_UNSUPPORTED;
}

// ---- cno::al_outer_loop (csrc/cno_auglag_host.h: the host side of cno_al_minimize) with an emulation backend ----
template <class Obj>
struct AlEmuBackend {
  using T = typename Obj::Scalar;
  Obj obj;
  long long B;
  cno::AlArrays<T> a;
  cno::AlView<T> view;
  cno::AlParams<T> p;
  int copy_or_zero(void* dst, const void* src, size_t bytes) {
    if (!bytes || src == dst) return 0;
    if (src) std::memcpy(dst, src, bytes); else std::memset(dst, 0, bytes);
    return 0;
  }
  int fill(void* dst, int byte, size_t bytes) { if (bytes) std::memset(dst, byte, bytes); return 0; }
  int autoscale() { launch(B, [&] { cno::al_autoscale_kernel<Obj>(obj, view, B, p, a); }); return 0; }
  int inner(const cno_stop_t& stop) {
    const cno::AugLagFn<Obj> fn{obj, view};
    cno_batch_out_t o{};
    o.x = a.x_work;
    o.nfev = const_cast<uint32_t*>(a.inner_nfev);
    unsigned long long queue = 0;
    emu::run_warp([&](int lane) {
      blockIdx.x = 0;
      threadIdx.x = (unsigned)lane;
      cno::lbfgs_minimize_kernel<cno::AugLagFn<Obj>, CNO_LBFGS_M>(fn, a.x, B, cno::make_stop<T>(stop), cno::make_out<T>(o),
                                                                 &queue, cno::ResumeArgs{nullptr, 0, 0, 0});
    });
    return 0;
  }
  int outer_step(int* remaining) {
    *a.remaining = 0;
    launch(B, [&] { cno::al_outer_step_kernel<Obj>(obj, view, B, p, a); });
    *remaining = *a.remaining;
    return 0;
  }
  int finalize() { launch(B, [&] { cno::al_finalize_kernel<T, Obj::Dim>(B, view.n_eq, view.n_ineq, a); }); return 0; }
};

template <class Obj>
int run_al_minimize(const Obj& obj, const cno_constraints_t* k, long long B, const void* x0, const void* eq0, const void* ineq0,
                    const void* penalty0, const cno_stop_t* inner_stop, const cno_al_stop_t* outer_stop,
                    const cno_al_config_t* config, const cno_al_out_t* out, int* launches) {
  using T = typename Obj::Scalar;
  const cno::AlLayout L((size_t)B, Obj::Dim, (size_t)k->n_eq, (size_t)k->n_ineq, sizeof(T));
  std::vector<unsigned char> storage(L.total + 256);
  unsigned char* ws = storage.data() + (256 - ((uintptr_t)storage.data() & 255)) % 256;
  AlEmuBackend<Obj> be{obj, B, cno::al_make_arrays<T>(*out, ws, L), {}, {}};
  be.view = cno::al_make_view<T>(*k, be.a);
  be.p = cno::al_make_params<T>(*config, *outer_stop);
  return cno::al_outer_loop<T>(be, be.a, B, Obj::Dim, k->n_eq, k->n_ineq, x0, eq0, ineq0, penalty0, *inner_stop, *config,
                               launches);
}

// cno_al_minimize's host logic (outer loop, scratch layout) with every kernel under emulation.  Host pointers.
extern "C" int emu_al_minimize(const cno_problem_t* objective, const cno_constraints_t* constraints, long long batch,
                               const void* x0, const void* eq0, const void* ineq0, const void* penalty0,
                               const cno_stop_t* inner_stop, const cno_al_stop_t* outer_stop,
                               const cno_al_config_t* config, const cno_al_out_t* out, int* launches) {
#define AL_CASE(FAM, DT, TY, DIM, FN)                                                                  \
  if (objective->family == FAM && objective->dtype == DT && objective->d == DIM)                       \
    return run_al_minimize(cno::FN<TY, DIM>{}, constraints, batch, x0, eq0, ineq0, penalty0, inner_stop, outer_stop, \
                           config, out, launches);
  AL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 2, RosenbrockFn)
  AL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 8, RosenbrockFn)
  AL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 37, RosenbrockFn)
  AL_CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 128, RosenbrockFn)
  AL_CASE(CNO_FN_ROSENBROCK, CNO_F32, float, 8, RosenbrockFn)
  AL_CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, double, 2, HalfSquaredNormFn)
  AL_CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, double, 8, HalfSquaredNormFn)
#undef AL_CASE
  if (objective->family == CNO_FN_DENSE_QUADRATIC && objective->dtype == CNO_F64 && (objective->d == 2 || objective->d == 8)) {
    const double* data = (const double*)objective->data;
    const long long stride = (long long)objective->data_stride;
    if (objective->d == 2)
      return run_al_minimize(cno::DenseQuadraticGlobalFn<double, 2>{data, stride}, constraints, batch, x0, eq0, ineq0,
                             penalty0, inner_stop, outer_stop, config, out, launches);
    return run_al_minimize(cno::DenseQuadraticGlobalFn<double, 8>{data, stride}, constraints, batch, x0, eq0, ineq0,
                           penalty0, inner_stop, outer_stop, config, out, launches);
  }
  return CNO_ERR_UNSUPPORTED;
}

// cno_minimize_steps under emulation: rounds of `every` iterations with the solver state parked in between
// (lbfgs_minimize_kernel<Fn, M, /*kResume=*/true>), until every instance has stopped.  Host pointers.
template <class Fn>
int run_steps(long long B, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out, int every, int* rounds) {
  using T = typename Fn::Scalar;
  using RL = cno::ResumeLayout<T, cno::Shape<Fn::Dim>::E, CNO_LBFGS_M>;
  std::vector<unsigned char> state((size_t)B * RL::kBytes + 16);
  unsigned char* st = state.data() + (16 - ((uintptr_t)state.data() & 15)) % 16;
  const Fn fn{};
  int n = 0;
  for (int first = 1;; first = 0) {
    unsigned long long queue = 0;
    emu::run_warp([&](int lane) {
      blockIdx.x = 0;
      threadIdx.x = (unsigned)lane;
      cno::lbfgs_minimize_kernel<Fn, CNO_LBFGS_M, true>(fn, (const T*)x0, B, cno::make_stop<T>(*stop), cno::make_out<T>(*out),
                                                        &queue, cno::ResumeArgs{st, (long long)RL::kBytes, every, first});
    });
    ++n;
    bool done = true;
    for (long long b = 0; b < B; ++b) done = done && (out->status[b] != CNO_STATUS_CONTINUE);
    if (done) break;
  }
  if (rounds) *rounds = n;
  return 0;
}

extern "C" int emu_minimize_steps(const cno_problem_t* p, long long batch, const void* x0, const cno_stop_t* stop,
                                  const cno_batch_out_t* out, int every, int* rounds) {
  if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 2)
    return run_steps<cno::RosenbrockFn<double, 2>>(batch, x0, stop, out, every, rounds);
  if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 128)
    return run_steps<cno::RosenbrockFn<double, 128>>(batch, x0, stop, out, every, rounds);
  return CNO_ERR_UNSUPPORTED;
}

extern "C" int emu_al(int op, const cno_problem_t* objective, const cno_constraints_t* constraints, long long batch,
                      const EmuArrays* arrays_, const cno_al_config_t* config, const cno_al_stop_t* stop,
                      const void* x_in, void* value_out, void* grad_out) {
#define CASE(FAM, DT, TY, DIM, FN)                                                                  \
  if (objective->family == FAM && objective->dtype == DT && objective->d == DIM)                    \
    return run(cno::FN<TY, DIM>{}, op, constraints, batch, *arrays_, config, stop, x_in, value_out, grad_out);
  CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 2, RosenbrockFn)
  CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 8, RosenbrockFn)
  CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 37, RosenbrockFn)
  CASE(CNO_FN_ROSENBROCK, CNO_F64, double, 128, RosenbrockFn)
  CASE(CNO_FN_ROSENBROCK, CNO_F32, float, 8, RosenbrockFn)
  CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, double, 2, HalfSquaredNormFn)
  CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, double, 8, HalfSquaredNormFn)
#undef CASE
  if (objective->family == CNO_FN_DENSE_QUADRATIC && objective->dtype == CNO_F64 && objective->d == 8)
    return run(cno::DenseQuadraticGlobalFn<double, 8>{(const double*)objective->data, (long long)objective->data_stride}, op,
               constraints, batch, *arrays_, config, stop, x_in, value_out, grad_out);
  return CNO_ERR_UNSUPPORTED;
}


// Lbfgsb<F, 5> (csrc/cno_lbfgsb.cuh) under emulation.  lower / upper: host arrays [d] (stride 0) or [B, d].
template <class Fn, int M = 5>
int run_lbfgsb(long long B, const void* x0, const void* lower, const void* upper, long long stride, const cno_stop_t* stop,
               const cno_batch_out_t* out) {
  using T = typename Fn::Scalar;
  unsigned long long queue = 0;
  emu::run_warp([&](int lane) {
    blockIdx.x = 0;
    threadIdx.x = (unsigned)lane;
    cno::lbfgsb_minimize_kernel<Fn, M>(Fn{}, (const T*)x0, B, cno::make_stop<T>(*stop), cno::make_out<T>(*out), &queue,
                                        cno::BoundsArgs<T>{(const T*)lower, (const T*)upper, stride});
  });
  return 0;
}
extern "C" int emu_lbfgsb(const cno_problem_t* p, long long batch, const void* x0, const void* lower, const void* upper,
                          long long stride, const cno_stop_t* stop, const cno_batch_out_t* out) {
  if (p->lbfgs_m == 10) {  // Lbfgsb<F, 10>
    if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 8)
      return run_lbfgsb<cno::RosenbrockFn<double, 8>, 10>(batch, x0, lower, upper, stride, stop, out);
    if (p->family == CNO_FN_ROSENBROCK && p->dtype == CNO_F64 && p->d == 37)
      return run_lbfgsb<cno::RosenbrockFn<double, 37>, 10>(batch, x0, lower, upper, stride, stop, out);
    return CNO_ERR_UNSUPPORTED;
  }
#define LB_CASE(FAM, DT, FN)                                   \
  if (p->family == FAM && p->dtype == DT) return run_lbfgsb<FN>(batch, x0, lower, upper, stride, stop, out);
  if (p->d == 2) { LB_CASE(CNO_FN_ROSENBROCK, CNO_F64, cno::RosenbrockFn<double CNO_EMU_COMMA 2>) }
  if (p->d == 8) { LB_CASE(CNO_FN_ROSENBROCK, CNO_F64, cno::RosenbrockFn<double CNO_EMU_COMMA 8>) }
  if (p->d == 37) { LB_CASE(CNO_FN_ROSENBROCK, CNO_F64, cno::RosenbrockFn<double CNO_EMU_COMMA 37>) }
  if (p->d == 128) { LB_CASE(CNO_FN_ROSENBROCK, CNO_F64, cno::RosenbrockFn<double CNO_EMU_COMMA 128>) }
  if (p->d == 8) { LB_CASE(CNO_FN_HALF_SQUARED_NORM, CNO_F64, cno::HalfSquaredNormFn<double CNO_EMU_COMMA 8>) }
#undef LB_CASE
  return CNO_ERR_UNSUPPORTED;
}
