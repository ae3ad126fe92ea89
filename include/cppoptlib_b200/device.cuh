// cppoptlib_b200/device.cuh -- compile a USER objective (or a composite of objectives) for the device.
//
// In an nvcc translation unit (-gencode arch=compute_90a,code=sm_90a -fmad=false, include path =
// cppnumericalsolvers_b200/csrc; include THIS header before any other cppoptlib_b200 header):
//
//   struct MyF : cppoptlib::function::FunctionCRTP<MyF, double, First, 64> {
//     double shift;   // POD parameters, passed to the kernel by value
//     __device__ double operator()(const cno::EvalCtx& ctx, const double (&x)[2],
//                                  double (*grad)[2]) const { ... }
//     // Second mode only (function_base.h:103-120, the 3-argument operator()):
//     __device__ void hess_diag(const cno::EvalCtx&, const double (&x)[2], double (&h)[2]) const;
//     __device__ void hess_col(const cno::EvalCtx&, const double (&x)[2], int j, bool transposed,
//                              double (&col)[2]) const;
//   };
//   using H = decltype(MyF{} + 0.5 * cppoptlib::function::HalfSquaredNorm<double, 64>{});   // expressions.h
//   CNO_DECLARE_FUNCTION(myf, MyF)        // host side: binds MyF to the symbols
//   CNO_INSTANTIATE_FUNCTION(myf, MyF)    // device side: defines the symbols
//
// Any Dim compiles.  A solver whose plan does not fit one SM for it (in fp64: Bfgs past d = 128, NewtonDescent past
// d = 169, the condition number past d = 120) returns CNO_ERR_UNSUPPORTED at run time; Lbfgs runs at every d.
//
// At d = 1024 (fp64) a functor may also have the group form of the functor concept (cno_functors.cuh), which the
// mirror's Rosenbrock and HalfSquaredNorm and every composite of group-form functors have:
//     __device__ double operator()(const cno::GroupEvalCtx<8>& c, const double (&x)[4], double (*grad)[4]) const;
// with the helpers cno::group_sum_terms, cno::group_neighbours and cno::group_first_elem (cno_lbfgs_group.cuh).  Lbfgs
// (MoreThuente, First mode, the default policy, nothing staged) on such a functor then runs the group kernel, d / 128
// warps per instance, which was measured faster there than the one-warp kernel (DESIGN.md 2.10); every other case
// runs the one-warp kernel as before.
//
// This is the "thin extern-C layer": one symbol set per instantiated functor (SURVEY.md 8(b)), behind
// which Lbfgs / Bfgs / NewtonDescent / GradientDescent / ConjugatedGradientDescent<MyF>::Minimize,
// SetCallback (stepwise solves) and FunctionExpr::operator() launch the same persistent kernels as the
// built-in families:
//   cno_<tag>_minimize        Solver::Minimize                    (solver.h:181-224)
//   cno_<tag>_state_bytes /
//   cno_<tag>_minimize_steps  OptimizationStep rounds + callback  (solver.h:163-176, 226-228; Lbfgs)
//   cno_<tag>_evaluate        F::operator()(x, &grad) per instance (function_base.h:103-120)
//   cno_<tag>_condition_hessian   Progress::condition_hessian at x per instance (progress.h:203-210; Second mode)
//
// A constrained problem with functor constraints (cppoptlib.h: ConstrainedOptimizationProblem<Objective,
// Equalities<C...>, Inequalities<C...>>; objective and constraints any functors or composites of one Scalar and
// Dim <= 128):
//   CNO_DECLARE_CONSTRAINED(tag, P)       host side (cppoptlib.h)
//   CNO_INSTANTIATE_CONSTRAINED(tag, P)   device side: defines
//   cno_<tag>_al_workspace_bytes / cno_<tag>_al_minimize   AugmentedLagrangian<P, Lbfgs>::Minimize
//        (augmented_lagrangian.h:278-449), with the contract of cno_al_minimize (include/cno_al.h) and its kernels,
//        the constraint set being P's functors instead of [a | t] rows
#ifndef CPPOPTLIB_B200_DEVICE_CUH_
#define CPPOPTLIB_B200_DEVICE_CUH_

#ifdef CPPOPTLIB_B200_CPPOPTLIB_H_
#error "include cppoptlib_b200/device.cuh BEFORE cppoptlib_b200/cppoptlib.h in nvcc translation units"
#endif
#include "cno_device.cuh"
#include "cno_functors.cuh"
#include "cno_lbfgs_group.cuh"
#define CPPOPTLIB_B200_WITH_DEVICE 1
#include "cppoptlib.h"
#include "expressions.h"
#include "cno_auglag_launch.cuh"
#include "cno_bfgs.cuh"
#include "cno_descent.cuh"
#include "cno_evaluate.cuh"
#include "cno_launch.cuh"
#include "cno_lbfgs.cuh"
#include "cno_newton.cuh"

namespace cno {
template <class Fn, class Plan, class Kernel, class... Extra>
inline int launch_user(Kernel kernel, const Fn& fn, int64_t batch, const void* x0,
                       const cno_stop_t* stop, const cno_batch_out_t* out, void* workspace,
                       size_t workspace_bytes, void* stream, cno_launch_info_t* info, Extra... extra) {
  using T = typename Fn::Scalar;
  // one warp per instance: the helper-warp extension of the functor concept (kHelperWarps, csrc/cno_logistic.cuh) is
  // launched by the library's own launcher only (its CTA has two warps per instance)
  static_assert(FnHelperWarps<Fn>::value == 0, "user functors run one warp per instance");
  if (batch < 0 || !out || !workspace || workspace_bytes < 8) return CNO_ERR_INVALID_ARGUMENT;
  if (info) *info = cno_launch_info_t{};
  if (batch == 0) return CNO_OK;
  cno_stop_t dflt;
  if (!stop) { cno_default_stop(&dflt); stop = &dflt; }
  // the kernels' past-f ring is CNO_MAX_PAST warp-private scalars (same check as cno_minimize)
  if (stop->past > CNO_MAX_PAST || stop->past < 0) return CNO_ERR_INVALID_ARGUMENT;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return CNO_ERR_NO_DEVICE;
  cudaError_t last_error = cudaSuccess;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  unsigned long long* queue = static_cast<unsigned long long*>(workspace);
  LaunchTimer timer(s, info);
  int rc = timer.start(last_error);
  if (!rc)
    rc = launch_persistent<Plan>(kernel, (long long)batch, queue, s, info, last_error, fn, static_cast<const T*>(x0),
                                 (long long)batch, make_stop<T>(*stop), make_out<T>(*out), queue, extra...);
  return rc ? rc : timer.stop(last_error);
}
// ---- which optional members a functor has ----
template <class F, class = void>
struct HasHessDiag : std::false_type {};
template <class F>
struct HasHessDiag<F, std::void_t<decltype(&F::hess_diag)>> : std::true_type {};
template <class F, class = void>
struct HasHessCol : std::false_type {};
template <class F>
struct HasHessCol<F, std::void_t<decltype(&F::hess_col)>> : std::true_type {};

template <class F, class LS, int M>
inline int user_lbfgs(const F& fn, int mode, int lbfgs_m, int64_t batch, const void* x0, const cno_stop_t* stop,
                      const cno_batch_out_t* out, void* workspace, size_t workspace_bytes, void* stream,
                      cno_launch_info_t* info) {
  if (lbfgs_m != 0 && lbfgs_m != M) return CNO_ERR_UNSUPPORTED;  // this tag was compiled for Lbfgs<F, M>
  // Lbfgs on a Second-mode function takes the diagonal-preconditioner branch (lbfgs.h:116-139), unless
  // the function was bound through a First-mode FunctionExpr (function_base.h:210-230: downgrade)
  if constexpr (F::Mode == 2 && HasHessDiag<F>::value) {
    if (mode == 2) {
      using F2 = SecondMode<F>;
      if (stop && stop->condition_hessian > 0) return CNO_ERR_UNSUPPORTED;
      const F2 f2(fn);
      return launch_user<F2, typename LbfgsPlan<F2, M, false, LS>::SM>(lbfgs_minimize_kernel<F2, M, false, LS>, f2, batch, x0, stop,
                                                out, workspace, workspace_bytes, stream, info,
                                                ResumeArgs{nullptr, 0, 0, 0});
    }
  }
  return launch_user<F, typename LbfgsPlan<F, M, false, LS>::SM>(lbfgs_minimize_kernel<F, M, false, LS>, fn, batch, x0, stop, out,
                                          workspace, workspace_bytes, stream, info, ResumeArgs{nullptr, 0, 0, 0});
}

// Lbfgs (MoreThuente) on the group kernel (cno_lbfgs_group.cuh) where it was measured faster than the one-warp kernel
// (DESIGN.md 2.10): fp64 functors with the group form at d = 1024, the default policy, nothing staged, and m such that
// one group's history fits one SM.  At d = 512 the one-warp kernel was faster; it keeps every other case.
template <class F, int M>
struct GroupLbfgsRoute {
  static constexpr bool value = F::Dim == 1024 && std::is_same<typename F::Scalar, double>::value &&
                                std::is_same<typename PolicyOf<F>::type, PolicyFast>::value &&
                                StageElems<F>::value == 0 && HasGroupForm<F, F::Dim / 128>::value &&
                                LbfgsGroupPlan<double, 1024, M>::kFit >= 1;
};

template <class F, class LS>
inline int user_bfgs(const F& fn, int64_t batch, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out,
                     void* workspace, size_t workspace_bytes, void* stream, cno_launch_info_t* info) {
  using P = BfgsPlan<F, LS>;
  if constexpr (P::kFits)
    return launch_user<F, typename P::SM>(P::kernel(), fn, batch, x0, stop, out, workspace, workspace_bytes, stream, info);
  else
    return CNO_ERR_UNSUPPORTED;  // the inverse Hessian does not fit one SM's shared memory
}

template <class F>
inline int user_newton(const F& fn, int64_t batch, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out,
                       void* workspace, size_t workspace_bytes, void* stream, cno_launch_info_t* info) {
  if constexpr (F::Mode == 2 && HasHessCol<F>::value && NewtonSmem<typename F::Scalar, F::Dim>::kWarpsFit >= 1) {
    using A = SecondOrderAdapter<F>;
    if (stop && stop->condition_hessian > 0) return CNO_ERR_UNSUPPORTED;
    return launch_user<A, NewtonSmem<typename F::Scalar, F::Dim>>(newton_minimize_kernel<A>, A{fn}, batch, x0, stop, out,
                                                                   workspace, workspace_bytes, stream, info);
  } else {
    return CNO_ERR_UNSUPPORTED;  // second-order differentiable functions whose Hessian fits one SM's shared memory
  }
}

// Progress::condition_hessian on request (solver/progress.h:203-210; csrc/cno_newton.cuh: condition_hessian_kernel) for a
// Second-mode user functor or composite: H(x) through hess_col, as NewtonDescent stages it.
template <class F>
inline int user_condition(const F& fn, int64_t batch, const void* x, void* condition, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if constexpr (F::Mode == 2 && HasHessCol<F>::value && ConditionSmem<typename F::Scalar, F::Dim>::kWarpsFit >= 1) {
    using A = SecondOrderAdapter<F>;
    using T = typename F::Scalar;
    if (batch < 0) return CNO_ERR_INVALID_ARGUMENT;
    if (batch == 0) return CNO_OK;
    if (!x || !condition || !workspace || workspace_bytes < sizeof(unsigned long long) || ((uintptr_t)workspace & 7))
      return CNO_ERR_INVALID_ARGUMENT;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return CNO_ERR_NO_DEVICE;
    cudaError_t last_error = cudaSuccess;
    unsigned long long* queue = static_cast<unsigned long long*>(workspace);
    return launch_persistent<ConditionSmem<T, F::Dim>>(condition_hessian_kernel<A>, (long long)batch, queue,
                                                       static_cast<cudaStream_t>(stream), nullptr, last_error, A{fn},
                                                       static_cast<const T*>(x), (long long)batch,
                                                       static_cast<T*>(condition), queue);
  } else {
    return CNO_ERR_UNSUPPORTED;  // second-order differentiable functions whose Hessian fits one SM's shared memory
  }
}

template <class F, int M>
inline int user_minimize(int solver, int mode, int lbfgs_m, const F& fn, int64_t batch, const void* x0, const cno_stop_t* stop,
                         const cno_batch_out_t* out, void* workspace, size_t workspace_bytes, void* stream,
                         cno_launch_info_t* info) {
  using T = typename F::Scalar;
  switch (solver) {
    case CNO_LBFGS:
      if constexpr (GroupLbfgsRoute<F, M>::value) {
        // First mode used: not Lbfgs's Second-mode preconditioner branch (user_lbfgs)
        const bool second = F::Mode == 2 && HasHessDiag<F>::value && mode == 2;
        if (!second && (lbfgs_m == 0 || lbfgs_m == M))
          return launch_user<F, LbfgsGroupPlan<double, 1024, M>>(lbfgs_group_minimize_kernel<F, M>, fn, batch, x0, stop,
                                                                 out, workspace, workspace_bytes, stream, info);
      }
      return user_lbfgs<F, LsMoreThuente, M>(fn, mode, lbfgs_m, batch, x0, stop, out, workspace, workspace_bytes, stream, info);
    case CNO_LBFGS_HAGER_ZHANG:
      return user_lbfgs<F, LsHagerZhang, M>(fn, mode, lbfgs_m, batch, x0, stop, out, workspace, workspace_bytes, stream, info);
    case CNO_BFGS:
      return user_bfgs<F, LsMoreThuente>(fn, batch, x0, stop, out, workspace, workspace_bytes, stream, info);
    case CNO_BFGS_HAGER_ZHANG:
      return user_bfgs<F, LsHagerZhang>(fn, batch, x0, stop, out, workspace, workspace_bytes, stream, info);
    case CNO_NEWTON:
      return user_newton<F>(fn, batch, x0, stop, out, workspace, workspace_bytes, stream, info);
    case CNO_GRADIENT_DESCENT:
      return launch_user<F, DescentSmem<T>>(descent_minimize_kernel<F, false>, fn, batch, x0, stop, out, workspace,
                                            workspace_bytes, stream, info);
    case CNO_GRADIENT_DESCENT_HAGER_ZHANG:
      return launch_user<F, DescentSmem<T>>(descent_minimize_kernel<F, false, LsHagerZhang>, fn, batch, x0, stop, out,
                                            workspace, workspace_bytes, stream, info);
    case CNO_CONJUGATED_GRADIENT_DESCENT:
      if constexpr (sizeof(T) == 8)  // fp64 only: the reference computes beta in double
        return launch_user<F, DescentSmem<T>>(descent_minimize_kernel<F, true>, fn, batch, x0, stop, out, workspace,
                                              workspace_bytes, stream, info);
      else
        return CNO_ERR_UNSUPPORTED;
  }
  return CNO_ERR_UNSUPPORTED;
}

// stepwise Lbfgs (MoreThuente) for a user functor: the kResume build of the same kernel
template <class F, int M>
inline int user_minimize_steps(int solver, int mode, int lbfgs_m, const F& fn, int64_t batch, const void* x0, const cno_stop_t* stop,
                               const cno_batch_out_t* out, void* state, size_t state_bytes, int32_t max_iterations,
                               int32_t first_call, void* workspace, size_t workspace_bytes, void* stream,
                               cno_launch_info_t* info) {
  using T = typename F::Scalar;
  using RL = ResumeLayout<T, Shape<F::Dim>::E, M>;
  if (solver != CNO_LBFGS || (mode == 2 && F::Mode == 2) || (lbfgs_m != 0 && lbfgs_m != M)) return CNO_ERR_UNSUPPORTED;
  if (batch < 0 || !out || max_iterations <= 0) return CNO_ERR_INVALID_ARGUMENT;
  if (!out->x || !out->value || !out->gradient || !out->status || !out->num_iterations) return CNO_ERR_INVALID_ARGUMENT;
  if (batch > 0 && (!state || state_bytes < (size_t)batch * RL::kBytes || ((uintptr_t)state & 15))) return CNO_ERR_WORKSPACE;
  if (!x0 && first_call) return CNO_ERR_INVALID_ARGUMENT;
  return launch_user<F, typename LbfgsPlan<F, M, true, LsMoreThuente>::SM>(lbfgs_minimize_kernel<F, M, true, LsMoreThuente>, fn, batch, x0, stop,
                                          out, workspace, workspace_bytes, stream, info,
                                          ResumeArgs{static_cast<unsigned char*>(state), (long long)RL::kBytes,
                                                     max_iterations, first_call ? 1 : 0});
}
template <class F, int M>
inline int user_state_bytes(int solver, int64_t batch, size_t* bytes) {
  using RL = ResumeLayout<typename F::Scalar, Shape<F::Dim>::E, M>;
  if (solver != CNO_LBFGS) return CNO_ERR_UNSUPPORTED;
  if (!bytes || batch < 0) return CNO_ERR_INVALID_ARGUMENT;
  *bytes = (size_t)batch * RL::kBytes;
  return CNO_OK;
}
// AugmentedLagrangian<P, Lbfgs>::Minimize for a functor-constrained problem P: cno_al_minimize's checks, workspace
// layout and kernels, with AlFunctors over P's lists as the constraint set.
template <class P>
inline int user_al_workspace_bytes(int64_t batch, size_t* bytes) {
  if (!bytes || batch < 0) return CNO_ERR_INVALID_ARGUMENT;
  *bytes = AlLayout((size_t)batch, P::Dimension, P::kNumEq, P::kNumIneq, sizeof(typename P::ScalarType)).total;
  return CNO_OK;
}
template <class P>
inline int user_al_minimize(const P& prob, int64_t batch, const void* x0, const void* eq0, const void* ineq0,
                            const void* penalty0, const cno_stop_t* inner_stop, const cno_al_stop_t* outer_stop,
                            const cno_al_config_t* config, const cno_al_out_t* out, void* workspace,
                            size_t workspace_bytes, void* stream, cno_launch_info_t* info) {
  using Cons = AlFunctors<decltype(prob.equality_constraints), decltype(prob.inequality_constraints)>;
  if (batch < 0 || !out) return CNO_ERR_INVALID_ARGUMENT;
  if (info) *info = cno_launch_info_t{};
  if (batch == 0) return CNO_OK;
  AlArgs a{(long long)batch, x0, eq0, ineq0, penalty0, inner_stop, outer_stop, config, out,
           static_cast<unsigned char*>(workspace), workspace_bytes, static_cast<cudaStream_t>(stream), info};
  cno_stop_t idflt;
  cno_al_stop_t odflt;
  cno_al_config_t cdflt;
  int rc = al_check_args(a, P::Dimension, Cons::kNumEq, Cons::kNumIneq, sizeof(typename P::ScalarType), &idflt, &odflt,
                         &cdflt);
  if (rc) return rc;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return CNO_ERR_NO_DEVICE;
  cudaError_t last_error = cudaSuccess;
  const cno_constraints_t k{Cons::kNumEq, Cons::kNumIneq, nullptr, nullptr, 0};
  return al_run(prob.objective, Cons{prob.equality_constraints, prob.inequality_constraints}, k, a, last_error);
}
}  // namespace cno

// CNO_INSTANTIATE_CONSTRAINED(tag, P): the AugmentedLagrangian symbols of a functor-constrained problem P.
#define CNO_INSTANTIATE_CONSTRAINED(tag, P)                                                                    \
  static_assert(std::is_trivially_copyable<P>::value, "the problem is passed to the kernels by value");       \
  extern "C" int cno_##tag##_al_workspace_bytes(int64_t batch, size_t* bytes) {                                \
    return cno::user_al_workspace_bytes<P>(batch, bytes);                                                      \
  }                                                                                                            \
  extern "C" int cno_##tag##_al_minimize(const void* problem_bytes, int64_t batch, const void* x0, const void* eq0, \
                                         const void* ineq0, const void* penalty0, const cno_stop_t* inner_stop, \
                                         const cno_al_stop_t* outer_stop, const cno_al_config_t* config,        \
                                         const cno_al_out_t* out, void* workspace, size_t workspace_bytes,      \
                                         void* stream, cno_launch_info_t* info) {                               \
    if (!problem_bytes) return CNO_ERR_INVALID_ARGUMENT;                                                       \
    alignas(P) unsigned char raw__[sizeof(P)];                                                                 \
    memcpy(raw__, problem_bytes, sizeof(P));                                                                   \
    return cno::user_al_minimize<P>(*reinterpret_cast<const P*>(raw__), batch, x0, eq0, ineq0, penalty0,       \
                                    inner_stop, outer_stop, config, out, workspace, workspace_bytes, stream,   \
                                    info);                                                                     \
  }

// CNO_INSTANTIATE_FUNCTION_M(tag, F, M): the same with the L-BFGS kernels compiled for Lbfgs<F, M> (lbfgs.h:40-41).
#define CNO_INSTANTIATE_FUNCTION(tag, F) CNO_INSTANTIATE_FUNCTION_M(tag, F, CNO_LBFGS_M)
#define CNO_INSTANTIATE_FUNCTION_M(tag, F, M)                                                                 \
  static_assert(std::is_trivially_copyable<F>::value, "device functors are passed to the kernel by value");   \
  extern "C" int cno_##tag##_minimize(int solver, int mode, int lbfgs_m, const void* functor_bytes, int64_t batch, \
                                      const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out,      \
                                      void* workspace, size_t workspace_bytes, void* stream,                   \
                                      cno_launch_info_t* info) {                                               \
    alignas(F) unsigned char raw__[sizeof(F)];                                                                 \
    memcpy(raw__, functor_bytes, sizeof(F));                                                                   \
    return cno::user_minimize<F, M>(solver, mode, lbfgs_m, *reinterpret_cast<const F*>(raw__), batch, x0, stop, out, \
                                    workspace, workspace_bytes, stream, info);                                 \
  }                                                                                                            \
  extern "C" int cno_##tag##_state_bytes(int solver, int64_t batch, size_t* bytes) {                           \
    return cno::user_state_bytes<F, M>(solver, batch, bytes);                                                  \
  }                                                                                                            \
  extern "C" int cno_##tag##_minimize_steps(int solver, int mode, int lbfgs_m, const void* functor_bytes, int64_t batch, \
                                            const void* x0, const cno_stop_t* stop,                            \
                                            const cno_batch_out_t* out, void* state, size_t state_bytes,       \
                                            int32_t max_iterations, int32_t first_call, void* workspace,       \
                                            size_t workspace_bytes, void* stream, cno_launch_info_t* info) {   \
    alignas(F) unsigned char raw__[sizeof(F)];                                                                 \
    memcpy(raw__, functor_bytes, sizeof(F));                                                                   \
    return cno::user_minimize_steps<F, M>(solver, mode, lbfgs_m, *reinterpret_cast<const F*>(raw__), batch, x0, stop, \
                                          out, state, state_bytes, max_iterations, first_call, workspace,      \
                                          workspace_bytes, stream, info);                                      \
  }                                                                                                            \
  extern "C" int cno_##tag##_evaluate(const void* functor_bytes, int64_t batch, const void* x, void* value,    \
                                      void* gradient, void* stream) {                                          \
    alignas(F) unsigned char raw__[sizeof(F)];                                                                 \
    memcpy(raw__, functor_bytes, sizeof(F));                                                                   \
    return cno::launch_evaluate<F>(*reinterpret_cast<const F*>(raw__), batch, x, value, gradient, stream);     \
  }                                                                                                            \
  extern "C" int cno_##tag##_condition_hessian(const void* functor_bytes, int64_t batch, const void* x,        \
                                               void* condition, void* workspace, size_t workspace_bytes,      \
                                               void* stream) {                                                \
    alignas(F) unsigned char raw__[sizeof(F)];                                                                 \
    memcpy(raw__, functor_bytes, sizeof(F));                                                                   \
    return cno::user_condition<F>(*reinterpret_cast<const F*>(raw__), batch, x, condition, workspace,          \
                                  workspace_bytes, stream);                                                    \
  }

#endif  // CPPOPTLIB_B200_DEVICE_CUH_
