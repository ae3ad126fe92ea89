// cppoptlib_b200/cppoptlib.h -- C++17 host-side mirror of cppoptlib's solver
// interface with a batch axis, over the extern "C" layer of libcno.so
// (include/cno.h).  Header only; compiles with g++ -std=c++17 (no nvcc), links
// against libcno.so and libcudart.
//
//   reference (include/cppoptlib/...)            here
//   -------------------------------------------  --------------------------------
//   function_base.h:42-46  DifferentiabilityMode  function::DifferentiabilityMode
//   function_base.h:96-126 FunctionCRTP           function::FunctionCRTP (static
//                                                 members; the device operator()
//                                                 lives in the functor's .cuh)
//   function_base.h:194-260 FunctionExpr          function::FunctionExpr (erases
//                                                 the LAUNCHER, not a virtual call:
//                                                 SURVEY.md 7 hard part 3)
//   function_base.h:298-332 FunctionState         function::BatchedFunctionState
//   solver/progress.h:37-47 Status                solver::Status
//   solver/progress.h:82-140 Progress             solver::Progress /
//                                                 solver::BatchedProgress
//   solver/progress.h:353-464 presets             solver::DefaultStopping...,
//                                                 solver::ConservativeStopping...
//   solver/solver.h:156-231 Solver<F,State>       solver::Solver<F>
//   solver/lbfgs.h / bfgs.h / newton_descent.h    solver::Lbfgs / Bfgs / NewtonDescent
//
// Error behaviour follows the reference: numerical outcomes are per-instance
// Status codes; only API misuse / CUDA failures throw std::runtime_error.
#ifndef CPPOPTLIB_B200_CPPOPTLIB_H_
#define CPPOPTLIB_B200_CPPOPTLIB_H_

#include <cuda_runtime_api.h>

#include <cstdint>
#include <cstdio>
#include <functional>
#include <iomanip>
#include <memory>
#include <ostream>
#include <sstream>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include "../cno.h"
#include "../cno_al.h"
#include "modes.h"

namespace cppoptlib {

namespace detail {
inline void check_cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
inline void check_cno(int rc, const char* what) {
  if (rc == CNO_OK) return;
  std::string msg = std::string(what) + ": " + cno_error_string(rc);
  if (rc == CNO_ERR_CUDA) {
    const char* m = nullptr;
    cno_last_cuda_error(&m);
    if (m) msg += std::string(" (") + m + ")";
  }
  throw std::runtime_error(msg);
}
// RAII device array (values everywhere, like the reference's Eigen members).
template <class T>
class DeviceArray {
 public:
  DeviceArray() = default;
  explicit DeviceArray(size_t n) : n_(n) {
    if (n) check_cuda(cudaMalloc(&p_, n * sizeof(T)), "cudaMalloc");
  }
  DeviceArray(const DeviceArray& o) : DeviceArray(o.n_) {
    if (n_) check_cuda(cudaMemcpy(p_, o.p_, n_ * sizeof(T), cudaMemcpyDeviceToDevice), "cudaMemcpy");
  }
  DeviceArray(DeviceArray&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  DeviceArray& operator=(DeviceArray o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
  ~DeviceArray() { if (p_) cudaFree(p_); }
  static DeviceArray FromHost(const std::vector<T>& h) {
    DeviceArray a(h.size());
    if (!h.empty()) check_cuda(cudaMemcpy(a.p_, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice), "H2D");
    return a;
  }
  std::vector<T> ToHost() const {
    std::vector<T> h(n_);
    if (n_) check_cuda(cudaMemcpy(h.data(), p_, n_ * sizeof(T), cudaMemcpyDeviceToHost), "D2H");
    return h;
  }
  // elements [first, first + count) only
  std::vector<T> ToHost(size_t first, size_t count) const {
    if (first + count > n_) throw std::out_of_range("DeviceArray::ToHost: range");
    std::vector<T> h(count);
    if (count)
      check_cuda(cudaMemcpy(h.data(), static_cast<const T*>(p_) + first, count * sizeof(T), cudaMemcpyDeviceToHost), "D2H");
    return h;
  }
  T* data() const { return static_cast<T*>(p_); }
  size_t size() const { return n_; }

 private:
  void* p_ = nullptr;
  size_t n_ = 0;
};
template <class T> struct DType;
template <> struct DType<double> { static constexpr int value = CNO_F64; };
template <> struct DType<float> { static constexpr int value = CNO_F32; };
}  // namespace detail

namespace function {


// function_base.h:96-126.  A user objective derives from FunctionCRTP exactly as
// with the reference; its operator() is the warp-cooperative __device__ form
// documented in cppnumericalsolvers_b200/csrc/cno_functors.cuh and is compiled by
// nvcc in the translation unit that says CNO_INSTANTIATE_FUNCTION (device.cuh).
template <class Derived, class TScalar, DifferentiabilityMode TMode, int TDimension>
struct FunctionCRTP {
  static constexpr int Dimension = TDimension;
  using ScalarType = TScalar;
  static constexpr DifferentiabilityMode Differentiability = TMode;
  // device functor concept names (cno_functors.cuh)
  using Scalar = TScalar;
  static constexpr int Dim = TDimension;
  static constexpr int Mode = static_cast<int>(TMode);
};

// What a solver needs to know about an objective: which kernels to launch.
// Built-in families go through cno_minimize's table; user functors (and composites of functors,
// expressions.h) through the extern "C" symbols generated by CNO_INSTANTIATE_FUNCTION(tag, F).
// `mode` = the DifferentiabilityMode the function is USED with (a Second-mode functor bound through a
// First-mode FunctionExpr is minimised as a First-mode function: function_base.h:210-230).
typedef int (*RawMinimizeFn)(int solver, int mode, int lbfgs_m, const void* functor_bytes, int64_t batch, const void* x0,
                             const cno_stop_t* stop, const cno_batch_out_t* out, void* workspace,
                             size_t workspace_bytes, void* stream, cno_launch_info_t* info);
typedef int (*RawStateBytesFn)(int solver, int64_t batch, size_t* bytes);
typedef int (*RawMinimizeStepsFn)(int solver, int mode, int lbfgs_m, const void* functor_bytes, int64_t batch, const void* x0,
                                  const cno_stop_t* stop, const cno_batch_out_t* out, void* state,
                                  size_t state_bytes, int32_t max_iterations, int32_t first_call, void* workspace,
                                  size_t workspace_bytes, void* stream, cno_launch_info_t* info);
typedef int (*RawEvaluateFn)(const void* functor_bytes, int64_t batch, const void* x, void* value, void* gradient,
                             void* stream);

typedef int (*RawConditionFn)(const void* functor_bytes, int64_t batch, const void* x, void* condition, void* workspace,
                              size_t workspace_bytes, void* stream);

template <class F, class = void>
struct LauncherTraits;  // specialised by CNO_DECLARE_FUNCTION / the built-ins below

// function_base.h:194-260: value-semantic, type-erased handle.  Erasure happens
// at the launcher (a function pointer + the functor's POD bytes), so nothing
// virtual ever has to cross to the device.
template <class TScalar, DifferentiabilityMode TMode = DifferentiabilityMode::First, int TDimension = -1>
struct FunctionExpr {
  using ScalarType = TScalar;
  static constexpr int Dimension = TDimension;
  static constexpr DifferentiabilityMode Differentiability = TMode;

  cno_problem_t problem{};          // built-in family (raw == nullptr)
  RawMinimizeFn raw = nullptr;      // user functor launchers (CNO_DECLARE_FUNCTION)
  RawStateBytesFn raw_state_bytes = nullptr;
  RawMinimizeStepsFn raw_steps = nullptr;
  RawEvaluateFn raw_evaluate = nullptr;
  RawConditionFn raw_condition = nullptr;
  std::vector<unsigned char> pod;   // the user functor's bytes
  int dimension = TDimension;       // (TDimension == -1: taken from the bound function)

  FunctionExpr() = default;
  // function_base.h:210-230: accepts any source at least as differentiable as TMode.  A stronger source
  // is used AS a TMode function (the reference wraps it in ModeDowngradeAdapter, :151-189; here the
  // launcher is told the mode, so e.g. Lbfgs does not take its Second-mode preconditioner branch).
  template <class F, class = std::enable_if_t<!std::is_same_v<std::decay_t<F>, FunctionExpr>>>
  FunctionExpr(const F& f) {  // NOLINT (converting, like function_base.h:210)
    static_assert(static_cast<int>(F::Differentiability) >= static_cast<int>(TMode),
                  "Differentiability mode mismatch: source must supply at least as much derivative information "
                  "as the target mode requires (downgrades are accepted, upgrades are not).");
    static_assert(std::is_same_v<typename F::ScalarType, TScalar>, "Compile-time scalar-type mismatch");
    static_assert(TDimension == -1 || F::Dimension == TDimension, "Dimension mismatch");
    LauncherTraits<F>::Bind(f, *this);
    dimension = F::Dimension;
    problem.mode = static_cast<int>(TMode);
  }
  int mode() const { return static_cast<int>(TMode); }

  // function_base.h:247-250 with a batch axis: value [B] (and gradient [B, d]) of the bound function at
  // x [B, d]; all three are device arrays.
  void operator()(int64_t batch, const TScalar* x, TScalar* value, TScalar* gradient = nullptr,
                  cudaStream_t stream = nullptr) const {
    const int rc = raw_evaluate ? raw_evaluate(pod.data(), batch, x, value, gradient, stream)
                                : cno_evaluate(&problem, batch, x, value, gradient, stream);
    detail::check_cno(rc, "FunctionExpr::operator()");
  }

  // Progress::condition_hessian (solver/progress.h:203-210) on request: condition[b] = H(x_b).norm() *
  // H(x_b).inverse().norm() for x [B, d] -- the value the reference's Progress::Update computes at every
  // iteration of a Second-mode function.  On the x a solve returned it is the reference's final
  // progress.condition_hessian.  Device arrays; built-in Second-mode families (cno_condition_hessian).
  void ConditionHessian(int64_t batch, const TScalar* x, TScalar* condition, cudaStream_t stream = nullptr) const {
    static_assert(TMode == DifferentiabilityMode::Second, "condition_hessian is defined for Second-mode functions");
    detail::DeviceArray<unsigned long long> ws(32);
    const size_t wsb = ws.size() * sizeof(unsigned long long);
    const int rc = raw ? (raw_condition ? raw_condition(pod.data(), batch, x, condition, ws.data(), wsb, stream) : CNO_ERR_UNSUPPORTED)
                       : cno_condition_hessian(&problem, batch, x, condition, ws.data(), wsb, stream);
    detail::check_cno(rc, "FunctionExpr::ConditionHessian");
    detail::check_cuda(cudaStreamSynchronize(stream), "FunctionExpr::ConditionHessian");
  }
};

// function_base.h:298-332 as in the reference: one instance, host vectors (the B = 1 signature of
// Solver::Minimize takes and returns it).
template <class TScalar, int TDimension>
struct FunctionState {
  using ScalarType = TScalar;
  static constexpr bool IsConstrained = false;
  std::vector<TScalar> x;
  TScalar value = TScalar(0);
  std::vector<TScalar> gradient;
  FunctionState() = default;
  explicit FunctionState(const std::vector<TScalar>& x_) : x(x_) {  // "legacy x-only constructor" (:315)
    if (static_cast<int>(x.size()) != TDimension) throw std::runtime_error("x must have Dimension entries");
  }
};

// FunctionState with a batch axis (function_base.h:298-332): x [B, d] row-major,
// value [B], gradient [B, d], all on the device.
template <class TScalar, int TDimension>
struct BatchedFunctionState {
  using ScalarType = TScalar;
  static constexpr bool IsConstrained = false;
  int64_t batch = 0;
  detail::DeviceArray<TScalar> x, value, gradient;

  BatchedFunctionState() = default;
  // "legacy x-only constructor" (:315): Minimize evaluates the function itself.
  static BatchedFunctionState FromHost(const std::vector<TScalar>& x_host, int64_t batch) {
    if ((int64_t)x_host.size() != batch * TDimension) throw std::runtime_error("x0 must be [B, d]");
    BatchedFunctionState s;
    s.batch = batch;
    s.x = detail::DeviceArray<TScalar>::FromHost(x_host);
    return s;
  }
};

// ---- objective families compiled into libcno.so --------------------------------
// In nvcc translation units (device.cuh) the tags are also DEVICE functors (they forward to the
// functors of csrc/cno_functors.cuh), so they can be operands of the expression templates
// (expressions.h): decltype(Rosenbrock<double, 8>{} + 0.5 * HalfSquaredNorm<double, 8>{}).
#ifdef CPPOPTLIB_B200_WITH_DEVICE
#define CNO_BUILTIN_DEVICE_MEMBERS(...)                                                                           \
  using DeviceFn = __VA_ARGS__;                                                                                   \
  static constexpr int E = cno::Shape<DeviceFn::Dim>::E;                                                          \
  __device__ __forceinline__ typename DeviceFn::Scalar operator()(const cno::EvalCtx& c,                          \
                                                                  const typename DeviceFn::Scalar (&x)[E],        \
                                                                  typename DeviceFn::Scalar (*grad)[E]) const {   \
    return DeviceFn{}(c, x, grad);                                                                                \
  }                                                                                                               \
  __device__ __forceinline__ void hess_diag(const cno::EvalCtx& c, const typename DeviceFn::Scalar (&x)[E],       \
                                            typename DeviceFn::Scalar (&h)[E]) const {                            \
    DeviceFn{}.hess_diag(c, x, h);                                                                                \
  }                                                                                                               \
  __device__ __forceinline__ void hess_col(const cno::EvalCtx& c, const typename DeviceFn::Scalar (&x)[E], int j, \
                                           bool transposed, typename DeviceFn::Scalar (&col)[E]) const {          \
    DeviceFn{}.hess_col(c, x, j, transposed, col);                                                                \
  }
#else
#define CNO_BUILTIN_DEVICE_MEMBERS(...)
#endif
template <class T, int D>
struct Rosenbrock : FunctionCRTP<Rosenbrock<T, D>, T, DifferentiabilityMode::First, D> {
  CNO_BUILTIN_DEVICE_MEMBERS(cno::RosenbrockFn<T, D>)
};
template <class T, int D>
struct RosenbrockFull : FunctionCRTP<RosenbrockFull<T, D>, T, DifferentiabilityMode::Second, D> {
  CNO_BUILTIN_DEVICE_MEMBERS(cno::RosenbrockFn<T, D>)
};
template <class T>
struct DiagQuadratic : FunctionCRTP<DiagQuadratic<T>, T, DifferentiabilityMode::First, 2> {
  CNO_BUILTIN_DEVICE_MEMBERS(cno::DiagQuadraticFn<T>)
};
template <class T, int D>
struct HalfSquaredNorm : FunctionCRTP<HalfSquaredNorm<T, D>, T, DifferentiabilityMode::First, D> {
  CNO_BUILTIN_DEVICE_MEMBERS(cno::HalfSquaredNormFn<T, D>)
};
// The Second-mode twins of the two families above (function_base.h:96-126 with Mode = Second), for
// composites that need Hessians (NewtonDescent, Lbfgs's preconditioner branch).
template <class T>
struct DiagQuadraticSecond : FunctionCRTP<DiagQuadraticSecond<T>, T, DifferentiabilityMode::Second, 2> {
  CNO_BUILTIN_DEVICE_MEMBERS(cno::DiagQuadraticFn<T>)
};
template <class T, int D>
struct HalfSquaredNormSecond : FunctionCRTP<HalfSquaredNormSecond<T, D>, T, DifferentiabilityMode::Second, D> {
  CNO_BUILTIN_DEVICE_MEMBERS(cno::HalfSquaredNormFn<T, D>)
};
// 0.5 x'Ax - b'x; data[b] = [A (d x d col-major, symmetric) | b] on the device.
template <class T, int D>
struct DenseQuadratic : FunctionCRTP<DenseQuadratic<T, D>, T, DifferentiabilityMode::Second, D> {
  const T* data = nullptr;
  int64_t data_stride = 0;
  // -1 = the default arithmetic of the dtype; CNO_POLICY_DMMA_LU (D = 64, double): NewtonDescent's factorisation with
  // fused multiply-subtracts, the trailing update on the FP64 tensor core (include/cno.h)
  int policy = -1;
};

namespace detail_builtin {
template <class T, int D>
inline cno_problem_t make(int family) {
  cno_problem_t p{};
  p.family = family;
  p.dtype = detail::DType<T>::value;
  p.d = D;
  p.policy = std::is_same_v<T, double> ? CNO_POLICY_DMMA_TREE : CNO_POLICY_WARP_TREE;
  return p;
}
}  // namespace detail_builtin

template <class T, int D>
struct LauncherTraits<Rosenbrock<T, D>> {
  template <class E> static void Bind(const Rosenbrock<T, D>&, E& e) { e.problem = detail_builtin::make<T, D>(CNO_FN_ROSENBROCK); }
};
template <class T, int D>
struct LauncherTraits<RosenbrockFull<T, D>> {
  template <class E> static void Bind(const RosenbrockFull<T, D>&, E& e) {
    e.problem = detail_builtin::make<T, D>(CNO_FN_ROSENBROCK);
    e.problem.mode = 2;  // Second mode: Lbfgs takes its diagonal-preconditioner branch (lbfgs.h:116-139)
  }
};
template <class T>
struct LauncherTraits<DiagQuadratic<T>> {
  template <class E> static void Bind(const DiagQuadratic<T>&, E& e) { e.problem = detail_builtin::make<T, 2>(CNO_FN_DIAG_QUADRATIC); }
};
template <class T, int D>
struct LauncherTraits<HalfSquaredNorm<T, D>> {
  template <class E> static void Bind(const HalfSquaredNorm<T, D>&, E& e) { e.problem = detail_builtin::make<T, D>(CNO_FN_HALF_SQUARED_NORM); }
};
template <class T, int D>
struct LauncherTraits<DenseQuadratic<T, D>> {
  template <class E> static void Bind(const DenseQuadratic<T, D>& f, E& e) {
    e.problem = detail_builtin::make<T, D>(CNO_FN_DENSE_QUADRATIC);
    e.problem.data = f.data;
    e.problem.data_stride = f.data_stride;
    if (f.policy >= 0) e.problem.policy = f.policy;
  }
};

}  // namespace function

namespace solver {

enum class Status {  // solver/progress.h:37-47
  NotStarted = -1, Continue = 0, IterationLimit, XDeltaViolation, FDeltaViolation,
  GradientNormViolation, HessianConditionViolation, Finished
};

// Stopping thresholds (solver/progress.h:82-140; same field names).
template <class FunctionType = void, class StateType = void>
struct Progress {
  size_t num_iterations = 0;
  double x_delta = 0;
  int x_delta_violations = 0;
  double f_delta = 0;
  int f_delta_violations = 0;
  bool f_delta_relative = false;
  double gradient_norm = 0;
  bool gradient_norm_relative = true;
  double condition_hessian = 0;
  int past = 0;
  double past_delta = 1e-6;
  Status status = Status::NotStarted;

  cno_stop_t to_c() const {
    cno_stop_t s{};
    s.num_iterations = num_iterations;
    s.x_delta = x_delta;
    s.x_delta_violations = x_delta_violations;
    s.f_delta = f_delta;
    s.f_delta_violations = f_delta_violations;
    s.f_delta_relative = f_delta_relative;
    s.gradient_norm = gradient_norm;
    s.gradient_norm_relative = gradient_norm_relative;
    s.condition_hessian = condition_hessian;
    s.past = past;
    s.past_delta = past_delta;
    return s;
  }
  static Progress from_c(const cno_stop_t& s) {
    Progress p;
    p.num_iterations = s.num_iterations;
    p.x_delta = s.x_delta;
    p.x_delta_violations = s.x_delta_violations;
    p.f_delta = s.f_delta;
    p.f_delta_violations = s.f_delta_violations;
    p.f_delta_relative = s.f_delta_relative != 0;
    p.gradient_norm = s.gradient_norm;
    p.gradient_norm_relative = s.gradient_norm_relative != 0;
    p.condition_hessian = s.condition_hessian;
    p.past = s.past;
    p.past_delta = s.past_delta;
    return p;
  }
};

template <class FunctionType = void, class StateType = void>
Progress<FunctionType, StateType> DefaultStoppingSolverProgress() {  // solver/progress.h:353-431
  cno_stop_t s;
  cno_default_stop(&s);
  return Progress<FunctionType, StateType>::from_c(s);
}
template <class FunctionType = void, class StateType = void>
Progress<FunctionType, StateType> ConservativeStoppingSolverProgress() {  // :456-464
  cno_stop_t s;
  cno_conservative_stop(&s);
  return Progress<FunctionType, StateType>::from_c(s);
}

// Per-instance Progress values (device arrays).
template <class T>
struct BatchedProgress {
  int64_t batch = 0;
  detail::DeviceArray<uint32_t> num_iterations, nfev;
  detail::DeviceArray<int8_t> status;
  detail::DeviceArray<T> x_delta, f_delta, gradient_norm;
  cno_launch_info_t launch{};
};

// solver/solver.h:156-231 with a batch axis.
template <class FunctionTypeT, int SolverId>
class Solver {
 public:
  using FunctionType = FunctionTypeT;
  using ScalarType = typename FunctionType::ScalarType;
  using StateType = function::BatchedFunctionState<ScalarType, FunctionType::Dimension>;
  using ProgressType = Progress<FunctionType, StateType>;

  using CallbackType =
      std::function<void(const FunctionType&, const StateType&, const BatchedProgress<ScalarType>&)>;

  ProgressType stopping_progress;

  explicit Solver(const ProgressType& progress = DefaultStoppingSolverProgress<FunctionType, StateType>())
      : stopping_progress(progress) {}
  virtual ~Solver() = default;

  // solver/solver.h:176.  The callback runs on the host after every `every` iterations:
  // Minimize then proceeds in rounds (cno_minimize_steps, solver state parked on the device
  // in between) -- the same trajectory, bit for bit, as the fused solve.
  void SetCallback(CallbackType callback, int every = 1) {
    step_callback_ = std::move(callback);
    callback_every_ = every < 1 ? 1 : every;
  }

  // Batched Minimize: returns {state at the solution, per-instance progress}.
  virtual std::tuple<StateType, BatchedProgress<ScalarType>> Minimize(const FunctionType& function,
                                                                      const StateType& function_state,
                                                                      cudaStream_t stream = nullptr) {
    using T = ScalarType;
    constexpr int D = FunctionType::Dimension;
    const int64_t B = function_state.batch;
    function::FunctionExpr<T, FunctionType::Differentiability, D> expr(function);
    expr.problem.lbfgs_m = lbfgs_m();

    StateType result;
    result.batch = B;
    result.x = detail::DeviceArray<T>(B * D);
    result.gradient = detail::DeviceArray<T>(B * D);
    result.value = detail::DeviceArray<T>(B);
    BatchedProgress<T> prog;
    prog.batch = B;
    prog.num_iterations = detail::DeviceArray<uint32_t>(B);
    prog.nfev = detail::DeviceArray<uint32_t>(B);
    prog.status = detail::DeviceArray<int8_t>(B);
    prog.x_delta = detail::DeviceArray<T>(B);
    prog.f_delta = detail::DeviceArray<T>(B);
    prog.gradient_norm = detail::DeviceArray<T>(B);

    cno_batch_out_t out{};
    out.x = result.x.data();
    out.value = result.value.data();
    out.gradient = result.gradient.data();
    out.num_iterations = prog.num_iterations.data();
    out.status = prog.status.data();
    out.nfev = prog.nfev.data();
    out.x_delta = prog.x_delta.data();
    out.f_delta = prog.f_delta.data();
    out.gradient_norm = prog.gradient_norm.data();

    detail::DeviceArray<unsigned char> workspace(256);
    const cno_stop_t stop = stopping_progress.to_c();
    int rc;
    if (step_callback_) {
      // solver.h:197 per-iteration callback: rounds of `callback_every_` iterations, the solver's members
      // parked on the device in between.  A (solver, function) pair without a stepwise kernel THROWS
      // (CNO_ERR_UNSUPPORTED) -- the callback is never silently dropped.
      if (expr.raw && (!expr.raw_steps || !expr.raw_state_bytes))
        throw std::runtime_error("SetCallback: this function has no stepwise launcher (CNO_DECLARE_FUNCTION)");
      size_t nbytes = 0;
      detail::check_cno(expr.raw ? expr.raw_state_bytes(SolverId, B, &nbytes)
                                 : cno_state_bytes(SolverId, &expr.problem, B, &nbytes),
                        "SetCallback (stepwise solves: cno_state_bytes)");
      detail::DeviceArray<unsigned char> state(nbytes < 16 ? 16 : nbytes);
      for (int first = 1;; first = 0) {
        rc = expr.raw ? expr.raw_steps(SolverId, expr.mode(), lbfgs_m(), expr.pod.data(), B, function_state.x.data(), &stop, &out,
                                       state.data(), state.size(), callback_every_, first, workspace.data(),
                                       workspace.size(), stream, nullptr)
                      : cno_minimize_steps(SolverId, &expr.problem, B, function_state.x.data(), &stop, &out,
                                           state.data(), state.size(), callback_every_, first, workspace.data(),
                                           workspace.size(), stream, nullptr);
        detail::check_cno(rc, "cno_minimize_steps");
        detail::check_cuda(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
        step_callback_(function, result, prog);
        bool done = true;
        for (int8_t s : prog.status.ToHost()) done = done && (s != CNO_STATUS_CONTINUE);
        if (done) break;
      }
      return {std::move(result), std::move(prog)};
    }
    if (expr.raw) {
      rc = expr.raw(SolverId, expr.mode(), lbfgs_m(), expr.pod.data(), B, function_state.x.data(), &stop, &out,
                    workspace.data(), workspace.size(), stream, &prog.launch);
    } else {
      rc = cno_minimize(SolverId, &expr.problem, B, function_state.x.data(), &stop, &out,
                        workspace.data(), workspace.size(), stream, &prog.launch);
    }
    detail::check_cno(rc, "Minimize");
    return {std::move(result), std::move(prog)};
  }

  // Multi-GPU Minimize (SURVEY.md 8(e)): one process (or thread) per GPU, the batch sharded contiguously.  This
  // rank's shard advances `every` iterations per round (cno_minimize_steps); after each round the ranks'
  // convergence bitmaps are all-gathered -- the ONE NCCL collective of the path (cno_allgather_done) -- and all
  // ranks leave the loop together once every instance of every shard has terminated.  `nccl_comm` is the caller's
  // ncclComm_t (one rank per GPU); shard_sizes[r] = instances of rank r.  Results per instance are bit-identical to
  // an unsharded Minimize.
  std::tuple<StateType, BatchedProgress<ScalarType>> MinimizeSharded(const FunctionType& function,
                                                                     const StateType& shard_state, void* nccl_comm,
                                                                     int rank, const std::vector<int64_t>& shard_sizes,
                                                                     int every = 64, cudaStream_t stream = nullptr) {
    using T = ScalarType;
    constexpr int D = FunctionType::Dimension;
    const int world = static_cast<int>(shard_sizes.size());
    if (rank < 0 || rank >= world || shard_sizes[rank] != shard_state.batch)
      throw std::invalid_argument("MinimizeSharded: shard_sizes[rank] must equal the shard's batch");
    const int64_t B = shard_state.batch;
    int64_t max_shard = 0, global = 0;
    for (int64_t n : shard_sizes) { max_shard = n > max_shard ? n : max_shard; global += n; }
    const size_t words = static_cast<size_t>((max_shard + 31) / 32);
    function::FunctionExpr<T, FunctionType::Differentiability, D> expr(function);
    expr.problem.lbfgs_m = lbfgs_m();
    if (expr.raw && (!expr.raw_steps || !expr.raw_state_bytes))
      throw std::runtime_error("MinimizeSharded: this function has no stepwise launcher");

    StateType result;
    result.batch = B;
    result.x = detail::DeviceArray<T>(B * D);
    result.gradient = detail::DeviceArray<T>(B * D);
    result.value = detail::DeviceArray<T>(B);
    BatchedProgress<T> prog;
    prog.batch = B;
    prog.num_iterations = detail::DeviceArray<uint32_t>(B);
    prog.nfev = detail::DeviceArray<uint32_t>(B);
    prog.status = detail::DeviceArray<int8_t>(B);
    prog.x_delta = detail::DeviceArray<T>(B);
    prog.f_delta = detail::DeviceArray<T>(B);
    prog.gradient_norm = detail::DeviceArray<T>(B);
    cno_batch_out_t out{};
    out.x = result.x.data();
    out.value = result.value.data();
    out.gradient = result.gradient.data();
    out.num_iterations = prog.num_iterations.data();
    out.status = prog.status.data();
    out.nfev = prog.nfev.data();
    out.x_delta = prog.x_delta.data();
    out.f_delta = prog.f_delta.data();
    out.gradient_norm = prog.gradient_norm.data();

    detail::DeviceArray<unsigned char> workspace(256);
    auto local = detail::DeviceArray<uint32_t>::FromHost(std::vector<uint32_t>(words, 0u));
    detail::DeviceArray<uint32_t> all(words * static_cast<size_t>(world));
    const cno_stop_t stop = stopping_progress.to_c();
    size_t nbytes = 0;
    detail::check_cno(expr.raw ? expr.raw_state_bytes(SolverId, B, &nbytes)
                               : cno_state_bytes(SolverId, &expr.problem, B, &nbytes),
                      "MinimizeSharded (stepwise solves: cno_state_bytes)");
    detail::DeviceArray<unsigned char> state(nbytes < 16 ? 16 : nbytes);
    int rounds = 0;
    for (int first = 1;; first = 0) {
      const int rc =
          expr.raw ? expr.raw_steps(SolverId, expr.mode(), lbfgs_m(), expr.pod.data(), B, shard_state.x.data(), &stop, &out,
                                    state.data(), state.size(), every, first, workspace.data(), workspace.size(), stream,
                                    nullptr)
                   : cno_minimize_steps(SolverId, &expr.problem, B, shard_state.x.data(), &stop, &out, state.data(),
                                        state.size(), every, first, workspace.data(), workspace.size(), stream, nullptr);
      detail::check_cno(rc, "cno_minimize_steps");
      ++rounds;
      detail::check_cno(cno_done_bitmap(prog.status.data(), B, local.data(), stream), "cno_done_bitmap");
      detail::check_cno(cno_allgather_done(nccl_comm, local.data(), all.data(), words, stream), "cno_allgather_done");
      int64_t done = 0;
      detail::check_cno(cno_count_done(all.data(), world, words, shard_sizes.data(), &done, stream), "cno_count_done");
      if (done == global) break;  // the same count on every rank: all leave together
    }
    prog.launch.kernel_launches = rounds;
    return {std::move(result), std::move(prog)};
  }

  // The reference's own signature (solver.h:181-182): ONE problem instance, host vectors in and out.
  // A batch of one through the same kernels (C1 plumbing: `Lbfgs<F> s; auto [sol, prog] = s.Minimize(f, FunctionState(x0));`).
  std::tuple<function::FunctionState<ScalarType, FunctionType::Dimension>, ProgressType> Minimize(
      const FunctionType& function, const function::FunctionState<ScalarType, FunctionType::Dimension>& initial) {
    auto [state, prog] = Minimize(function, StateType::FromHost(initial.x, 1), nullptr);
    function::FunctionState<ScalarType, FunctionType::Dimension> sol;
    sol.x = state.x.ToHost();
    sol.gradient = state.gradient.ToHost();
    sol.value = state.value.ToHost()[0];
    ProgressType p = stopping_progress;  // thresholds stay; the counters are the run's
    p.num_iterations = prog.num_iterations.ToHost()[0];
    p.x_delta = prog.x_delta.ToHost()[0];
    p.f_delta = prog.f_delta.ToHost()[0];
    p.gradient_norm = prog.gradient_norm.ToHost()[0];
    p.status = static_cast<Status>(prog.status.ToHost()[0]);
    return {std::move(sol), p};
  }

 protected:
  virtual int lbfgs_m() const { return 0; }  // Lbfgs<F, m>: pairs kept (0 = not an L-BFGS solver / the default)
  CallbackType step_callback_;
  int callback_every_ = 1;
};

// solver/solver.h:59-130 with a batch axis: prints the reference's per-iteration block (label
// width 18, numeric width 15, fixed 6 decimals; vectors through Eigen's default IOFormat) for ONE
// instance of the batch and a line summarising the batch.  Use with
//   solver.SetCallback(PrintProgressCallback<F>(std::cout), /*every=*/K);
// each call reads that instance's row and the status array back from the device.
template <class FunctionType>
auto PrintProgressCallback(std::ostream& output_stream, int64_t instance = 0) {
  using T = typename FunctionType::ScalarType;
  using StateType = function::BatchedFunctionState<T, FunctionType::Dimension>;
  return [&output_stream, instance](const FunctionType&, const StateType& state,
                                    const BatchedProgress<T>& progress) {
    constexpr int label_width = 18, num_width = 15, precision = 6;
    constexpr size_t D = FunctionType::Dimension;
    const size_t i = static_cast<size_t>(instance);
    auto eigen_row = [](const std::vector<T>& v) {  // `ss << vector.transpose()`, default stream
      std::vector<std::string> cells;
      size_t width = 0;
      for (T c : v) {
        char buf[64];
        std::snprintf(buf, sizeof(buf), "%g", static_cast<double>(c));
        cells.emplace_back(buf);
        if (cells.back().size() > width) width = cells.back().size();
      }
      std::string row;
      for (size_t k = 0; k < cells.size(); ++k)
        row += (k ? " " : "") + std::string(width - cells[k].size(), ' ') + cells[k];
      return row;
    };
    std::ostream& os = output_stream;
    os << std::fixed << std::setprecision(precision);
    os << "--- Iteration: " << std::setw(5) << std::right << progress.num_iterations.ToHost(i, 1)[0] << " ---\n";
    if (state.value.size() > i)
      os << std::left << std::setw(label_width) << "  Value:" << std::right << std::setw(num_width)
         << state.value.ToHost(i, 1)[0] << "\n";
    os << std::left << std::setw(label_width) << "  X:" << " " << eigen_row(state.x.ToHost(i * D, D)) << "\n";
    if (state.gradient.size() >= (i + 1) * D) {
      os << std::left << std::setw(label_width) << "  Gradient:" << " " << eigen_row(state.gradient.ToHost(i * D, D)) << "\n";
      os << std::left << std::setw(label_width) << "  Gradient Norm:" << std::right << std::setw(num_width)
         << progress.gradient_norm.ToHost(i, 1)[0] << "\n";
    }
    os << std::left << std::setw(label_width) << "  X Delta:" << std::right << std::setw(num_width)
       << progress.x_delta.ToHost(i, 1)[0] << "\n";
    os << std::left << std::setw(label_width) << "  F Delta:" << std::right << std::setw(num_width)
       << progress.f_delta.ToHost(i, 1)[0] << "\n";
    if (FunctionType::Differentiability == function::DifferentiabilityMode::Second)
      os << std::left << std::setw(label_width) << "  Hessian Cond.:" << std::right << std::setw(num_width) << "N/A"
         << "\n";  // not computed (DESIGN.md 2.3)
    size_t running = 0;
    for (int8_t st : progress.status.ToHost()) running += (st == static_cast<int8_t>(Status::Continue));
    os << std::left << std::setw(label_width) << "  Batch:" << " " << running << " of " << progress.batch
       << " instances still running\n";
    os << "-------------------------" << std::endl;
  };
}

// The LineSearch policies (linesearch/more_thuente.h, linesearch/hager_zhang.h:54-552).  The
// reference takes them as `template <class, int> class LineSearch`; here they are tags that
// select the kernel compiled with that search (C ABI solver ids CNO_*_HAGER_ZHANG).
namespace linesearch {
struct MoreThuente {
  static constexpr int solver_id(int base) { return base; }
};
struct HagerZhang {
  static constexpr int solver_id(int base) {
    return base == CNO_LBFGS ? CNO_LBFGS_HAGER_ZHANG
                             : (base == CNO_BFGS ? CNO_BFGS_HAGER_ZHANG : CNO_GRADIENT_DESCENT_HAGER_ZHANG);
  }
};
}  // namespace linesearch

// solver/lbfgs.h:40-42: Lbfgs<F, m = 10, LineSearch = MoreThuente>
// (built-in families: m = 5, 10, 20 are compiled into libcno.so; user functors: the m given to
// CNO_INSTANTIATE_FUNCTION_M -- any other combination throws CNO_ERR_UNSUPPORTED)
template <class F, int m = CNO_LBFGS_M, class LineSearch = linesearch::MoreThuente>
class Lbfgs : public Solver<F, LineSearch::solver_id(CNO_LBFGS)> {
  static_assert(m >= 1 && m <= 24, "Lbfgs<F, m>: 1 <= m <= 24");
 public:
  using Solver<F, LineSearch::solver_id(CNO_LBFGS)>::Solver;
 protected:
  int lbfgs_m() const override { return m; }
};
// solver/lbfgsb.h:44-538: Lbfgsb<F, m = 5, MoreThuente> -- L-BFGS-B (box constraints).  The constructor carries the
// reference's preset (default + f_delta = 2.22e-9 relative, :78-81); SetBounds (:88-92) takes device arrays [d]
// (one box for the batch) or [B, d].
template <class F, int m = 5>
class Lbfgsb {
  static_assert(m == 5 || m == 10, "Lbfgsb<F, m>: kernels are compiled for m = 5 (every built-in) and m = 10 (Rosenbrock)");

 public:
  using FunctionType = F;
  using ScalarType = typename F::ScalarType;
  using StateType = function::BatchedFunctionState<ScalarType, F::Dimension>;
  using ProgressType = Progress<F, StateType>;
  ProgressType stopping_progress;

  Lbfgsb() {
    cno_stop_t s;
    cno_lbfgsb_default_stop(&s);
    stopping_progress = ProgressType::from_c(s);
  }
  explicit Lbfgsb(const ProgressType& progress) : stopping_progress(progress) {}

  // lower / upper: host vectors of d (one box) or B*d (per instance) entries; empty = unbounded on that side
  void SetBounds(const std::vector<ScalarType>& lower_bound, const std::vector<ScalarType>& upper_bound) {
    lower_ = detail::DeviceArray<ScalarType>::FromHost(lower_bound);
    upper_ = detail::DeviceArray<ScalarType>::FromHost(upper_bound);
  }

  std::tuple<StateType, BatchedProgress<ScalarType>> Minimize(const F& function, const StateType& function_state,
                                                              cudaStream_t stream = nullptr) {
    using T = ScalarType;
    constexpr int D = F::Dimension;
    const int64_t B = function_state.batch;
    function::FunctionExpr<T, function::DifferentiabilityMode::First, D> expr(function);
    if (expr.raw) throw std::runtime_error("Lbfgsb: built-in objective families only");
    expr.problem.lbfgs_m = m;
    cno_bounds_t bounds{};
    bounds.lower = lower_.size() ? lower_.data() : nullptr;
    bounds.upper = upper_.size() ? upper_.data() : nullptr;
    for (size_t n : {lower_.size(), upper_.size()}) {
      if (n == 0) continue;
      if (n == static_cast<size_t>(B) * D && B != 1) bounds.stride = D;
      else if (n != static_cast<size_t>(D)) throw std::invalid_argument("SetBounds: d or B*d entries");
    }
    StateType result;
    result.batch = B;
    result.x = detail::DeviceArray<T>(B * D);
    result.gradient = detail::DeviceArray<T>(B * D);
    result.value = detail::DeviceArray<T>(B);
    BatchedProgress<T> prog;
    prog.batch = B;
    prog.num_iterations = detail::DeviceArray<uint32_t>(B);
    prog.nfev = detail::DeviceArray<uint32_t>(B);
    prog.status = detail::DeviceArray<int8_t>(B);
    prog.x_delta = detail::DeviceArray<T>(B);
    prog.f_delta = detail::DeviceArray<T>(B);
    prog.gradient_norm = detail::DeviceArray<T>(B);
    cno_batch_out_t out{};
    out.x = result.x.data();
    out.value = result.value.data();
    out.gradient = result.gradient.data();
    out.num_iterations = prog.num_iterations.data();
    out.status = prog.status.data();
    out.nfev = prog.nfev.data();
    out.x_delta = prog.x_delta.data();
    out.f_delta = prog.f_delta.data();
    out.gradient_norm = prog.gradient_norm.data();
    detail::DeviceArray<unsigned char> workspace(256);
    const cno_stop_t stop = stopping_progress.to_c();
    detail::check_cno(cno_lbfgsb_minimize(&expr.problem, &bounds, B, function_state.x.data(), &stop, &out, workspace.data(),
                                          workspace.size(), stream, &prog.launch),
                      "Lbfgsb::Minimize");
    return {std::move(result), std::move(prog)};
  }

 private:
  detail::DeviceArray<ScalarType> lower_, upper_;
};
// solver/bfgs.h:39-41: Bfgs<F, LineSearch = MoreThuente>
template <class F, class LineSearch = linesearch::MoreThuente>
class Bfgs : public Solver<F, LineSearch::solver_id(CNO_BFGS)> {
  using Solver<F, LineSearch::solver_id(CNO_BFGS)>::Solver;
};
template <class F> class NewtonDescent : public Solver<F, CNO_NEWTON> {
  static_assert(F::Differentiability == function::DifferentiabilityMode::Second,
                "NewtonDescent only supports second-order differentiable functions");
  using Solver<F, CNO_NEWTON>::Solver;
};
// solver/gradient_descent.h:37-75 (LineSearch = MoreThuente, the reference's default policy)
template <class F, class LineSearch = linesearch::MoreThuente>
class GradientDescent : public Solver<F, LineSearch::solver_id(CNO_GRADIENT_DESCENT)> {
  using Solver<F, LineSearch::solver_id(CNO_GRADIENT_DESCENT)>::Solver;
};
// solver/conjugated_gradient_descent.h:38-92 (Fletcher-Reeves beta, Armijo<F,1>)
template <class F> class ConjugatedGradientDescent : public Solver<F, CNO_CONJUGATED_GRADIENT_DESCENT> {
  static_assert(sizeof(typename F::ScalarType) == 8,
                "ConjugatedGradientDescent: fp64 only (the reference computes beta in double)");
  using Solver<F, CNO_CONJUGATED_GRADIENT_DESCENT>::Solver;
};


// ---- the constrained caller of the path (solver/augmented_lagrangian.h, function_problem.h) ----
// Parity: tests/cpp/al_host.cc, run on the GPU by tests/test_al_gpu.py.
}  // namespace solver

namespace function {
// function_problem.h:38-60 with the two device constraint families (include/cno_al.h):
// a constraint is a row [a (d) | t]; AFFINE c(x) = a.x - t, SQNORM c(x) = t - x.x; equalities
// (c == 0) first, then inequalities (c >= 0).  `rows` is one set shared by the batch
// ([n_con][d+1]) or per instance ([B][n_con][d+1]).
template <class Objective>
struct ConstrainedOptimizationProblem {
  using ScalarType = typename Objective::ScalarType;
  static constexpr int Dimension = Objective::Dimension;
  static constexpr DifferentiabilityMode Differentiability = Objective::Differentiability;
  Objective objective;
  std::vector<int32_t> kinds;
  std::vector<ScalarType> rows;
  int n_eq = 0;
  bool per_instance = false;
  int n_ineq() const { return static_cast<int>(kinds.size()) - n_eq; }
};
}  // namespace function

namespace solver {

template <class TScalar>
struct AugmentedLagrangianConfig {  // solver/augmented_lagrangian.h:63-239, same names and defaults
  TScalar penalty_growth_factor = TScalar{10};
  TScalar violation_shrink_ratio = TScalar{0.25};
  bool auto_scale_initial_penalty = true;
  TScalar penalty_auto_objective_scale = TScalar{10};
  TScalar penalty_auto_min = TScalar{1e-8};
  TScalar penalty_auto_max = TScalar{1e8};
  int warmup_max_inner_iterations = 10;
  TScalar warmup_inner_gradient_tolerance = TScalar{1e-2};
  TScalar multiplier_max = TScalar{1e20};
  TScalar kkt_gradient_tolerance = TScalar{1e-4};
};

// AugmentedLagrangeState (solver/augmented_lagrangian.h:241-276), one row per instance.
template <class TScalar, int TDimension>
struct BatchedAugmentedLagrangeState {
  static constexpr bool IsConstrained = true;
  int64_t batch = 0;
  detail::DeviceArray<TScalar> x, equality_multipliers, inequality_multipliers, penalty, max_violation,
      max_lagrangian_gradient;
  // (x, num_eq, num_ineq, penalty = 0): zero multipliers; penalty 0 = auto-scale (:263-275, 312-318)
  static BatchedAugmentedLagrangeState FromHost(const std::vector<TScalar>& x_host, int64_t batch, size_t num_eq,
                                                size_t num_ineq, TScalar penalty = TScalar(0)) {
    if (static_cast<int64_t>(x_host.size()) != batch * TDimension) throw std::invalid_argument("x0 must be [B, d]");
    BatchedAugmentedLagrangeState s;
    s.batch = batch;
    s.x = detail::DeviceArray<TScalar>::FromHost(x_host);
    s.equality_multipliers = detail::DeviceArray<TScalar>::FromHost(std::vector<TScalar>(batch * num_eq, TScalar(0)));
    s.inequality_multipliers = detail::DeviceArray<TScalar>::FromHost(std::vector<TScalar>(batch * num_ineq, TScalar(0)));
    s.penalty = detail::DeviceArray<TScalar>::FromHost(std::vector<TScalar>(batch, penalty));
    return s;
  }
};

// AugmentedLagrangian<Problem, Lbfgs<...>> (solver/augmented_lagrangian.h:278-449).
template <class ProblemType, class solver_t>
class AugmentedLagrangian {
 public:
  using ScalarType = typename ProblemType::ScalarType;
  using StateType = BatchedAugmentedLagrangeState<ScalarType, ProblemType::Dimension>;
  // the fields of the outer stopping_progress the constrained branch of Progress::Update reads
  struct OuterProgress {
    size_t num_iterations = 10000;
    ScalarType constraint_threshold = ScalarType(1e-5);
    ScalarType kkt_stationarity_threshold = ScalarType(1e-4);
  } stopping_progress;

  AugmentedLagrangian(const ProblemType& problem, const solver_t& unconstrained_solver,
                      AugmentedLagrangianConfig<ScalarType> config = {})
      : problem_(problem), unconstrained_solver_template_(unconstrained_solver), config_(config) {}

  std::tuple<StateType, BatchedProgress<ScalarType>> Minimize(const StateType& state, cudaStream_t stream = nullptr) {
    using T = ScalarType;
    constexpr int D = ProblemType::Dimension;
    const int64_t B = state.batch;
    const int ne = problem_.n_eq, ni = problem_.n_ineq();
    function::FunctionExpr<T, ProblemType::Differentiability, D> expr(problem_.objective);
    if (expr.raw) throw std::runtime_error("AugmentedLagrangian: built-in objective families only");
    auto kinds = detail::DeviceArray<int32_t>::FromHost(problem_.kinds);
    auto rows = detail::DeviceArray<T>::FromHost(problem_.rows);
    cno_constraints_t k{};
    k.n_eq = ne;
    k.n_ineq = ni;
    k.kinds = kinds.data();
    k.data = rows.data();
    k.data_stride = problem_.per_instance ? static_cast<int64_t>(problem_.kinds.size()) * (D + 1) : 0;

    StateType result;
    result.batch = B;
    result.x = detail::DeviceArray<T>(B * D);
    result.equality_multipliers = detail::DeviceArray<T>(B * ne);
    result.inequality_multipliers = detail::DeviceArray<T>(B * ni);
    result.penalty = detail::DeviceArray<T>(B);
    result.max_violation = detail::DeviceArray<T>(B);
    result.max_lagrangian_gradient = detail::DeviceArray<T>(B);
    BatchedProgress<T> prog;
    prog.batch = B;
    prog.num_iterations = detail::DeviceArray<uint32_t>(B);
    prog.nfev = detail::DeviceArray<uint32_t>(B);
    prog.status = detail::DeviceArray<int8_t>(B);
    prog.x_delta = detail::DeviceArray<T>(B);
    prog.f_delta = detail::DeviceArray<T>(B);
    prog.gradient_norm = detail::DeviceArray<T>(B);
    cno_al_out_t out{};
    out.x = result.x.data();
    out.equality_multipliers = result.equality_multipliers.data();
    out.inequality_multipliers = result.inequality_multipliers.data();
    out.penalty = result.penalty.data();
    out.max_violation = result.max_violation.data();
    out.max_lagrangian_gradient = result.max_lagrangian_gradient.data();
    out.num_iterations = prog.num_iterations.data();
    out.status = prog.status.data();
    out.nfev = prog.nfev.data();
    out.x_delta = prog.x_delta.data();
    out.f_delta = prog.f_delta.data();
    out.gradient_norm = prog.gradient_norm.data();

    size_t nbytes = 0;
    detail::check_cno(cno_al_workspace_bytes(&expr.problem, &k, B, &nbytes), "cno_al_workspace_bytes");
    detail::DeviceArray<unsigned char> workspace(nbytes < 256 ? 256 : nbytes);
    const cno_stop_t inner = unconstrained_solver_template_.stopping_progress.to_c();
    cno_al_stop_t outer{};
    outer.num_iterations = stopping_progress.num_iterations;
    outer.constraint_threshold = stopping_progress.constraint_threshold;
    outer.kkt_stationarity_threshold = stopping_progress.kkt_stationarity_threshold;
    cno_al_config_t cfg{};
    cfg.penalty_growth_factor = config_.penalty_growth_factor;
    cfg.violation_shrink_ratio = config_.violation_shrink_ratio;
    cfg.auto_scale_initial_penalty = config_.auto_scale_initial_penalty;
    cfg.penalty_auto_objective_scale = config_.penalty_auto_objective_scale;
    cfg.penalty_auto_min = config_.penalty_auto_min;
    cfg.penalty_auto_max = config_.penalty_auto_max;
    cfg.warmup_max_inner_iterations = config_.warmup_max_inner_iterations;
    cfg.warmup_inner_gradient_tolerance = config_.warmup_inner_gradient_tolerance;
    cfg.multiplier_max = config_.multiplier_max;
    cfg.kkt_gradient_tolerance = config_.kkt_gradient_tolerance;
    detail::check_cno(
        cno_al_minimize(&expr.problem, &k, B, state.x.data(),
                        ne ? state.equality_multipliers.data() : nullptr,
                        ni ? state.inequality_multipliers.data() : nullptr, state.penalty.data(), &inner, &outer, &cfg,
                        &out, workspace.data(), workspace.size(), stream, &prog.launch),
        "cno_al_minimize");
    return {std::move(result), std::move(prog)};
  }

 private:
  ProblemType problem_;
  solver_t unconstrained_solver_template_;
  AugmentedLagrangianConfig<ScalarType> config_;
};

}  // namespace solver
}  // namespace cppoptlib

// Declares (for a host translation unit) the extern "C" launchers that
// CNO_INSTANTIATE_FUNCTION(tag, F) defines in an nvcc translation unit, and
// binds F to them.
#define CNO_DECLARE_FUNCTION(tag, F)                                                                             \
  extern "C" int cno_##tag##_minimize(int solver, int mode, int lbfgs_m, const void* functor_bytes, int64_t batch, \
                                      const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out,         \
                                      void* workspace, size_t workspace_bytes, void* stream,                      \
                                      cno_launch_info_t* info);                                                   \
  extern "C" int cno_##tag##_state_bytes(int solver, int64_t batch, size_t* bytes);                               \
  extern "C" int cno_##tag##_minimize_steps(int solver, int mode, int lbfgs_m, const void* functor_bytes, int64_t batch, \
                                            const void* x0, const cno_stop_t* stop,                               \
                                            const cno_batch_out_t* out, void* state, size_t state_bytes,          \
                                            int32_t max_iterations, int32_t first_call, void* workspace,          \
                                            size_t workspace_bytes, void* stream, cno_launch_info_t* info);       \
  extern "C" int cno_##tag##_evaluate(const void* functor_bytes, int64_t batch, const void* x, void* value,       \
                                      void* gradient, void* stream);                                              \
  extern "C" int cno_##tag##_condition_hessian(const void* functor_bytes, int64_t batch, const void* x,           \
                                               void* condition, void* workspace, size_t workspace_bytes,         \
                                               void* stream);                                                    \
  namespace cppoptlib::function {                                                                                 \
  template <>                                                                                                     \
  struct LauncherTraits<F> {                                                                                      \
    template <class E>                                                                                            \
    static void Bind(const F& f, E& e) {                                                                          \
      static_assert(std::is_trivially_copyable_v<F>, "device functors are passed by value");                     \
      e.raw = &cno_##tag##_minimize;                                                                              \
      e.raw_state_bytes = &cno_##tag##_state_bytes;                                                               \
      e.raw_steps = &cno_##tag##_minimize_steps;                                                                  \
      e.raw_evaluate = &cno_##tag##_evaluate;                                                                     \
      e.raw_condition = &cno_##tag##_condition_hessian;                                                           \
      e.pod.assign(reinterpret_cast<const unsigned char*>(&f),                                                   \
                   reinterpret_cast<const unsigned char*>(&f) + sizeof(F));                                      \
    }                                                                                                             \
  };                                                                                                              \
  }

#include "expressions.h"

#endif  // CPPOPTLIB_B200_CPPOPTLIB_H_
