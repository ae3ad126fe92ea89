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
// This is the "thin extern-C layer": one symbol set per instantiated functor (SURVEY.md 8(b)), behind
// which Lbfgs / Bfgs / NewtonDescent / GradientDescent / ConjugatedGradientDescent<MyF>::Minimize,
// SetCallback (stepwise solves) and FunctionExpr::operator() launch the same persistent kernels as the
// built-in families:
//   cno_<tag>_minimize        Solver::Minimize                    (solver.h:181-224)
//   cno_<tag>_state_bytes /
//   cno_<tag>_minimize_steps  OptimizationStep rounds + callback  (solver.h:163-176, 226-228; Lbfgs)
//   cno_<tag>_evaluate        F::operator()(x, &grad) per instance (function_base.h:103-120)
//   cno_<tag>_condition_hessian   Progress::condition_hessian at x per instance (progress.h:203-210; Second mode)
#ifndef CPPOPTLIB_B200_DEVICE_CUH_
#define CPPOPTLIB_B200_DEVICE_CUH_

#ifdef CPPOPTLIB_B200_CPPOPTLIB_H_
#error "include cppoptlib_b200/device.cuh BEFORE cppoptlib_b200/cppoptlib.h in nvcc translation units"
#endif
#include "cno_device.cuh"
#include "cno_functors.cuh"
#define CPPOPTLIB_B200_WITH_DEVICE 1
#include "cppoptlib.h"
#include "expressions.h"
#include "cno_bfgs.cuh"
#include "cno_descent.cuh"
#include "cno_evaluate.cuh"
#include "cno_lbfgs.cuh"
#include "cno_newton.cuh"

namespace cno {
template <class Fn, class Smem, class Kernel, class... Extra>
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
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return CNO_ERR_NO_DEVICE;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t smem = Smem::kWarpBytes * Smem::kWarps;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return CNO_ERR_CUDA;
  long long ctas = (batch + Smem::kWarps - 1) / Smem::kWarps;
  const int grid = (int)(ctas < sms ? ctas : sms);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(workspace, 0, 8, s);
  struct Event {  // released on every return path
    cudaEvent_t e = nullptr;
    ~Event() { if (e) cudaEventDestroy(e); }
  } e0, e1;
  if (info) {
    if (cudaEventCreate(&e0.e) != cudaSuccess || cudaEventCreate(&e1.e) != cudaSuccess) return CNO_ERR_CUDA;
    cudaEventRecord(e0.e, s);
  }
  kernel<<<grid, Smem::kWarps * 32, smem, s>>>(fn, static_cast<const T*>(x0), (long long)batch,
                                               make_stop<T>(*stop), make_out<T>(*out),
                                               static_cast<unsigned long long*>(workspace), extra...);
  if (cudaGetLastError() != cudaSuccess) return CNO_ERR_CUDA;
  if (info) {
    cudaEventRecord(e1.e, s);
    if (cudaEventSynchronize(e1.e) != cudaSuccess) return CNO_ERR_CUDA;
    cudaEventElapsedTime(&info->kernel_ms, e0.e, e1.e);
    info->total_ms = info->kernel_ms;
    info->kernel_launches = 1;
    info->grid = grid;
    info->block = Smem::kWarps * 32;
    info->warps_per_cta = Smem::kWarps;
    info->dynamic_smem = (int64_t)smem;
  }
  return CNO_OK;
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

template <class F, class LS>
inline int user_bfgs(const F& fn, int64_t batch, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out,
                     void* workspace, size_t workspace_bytes, void* stream, cno_launch_info_t* info) {
  if constexpr (F::Dim <= 32) {  // the register-resident inverse Hessian (cno_bfgs.cuh)
    return launch_user<F, BfgsSmem<typename F::Scalar, F::Dim>>(bfgs_minimize_kernel<F, LS>, fn, batch, x0, stop, out,
                                                                 workspace, workspace_bytes, stream, info);
  } else {  // the inverse Hessian in shared memory
    return launch_user<F, BfgsBigSmem<typename F::Scalar, F::Dim>>(bfgs_smem_minimize_kernel<F, LS>, fn, batch, x0, stop,
                                                                    out, workspace, workspace_bytes, stream, info);
  }
}

template <class F>
inline int user_newton(const F& fn, int64_t batch, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out,
                       void* workspace, size_t workspace_bytes, void* stream, cno_launch_info_t* info) {
  if constexpr (F::Mode == 2 && HasHessCol<F>::value) {
    using A = SecondOrderAdapter<F>;
    if (stop && stop->condition_hessian > 0) return CNO_ERR_UNSUPPORTED;
    return launch_user<A, NewtonSmem<typename F::Scalar, F::Dim>>(newton_minimize_kernel<A>, A{fn}, batch, x0, stop, out,
                                                                   workspace, workspace_bytes, stream, info);
  } else {
    return CNO_ERR_UNSUPPORTED;  // NewtonDescent only supports second-order differentiable functions
  }
}

// Progress::condition_hessian on request (solver/progress.h:203-210; csrc/cno_newton.cuh: condition_hessian_kernel) for a
// Second-mode user functor or composite: H(x) through hess_col, as NewtonDescent stages it.
template <class F>
inline int user_condition(const F& fn, int64_t batch, const void* x, void* condition, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if constexpr (F::Mode == 2 && HasHessCol<F>::value) {
    using A = SecondOrderAdapter<F>;
    using T = typename F::Scalar;
    using CS = ConditionSmem<T, F::Dim>;
    if (batch < 0) return CNO_ERR_INVALID_ARGUMENT;
    if (batch == 0) return CNO_OK;
    if (!x || !condition || !workspace || workspace_bytes < sizeof(unsigned long long) || ((uintptr_t)workspace & 7))
      return CNO_ERR_INVALID_ARGUMENT;
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return CNO_ERR_NO_DEVICE;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    auto kernel = condition_hessian_kernel<A>;
    const size_t smem = CS::kWarpBytes * CS::kWarps;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return CNO_ERR_CUDA;
    long long ctas = (batch + CS::kWarps - 1) / CS::kWarps;
    const int grid = (int)(ctas < sms ? (ctas < 1 ? 1 : ctas) : sms);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    unsigned long long* queue = static_cast<unsigned long long*>(workspace);
    if (cudaMemsetAsync(queue, 0, sizeof(unsigned long long), s) != cudaSuccess) return CNO_ERR_CUDA;
    kernel<<<grid, CS::kWarps * 32, smem, s>>>(A{fn}, static_cast<const T*>(x), (long long)batch, static_cast<T*>(condition), queue);
    return cudaGetLastError() == cudaSuccess ? CNO_OK : CNO_ERR_CUDA;
  } else {
    return CNO_ERR_UNSUPPORTED;  // defined for second-order differentiable functions
  }
}

template <class F, int M>
inline int user_minimize(int solver, int mode, int lbfgs_m, const F& fn, int64_t batch, const void* x0, const cno_stop_t* stop,
                         const cno_batch_out_t* out, void* workspace, size_t workspace_bytes, void* stream,
                         cno_launch_info_t* info) {
  using T = typename F::Scalar;
  switch (solver) {
    case CNO_LBFGS:
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
}  // namespace cno

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
