// cno_api.cu -- the extern "C" layer of libcno.so (include/cno.h) and the
// table of kernels instantiated for the built-in objective families.
//
// Build (see cppnumericalsolvers_b200/build.py):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false ...
// -fmad=false is part of the arithmetic specification: the reference's
// canonical build forms no FMAs (generator.bzl:13, Dockerfile.test:111).
#include <cuda_runtime.h>

#include <dlfcn.h>

#include <cstdio>
#include <cstring>
#include <mutex>

#include "../../include/cno.h"
#include "cno_functors.cuh"
#include "cno_kernel_params.h"
#include "cno_lbfgs.cuh"
#include "cno_lbfgs_group.cuh"
#include "cno_lbfgsb.cuh"
#include "cno_lbfgsb_group.cuh"
#include "cno_bfgs.cuh"
#include "cno_descent.cuh"
#include "cno_evaluate.cuh"
#include "cno_launch.cuh"
#include "cno_newton.cuh"
#include "cno_newton_dmma.cuh"
#include "cno_logistic.cuh"
#include "cno_auglag_launch.cuh"
#include "../../include/cno_al.h"

namespace {

thread_local cudaError_t g_last_cuda = cudaSuccess;

#define CNO_CUDA(expr)                       \
  do {                                       \
    cudaError_t e__ = (expr);                \
    if (e__ != cudaSuccess) {                \
      g_last_cuda = e__;                     \
      return CNO_ERR_CUDA;                   \
    }                                        \
  } while (0)

// Owners for the CUDA objects the entry points create, so that every early return
// (CNO_CUDA, a failing launcher) releases them.
struct EventOwner {
  cudaEvent_t e = nullptr;
  ~EventOwner() { if (e) cudaEventDestroy(e); }
  cudaError_t create() { return cudaEventCreate(&e); }
};
struct StreamOwner {
  cudaStream_t s = nullptr;
  ~StreamOwner() { if (s) cudaStreamDestroy(s); }
  cudaError_t create() { return cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); }
};
struct DeviceBuffer {
  void* p = nullptr;
  ~DeviceBuffer() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes); }
};

// The device arena of cno_minimize_host, kept between calls (a 4 GiB cudaMalloc + cudaFree per call is
// ~70 ms of the end-to-end time at the headline size).  One arena per process, owned by whichever call
// holds the lock; a concurrent call on another thread allocates its own.  cno_release_host_arena() frees it.
struct HostArena {
  std::mutex m;
  void* p = nullptr;
  size_t bytes = 0;
  int device = -1;
};
HostArena g_host_arena;

int default_policy(int dtype) { return dtype == CNO_F64 ? CNO_POLICY_DMMA_TREE : CNO_POLICY_WARP_TREE; }

// problem->data holds a block of at least `elems` scalars per instance; blocks that TMA bulk copies read must also
// be 16-byte aligned.
template <class T>
bool data_block_ok(const cno_problem_t* p, int64_t elems, bool tma_aligned) {
  if (!p->data || p->data_stride < elems) return false;
  return !tma_aligned || (((uintptr_t)p->data & 15) == 0 && ((size_t)p->data_stride * sizeof(T)) % 16 == 0);
}

struct LaunchArgs {
  const cno_problem_t* problem;
  long long batch;
  const void* x0;
  const cno_stop_t* stop;
  const cno_batch_out_t* out;
  void* workspace;
  cudaStream_t stream;
  cno_launch_info_t* info;
  cno::ResumeArgs resume = cno::ResumeArgs{nullptr, 0, 0, 0};  // stepwise solves only
};

// One persistent launch of a solve kernel(fn, x0, batch, stop, out, queue, extra...); the queue counter is the
// first 8 bytes of the workspace.  A is LaunchArgs or LbfgsbArgs.
template <class Plan, class Fn, class Kernel, class A, class... Extra>
int launch_solve(Kernel kernel, const Fn& fn, const A& a, const Extra&... extra) {
  using T = typename Fn::Scalar;
  unsigned long long* queue = static_cast<unsigned long long*>(a.workspace);
  return cno::launch_persistent<Plan>(kernel, a.batch, queue, a.stream, a.info, g_last_cuda, fn,
                                      static_cast<const T*>(a.x0), a.batch, cno::make_stop<T>(*a.stop),
                                      cno::make_out<T>(*a.out), queue, extra...);
}

template <class Fn, int M = CNO_LBFGS_M, bool kResume = false, class LS = cno::LsMoreThuente>
int lbfgs(const Fn& fn, const LaunchArgs& a) {
  return launch_solve<typename cno::LbfgsPlan<Fn, M, kResume, LS>::SM>(cno::lbfgs_minimize_kernel<Fn, M, kResume, LS>,
                                                                      fn, a, a.resume);
}
template <class Fn, class LS = cno::LsMoreThuente>
int bfgs(const Fn& fn, const LaunchArgs& a) {
  return launch_solve<typename cno::BfgsPlan<Fn, LS>::SM>(cno::BfgsPlan<Fn, LS>::kernel(), fn, a);
}
// GradientDescent (kConjugate = false) / ConjugatedGradientDescent
template <class Fn, bool kConjugate, class LS = cno::LsMoreThuente>
int descent(const Fn& fn, const LaunchArgs& a) {
  return launch_solve<cno::DescentSmem<typename Fn::Scalar>>(cno::descent_minimize_kernel<Fn, kConjugate, LS>, fn, a);
}
template <class Fn>
int newton(const Fn& fn, const LaunchArgs& a) {
  if (a.stop->condition_hessian > 0) return CNO_ERR_UNSUPPORTED;  // see cno_newton.cuh
  return launch_solve<cno::NewtonSmem<typename Fn::Scalar, Fn::Dim>>(cno::newton_minimize_kernel<Fn>, fn, a);
}

template <class T, int D>
int newton_dense_quadratic(const LaunchArgs& a) {
  const cno_problem_t* p = a.problem;
  if (!data_block_ok<T>(p, (int64_t)D * D + D, true)) return CNO_ERR_INVALID_ARGUMENT;
  return newton(cno::DenseQuadraticFn<T, D>{static_cast<const T*>(p->data), (long long)p->data_stride}, a);
}
// CNO_POLICY_DMMA_LU: d = 64 fp64 dense quadratic, blocked LU with the trailing update on the FP64 tensor core
// (csrc/cno_newton_dmma.cuh).
int newton_dense_quadratic_dmma(const LaunchArgs& a) {
  using Fn = cno::DenseQuadraticDmmaFn;
  const cno_problem_t* p = a.problem;
  if (!data_block_ok<double>(p, (int64_t)64 * 64 + 64, true)) return CNO_ERR_INVALID_ARGUMENT;
  if (a.stop->condition_hessian > 0) return CNO_ERR_UNSUPPORTED;  // see cno_newton.cuh
  Fn fn;
  fn.data = static_cast<const double*>(p->data);
  fn.stride = (long long)p->data_stride;
  return launch_solve<cno::NewtonDmmaSmem>(cno::newton_dmma_minimize_kernel<Fn>, fn, a);
}
template <class T, int D>
int newton_rosenbrock(const LaunchArgs& a) { return newton(cno::RosenbrockFullFn<T, D>{}, a); }

template <class T, int D>
int bfgs_rosenbrock(const LaunchArgs& a) { return bfgs(cno::RosenbrockFn<T, D>{}, a); }
template <class T, int D>
int bfgs_half_sq_norm(const LaunchArgs& a) { return bfgs(cno::HalfSquaredNormFn<T, D>{}, a); }
template <class T>
int bfgs_diag_quadratic(const LaunchArgs& a) { return bfgs(cno::DiagQuadraticFn<T>{}, a); }

// LineSearch = HagerZhang variants (CNO_*_HAGER_ZHANG)
template <class T, int D>
int lbfgs_rosenbrock_hz(const LaunchArgs& a) {
  return lbfgs<cno::RosenbrockFn<T, D>, CNO_LBFGS_M, false, cno::LsHagerZhang>(cno::RosenbrockFn<T, D>{}, a);
}
template <class T, int D>
int bfgs_rosenbrock_hz(const LaunchArgs& a) { return bfgs<cno::RosenbrockFn<T, D>, cno::LsHagerZhang>({}, a); }
template <class T, int D>
int gd_rosenbrock_hz(const LaunchArgs& a) { return descent<cno::RosenbrockFn<T, D>, false, cno::LsHagerZhang>({}, a); }

template <class T, int D, bool kConjugate>
int descent_rosenbrock(const LaunchArgs& a) { return descent<cno::RosenbrockFn<T, D>, kConjugate>({}, a); }
template <class T, bool kConjugate>
int descent_diag_quadratic(const LaunchArgs& a) { return descent<cno::DiagQuadraticFn<T>, kConjugate>({}, a); }

template <class T, int D>
int lbfgs_rosenbrock(const LaunchArgs& a) { return lbfgs(cno::RosenbrockFn<T, D>{}, a); }
// Lbfgs<F, m> for m other than the default (lbfgs.h:40-41)
template <class T, int D, int M>
int lbfgs_rosenbrock_m(const LaunchArgs& a) { return lbfgs<cno::RosenbrockFn<T, D>, M>({}, a); }
// "parity mode": Eigen-SSE2-model reduction order (CNO_POLICY_EIGEN_SSE2), d = 128 fp64
int lbfgs_rosenbrock_d128_eigen(const LaunchArgs& a) {
  return lbfgs(cno::RosenbrockFn<double, 128, cno::PolicyEigenSSE2>{}, a);
}
// d = 512 / 1024 fp64 (cno_lbfgs_group.cuh): one group of d / 128 warps per instance, the history in the group's shared
// memory; MoreThuente, First mode, the default m and policy only (no stepwise variant).  No row at d = 256: there the
// group kernel was measured slower than the one-warp kernel (DESIGN.md 2.10).
template <int D>
int lbfgs_group_rosenbrock(const LaunchArgs& a) {
  using Fn = cno::GroupRosenbrockFn<double, D>;
  return launch_solve<cno::LbfgsGroupPlan<double, D, CNO_LBFGS_M>>(cno::lbfgs_group_minimize_kernel<Fn, CNO_LBFGS_M>,
                                                                   Fn{}, a);
}
// Lbfgs on a Second-mode function: diagonal-preconditioner branch (lbfgs.h:116-139)
template <class T, int D>
int lbfgs_rosenbrock_second(const LaunchArgs& a) {
  if (a.stop->condition_hessian > 0) return CNO_ERR_UNSUPPORTED;  // not computed (cno_newton.cuh)
  return lbfgs(cno::SecondMode<cno::RosenbrockFn<T, D>>{}, a);
}
// First-mode dense quadratic ([A | b] read from global memory per evaluation)
template <class T, int D>
int lbfgs_dense_quadratic(const LaunchArgs& a) {
  const cno_problem_t* p = a.problem;
  if (!data_block_ok<T>(p, (int64_t)D * D + D, false)) return CNO_ERR_INVALID_ARGUMENT;
  return lbfgs(cno::DenseQuadraticGlobalFn<T, D>{static_cast<const T*>(p->data), (long long)p->data_stride}, a);
}
template <class T, int D>
int lbfgs_half_sq_norm(const LaunchArgs& a) { return lbfgs(cno::HalfSquaredNormFn<T, D>{}, a); }
template <class T>
int lbfgs_diag_quadratic(const LaunchArgs& a) { return lbfgs(cno::DiagQuadraticFn<T>{}, a); }

// Stepwise variants (cno_minimize_steps): same kernel with park / un-park code.
template <class T, int D>
int lbfgs_rosenbrock_steps(const LaunchArgs& a) { return lbfgs<cno::RosenbrockFn<T, D>, CNO_LBFGS_M, true>({}, a); }
template <class Fn>
int lbfgs_steps_stateless(const LaunchArgs& a) { return lbfgs<Fn, CNO_LBFGS_M, true>({}, a); }  // functors without parameters
template <class T, int D>
size_t lbfgs_state_stride() {
  return cno::ResumeLayout<T, cno::Shape<D>::E, CNO_LBFGS_M>::kBytes;
}

template <class T, int D, int N>
int lbfgs_logistic(const LaunchArgs& a) {
  const cno_problem_t* p = a.problem;
  using Fn = cno::LogisticFn<T, D, N>;
  if (p->n != N || !data_block_ok<T>(p, Fn::kBlockElems, true)) return CNO_ERR_INVALID_ARGUMENT;
  return lbfgs(Fn{static_cast<const T*>(p->data), (long long)p->data_stride, (T)p->param}, a);
}

// ---- Progress::condition_hessian on request (csrc/cno_newton.cuh: condition_hessian_kernel) ----
struct CondArgs {
  const cno_problem_t* problem;
  long long batch;
  const void* x;
  void* out;
  void* workspace;
  cudaStream_t stream;
};
template <class Fn>
int launch_condition(const Fn& fn, const CondArgs& a) {
  using T = typename Fn::Scalar;
  unsigned long long* queue = static_cast<unsigned long long*>(a.workspace);
  return cno::launch_persistent<cno::ConditionSmem<T, Fn::Dim>>(cno::condition_hessian_kernel<Fn>, a.batch, queue,
                                                                a.stream, nullptr, g_last_cuda, fn,
                                                                static_cast<const T*>(a.x), a.batch,
                                                                static_cast<T*>(a.out), queue);
}
template <class T, int D>
int condition_dense_quadratic(const CondArgs& a) {
  const cno_problem_t* p = a.problem;
  if (!data_block_ok<T>(p, (int64_t)D * D + D, true)) return CNO_ERR_INVALID_ARGUMENT;
  return launch_condition(cno::DenseQuadraticFn<T, D>{static_cast<const T*>(p->data), (long long)p->data_stride}, a);
}
template <class T, int D>
int condition_rosenbrock(const CondArgs& a) {
  return launch_condition(cno::RosenbrockFullFn<T, D>{}, a);
}
struct CondEntry { int family, dtype, d; int (*fn)(const CondArgs&); };
const CondEntry kCondTable[] = {  // the Second-mode built-ins of NewtonDescent
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 64, condition_dense_quadratic<double, 64>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 12, condition_dense_quadratic<double, 12>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F32, 64, condition_dense_quadratic<float, 64>},
    {CNO_FN_ROSENBROCK, CNO_F64, 2, condition_rosenbrock<double, 2>},
    {CNO_FN_ROSENBROCK, CNO_F64, 8, condition_rosenbrock<double, 8>},
};

typedef int (*launcher_t)(const LaunchArgs&);

struct Entry {
  int solver, family, dtype, d;
  launcher_t fn;
  int policy = -1;  // -1 = the default policy of the dtype (fp64: DMMA tree, fp32: butterfly)
  int mode = 0;     // 2 = Lbfgs on a Second-mode function (cno_problem_t::mode)
  launcher_t steps_fn = nullptr;          // stepwise variant (cno_minimize_steps), if instantiated
  size_t (*state_stride)() = nullptr;     // bytes of one parked instance
  int m = CNO_LBFGS_M;                    // Lbfgs<F, m>: pairs kept (cno_problem_t::lbfgs_m)
};

// Every (solver, functor, T, D) compiled into this library.
const Entry kTable[] = {
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 2, lbfgs_rosenbrock<double, 2>, -1, 0,
     lbfgs_rosenbrock_steps<double, 2>, lbfgs_state_stride<double, 2>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 3, lbfgs_rosenbrock<double, 3>, -1, 0,
     lbfgs_rosenbrock_steps<double, 3>, lbfgs_state_stride<double, 3>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 8, lbfgs_rosenbrock<double, 8>, -1, 0,
     lbfgs_rosenbrock_steps<double, 8>, lbfgs_state_stride<double, 8>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 32, lbfgs_rosenbrock<double, 32>, -1, 0,
     lbfgs_rosenbrock_steps<double, 32>, lbfgs_state_stride<double, 32>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 37, lbfgs_rosenbrock<double, 37>, -1, 0,
     lbfgs_rosenbrock_steps<double, 37>, lbfgs_state_stride<double, 37>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 64, lbfgs_rosenbrock<double, 64>, -1, 0,
     lbfgs_rosenbrock_steps<double, 64>, lbfgs_state_stride<double, 64>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgs_rosenbrock<double, 128>, -1, 0,
     lbfgs_rosenbrock_steps<double, 128>, lbfgs_state_stride<double, 128>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgs_rosenbrock_d128_eigen, CNO_POLICY_EIGEN_SSE2},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 512, lbfgs_group_rosenbrock<512>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 1024, lbfgs_group_rosenbrock<1024>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 2, lbfgs_rosenbrock_second<double, 2>, -1, 2},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 37, lbfgs_rosenbrock_second<double, 37>, -1, 2},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgs_rosenbrock_second<double, 128>, -1, 2},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 8, lbfgs_rosenbrock_m<double, 8, 5>, -1, 0, nullptr, nullptr, 5},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 37, lbfgs_rosenbrock_m<double, 37, 5>, -1, 0, nullptr, nullptr, 5},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgs_rosenbrock_m<double, 128, 5>, -1, 0, nullptr, nullptr, 5},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 8, lbfgs_rosenbrock_m<double, 8, 20>, -1, 0, nullptr, nullptr, 20},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 37, lbfgs_rosenbrock_m<double, 37, 20>, -1, 0, nullptr, nullptr, 20},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgs_rosenbrock_m<double, 128, 20>, -1, 0, nullptr, nullptr, 20},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F32, 37, lbfgs_rosenbrock_m<float, 37, 5>, -1, 0, nullptr, nullptr, 5},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F32, 2, lbfgs_rosenbrock<float, 2>, -1, 0,
     lbfgs_rosenbrock_steps<float, 2>, lbfgs_state_stride<float, 2>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F32, 37, lbfgs_rosenbrock<float, 37>, -1, 0,
     lbfgs_rosenbrock_steps<float, 37>, lbfgs_state_stride<float, 37>},
    {CNO_LBFGS, CNO_FN_ROSENBROCK, CNO_F32, 128, lbfgs_rosenbrock<float, 128>, -1, 0,
     lbfgs_rosenbrock_steps<float, 128>, lbfgs_state_stride<float, 128>},
    {CNO_LBFGS, CNO_FN_DIAG_QUADRATIC, CNO_F64, 2, lbfgs_diag_quadratic<double>, -1, 0,
     lbfgs_steps_stateless<cno::DiagQuadraticFn<double>>, lbfgs_state_stride<double, 2>},
    {CNO_LBFGS, CNO_FN_HALF_SQUARED_NORM, CNO_F64, 2, lbfgs_half_sq_norm<double, 2>, -1, 0,
     lbfgs_steps_stateless<cno::HalfSquaredNormFn<double, 2>>, lbfgs_state_stride<double, 2>},
    {CNO_LBFGS, CNO_FN_HALF_SQUARED_NORM, CNO_F64, 50, lbfgs_half_sq_norm<double, 50>, -1, 0,
     lbfgs_steps_stateless<cno::HalfSquaredNormFn<double, 50>>, lbfgs_state_stride<double, 50>},
    {CNO_LBFGS, CNO_FN_LOGISTIC, CNO_F32, 64, lbfgs_logistic<float, 64, 256>},
    {CNO_LBFGS, CNO_FN_DENSE_QUADRATIC, CNO_F64, 2, lbfgs_dense_quadratic<double, 2>},
    {CNO_LBFGS, CNO_FN_DENSE_QUADRATIC, CNO_F64, 8, lbfgs_dense_quadratic<double, 8>},
    {CNO_LBFGS, CNO_FN_DENSE_QUADRATIC, CNO_F64, 64, lbfgs_dense_quadratic<double, 64>},
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F64, 2, bfgs_rosenbrock<double, 2>},
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F64, 8, bfgs_rosenbrock<double, 8>},
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F64, 32, bfgs_rosenbrock<double, 32>},
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F32, 32, bfgs_rosenbrock<float, 32>},
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F64, 37, bfgs_rosenbrock<double, 37>},    // D > 32: H in shared memory
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F64, 64, bfgs_rosenbrock<double, 64>},
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F64, 128, bfgs_rosenbrock<double, 128>},
    {CNO_BFGS, CNO_FN_ROSENBROCK, CNO_F32, 128, bfgs_rosenbrock<float, 128>},
    {CNO_BFGS, CNO_FN_DIAG_QUADRATIC, CNO_F64, 2, bfgs_diag_quadratic<double>},
    {CNO_BFGS, CNO_FN_HALF_SQUARED_NORM, CNO_F64, 2, bfgs_half_sq_norm<double, 2>},
    {CNO_NEWTON, CNO_FN_DENSE_QUADRATIC, CNO_F64, 64, newton_dense_quadratic<double, 64>},
    {CNO_NEWTON, CNO_FN_DENSE_QUADRATIC, CNO_F64, 64, newton_dense_quadratic_dmma, CNO_POLICY_DMMA_LU},
    {CNO_NEWTON, CNO_FN_DENSE_QUADRATIC, CNO_F64, 12, newton_dense_quadratic<double, 12>},
    {CNO_NEWTON, CNO_FN_DENSE_QUADRATIC, CNO_F32, 64, newton_dense_quadratic<float, 64>},
    {CNO_NEWTON, CNO_FN_ROSENBROCK, CNO_F64, 2, newton_rosenbrock<double, 2>},
    {CNO_NEWTON, CNO_FN_ROSENBROCK, CNO_F64, 8, newton_rosenbrock<double, 8>},
    {CNO_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 2, descent_rosenbrock<double, 2, false>},
    {CNO_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 8, descent_rosenbrock<double, 8, false>},
    {CNO_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 37, descent_rosenbrock<double, 37, false>},
    {CNO_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 128, descent_rosenbrock<double, 128, false>},
    {CNO_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F32, 37, descent_rosenbrock<float, 37, false>},
    {CNO_GRADIENT_DESCENT, CNO_FN_DIAG_QUADRATIC, CNO_F64, 2, descent_diag_quadratic<double, false>},
    {CNO_CONJUGATED_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 2, descent_rosenbrock<double, 2, true>},
    {CNO_CONJUGATED_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 8, descent_rosenbrock<double, 8, true>},
    {CNO_CONJUGATED_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 37, descent_rosenbrock<double, 37, true>},
    {CNO_CONJUGATED_GRADIENT_DESCENT, CNO_FN_ROSENBROCK, CNO_F64, 128, descent_rosenbrock<double, 128, true>},
    {CNO_CONJUGATED_GRADIENT_DESCENT, CNO_FN_DIAG_QUADRATIC, CNO_F64, 2, descent_diag_quadratic<double, true>},
    {CNO_LBFGS_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 2, lbfgs_rosenbrock_hz<double, 2>},
    {CNO_LBFGS_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 37, lbfgs_rosenbrock_hz<double, 37>},
    {CNO_LBFGS_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgs_rosenbrock_hz<double, 128>},
    {CNO_LBFGS_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F32, 37, lbfgs_rosenbrock_hz<float, 37>},
    {CNO_BFGS_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 8, bfgs_rosenbrock_hz<double, 8>},
    {CNO_BFGS_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 32, bfgs_rosenbrock_hz<double, 32>},
    {CNO_BFGS_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 64, bfgs_rosenbrock_hz<double, 64>},
    {CNO_GRADIENT_DESCENT_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 8, gd_rosenbrock_hz<double, 8>},
    {CNO_GRADIENT_DESCENT_HAGER_ZHANG, CNO_FN_ROSENBROCK, CNO_F64, 37, gd_rosenbrock_hz<double, 37>},
};

// ---- Lbfgsb (solver/lbfgsb.h) ----
struct LbfgsbArgs {
  const cno_problem_t* problem;
  const cno_bounds_t* bounds;
  long long batch;
  const void* x0;
  const cno_stop_t* stop;
  const cno_batch_out_t* out;
  void* workspace;
  cudaStream_t stream;
  cno_launch_info_t* info;
};
template <class T>
cno::BoundsArgs<T> bounds_args(const LbfgsbArgs& a) {
  return cno::BoundsArgs<T>{a.bounds ? static_cast<const T*>(a.bounds->lower) : nullptr,
                            a.bounds ? static_cast<const T*>(a.bounds->upper) : nullptr,
                            a.bounds ? (long long)a.bounds->stride : 0};
}
template <class Fn, int M = 5>
int lbfgsb(const Fn& fn, const LbfgsbArgs& a) {
  using T = typename Fn::Scalar;
  return launch_solve<cno::LbfgsbSmem<T, Fn::Dim, M>>(cno::lbfgsb_minimize_kernel<Fn, M>, fn, a, bounds_args<T>(a));
}
// d = 256 / 512 / 1024 fp64 (cno_lbfgsb_group.cuh): one group of d / 128 warps per instance, the history in the group's
// shared memory; m = 5 and the default policy only.
template <int D>
int lbfgsb_group_rosenbrock(const LbfgsbArgs& a) {
  using Fn = cno::GroupRosenbrockFn<double, D>;
  return launch_solve<cno::LbfgsbGroupPlan<double, D, 5>>(cno::lbfgsb_group_minimize_kernel<Fn, 5>, Fn{}, a,
                                                          bounds_args<double>(a));
}
template <class T, int D>
int lbfgsb_rosenbrock(const LbfgsbArgs& a) { return lbfgsb(cno::RosenbrockFn<T, D>{}, a); }
template <class T, int D>
int lbfgsb_half_sq_norm(const LbfgsbArgs& a) { return lbfgsb(cno::HalfSquaredNormFn<T, D>{}, a); }
template <class T>
int lbfgsb_diag_quadratic(const LbfgsbArgs& a) { return lbfgsb(cno::DiagQuadraticFn<T>{}, a); }
template <class T, int D>
int lbfgsb_dense_quadratic(const LbfgsbArgs& a) {
  const cno_problem_t* p = a.problem;
  if (!data_block_ok<T>(p, (int64_t)D * D + D, false)) return CNO_ERR_INVALID_ARGUMENT;
  return lbfgsb(cno::DenseQuadraticGlobalFn<T, D>{static_cast<const T*>(p->data), (long long)p->data_stride}, a);
}
// Lbfgsb<F, m> for m other than the default 5 (lbfgsb.h:44-45)
template <class T, int D, int M>
int lbfgsb_rosenbrock_m(const LbfgsbArgs& a) { return lbfgsb<cno::RosenbrockFn<T, D>, M>({}, a); }
struct LbfgsbEntry { int family, dtype, d; int (*fn)(const LbfgsbArgs&); int m = 5; };
const LbfgsbEntry kLbfgsbTable[] = {
    {CNO_FN_ROSENBROCK, CNO_F64, 8, lbfgsb_rosenbrock_m<double, 8, 10>, 10},
    {CNO_FN_ROSENBROCK, CNO_F64, 37, lbfgsb_rosenbrock_m<double, 37, 10>, 10},
    {CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgsb_rosenbrock_m<double, 128, 10>, 10},
    {CNO_FN_ROSENBROCK, CNO_F64, 2, lbfgsb_rosenbrock<double, 2>},
    {CNO_FN_ROSENBROCK, CNO_F64, 8, lbfgsb_rosenbrock<double, 8>},
    {CNO_FN_ROSENBROCK, CNO_F64, 37, lbfgsb_rosenbrock<double, 37>},
    {CNO_FN_ROSENBROCK, CNO_F64, 64, lbfgsb_rosenbrock<double, 64>},
    {CNO_FN_ROSENBROCK, CNO_F64, 128, lbfgsb_rosenbrock<double, 128>},
    {CNO_FN_ROSENBROCK, CNO_F64, 256, lbfgsb_group_rosenbrock<256>},
    {CNO_FN_ROSENBROCK, CNO_F64, 512, lbfgsb_group_rosenbrock<512>},
    {CNO_FN_ROSENBROCK, CNO_F64, 1024, lbfgsb_group_rosenbrock<1024>},
    {CNO_FN_ROSENBROCK, CNO_F32, 37, lbfgsb_rosenbrock<float, 37>},
    {CNO_FN_DIAG_QUADRATIC, CNO_F64, 2, lbfgsb_diag_quadratic<double>},
    {CNO_FN_HALF_SQUARED_NORM, CNO_F64, 2, lbfgsb_half_sq_norm<double, 2>},
    {CNO_FN_HALF_SQUARED_NORM, CNO_F64, 8, lbfgsb_half_sq_norm<double, 8>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 8, lbfgsb_dense_quadratic<double, 8>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 64, lbfgsb_dense_quadratic<double, 64>},
};
const LbfgsbEntry* lbfgsb_find(const cno_problem_t* p) {
  if (!p || p->policy != default_policy(p->dtype)) return nullptr;
  const int m = p->lbfgs_m > 0 ? p->lbfgs_m : 5;  // cno_problem_t::lbfgs_m: pairs kept (0 = the reference's default, 5)
  for (const LbfgsbEntry& e : kLbfgsbTable)
    if (e.family == p->family && e.dtype == p->dtype && e.d == p->d && e.m == m) return &e;
  return nullptr;
}

// ---- cno_evaluate: F::operator()(x, &gradient) of the built-in families ----
typedef int (*evaluator_t)(const cno_problem_t*, int64_t, const void*, void*, void*, void*);
template <class T, int D>
int eval_rosenbrock(const cno_problem_t*, int64_t b, const void* x, void* f, void* g, void* s) {
  return cno::launch_evaluate(cno::RosenbrockFn<T, D>{}, b, x, f, g, s);
}
template <class T>
int eval_diag_quadratic(const cno_problem_t*, int64_t b, const void* x, void* f, void* g, void* s) {
  return cno::launch_evaluate(cno::DiagQuadraticFn<T>{}, b, x, f, g, s);
}
template <class T, int D>
int eval_half_sq_norm(const cno_problem_t*, int64_t b, const void* x, void* f, void* g, void* s) {
  return cno::launch_evaluate(cno::HalfSquaredNormFn<T, D>{}, b, x, f, g, s);
}
template <class T, int D>
int eval_dense_quadratic(const cno_problem_t* p, int64_t b, const void* x, void* f, void* g, void* s) {
  if (!data_block_ok<T>(p, (int64_t)D * D + D, false)) return CNO_ERR_INVALID_ARGUMENT;
  return cno::launch_evaluate(cno::DenseQuadraticGlobalFn<T, D>{static_cast<const T*>(p->data), (long long)p->data_stride},
                              b, x, f, g, s);
}
struct EvalEntry { int family, dtype, d; evaluator_t fn; };
const EvalEntry kEvalTable[] = {
    {CNO_FN_ROSENBROCK, CNO_F64, 2, eval_rosenbrock<double, 2>},   {CNO_FN_ROSENBROCK, CNO_F64, 3, eval_rosenbrock<double, 3>},
    {CNO_FN_ROSENBROCK, CNO_F64, 8, eval_rosenbrock<double, 8>},   {CNO_FN_ROSENBROCK, CNO_F64, 32, eval_rosenbrock<double, 32>},
    {CNO_FN_ROSENBROCK, CNO_F64, 37, eval_rosenbrock<double, 37>}, {CNO_FN_ROSENBROCK, CNO_F64, 64, eval_rosenbrock<double, 64>},
    {CNO_FN_ROSENBROCK, CNO_F64, 128, eval_rosenbrock<double, 128>},
    {CNO_FN_ROSENBROCK, CNO_F32, 2, eval_rosenbrock<float, 2>},    {CNO_FN_ROSENBROCK, CNO_F32, 32, eval_rosenbrock<float, 32>},
    {CNO_FN_ROSENBROCK, CNO_F32, 37, eval_rosenbrock<float, 37>},  {CNO_FN_ROSENBROCK, CNO_F32, 128, eval_rosenbrock<float, 128>},
    {CNO_FN_DIAG_QUADRATIC, CNO_F64, 2, eval_diag_quadratic<double>},
    {CNO_FN_HALF_SQUARED_NORM, CNO_F64, 2, eval_half_sq_norm<double, 2>},
    {CNO_FN_HALF_SQUARED_NORM, CNO_F64, 8, eval_half_sq_norm<double, 8>},
    {CNO_FN_HALF_SQUARED_NORM, CNO_F64, 50, eval_half_sq_norm<double, 50>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 2, eval_dense_quadratic<double, 2>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 8, eval_dense_quadratic<double, 8>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 64, eval_dense_quadratic<double, 64>},
};

const Entry* find_entry(int solver, const cno_problem_t* p) {
  const int dflt = default_policy(p->dtype);
  const bool is_lbfgs = (solver == CNO_LBFGS || solver == CNO_LBFGS_HAGER_ZHANG);
  const int m = (is_lbfgs && p->lbfgs_m > 0) ? p->lbfgs_m : CNO_LBFGS_M;
  for (const Entry& e : kTable)
    if (e.solver == solver && e.family == p->family && e.dtype == p->dtype && e.d == p->d && e.m == m &&
        ((e.policy < 0) ? dflt : e.policy) == p->policy &&
        ((solver == CNO_BFGS || solver == CNO_NEWTON) || (e.mode == 2) == (p->mode == 2)))
      return &e;
  return nullptr;
}

int check_args(int solver, const cno_problem_t* p) {
  if (!p) return CNO_ERR_INVALID_ARGUMENT;
  if (solver < CNO_LBFGS || solver > CNO_GRADIENT_DESCENT_HAGER_ZHANG) return CNO_ERR_INVALID_ARGUMENT;
  if (p->dtype != CNO_F64 && p->dtype != CNO_F32) return CNO_ERR_INVALID_ARGUMENT;
  if (p->d <= 0) return CNO_ERR_INVALID_ARGUMENT;
  // the reduction policy is compiled into the kernels (find_entry matches it):
  // fp64 = tensor-core tree, fp32 = butterfly, plus the Eigen-SSE2 parity mode where listed
  if (!find_entry(solver, p)) return CNO_ERR_UNSUPPORTED;
  return CNO_OK;
}

constexpr size_t kWorkspaceBytes = 256;

// ---- small utility kernels ---------------------------------------------------

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z ^= z >> 30;
  z *= 0xBF58476D1CE4E5B9ULL;
  z ^= z >> 27;
  z *= 0x94D049BB133111EBULL;
  z ^= z >> 31;
  return z;
}

template <class T>
__global__ void fill_uniform_kernel(T* dst, long long first, long long count,
                                    unsigned long long seed, T lo, T hi) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride) {
    const unsigned long long n = (unsigned long long)(first + k) + 1ULL;
    const unsigned long long z = mix64(seed + n * 0x9E3779B97F4A7C15ULL);
    T u;
    if (sizeof(T) == 8)
      u = (T)((double)(z >> 11) * 0x1.0p-53);
    else
      u = (T)((float)(z >> 40) * 0x1.0p-24f);
    dst[k] = lo + (hi - lo) * u;
  }
}

__global__ void done_bitmap_kernel(const int8_t* status, long long batch, uint32_t* words) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool done = (i < batch) && (status[i] != CNO_STATUS_CONTINUE) &&
                    (status[i] != CNO_STATUS_NOT_STARTED);
  const unsigned m = __ballot_sync(0xffffffffu, done);
  if ((threadIdx.x & 31) == 0 && i < batch) words[i >> 5] = m;
}

// set bits among the first `bits` bits of a bitmap
__global__ void count_bits_kernel(const uint32_t* words, long long bits, unsigned long long* total) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nw = (bits + 31) / 32;
  unsigned c = 0;
  if (w < nw) {
    uint32_t v = words[w];
    const long long rem = bits - w * 32;
    if (rem < 32) v &= (rem <= 0) ? 0u : ((1u << rem) - 1u);
    c = __popc(v);
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(total, (unsigned long long)c);
}

__global__ void div_check_kernel(const double* a, const double* b, long long n, double* helper, double* plain,
                                 int* accepted) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool ok;
  const double q = cno::div_with(a[i], b[i], cno::div_rcp(b[i]), ok);
  const double p = a[i] / b[i];
  helper[i] = ok ? q : p;
  plain[i] = p;
  accepted[i] = ok ? 1 : 0;
}

__global__ void cstep_kernel(double* io, int* flags) {
  bool brackt = flags[0] != 0;
  int info = flags[1];
  const int ret = cno::cstep<double>(io[0], io[1], io[2], io[3], io[4], io[5], io[6], io[7],
                                     io[8], brackt, io[9], io[10], info);
  flags[0] = brackt ? 1 : 0;
  flags[1] = info;
  flags[2] = ret;
}

// ---- AugmentedLagrangian (include/cno_al.h; csrc/cno_auglag.cuh, csrc/cno_auglag_launch.cuh) ----
template <class Obj>
int al_rows(const Obj& obj, const cno_constraints_t* k, const cno::AlArgs& a) {
  return cno::al_run(obj, cno::AlRows{}, *k, a, g_last_cuda);
}
template <class T, int D>
int al_rosenbrock(const cno_problem_t*, const cno_constraints_t* k, const cno::AlArgs& a) {
  return al_rows(cno::RosenbrockFn<T, D>{}, k, a);
}
template <class T, int D>
int al_half_sq_norm(const cno_problem_t*, const cno_constraints_t* k, const cno::AlArgs& a) {
  return al_rows(cno::HalfSquaredNormFn<T, D>{}, k, a);
}
template <class T, int D>
int al_dense_quadratic(const cno_problem_t* p, const cno_constraints_t* k, const cno::AlArgs& a) {
  // the batched "QP with affine / ball constraints"
  if (!data_block_ok<T>(p, (int64_t)D * D + D, false)) return CNO_ERR_INVALID_ARGUMENT;
  return al_rows(cno::DenseQuadraticGlobalFn<T, D>{static_cast<const T*>(p->data), (long long)p->data_stride}, k, a);
}

struct AlEntry {
  int family, dtype, d;
  int (*fn)(const cno_problem_t*, const cno_constraints_t*, const cno::AlArgs&);
};
const AlEntry kAlTable[] = {
    {CNO_FN_ROSENBROCK, CNO_F64, 2, al_rosenbrock<double, 2>},
    {CNO_FN_ROSENBROCK, CNO_F64, 8, al_rosenbrock<double, 8>},
    {CNO_FN_ROSENBROCK, CNO_F64, 37, al_rosenbrock<double, 37>},
    {CNO_FN_ROSENBROCK, CNO_F64, 128, al_rosenbrock<double, 128>},
    {CNO_FN_ROSENBROCK, CNO_F32, 8, al_rosenbrock<float, 8>},
    {CNO_FN_HALF_SQUARED_NORM, CNO_F64, 2, al_half_sq_norm<double, 2>},
    {CNO_FN_HALF_SQUARED_NORM, CNO_F64, 8, al_half_sq_norm<double, 8>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 2, al_dense_quadratic<double, 2>},
    {CNO_FN_DENSE_QUADRATIC, CNO_F64, 8, al_dense_quadratic<double, 8>},
};

const AlEntry* al_find(const cno_problem_t* p) {
  if (p->policy != default_policy(p->dtype) || p->mode == 2) return nullptr;
  for (const AlEntry& e : kAlTable)
    if (e.family == p->family && e.dtype == p->dtype && e.d == p->d) return &e;
  return nullptr;
}

int al_check(const cno_problem_t* p, const cno_constraints_t* k) {
  if (!p || !k) return CNO_ERR_INVALID_ARGUMENT;
  if (p->dtype != CNO_F64 && p->dtype != CNO_F32) return CNO_ERR_INVALID_ARGUMENT;
  if (k->n_eq < 0 || k->n_ineq < 0) return CNO_ERR_INVALID_ARGUMENT;
  if (k->n_eq > cno::kAlMaxCon || k->n_ineq > cno::kAlMaxCon) return CNO_ERR_UNSUPPORTED;
  if (k->n_eq + k->n_ineq > 0 && (!k->kinds || !k->data)) return CNO_ERR_INVALID_ARGUMENT;
  if (!al_find(p)) return CNO_ERR_UNSUPPORTED;
  return CNO_OK;
}

bool have_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) { g_last_cuda = e; (void)cudaGetLastError(); return false; }
  return n > 0;
}

// NULL stop = the preset `dflt` writes into *local; a `past` beyond the kernels' CNO_MAX_PAST ring is rejected.
int resolve_stop(const cno_stop_t*& stop, cno_stop_t* local, void (*dflt)(cno_stop_t*)) {
  if (!stop) {
    dflt(local);
    stop = local;
  }
  return (stop->past > CNO_MAX_PAST || stop->past < 0) ? CNO_ERR_INVALID_ARGUMENT : CNO_OK;
}

// the queue counter: 8-byte aligned, kWorkspaceBytes at least
bool queue_workspace_ok(const void* workspace, size_t bytes) {
  return workspace && bytes >= kWorkspaceBytes && !((uintptr_t)workspace & 7);
}

// the kernels load and store x and the gradient as 16-byte vectors
bool io_aligned(const void* x0, const cno_batch_out_t* out) {
  return !(((uintptr_t)x0 & 15) || ((uintptr_t)out->x & 15) || ((uintptr_t)out->gradient & 15));
}

}  // namespace

extern "C" {

void cno_version(int* major, int* minor) {
  if (major) *major = CNO_VERSION_MAJOR;
  if (minor) *minor = CNO_VERSION_MINOR;
}

const char* cno_error_string(int err) {
  switch (err) {
    case CNO_OK: return "ok";
    case CNO_ERR_INVALID_ARGUMENT: return "invalid argument";
    case CNO_ERR_UNSUPPORTED: return "no kernel instantiated for this (solver, functor, dtype, d, policy)";
    case CNO_ERR_NO_DEVICE: return "no CUDA device (there is no CPU fallback)";
    case CNO_ERR_CUDA: return "CUDA error (see cno_last_cuda_error)";
    case CNO_ERR_WORKSPACE: return "workspace too small or misaligned";
  }
  return "unknown error";
}

int cno_last_cuda_error(const char** msg) {
  if (msg) *msg = cudaGetErrorString(g_last_cuda);
  return (int)g_last_cuda;
}

void cno_default_stop(cno_stop_t* s) {  // solver/progress.h:353-431
  if (!s) return;
  memset(s, 0, sizeof(*s));
  s->num_iterations = 10000;
  s->x_delta = 1e-9;
  s->x_delta_violations = 1;
  s->f_delta = 0;
  s->f_delta_violations = 1;
  s->f_delta_relative = 0;
  s->gradient_norm = 1e-5;
  s->gradient_norm_relative = 1;
  s->condition_hessian = 0;
  s->past = 3;
  s->past_delta = 1e-6;
}

void cno_conservative_stop(cno_stop_t* s) {  // solver/progress.h:456-464
  if (!s) return;
  cno_default_stop(s);
  s->gradient_norm = 5e-6;
  s->past = 5;
  s->past_delta = 1e-10;
}

int cno_supported(int solver, const cno_problem_t* problem) { return check_args(solver, problem); }

int cno_workspace_bytes(int solver, const cno_problem_t* problem, int64_t batch, size_t* bytes) {
  (void)batch;
  int rc = check_args(solver, problem);
  if (rc) return rc;
  if (!bytes) return CNO_ERR_INVALID_ARGUMENT;
  *bytes = kWorkspaceBytes;
  return CNO_OK;
}

int cno_minimize(int solver, const cno_problem_t* problem, int64_t batch, const void* x0,
                 const cno_stop_t* stop, const cno_batch_out_t* out, void* workspace,
                 size_t workspace_bytes, void* stream, cno_launch_info_t* info) {
  int rc = check_args(solver, problem);
  if (rc) return rc;
  if (batch < 0 || !out) return CNO_ERR_INVALID_ARGUMENT;
  if (batch == 0) {
    if (info) memset(info, 0, sizeof(*info));
    return have_device() ? CNO_OK : CNO_ERR_NO_DEVICE;
  }
  if (!x0) return CNO_ERR_INVALID_ARGUMENT;
  if (!queue_workspace_ok(workspace, workspace_bytes)) return CNO_ERR_WORKSPACE;
  if (!io_aligned(x0, out)) return CNO_ERR_INVALID_ARGUMENT;
  cno_stop_t local;
  if ((rc = resolve_stop(stop, &local, cno_default_stop))) return rc;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  if (info) memset(info, 0, sizeof(*info));

  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cno::LaunchTimer timer(s, info);
  if ((rc = timer.start(g_last_cuda))) return rc;
  const LaunchArgs a{problem, (long long)batch, x0, stop, out, workspace, s, info};
  if ((rc = find_entry(solver, problem)->fn(a))) return rc;
  return timer.stop(g_last_cuda);
}

int cno_state_bytes(int solver, const cno_problem_t* problem, int64_t batch, size_t* bytes) {
  int rc = check_args(solver, problem);
  if (rc) return rc;
  if (!bytes || batch < 0) return CNO_ERR_INVALID_ARGUMENT;
  const Entry* e = find_entry(solver, problem);
  if (!e->steps_fn) return CNO_ERR_UNSUPPORTED;
  *bytes = (size_t)batch * e->state_stride();
  return CNO_OK;
}

int cno_minimize_steps(int solver, const cno_problem_t* problem, int64_t batch, const void* x0,
                       const cno_stop_t* stop, const cno_batch_out_t* out, void* state,
                       size_t state_bytes, int32_t max_iterations, int32_t first_call,
                       void* workspace, size_t workspace_bytes, void* stream,
                       cno_launch_info_t* info) {
  int rc = check_args(solver, problem);
  if (rc) return rc;
  const Entry* e = find_entry(solver, problem);
  if (!e->steps_fn) return CNO_ERR_UNSUPPORTED;
  if (batch < 0 || !out || max_iterations <= 0) return CNO_ERR_INVALID_ARGUMENT;
  if (!out->x || !out->value || !out->gradient || !out->status || !out->num_iterations)
    return CNO_ERR_INVALID_ARGUMENT;  // the parked state continues from these arrays
  if (info) memset(info, 0, sizeof(*info));
  if (batch == 0) return have_device() ? CNO_OK : CNO_ERR_NO_DEVICE;
  if (!x0 && first_call) return CNO_ERR_INVALID_ARGUMENT;
  const size_t stride = e->state_stride();
  if (!state || state_bytes < (size_t)batch * stride || ((uintptr_t)state & 15)) return CNO_ERR_WORKSPACE;
  if (!queue_workspace_ok(workspace, workspace_bytes)) return CNO_ERR_WORKSPACE;
  if (!io_aligned(x0, out)) return CNO_ERR_INVALID_ARGUMENT;
  cno_stop_t local;
  if ((rc = resolve_stop(stop, &local, cno_default_stop))) return rc;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cno::LaunchTimer timer(s, info);
  if ((rc = timer.start(g_last_cuda))) return rc;
  LaunchArgs a{problem, (long long)batch, x0, stop, out, workspace, s, info};
  a.resume = cno::ResumeArgs{static_cast<unsigned char*>(state), (long long)stride, max_iterations,
                             first_call ? 1 : 0};
  if ((rc = e->steps_fn(a))) return rc;
  return timer.stop(g_last_cuda);
}

int cno_minimize_host(int solver, const cno_problem_t* problem, int64_t batch, const void* x0,
                      const cno_stop_t* stop, const cno_batch_out_t* out,
                      cno_launch_info_t* info) {
  int rc = check_args(solver, problem);
  if (rc) return rc;
  if (batch < 0 || !x0 || !out) return CNO_ERR_INVALID_ARGUMENT;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  cno_launch_info_t local;
  memset(&local, 0, sizeof(local));
  if (batch == 0) { if (info) *info = local; return CNO_OK; }
  cno_stop_t local_stop;
  if ((rc = resolve_stop(stop, &local_stop, cno_default_stop))) return rc;

  const size_t ts = problem->dtype == CNO_F64 ? 8 : 4;
  const size_t d = (size_t)problem->d;
  const size_t vec_bytes = (size_t)batch * d * ts, sc_bytes = (size_t)batch * ts;
  // declared before the arena: destroyed after it (cudaFree waits for the device)
  StreamOwner so, so2;
  EventOwner eo0, eo1, eo_join;
  CNO_CUDA(so.create());
  CNO_CUDA(so2.create());
  CNO_CUDA(eo0.create());
  CNO_CUDA(eo1.create());
  CNO_CUDA(eo_join.create());
  const cudaStream_t s = so.s, s2 = so2.s;
  const cudaEvent_t e0 = eo0.e, e1 = eo1.e, e_start2 = eo_join.e;

  // One device arena: x0 | x | g | value | x_delta | f_delta | gnorm | iters | nfev | status | ws | data
  const size_t data_bytes = problem->data ? (size_t)batch * (size_t)problem->data_stride * ts : 0;
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  size_t off = 0;
  const size_t o_x0 = off; off += up(vec_bytes);
  const size_t o_x = off; off += out->x ? up(vec_bytes) : 0;
  const size_t o_g = off; off += out->gradient ? up(vec_bytes) : 0;
  const size_t o_f = off; off += out->value ? up(sc_bytes) : 0;
  const size_t o_xd = off; off += out->x_delta ? up(sc_bytes) : 0;
  const size_t o_fd = off; off += out->f_delta ? up(sc_bytes) : 0;
  const size_t o_gn = off; off += out->gradient_norm ? up(sc_bytes) : 0;
  const size_t o_it = off; off += out->num_iterations ? up((size_t)batch * 4) : 0;
  const size_t o_nf = off; off += out->nfev ? up((size_t)batch * 4) : 0;
  const size_t o_st = off; off += out->status ? up((size_t)batch) : 0;
  const size_t o_ws = off; off += kWorkspaceBytes;  // one 16-byte queue slot per chunk
  const size_t o_data = off; off += up(data_bytes);
  DeviceBuffer arena_owner;  // (a private arena when another thread holds the cached one)
  std::unique_lock<std::mutex> arena_lock(g_host_arena.m, std::try_to_lock);
  struct Drain {  // on every return path: no copy or kernel of this call still uses the arena when it is handed on
    cudaStream_t a, b;
    ~Drain() { cudaStreamSynchronize(a); cudaStreamSynchronize(b); }
  } drain{s, s2};
  unsigned char* arena = nullptr;
  if (arena_lock.owns_lock()) {
    int dev = 0;
    CNO_CUDA(cudaGetDevice(&dev));
    if (g_host_arena.device != dev || g_host_arena.bytes < off) {
      if (g_host_arena.p) {
        int prev = dev;
        if (g_host_arena.device >= 0 && g_host_arena.device != dev) { cudaSetDevice(g_host_arena.device); prev = g_host_arena.device; }
        cudaFree(g_host_arena.p);
        if (prev != dev) cudaSetDevice(dev);
        g_host_arena.p = nullptr;
        g_host_arena.bytes = 0;
      }
      CNO_CUDA(cudaMalloc(&g_host_arena.p, off));
      g_host_arena.bytes = off;
      g_host_arena.device = dev;
    }
    arena = static_cast<unsigned char*>(g_host_arena.p);
  } else {
    CNO_CUDA(arena_owner.alloc(off));
    arena = static_cast<unsigned char*>(arena_owner.p);
  }

  // Chunked pipeline on two streams: H2D of chunk c+1 and D2H of chunk c-1 overlap
  // the solve of chunk c, so only ~1/kChunks of the copy time is exposed.
  cudaStream_t streams[2] = {s, s2};
  const int64_t min_chunk = 16384;
  int chunks = (int)((batch + min_chunk - 1) / min_chunk);
  if (chunks > 8) chunks = 8;
  if (chunks < 1) chunks = 1;
  const int64_t per = (batch + chunks - 1) / chunks;
  CNO_CUDA(cudaEventRecord(e0, s));
  CNO_CUDA(cudaStreamWaitEvent(s2, e0, 0));  // both streams start after e0
  cno_launch_info_t kinfo;
  memset(&kinfo, 0, sizeof(kinfo));
  const size_t stride_bytes = (size_t)problem->data_stride * ts;
  for (int c = 0; c < chunks; ++c) {
    const int64_t lo = c * per;
    const int64_t n = (lo + per <= batch) ? per : (batch - lo);
    if (n <= 0) break;
    cudaStream_t st = streams[c & 1];
    const size_t vlo = (size_t)lo * d * ts, vn = (size_t)n * d * ts, slo = (size_t)lo * ts, sn = (size_t)n * ts;
    CNO_CUDA(cudaMemcpyAsync(arena + o_x0 + vlo, (const char*)x0 + vlo, vn, cudaMemcpyHostToDevice, st));
    local.h2d_bytes += (int64_t)vn;
    cno_problem_t dprob = *problem;
    if (data_bytes) {
      CNO_CUDA(cudaMemcpyAsync(arena + o_data + (size_t)lo * stride_bytes,
                               (const char*)problem->data + (size_t)lo * stride_bytes,
                               (size_t)n * stride_bytes, cudaMemcpyHostToDevice, st));
      dprob.data = arena + o_data + (size_t)lo * stride_bytes;
      local.h2d_bytes += (int64_t)((size_t)n * stride_bytes);
    }
    cno_batch_out_t dout;
    dout.x = out->x ? arena + o_x + vlo : nullptr;
    dout.gradient = out->gradient ? arena + o_g + vlo : nullptr;
    dout.value = out->value ? arena + o_f + slo : nullptr;
    dout.x_delta = out->x_delta ? arena + o_xd + slo : nullptr;
    dout.f_delta = out->f_delta ? arena + o_fd + slo : nullptr;
    dout.gradient_norm = out->gradient_norm ? arena + o_gn + slo : nullptr;
    dout.num_iterations = out->num_iterations ? (uint32_t*)(arena + o_it) + lo : nullptr;
    dout.nfev = out->nfev ? (uint32_t*)(arena + o_nf) + lo : nullptr;
    dout.status = out->status ? (int8_t*)(arena + o_st) + lo : nullptr;
    const LaunchArgs a{&dprob, (long long)n, arena + o_x0 + vlo, stop, &dout,
                       arena + o_ws + (size_t)c * 16, st, &kinfo};
    rc = find_entry(solver, problem)->fn(a);
    if (rc) return rc;
    auto down = [&](void* host, size_t o, size_t off, size_t bytes) -> cudaError_t {
      if (!host) return cudaSuccess;
      local.d2h_bytes += (int64_t)bytes;
      return cudaMemcpyAsync((char*)host + off, arena + o + off, bytes, cudaMemcpyDeviceToHost, st);
    };
    CNO_CUDA(down(out->x, o_x, vlo, vn));
    CNO_CUDA(down(out->gradient, o_g, vlo, vn));
    CNO_CUDA(down(out->value, o_f, slo, sn));
    CNO_CUDA(down(out->x_delta, o_xd, slo, sn));
    CNO_CUDA(down(out->f_delta, o_fd, slo, sn));
    CNO_CUDA(down(out->gradient_norm, o_gn, slo, sn));
    CNO_CUDA(down(out->num_iterations, o_it, (size_t)lo * 4, (size_t)n * 4));
    CNO_CUDA(down(out->nfev, o_nf, (size_t)lo * 4, (size_t)n * 4));
    CNO_CUDA(down(out->status, o_st, (size_t)lo, (size_t)n));
  }
  CNO_CUDA(cudaEventRecord(e_start2, s2));
  CNO_CUDA(cudaStreamWaitEvent(s, e_start2, 0));  // join
  CNO_CUDA(cudaEventRecord(e1, s));
  CNO_CUDA(cudaEventSynchronize(e1));
  float ms = 0;
  CNO_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  const int64_t h2d = local.h2d_bytes, d2h = local.d2h_bytes;
  local = kinfo;
  local.h2d_bytes = h2d;
  local.d2h_bytes = d2h;
  local.total_ms = ms;
  local.kernel_ms = ms;
  if (info) *info = local;
  return CNO_OK;
}

void cno_lbfgsb_default_stop(cno_stop_t* s) {  // solver/lbfgsb.h:78-81
  if (!s) return;
  cno_default_stop(s);
  s->f_delta = 2.22e-9;
  s->f_delta_relative = 1;
}

int cno_lbfgsb_supported(const cno_problem_t* problem) {
  if (!problem) return CNO_ERR_INVALID_ARGUMENT;
  return lbfgsb_find(problem) ? CNO_OK : CNO_ERR_UNSUPPORTED;
}

int cno_lbfgsb_minimize(const cno_problem_t* problem, const cno_bounds_t* bounds, int64_t batch, const void* x0,
                        const cno_stop_t* stop, const cno_batch_out_t* out, void* workspace, size_t workspace_bytes,
                        void* stream, cno_launch_info_t* info) {
  if (!problem) return CNO_ERR_INVALID_ARGUMENT;
  const LbfgsbEntry* e = lbfgsb_find(problem);
  if (!e) return CNO_ERR_UNSUPPORTED;
  if (batch < 0 || !out) return CNO_ERR_INVALID_ARGUMENT;
  if (info) memset(info, 0, sizeof(*info));
  if (batch == 0) return have_device() ? CNO_OK : CNO_ERR_NO_DEVICE;
  if (!x0) return CNO_ERR_INVALID_ARGUMENT;
  if (bounds && bounds->stride != 0 && bounds->stride < problem->d) return CNO_ERR_INVALID_ARGUMENT;
  if (!queue_workspace_ok(workspace, workspace_bytes)) return CNO_ERR_WORKSPACE;
  if (!io_aligned(x0, out)) return CNO_ERR_INVALID_ARGUMENT;
  cno_stop_t local;
  int rc = resolve_stop(stop, &local, cno_lbfgsb_default_stop);
  if (rc) return rc;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cno::LaunchTimer timer(s, info);
  if ((rc = timer.start(g_last_cuda))) return rc;
  const LbfgsbArgs a{problem, bounds, (long long)batch, x0, stop, out, workspace, s, info};
  if ((rc = e->fn(a))) return rc;
  return timer.stop(g_last_cuda);
}

int cno_evaluate(const cno_problem_t* problem, int64_t batch, const void* x, void* value, void* gradient,
                 void* stream) {
  if (!problem || batch < 0) return CNO_ERR_INVALID_ARGUMENT;
  if (problem->dtype != CNO_F64 && problem->dtype != CNO_F32) return CNO_ERR_INVALID_ARGUMENT;
  if (problem->policy != default_policy(problem->dtype)) return CNO_ERR_UNSUPPORTED;
  for (const EvalEntry& e : kEvalTable)
    if (e.family == problem->family && e.dtype == problem->dtype && e.d == problem->d) {
      if (!have_device()) return CNO_ERR_NO_DEVICE;
      return e.fn(problem, batch, x, value, gradient, stream);
    }
  return CNO_ERR_UNSUPPORTED;
}

int cno_condition_hessian(const cno_problem_t* problem, int64_t batch, const void* x, void* condition,
                          void* workspace, size_t workspace_bytes, void* stream) {
  if (!problem || batch < 0) return CNO_ERR_INVALID_ARGUMENT;
  if (problem->dtype != CNO_F64 && problem->dtype != CNO_F32) return CNO_ERR_INVALID_ARGUMENT;
  if (problem->policy != default_policy(problem->dtype)) return CNO_ERR_UNSUPPORTED;  // (the fused-LU policy has no condition-number kernel)
  for (const CondEntry& e : kCondTable)
    if (e.family == problem->family && e.dtype == problem->dtype && e.d == problem->d) {
      if (batch == 0) return CNO_OK;
      if (!x || !condition || !workspace || workspace_bytes < sizeof(unsigned long long) ||
          ((uintptr_t)workspace & 7) || ((uintptr_t)x & 15))
        return CNO_ERR_INVALID_ARGUMENT;
      if (!have_device()) return CNO_ERR_NO_DEVICE;
      const CondArgs a{problem, (long long)batch, x, condition, workspace, static_cast<cudaStream_t>(stream)};
      return e.fn(a);
    }
  return CNO_ERR_UNSUPPORTED;
}

int cno_release_host_arena(void) {
  std::lock_guard<std::mutex> lk(g_host_arena.m);
  if (g_host_arena.p) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (g_host_arena.device >= 0 && g_host_arena.device != dev) cudaSetDevice(g_host_arena.device);
    cudaError_t e = cudaFree(g_host_arena.p);
    if (g_host_arena.device != dev) cudaSetDevice(dev);
    g_host_arena.p = nullptr;
    g_host_arena.bytes = 0;
    g_host_arena.device = -1;
    if (e != cudaSuccess) { g_last_cuda = e; return CNO_ERR_CUDA; }
  }
  return CNO_OK;
}

int cno_fill_uniform(int dtype, void* dst, int64_t first, int64_t count, uint64_t seed,
                     double lo, double hi, void* stream) {
  if (!dst || count < 0 || (dtype != CNO_F64 && dtype != CNO_F32)) return CNO_ERR_INVALID_ARGUMENT;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  if (count == 0) return CNO_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int block = 256;
  int sms = 0;
  const int rc = cno::device_sm_count(&sms, g_last_cuda);
  if (rc) return rc;
  long long blocks = (count + block - 1) / block;
  if (blocks > (long long)sms * 16) blocks = (long long)sms * 16;  // grid-stride loop: 16 blocks per SM
  if (dtype == CNO_F64)
    fill_uniform_kernel<double><<<(int)blocks, block, 0, s>>>((double*)dst, first, count, seed, lo, hi);
  else
    fill_uniform_kernel<float><<<(int)blocks, block, 0, s>>>((float*)dst, first, count, seed, (float)lo, (float)hi);
  CNO_CUDA(cudaGetLastError());
  return CNO_OK;
}

int cno_done_bitmap(const int8_t* status, int64_t batch, uint32_t* words, void* stream) {
  if (!status || !words || batch < 0) return CNO_ERR_INVALID_ARGUMENT;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  if (batch == 0) return CNO_OK;
  const int block = 256;
  const long long blocks = (batch + block - 1) / block;
  done_bitmap_kernel<<<(unsigned)blocks, block, 0, static_cast<cudaStream_t>(stream)>>>(status, batch, words);
  CNO_CUDA(cudaGetLastError());
  return CNO_OK;
}

// ncclAllGather(sendbuff, recvbuff, sendcount, datatype, comm, stream), resolved at first use so that libcno.so
// has no link-time dependency on NCCL (ncclUint32 = 3 in every NCCL 2.x nccl.h).
typedef int (*nccl_allgather_t)(const void*, void*, size_t, int, void*, cudaStream_t);
static nccl_allgather_t resolve_nccl_allgather() {
  static std::once_flag once;
  static nccl_allgather_t fn = nullptr;
  std::call_once(once, [] {
    void* sym = dlsym(RTLD_DEFAULT, "ncclAllGather");  // already in the process (e.g. loaded by PyTorch)
    if (!sym) {
      void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
      if (h) sym = dlsym(h, "ncclAllGather");
    }
    fn = reinterpret_cast<nccl_allgather_t>(sym);
  });
  return fn;
}

int cno_allgather_done(void* comm, const uint32_t* local_words, uint32_t* all_words, size_t words, void* stream) {
  if (!comm || !local_words || !all_words) return CNO_ERR_INVALID_ARGUMENT;
  if (words == 0) return CNO_OK;
  const nccl_allgather_t allgather = resolve_nccl_allgather();
  if (!allgather) return CNO_ERR_UNSUPPORTED;
  const int rc = allgather(local_words, all_words, words, /*ncclUint32*/ 3, comm, static_cast<cudaStream_t>(stream));
  if (rc != 0) { g_last_cuda = cudaErrorUnknown; return CNO_ERR_CUDA; }
  return CNO_OK;
}

int cno_count_done(const uint32_t* all_words, int32_t ranks, size_t words_per_rank, const int64_t* bits_per_rank,
                   int64_t* total_done, void* stream) {
  if (!all_words || ranks <= 0 || !bits_per_rank || !total_done) return CNO_ERR_INVALID_ARGUMENT;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DeviceBuffer dcount;
  CNO_CUDA(dcount.alloc(sizeof(unsigned long long)));
  CNO_CUDA(cudaMemsetAsync(dcount.p, 0, sizeof(unsigned long long), s));
  for (int r = 0; r < ranks; ++r) {
    const long long bits = (long long)bits_per_rank[r];
    if (bits < 0 || (size_t)((bits + 31) / 32) > words_per_rank) return CNO_ERR_INVALID_ARGUMENT;
    if (bits == 0) continue;
    const long long nw = (bits + 31) / 32;
    count_bits_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, s>>>(all_words + (size_t)r * words_per_rank, bits,
                                                                   static_cast<unsigned long long*>(dcount.p));
    CNO_CUDA(cudaGetLastError());
  }
  unsigned long long h = 0;
  CNO_CUDA(cudaMemcpyAsync(&h, dcount.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  CNO_CUDA(cudaStreamSynchronize(s));
  *total_done = (int64_t)h;
  return CNO_OK;
}

int cno_device_cstep(double io[11], int* brackt, int* info, int* ret) {
  if (!io || !brackt || !info || !ret) return CNO_ERR_INVALID_ARGUMENT;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  DeviceBuffer bio, bfl;
  CNO_CUDA(bio.alloc(11 * sizeof(double)));
  CNO_CUDA(bfl.alloc(3 * sizeof(int)));
  double* const dio = static_cast<double*>(bio.p);
  int* const dfl = static_cast<int*>(bfl.p);
  int fl[3] = {*brackt, *info, 0};
  CNO_CUDA(cudaMemcpy(dio, io, 11 * sizeof(double), cudaMemcpyHostToDevice));
  CNO_CUDA(cudaMemcpy(dfl, fl, sizeof(fl), cudaMemcpyHostToDevice));
  cstep_kernel<<<1, 1>>>(dio, dfl);
  CNO_CUDA(cudaGetLastError());
  CNO_CUDA(cudaMemcpy(io, dio, 11 * sizeof(double), cudaMemcpyDeviceToHost));
  CNO_CUDA(cudaMemcpy(fl, dfl, sizeof(fl), cudaMemcpyDeviceToHost));
  *brackt = fl[0];
  *info = fl[1];
  *ret = fl[2];
  return CNO_OK;
}

int cno_device_div_check(const double* a, const double* b, int64_t n, double* helper, double* plain,
                         int32_t* accepted) {
  if (!a || !b || !helper || !plain || !accepted || n < 0) return CNO_ERR_INVALID_ARGUMENT;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  if (n == 0) return CNO_OK;
  DeviceBuffer da, db, dh, dp, dk;
  const size_t bytes = (size_t)n * sizeof(double);
  CNO_CUDA(da.alloc(bytes));
  CNO_CUDA(db.alloc(bytes));
  CNO_CUDA(dh.alloc(bytes));
  CNO_CUDA(dp.alloc(bytes));
  CNO_CUDA(dk.alloc((size_t)n * sizeof(int)));
  CNO_CUDA(cudaMemcpy(da.p, a, bytes, cudaMemcpyHostToDevice));
  CNO_CUDA(cudaMemcpy(db.p, b, bytes, cudaMemcpyHostToDevice));
  div_check_kernel<<<(unsigned)((n + 255) / 256), 256>>>(static_cast<const double*>(da.p), static_cast<const double*>(db.p),
                                                         (long long)n, static_cast<double*>(dh.p),
                                                         static_cast<double*>(dp.p), static_cast<int*>(dk.p));
  CNO_CUDA(cudaGetLastError());
  CNO_CUDA(cudaMemcpy(helper, dh.p, bytes, cudaMemcpyDeviceToHost));
  CNO_CUDA(cudaMemcpy(plain, dp.p, bytes, cudaMemcpyDeviceToHost));
  CNO_CUDA(cudaMemcpy(accepted, dk.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  return CNO_OK;
}

void cno_al_default_config(cno_al_config_t* c) {  // augmented_lagrangian.h:63-239
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->penalty_growth_factor = 10;
  c->violation_shrink_ratio = 0.25;
  c->auto_scale_initial_penalty = 1;
  c->penalty_auto_objective_scale = 10;
  c->penalty_auto_min = 1e-8;
  c->penalty_auto_max = 1e8;
  c->warmup_max_inner_iterations = 10;
  c->warmup_inner_gradient_tolerance = 1e-2;
  c->multiplier_max = 1e20;
  c->kkt_gradient_tolerance = 1e-4;
}

void cno_al_default_stop(cno_al_stop_t* s) {  // progress.h:126, 353-431
  if (!s) return;
  s->num_iterations = 10000;
  s->constraint_threshold = 1e-5;
  s->kkt_stationarity_threshold = 1e-4;
}

int cno_al_supported(const cno_problem_t* objective, const cno_constraints_t* constraints) {
  return al_check(objective, constraints);
}

int cno_al_workspace_bytes(const cno_problem_t* objective, const cno_constraints_t* constraints,
                           int64_t batch, size_t* bytes) {
  int rc = al_check(objective, constraints);
  if (rc) return rc;
  if (!bytes || batch < 0) return CNO_ERR_INVALID_ARGUMENT;
  const size_t ts = objective->dtype == CNO_F64 ? 8 : 4;
  *bytes = cno::AlLayout((size_t)batch, (size_t)objective->d, (size_t)constraints->n_eq,
                         (size_t)constraints->n_ineq, ts).total;
  return CNO_OK;
}

int cno_al_minimize(const cno_problem_t* objective, const cno_constraints_t* constraints,
                    int64_t batch, const void* x0, const void* eq0, const void* ineq0,
                    const void* penalty0, const cno_stop_t* inner_stop,
                    const cno_al_stop_t* outer_stop, const cno_al_config_t* config,
                    const cno_al_out_t* out, void* workspace, size_t workspace_bytes, void* stream,
                    cno_launch_info_t* info) {
  int rc = al_check(objective, constraints);
  if (rc) return rc;
  if (batch < 0 || !out) return CNO_ERR_INVALID_ARGUMENT;
  if (info) memset(info, 0, sizeof(*info));
  if (batch == 0) return have_device() ? CNO_OK : CNO_ERR_NO_DEVICE;
  cno::AlArgs a{(long long)batch, x0, eq0, ineq0, penalty0, inner_stop, outer_stop, config, out,
                static_cast<unsigned char*>(workspace), workspace_bytes, static_cast<cudaStream_t>(stream), info};
  cno_stop_t idflt;
  cno_al_stop_t odflt;
  cno_al_config_t cdflt;
  if ((rc = cno::al_check_args(a, (size_t)objective->d, constraints->n_eq, constraints->n_ineq,
                               objective->dtype == CNO_F64 ? 8 : 4, &idflt, &odflt, &cdflt)))
    return rc;
  if (!have_device()) return CNO_ERR_NO_DEVICE;
  return al_find(objective)->fn(objective, constraints, a);
}

#ifdef CNO_LBFGS_PHASE_CLOCKS
// The phase probe's counters of lbfgs_minimize_kernel (cno_lbfgs.cuh), copied to out[0 .. n) and zeroed.  Only a
// measurement build compiled with -DCNO_LBFGS_PHASE_CLOCKS has it (tools/lbfgs_phase_clocks.py).
int cno_lbfgs_phase_clocks_take(unsigned long long* out, int n) {
  if (n != cno::kPhSlots) return CNO_ERR_INVALID_ARGUMENT;
  unsigned long long zero[cno::kPhSlots] = {};
  if (cudaMemcpyFromSymbol(out, cno::cno_lbfgs_phase_clocks, sizeof(zero)) != cudaSuccess ||
      cudaMemcpyToSymbol(cno::cno_lbfgs_phase_clocks, zero, sizeof(zero)) != cudaSuccess)
    return CNO_ERR_CUDA;
  return CNO_OK;
}
#endif

}  // extern "C"
