// cno_auglag_launch.cuh -- the CUDA side of AugmentedLagrangian::Minimize, shared by cno_al_minimize (libcno.so,
// cno_api.cu: built-in objectives on [a | t] rows) and cno_<tag>_al_minimize (include/cppoptlib_b200/device.cuh: user
// functors and composites with functor constraints).  Both run cno::al_outer_loop (cno_auglag_host.h) on this backend,
// so both check their arguments, lay out the workspace (AlLayout) and count kernel launches the same way.
// Errors: a failing CUDA call is CNO_ERR_CUDA, its cudaError_t goes to the caller's `last_error`.
#ifndef CNO_AUGLAG_LAUNCH_CUH_
#define CNO_AUGLAG_LAUNCH_CUH_

#include <cuda_runtime.h>

#include "../../include/cno_al.h"
#include "cno_auglag.cuh"
#include "cno_auglag_host.h"
#include "cno_launch.cuh"
#include "cno_lbfgs.cuh"

namespace cno {

// The arguments of cno_al_minimize that do not describe the problem.
struct AlArgs {
  long long batch;
  const void* x0;
  const void* eq0;
  const void* ineq0;
  const void* penalty0;
  const cno_stop_t* inner_stop;
  const cno_al_stop_t* outer_stop;
  const cno_al_config_t* config;
  const cno_al_out_t* out;
  unsigned char* workspace;
  size_t workspace_bytes;
  cudaStream_t stream;
  cno_launch_info_t* info;
};

// The checks of a call with batch > 0 on a problem of dimension d with ne / ni constraints and ts-byte scalars, in
// this order: the state arrays of cno_al_out_t, 16-byte aligned x0 / x, the workspace (AlLayout bytes, 256-byte
// aligned), the inner stop's `past`.  NULL inner_stop / outer_stop / config become the defaults in the *_local copies.
inline int al_check_args(AlArgs& A, size_t d, int ne, int ni, size_t ts, cno_stop_t* inner_local,
                         cno_al_stop_t* outer_local, cno_al_config_t* config_local) {
  const cno_al_out_t* out = A.out;
  if (!A.x0 || !out->x || !out->penalty || !out->max_violation || !out->max_lagrangian_gradient ||
      !out->num_iterations || !out->status || !out->nfev)
    return CNO_ERR_INVALID_ARGUMENT;  // they are the solver's state between outer iterations
  if ((ne > 0 && !out->equality_multipliers) || (ni > 0 && !out->inequality_multipliers))
    return CNO_ERR_INVALID_ARGUMENT;
  if (((uintptr_t)A.x0 & 15) || ((uintptr_t)out->x & 15)) return CNO_ERR_INVALID_ARGUMENT;
  const AlLayout L((size_t)A.batch, d, (size_t)ne, (size_t)ni, ts);
  if (!A.workspace || A.workspace_bytes < L.total || ((uintptr_t)A.workspace & 255)) return CNO_ERR_WORKSPACE;
  if (!A.inner_stop) {
    cno_default_stop(inner_local);
    A.inner_stop = inner_local;
  }
  // the kernels' past-f ring is CNO_MAX_PAST warp-private scalars
  if (A.inner_stop->past > CNO_MAX_PAST || A.inner_stop->past < 0) return CNO_ERR_INVALID_ARGUMENT;
  if (!A.outer_stop) {
    cno_al_default_stop(outer_local);
    A.outer_stop = outer_local;
  }
  if (!A.config) {
    cno_al_default_config(config_local);
    A.config = config_local;
  }
  return CNO_OK;
}

// The CUDA backend of cno::al_outer_loop: the three AL kernels on a grid of kAlWarps-warp blocks, the inner solve as
// the persistent lbfgs_minimize_kernel<AugLagFn<Obj, Cons>, CNO_LBFGS_M>.
template <class Obj, class Cons>
struct AlCudaBackend {
  using T = typename Obj::Scalar;
  const Obj& obj;
  const Cons& cons;
  const AlArgs& A;
  AlArrays<T> a;
  AlView<T> view;
  AlParams<T> p;
  unsigned long long* queue;
  cudaError_t& last_error;
  int blocks, threads;

  int copy_or_zero(void* dst, const void* src, size_t bytes) {
    if (!bytes || src == dst) return CNO_OK;  // (a caller may pass its state arrays as the initial values)
    return cuda_rc(src ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, A.stream)
                       : cudaMemsetAsync(dst, 0, bytes, A.stream),
                   last_error);
  }
  int fill(void* dst, int byte, size_t bytes) {
    return bytes ? cuda_rc(cudaMemsetAsync(dst, byte, bytes, A.stream), last_error) : CNO_OK;
  }
  int autoscale() {
    al_autoscale_kernel<Obj, Cons><<<blocks, threads, 0, A.stream>>>(obj, view, A.batch, p, a, cons);
    return cuda_rc(cudaGetLastError(), last_error);
  }
  int inner(const cno_stop_t& stop) {
    using Fn = AugLagFn<Obj, Cons>;
    const Fn composite(obj, view, cons);
    cno_batch_out_t inner_out{};
    inner_out.x = a.x_work;
    inner_out.nfev = const_cast<uint32_t*>(a.inner_nfev);
    cno_launch_info_t inner_info{};
    return launch_persistent<typename LbfgsPlan<Fn, CNO_LBFGS_M, false, LsMoreThuente>::SM>(
        lbfgs_minimize_kernel<Fn, CNO_LBFGS_M, false, LsMoreThuente>, A.batch, queue, A.stream, &inner_info, last_error,
        composite, static_cast<const T*>(a.x), A.batch, make_stop<T>(stop), make_out<T>(inner_out), queue,
        ResumeArgs{nullptr, 0, 0, 0});
  }
  int outer_step(int* remaining) {
    int rc = cuda_rc(cudaMemsetAsync(a.remaining, 0, sizeof(int), A.stream), last_error);
    if (rc) return rc;
    al_outer_step_kernel<Obj, Cons><<<blocks, threads, 0, A.stream>>>(obj, view, A.batch, p, a, cons);
    if ((rc = cuda_rc(cudaGetLastError(), last_error))) return rc;
    if ((rc = cuda_rc(cudaMemcpyAsync(remaining, a.remaining, sizeof(int), cudaMemcpyDeviceToHost, A.stream),
                      last_error)))
      return rc;
    return cuda_rc(cudaStreamSynchronize(A.stream), last_error);
  }
  int finalize() {
    al_finalize_kernel<T, Obj::Dim><<<blocks, threads, 0, A.stream>>>(A.batch, view.n_eq, view.n_ineq, a);
    return cuda_rc(cudaGetLastError(), last_error);
  }
};

// AugmentedLagrangian::Minimize for a batch that passed al_check_args: k gives the constraint counts (and, for
// AlRows, the rows), cons evaluates the constraints.  Fills info (timing, kernel_launches) when given.
template <class Obj, class Cons>
inline int al_run(const Obj& obj, const Cons& cons, const cno_constraints_t& k, const AlArgs& A,
                  cudaError_t& last_error) {
  using T = typename Obj::Scalar;
  constexpr int D = Obj::Dim;
  const int ne = k.n_eq, ni = k.n_ineq;
  const AlLayout L((size_t)A.batch, D, (size_t)ne, (size_t)ni, sizeof(T));
  LaunchTimer timer(A.stream, A.info);
  int rc = timer.start(last_error);
  if (rc) return rc;
  AlCudaBackend<Obj, Cons> be{obj,
                              cons,
                              A,
                              al_make_arrays<T>(*A.out, A.workspace, L),
                              {},
                              {},
                              reinterpret_cast<unsigned long long*>(A.workspace + L.queue),
                              last_error,
                              (int)((A.batch + kAlWarps - 1) / kAlWarps),
                              kAlWarps * 32};
  be.view = al_make_view<T>(k, be.a);
  be.p = al_make_params<T>(*A.config, *A.outer_stop);
  int launches = 0;
  rc = al_outer_loop<T>(be, be.a, A.batch, D, ne, ni, A.x0, A.eq0, A.ineq0, A.penalty0, *A.inner_stop, *A.config,
                        &launches);
  if (rc) return rc;
  if (A.info) A.info->kernel_launches = launches;
  return timer.stop(last_error);
}

}  // namespace cno

#endif  // CNO_AUGLAG_LAUNCH_CUH_
