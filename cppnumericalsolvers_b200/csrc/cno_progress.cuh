// cno_progress.cuh -- the per-instance life every persistent solver kernel shares around its solver step: claim the
// next instance from the work queue, start Progress, update it once per iteration (progress.h:153-327), and write
// the instance's result record (BatchOut).  The host half is launch_persistent (cno_launch.cuh), which zeroes the
// queue counter before each launch.
#ifndef CNO_PROGRESS_CUH_
#define CNO_PROGRESS_CUH_

#include "cno_device.cuh"
#include "cno_kernel_params.h"

namespace cno {

// The next instance index from the work queue, the same in every lane of the warp.
__device__ __forceinline__ unsigned long long claim_instance(unsigned long long* queue, const int lane) {
  unsigned long long b = 0;
  if (lane == 0) b = atomicAdd(queue, 1ULL);
  return __shfl_sync(kFullMask, b, 0);
}

// progress.h:153-327 on warp-uniform scalars (FunctionState branch).  The
// past-f ring (progress.h:138-140) lives in the warp's shared-memory slice.
template <class T>
struct ProgressState {
  uint32_t num_iterations;
  int x_delta_violations;
  int f_delta_violations;
  T x_delta, f_delta, gradient_norm;
  int ring_size, ring_pos;
  int status;
};

// Progress before the first iteration (progress.h:87-140).  Filled in place: returned by value, the state takes two
// more registers in some kernels (GradientDescent with HagerZhang).
template <class T>
__device__ __forceinline__ void progress_start(ProgressState<T>& p) {
  p.num_iterations = 0;
  p.x_delta_violations = 0;
  p.f_delta_violations = 0;
  p.x_delta = p.f_delta = p.gradient_norm = T(0);
  p.ring_size = 0;
  p.ring_pos = 0;
  p.status = CNO_STATUS_NOT_STARTED;
}

// progress.h:153-277: the counters and the tests before the plateau test.  Returns the status they decide.
template <class T>
__device__ __forceinline__ int progress_update_head(ProgressState<T>& p, const StopParams<T>& stop, T prev_value,
                                                    T cur_value, T x_delta, T gradient_norm) {
  p.num_iterations++;
  p.f_delta = cabs(cur_value - prev_value);
  p.x_delta = x_delta;
  p.gradient_norm = gradient_norm;
  int status = CNO_STATUS_CONTINUE;
  // Tests in the reference's order; the first that fires wins (each `return`
  // of progress.h becomes "status already set").
  if ((stop.num_iterations > 0) && ((unsigned long long)p.num_iterations > stop.num_iterations))
    status = CNO_STATUS_ITERATION_LIMIT;  // :212-216
  if (status == CNO_STATUS_CONTINUE) {    // :254-262
    if ((stop.x_delta > 0) && (p.x_delta < stop.x_delta)) {
      p.x_delta_violations++;
      if (p.x_delta_violations >= stop.x_delta_violations) status = CNO_STATUS_X_DELTA_VIOLATION;
    } else {
      p.x_delta_violations = 0;
    }
  }
  if (status == CNO_STATUS_CONTINUE) {  // :263-277
    if ((stop.f_delta > 0) &&
        (p.f_delta < stop.f_delta * (stop.f_delta_relative
                                         ? smax(smax(cabs(cur_value), cabs(prev_value)), T(1))
                                         : T(1)))) {
      p.f_delta_violations++;
      if (p.f_delta_violations >= stop.f_delta_violations) status = CNO_STATUS_F_DELTA_VIOLATION;
    } else {
      p.f_delta_violations = 0;
    }
  }
  return status;
}

// progress.h:299-317: the gradient-norm test, when no earlier test has fired.
template <class T>
__device__ __forceinline__ int progress_gradient_test(int status, const ProgressState<T>& p, const StopParams<T>& stop,
                                                      T x_inf) {
  if (status == CNO_STATUS_CONTINUE && stop.gradient_norm > 0) {  // :299-317
    const T scale = stop.gradient_norm_relative ? smax(T(1), x_inf) : T(1);
    if (p.gradient_norm < stop.gradient_norm * scale) status = CNO_STATUS_GRADIENT_NORM_VIOLATION;
  }
  return status;
}

template <class T>
__device__ __forceinline__ void progress_update(ProgressState<T>& p, const StopParams<T>& stop,
                                                T* __restrict__ ring, const int lane,
                                                T prev_value, T cur_value, T x_delta,
                                                T gradient_norm, T x_inf) {
  int status = progress_update_head(p, stop, prev_value, cur_value, x_delta, gradient_norm);
  if (uni(status == CNO_STATUS_CONTINUE && stop.past > 0)) {  // :280-298
    const int pp = stop.past;
    if (uni(p.ring_size != pp)) {
      if (lane < pp) ring[lane] = cur_value;
      p.ring_size = pp;
      p.ring_pos = 0;
      __syncwarp();
    }
    bool fired = false;
    if (uni((int)p.num_iterations > pp)) {
      const T past_f = ring[p.ring_pos];
      // rate = |past_f - f| / max(1, |f|) < past_delta (:287-290)?  A difference above twice (below half) the product
      // past_delta * max(1, |f|) decides it without the division: the quotient is then above 2 (below 0.5) past_delta
      // up to two roundings.  In between, or with a non-finite operand: the specification's expression.
      const T diff = cabs(past_f - cur_value), mag = smax(T(1), cabs(cur_value));
      const T bound = stop.past_delta * mag;
      if (cfinite(diff) && cfinite(bound) && bound > T(0) && diff > T(2) * bound) {
        fired = false;
      } else if (cfinite(diff) && cfinite(bound) && bound >= Num<T>::min_normal && diff < T(0.5) * bound) {
        fired = true;
      } else {
        const T rate = diff / mag;
        fired = rate < stop.past_delta;
      }
    }
    if (uni(fired)) {
      status = CNO_STATUS_F_DELTA_VIOLATION;
    } else {
      __syncwarp();
      if (lane == 0) ring[p.ring_pos] = cur_value;
      p.ring_pos = (p.ring_pos + 1 == pp) ? 0 : p.ring_pos + 1;
      __syncwarp();
    }
  }
  p.status = progress_gradient_test(status, p, stop, x_inf);
}

// The scalars of instance b's result record, written by one thread: the returned FunctionState's value and Progress.
template <class T>
__device__ __forceinline__ void store_result_scalars(const BatchOut<T>& out, const unsigned long long b, const T f,
                                                     const ProgressState<T>& prog, const uint32_t nfev) {
  if (out.value) out.value[b] = f;
  if (out.num_iterations) out.num_iterations[b] = prog.num_iterations;
  if (out.status) out.status[b] = (int8_t)prog.status;
  if (out.nfev) out.nfev[b] = nfev;
  if (out.x_delta) out.x_delta[b] = prog.x_delta;
  if (out.f_delta) out.f_delta[b] = prog.f_delta;
  if (out.gradient_norm) out.gradient_norm[b] = prog.gradient_norm;
}

// Instance b's whole result record from the warp that solved it (x and g: Shape<D>::E elements per lane).
template <class T, int D>
__device__ __forceinline__ void store_result(const BatchOut<T>& out, const unsigned long long b, const int lane,
                                             const T (&x)[Shape<D>::E], const T (&g)[Shape<D>::E], const T f,
                                             const ProgressState<T>& prog, const uint32_t nfev) {
  if (out.x) store_row<T, D>(out.x + b * D, lane, x);
  if (out.gradient) store_row<T, D>(out.gradient + b * D, lane, g);
  if (lane == 0) store_result_scalars<T>(out, b, f, prog, nfev);
  __syncwarp();
}

}  // namespace cno

#endif  // CNO_PROGRESS_CUH_
