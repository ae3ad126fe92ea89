// cno_descent.cuh -- batched GradientDescent<F>::Minimize and
// ConjugatedGradientDescent<F>::Minimize, one warp per instance, the whole
// Solver::Minimize loop in one persistent kernel (sm_90a).
//
// Reference path (include/cppoptlib/...):
//   solver/solver.h:181-224                      Solver::Minimize driver loop
//   solver/gradient_descent.h:64-73              d = -g, MoreThuente::Search, x - rate g
//   linesearch/more_thuente.h:63-77              Search(x, d, f): evaluate, cvsrch, return alpha
//   solver/conjugated_gradient_descent.h:62-86   Fletcher-Reeves beta, Armijo<F,1>::Search
//   linesearch/armijo.h:52-68                    Armijo<F,1> backtracking
//   solver/progress.h:153-327                    Progress::Update
//
// Both solvers hand the driver loop an x-only state, so the reference evaluates
// the objective again at the new point (solver.h:210-216), and both line
// searches start by evaluating it again at the old one.  Those are evaluations
// of the same function at the same point: the kernel reuses the bits it already
// holds (the accepted trial of the line search IS the new state -- x0 + stp*(-g)
// and x0 - stp*g are the same IEEE operation, x + alpha*d is the same
// expression) and only counts them in `nfev`.  State lives in registers
// (x, g, direction: E = ceil(D/32) elements per lane); shared memory holds only
// the Progress ring.
#ifndef CNO_DESCENT_CUH_
#define CNO_DESCENT_CUH_

#include "cno_device.cuh"
#include "cno_kernel_params.h"
#include "cno_lbfgs.cuh"  // ProgressState / progress_update
#include "cno_linesearch.cuh"

namespace cno {

template <class T>
struct DescentSmem {
  static constexpr int kWarpElems = CNO_MAX_PAST;
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  static constexpr int kWarps = 16;
};

// kConjugate = false: GradientDescent (MoreThuente); true: ConjugatedGradientDescent (Armijo<F,1>)
template <class Fn, bool kConjugate, class LS = LsMoreThuente>
__global__ void __launch_bounds__(DescentSmem<typename Fn::Scalar>::kWarps * 32, 1)
descent_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0, const long long batch,
                        const StopParams<typename Fn::Scalar> stop,
                        const BatchOut<typename Fn::Scalar> out,
                        unsigned long long* __restrict__ queue) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  constexpr int E = Shape<D>::E;
  using SMD = DescentSmem<T>;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T* const ring = reinterpret_cast<T*>(smem_raw) + (size_t)warp * SMD::kWarpElems;

  for (;;) {
    unsigned long long b = 0;
    if (lane == 0) b = atomicAdd(queue, 1ULL);
    b = __shfl_sync(kFullMask, b, 0);
    if (uni(b >= (unsigned long long)batch)) break;
    const EvalCtx ctx{lane, (long long)b, nullptr};

    // solver.h:189-192
    T x[E], g[E];
    load_row<T, D>(x0 + b * D, lane, x);
    T f = fn(ctx, x, &g);
    uint32_t nfev = 1;
    if (kConjugate) nfev++;  // InitializeSolver: function(x0, &previous_gradient_) (:62-65)

    T dir[E];
    T gg_prev = T(0);  // previous_gradient_.dot(previous_gradient_)
#pragma unroll
    for (int e = 0; e < E; ++e) dir[e] = T(0);

    ProgressState<T> prog;
    prog.num_iterations = 0;
    prog.x_delta_violations = 0;
    prog.f_delta_violations = 0;
    prog.x_delta = prog.f_delta = prog.gradient_norm = T(0);
    prog.ring_size = 0;
    prog.ring_pos = 0;
    prog.status = CNO_STATUS_NOT_STARTED;

    do {  // solver.h:196-220
      nfev++;  // function(current.x, &gradient): the state's gradient, bit for bit
      T xn[E], gn[E];
      T fn_val;
      const T gg = warp_sum(lane_dot<T, E>(g, g));
      if constexpr (!kConjugate) {
        // ---- gradient_descent.h:66-72 ----
#pragma unroll
        for (int e = 0; e < E; ++e) dir[e] = -g[e];
        nfev++;  // MoreThuente::Search evaluates (f, g) at x (more_thuente.h:69)
        // dginit = g.(-g) = -(g.g), bit for bit
        if constexpr (!LS::kStateMayDifferFromStep) {
          nfev += LS::template search<Fn, T, E>(fn, ctx, RedCtx<T>{nullptr, lane}, x, f, g, xn, fn_val, gn, T(1), dir, -gg);
        } else {
          // gradient_descent.h:72 builds the next point from the step width alone: after a failed
          // search that is x - 0 * g (NaN where g is not finite) or x - 1 * g, not the start state
          T rate;
          bool ls_ok;
          nfev += LS::template search_with_step<Fn, T, E>(fn, ctx, RedCtx<T>{nullptr, lane}, x, f, g, xn, fn_val, gn, T(1),
                                                          dir, -gg, rate, ls_ok);
          if (uni(!ls_ok)) {
#pragma unroll
            for (int e = 0; e < E; ++e) xn[e] = x[e] - rate * g[e];
            fn_val = fn(ctx, xn, &gn);  // = the driver's re-evaluation, counted below
          }
        }
      } else {
        // ---- conjugated_gradient_descent.h:70-84 ----
        if (uni(prog.num_iterations == 0)) {
#pragma unroll
          for (int e = 0; e < E; ++e) dir[e] = -g[e];
        } else {
          const T beta = gg / gg_prev;
#pragma unroll
          for (int e = 0; e < E; ++e) dir[e] = -g[e] + beta * dir[e];
        }
        gg_prev = gg;
        // ---- Armijo<F,1>::Search (armijo.h:52-68) ----
        nfev++;  // f_in = function(x, &gradient)
        const T cc = T(0.2), rho = T(0.9), alpha_min = T(1e-8);
        T alpha = T(1.0);
#pragma unroll
        for (int e = 0; e < E; ++e) xn[e] = x[e] + alpha * dir[e];
        fn_val = fn(ctx, xn, &gn);
        nfev++;
        const T cache = cc * warp_sum(lane_dot<T, E>(g, dir));
        while (uni((fn_val > f + alpha * cache) && (alpha > alpha_min))) {
          alpha *= rho;
#pragma unroll
          for (int e = 0; e < E; ++e) xn[e] = x[e] + alpha * dir[e];
          fn_val = fn(ctx, xn, &gn);
          nfev++;
        }
      }
      nfev++;  // re-evaluation of the x-only state (solver.h:210-216) = the accepted trial

      // ---- Progress::Update ----
      T sdx[E];
#pragma unroll
      for (int e = 0; e < E; ++e) sdx[e] = xn[e] - x[e];
      const T prev_value = f;
      const T x_delta = warp_maxabs<T, E>(sdx);
#pragma unroll
      for (int e = 0; e < E; ++e) { x[e] = xn[e]; g[e] = gn[e]; }
      f = fn_val;
      const T gnorm_inf = warp_maxabs<T, E>(g);
      const T x_inf = warp_maxabs<T, E>(x);
      progress_update<T>(prog, stop, ring, lane, prev_value, f, x_delta, gnorm_inf, x_inf);
    } while (uni(prog.status == CNO_STATUS_CONTINUE));

    if (out.x) store_row<T, D>(out.x + b * D, lane, x);
    if (out.gradient) store_row<T, D>(out.gradient + b * D, lane, g);
    if (lane == 0) {
      if (out.value) out.value[b] = f;
      if (out.num_iterations) out.num_iterations[b] = prog.num_iterations;
      if (out.status) out.status[b] = (int8_t)prog.status;
      if (out.nfev) out.nfev[b] = nfev;
      if (out.x_delta) out.x_delta[b] = prog.x_delta;
      if (out.f_delta) out.f_delta[b] = prog.f_delta;
      if (out.gradient_norm) out.gradient_norm[b] = prog.gradient_norm;
    }
    __syncwarp();
  }
}

}  // namespace cno

#endif  // CNO_DESCENT_CUH_
