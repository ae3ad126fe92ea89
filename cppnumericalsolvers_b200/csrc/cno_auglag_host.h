// cno_auglag_host.h -- the host side of AugmentedLagrangian::Minimize (solver/augmented_lagrangian.h:
// 295-449), independent of how memory is moved and kernels are launched: the outer loop, the scratch
// layout, the parameter narrowing.  csrc/cno_auglag_launch.cuh drives it with the CUDA backend (for cno_al_minimize and
// cno_<tag>_al_minimize); tests/emu drives the SAME code with the CPU warp emulation (the `-m "not gpu"` check of this
// logic; DESIGN.md 8).
//
// Backend concept (all return 0 or a cno_error_t):
//   int copy_or_zero(void* dst, const void* src, size_t bytes)   device copy, or zero fill when src == nullptr
//   int fill(void* dst, int byte, size_t bytes)
//   int autoscale()                                              al_autoscale_kernel
//   int inner(const cno_stop_t& stop)                            lbfgs_minimize_kernel<AugLagFn<Obj, Cons>>: x -> x_work, inner_nfev
//   int outer_step(int* remaining)                               al_outer_step_kernel; instances still running
//   int finalize()                                               al_finalize_kernel
#ifndef CNO_AUGLAG_HOST_H_
#define CNO_AUGLAG_HOST_H_

#include <stddef.h>
#include <stdint.h>

#include "../../include/cno_al.h"
#include "cno_auglag.cuh"

namespace cno {

inline size_t al_up(size_t v) { return (v + 255) & ~(size_t)255; }

// Scratch layout behind the workspace of cno_al_minimize (every region 256-byte aligned).
struct AlLayout {
  size_t queue, remaining, x_work, prev_penalty, inner_nfev, best_recorded, best_x, best_lambda, best_mu,
      best_penalty, best_objective, best_violation, best_kkt, total;
  AlLayout(size_t B, size_t d, size_t ne, size_t ni, size_t ts) {
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += al_up(bytes ? bytes : 1); return o; };
    queue = take(256);
    remaining = take(sizeof(int));
    x_work = take(B * d * ts);
    prev_penalty = take(B * ts);
    inner_nfev = take(B * 4);
    best_recorded = take(B);
    best_x = take(B * d * ts);
    best_lambda = take(B * ne * ts);
    best_mu = take(B * ni * ts);
    best_penalty = take(B * ts);
    best_objective = take(B * ts);
    best_violation = take(B * ts);
    best_kkt = take(B * ts);
    total = off;
  }
};

// The solver's arrays: results / state from cno_al_out_t, the rest carved out of the workspace.
template <class T>
inline AlArrays<T> al_make_arrays(const cno_al_out_t& o, unsigned char* ws, const AlLayout& L) {
  AlArrays<T> a{};
  a.x = static_cast<T*>(o.x);
  a.x_work = reinterpret_cast<T*>(ws + L.x_work);
  a.lambda = static_cast<T*>(o.equality_multipliers);
  a.mu = static_cast<T*>(o.inequality_multipliers);
  a.penalty = static_cast<T*>(o.penalty);
  a.prev_penalty = reinterpret_cast<T*>(ws + L.prev_penalty);
  a.max_violation = static_cast<T*>(o.max_violation);
  a.max_lagrangian_gradient = static_cast<T*>(o.max_lagrangian_gradient);
  a.num_iterations = o.num_iterations;
  a.status = o.status;
  a.nfev = o.nfev;
  a.inner_nfev = reinterpret_cast<uint32_t*>(ws + L.inner_nfev);
  a.x_delta = static_cast<T*>(o.x_delta);
  a.f_delta = static_cast<T*>(o.f_delta);
  a.gradient_norm = static_cast<T*>(o.gradient_norm);
  a.best_recorded = reinterpret_cast<int8_t*>(ws + L.best_recorded);
  a.best_x = reinterpret_cast<T*>(ws + L.best_x);
  a.best_lambda = reinterpret_cast<T*>(ws + L.best_lambda);
  a.best_mu = reinterpret_cast<T*>(ws + L.best_mu);
  a.best_penalty = reinterpret_cast<T*>(ws + L.best_penalty);
  a.best_objective = reinterpret_cast<T*>(ws + L.best_objective);
  a.best_violation = reinterpret_cast<T*>(ws + L.best_violation);
  a.best_kkt = reinterpret_cast<T*>(ws + L.best_kkt);
  a.remaining = reinterpret_cast<int*>(ws + L.remaining);
  return a;
}

template <class T>
inline AlView<T> al_make_view(const cno_constraints_t& k, const AlArrays<T>& a) {
  AlView<T> v{};
  v.rows = static_cast<const T*>(k.data);
  v.row_stride = (long long)k.data_stride;
  v.kinds = reinterpret_cast<const int*>(k.kinds);
  v.n_eq = k.n_eq;
  v.n_ineq = k.n_ineq;
  v.lambda = a.lambda;
  v.mu = a.mu;
  v.penalty = a.penalty;
  v.status = a.status;
  return v;
}

template <class T>
inline AlParams<T> al_make_params(const cno_al_config_t& c, const cno_al_stop_t& s) {
  AlParams<T> p{};
  p.penalty_growth_factor = (T)c.penalty_growth_factor;
  p.violation_shrink_ratio = (T)c.violation_shrink_ratio;
  p.auto_scale_initial_penalty = c.auto_scale_initial_penalty;
  p.penalty_auto_objective_scale = (T)c.penalty_auto_objective_scale;
  p.penalty_auto_min = (T)c.penalty_auto_min;
  p.penalty_auto_max = (T)c.penalty_auto_max;
  p.multiplier_max = (T)c.multiplier_max;
  p.num_iterations = s.num_iterations;
  p.constraint_threshold = (T)s.constraint_threshold;
  p.kkt_stationarity_threshold = s.kkt_stationarity_threshold;
  return p;
}

// AugmentedLagrangian::Minimize: initial state, the outer loop, the best-iterate epilogue.
template <class T, class Backend>
int al_outer_loop(Backend& be, const AlArrays<T>& a, long long B, int D, int ne, int ni, const void* x0,
                  const void* eq0, const void* ineq0, const void* penalty0, const cno_stop_t& inner_stop,
                  const cno_al_config_t& config, int* launches) {
  int rc;
#define CNO_AL_TRY(expr) do { rc = (expr); if (rc) return rc; } while (0)
  // ---- initial AugmentedLagrangeState (:241-276) + ResetBestIterateTracker (:536-543) ----
  CNO_AL_TRY(be.copy_or_zero(a.x, x0, (size_t)B * D * sizeof(T)));
  CNO_AL_TRY(be.copy_or_zero(a.lambda, eq0, (size_t)B * ne * sizeof(T)));
  CNO_AL_TRY(be.copy_or_zero(a.mu, ineq0, (size_t)B * ni * sizeof(T)));
  CNO_AL_TRY(be.copy_or_zero(a.penalty, penalty0, (size_t)B * sizeof(T)));
  CNO_AL_TRY(be.copy_or_zero(a.prev_penalty, a.penalty, (size_t)B * sizeof(T)));
  CNO_AL_TRY(be.fill(a.max_violation, 0, (size_t)B * sizeof(T)));
  CNO_AL_TRY(be.fill(a.max_lagrangian_gradient, 0, (size_t)B * sizeof(T)));
  CNO_AL_TRY(be.fill(a.num_iterations, 0, (size_t)B * 4));
  CNO_AL_TRY(be.fill(a.nfev, 0, (size_t)B * 4));
  CNO_AL_TRY(be.fill(a.status, 0xFF, (size_t)B));  // CNO_STATUS_NOT_STARTED
  CNO_AL_TRY(be.fill(a.best_recorded, 0, (size_t)B));
  int n = 0;
  for (unsigned long long outer = 1;; ++outer) {
    if (outer == 1 && config.auto_scale_initial_penalty) {  // :312-318
      CNO_AL_TRY(be.autoscale());
      ++n;
    }
    cno_stop_t inner = inner_stop;  // working copy of the template (:347), ConfigureInnerSubproblem (:477-490)
    inner.f_delta = 0;
    if (outer == 1 && (ne > 0 || ni > 0) && config.warmup_max_inner_iterations > 0) {
      inner.num_iterations = (uint64_t)config.warmup_max_inner_iterations;
      inner.gradient_norm = (double)(T)config.warmup_inner_gradient_tolerance;
    }
    CNO_AL_TRY(be.inner(inner));
    ++n;
    int remaining = 0;
    CNO_AL_TRY(be.outer_step(&remaining));
    ++n;
    if (remaining == 0) break;
  }
  CNO_AL_TRY(be.finalize());  // Minimize (:436-449)
  ++n;
#undef CNO_AL_TRY
  if (launches) *launches = n;
  return 0;
}

}  // namespace cno

#endif  // CNO_AUGLAG_HOST_H_
