// cno_auglag.cuh -- batched AugmentedLagrangian<Problem, Lbfgs>::Minimize: the
// composite device functor the fused L-BFGS kernel minimises, and the kernels of the
// outer loop (one warp per instance, sm_90a).
//
// Parity: bit-identical on the GPU to the pinned CPU oracle (oracle/cno_oracle_impl.inc:
// eval_auglag, al_minimize_one) and to the reference-headers fixtures tests/golden/al_*.npz
// (tests/test_al_gpu.py).  DESIGN.md 8.
//
// Reference path (include/cppoptlib/...):
//   function_penalty.h:97-250              ToAugmentedLagrangian = ((f + Lag) + Pen) + Ineq (PHR)
//   function_expressions.h:45-400          Const / Add / Sub / Mul (c == 0 short cut) / Prod / MaxZero:
//                                          the node-by-node evaluation order restated below
//   solver/augmented_lagrangian.h:295-434  OptimizationStep
//   solver/augmented_lagrangian.h:436-449  Minimize (best iterate restored)
//   solver/progress.h:162-252              Progress::Update, constrained branch
//
// One outer iteration on the device = [al_autoscale_kernel on the first] ->
// lbfgs_minimize_kernel<AugLagFn<Obj>> (the inner solve, skipping finished instances
// through AugLagFn::active) -> al_outer_step_kernel.  Everything per-instance lives in
// [B, .] arrays in HBM between launches; inside a launch it is registers only.
#ifndef CNO_AUGLAG_CUH_
#define CNO_AUGLAG_CUH_

#include "../../include/cno_al.h"
#include "cno_device.cuh"
#include "cno_kernel_params.h"

namespace cno {

constexpr int kAlMaxCon = 32;  // per kind; the outer-step kernel keeps one multiplier per lane

// The constrained problem + one multiplier/penalty state, as device pointers.
template <class T>
struct AlView {
  const T* rows;         // [B or 1][n_eq + n_ineq][D + 1]  rows [a | t]
  long long row_stride;  // scalars between instances (0 = one set shared by the batch)
  const int* kinds;      // [n_eq + n_ineq] cno_constraint_kind_t
  int n_eq, n_ineq;
  const T* lambda;        // [B, n_eq]   equality multipliers
  const T* mu;            // [B, n_ineq] inequality multipliers
  const T* penalty;       // [B]
  const int8_t* status;   // [B] outer status (finished instances are skipped) or nullptr
};

// One constraint functor: value, and this lane's slice of the gradient in gc.
template <class T, int D>
__device__ __forceinline__ T al_con_eval(const AlView<T>& v, long long instance, int idx, int lane,
                                         const T (&x)[Shape<D>::E], T (&gc)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
  const T* row = v.rows + instance * v.row_stride + (long long)idx * (D + 1);
  const T t = __ldg(row + D);
  if (uni(v.kinds[idx] == CNO_CON_AFFINE)) {
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int i = lane * E + j;
      gc[j] = (i < D) ? __ldg(row + i) : T(0);
    }
    return warp_sum(lane_dot<T, E>(x, gc)) - t;
  }
#pragma unroll
  for (int j = 0; j < E; ++j) gc[j] = T(-2) * x[j];
  return t - warp_sum(lane_dot<T, E>(x, x));
}

// ToAugmentedLagrangian(prob, multipliers, penalty) as a First-mode device functor.
template <class Obj>
struct AugLagFn {
  using Scalar = typename Obj::Scalar;
  static constexpr int Dim = Obj::Dim;
  static constexpr int Mode = 1;
  static constexpr int E = Shape<Dim>::E;
  using T = Scalar;
  Obj obj;
  AlView<T> v;

  // lbfgs_minimize_kernel skips instances whose outer loop has finished
  __device__ __forceinline__ bool active(long long b) const {
    if (v.status == nullptr) return true;
    const int s = v.status[b];
    return (s == CNO_STATUS_CONTINUE) | (s == CNO_STATUS_NOT_STARTED);
  }

  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E]) const {
    return eval_with(c, x, grad, v.lambda + c.instance * v.n_eq, v.mu + c.instance * v.n_ineq,
                     v.penalty[c.instance]);
  }

  // the composite under the given multipliers / penalty (any address space)
  __device__ __forceinline__ T eval_with(const EvalCtx& c, const T (&x)[E], T (*grad)[E], const T* lam,
                                         const T* mu, const T rho) const {
    T gf[E], gc[E], gL[E], gP[E], gI[E];
    const T vf = obj(c, x, &gf);

    // FormLagrangianPart (function_penalty.h:97-109): L <- L + lambda_i * c_i from Const(0)
    T vL = T(0);
#pragma unroll
    for (int k = 0; k < E; ++k) gL[k] = T(0);
#pragma unroll 1
    for (int i = 0; i < v.n_eq; ++i) {
      const T l = lam[i];
      T tv = T(0);
      if (uni(l == T(0))) {  // MulExpression: c == 0 -> (0, zeros)
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = T(0);
      } else {
        const T cv = al_con_eval<T, Dim>(v, c.instance, i, c.lane, x, gc);
        tv = l * cv;
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = l * gc[k];
      }
      vL = vL + tv;
#pragma unroll
      for (int k = 0; k < E; ++k) gL[k] = gL[k] + gc[k];
    }

    // FormPenaltyPart (:116-128): P <- P + rho * (0.5 * (c_i * c_i))
    T vP = T(0);
#pragma unroll
    for (int k = 0; k < E; ++k) gP[k] = T(0);
#pragma unroll 1
    for (int i = 0; i < v.n_eq; ++i) {
      T tv = T(0);
      if (uni(rho == T(0))) {
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = T(0);
      } else {
        const T cv = al_con_eval<T, Dim>(v, c.instance, i, c.lane, x, gc);
        const T pv = cv * cv;  // Prod: (f g, g * grad_f + f * grad_g)
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = cv * gc[k] + cv * gc[k];
        const T hv = T(0.5) * pv;
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = T(0.5) * gc[k];
        tv = rho * hv;
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = rho * gc[k];
      }
      vP = vP + tv;
#pragma unroll
      for (int k = 0; k < E; ++k) gP[k] = gP[k] + gc[k];
    }

    // FormInequalityPart (:156-199), Powell-Hestenes-Rockafellar
    T vI = T(0);
#pragma unroll
    for (int k = 0; k < E; ++k) gI[k] = T(0);
    if (uni(!(rho <= T(0)))) {
      const T half_inv_rho = T(1) / (T(2) * rho);
#pragma unroll 1
      for (int j = 0; j < v.n_ineq; ++j) {
        const T m = mu[j];
        const T gv = al_con_eval<T, Dim>(v, c.instance, v.n_eq + j, c.lane, x, gc);
        T av = m - rho * gv;  // argument = Const(mu) - rho * g
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = T(0) - rho * gc[k];
        if (uni(av <= T(0))) {  // MaxZero
          av = T(0);
#pragma unroll
          for (int k = 0; k < E; ++k) gc[k] = T(0);
        }
        const T qv = av * av;
#pragma unroll
        for (int k = 0; k < E; ++k) gc[k] = av * gc[k] + av * gc[k];
        T tv = T(0);
        if (uni(half_inv_rho == T(0))) {
#pragma unroll
          for (int k = 0; k < E; ++k) gc[k] = T(0);
        } else {
          tv = half_inv_rho * qv;
#pragma unroll
          for (int k = 0; k < E; ++k) gc[k] = half_inv_rho * gc[k];
        }
        vI = vI + tv;
#pragma unroll
        for (int k = 0; k < E; ++k) gI[k] = gI[k] + gc[k];
        const T constant_offset = m * m * half_inv_rho;
        vI = vI - constant_offset;  // Sub(I, Const): the gradient minus zeros
#pragma unroll
        for (int k = 0; k < E; ++k) gI[k] = gI[k] - T(0);
      }
    }
    if (grad) {
#pragma unroll
      for (int k = 0; k < E; ++k) (*grad)[k] = ((gf[k] + gL[k]) + gP[k]) + gI[k];
    }
    return ((vf + vL) + vP) + vI;
  }
};

// cno_al_config_t / cno_al_stop_t narrowed to the scalar type.
template <class T>
struct AlParams {
  T penalty_growth_factor, violation_shrink_ratio;
  int auto_scale_initial_penalty;
  T penalty_auto_objective_scale, penalty_auto_min, penalty_auto_max;
  T multiplier_max;
  unsigned long long num_iterations;
  T constraint_threshold;
  double kkt_stationarity_threshold;  // compared with <= 0 as a double, like the oracle
};

// The solver's per-instance state and results ([B, .] device arrays; cno_al_out_t + scratch).
template <class T>
struct AlArrays {
  T* x;        // [B, D] state x (AugmentedLagrangeState::x)
  T* x_work;   // [B, D] inner solve result
  T* lambda;   // [B, n_eq]
  T* mu;       // [B, n_ineq]
  T* penalty;  // [B]
  T* prev_penalty;  // [B] the penalty the previous outer iterate was built with (before auto-scaling on iteration 1)
  T* max_violation;
  T* max_lagrangian_gradient;
  uint32_t* num_iterations;
  int8_t* status;
  uint32_t* nfev;
  const uint32_t* inner_nfev;  // [B] evaluations of the last inner solve
  T* x_delta;
  T* f_delta;
  T* gradient_norm;
  // best-iterate tracker (augmented_lagrangian.h:529-604)
  int8_t* best_recorded;
  T* best_x;
  T* best_lambda;
  T* best_mu;
  T* best_penalty;
  T* best_objective;
  T* best_violation;
  T* best_kkt;
  int* remaining;  // number of instances still running after this outer step
};

template <class T, int D>
__device__ __forceinline__ void al_load(const T* row, int lane, T (&v)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
#pragma unroll
  for (int j = 0; j < E; ++j) {
    const int i = lane * E + j;
    v[j] = (i < D) ? row[i] : T(0);
  }
}
template <class T, int D>
__device__ __forceinline__ void al_store(T* row, int lane, const T (&v)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
#pragma unroll
  for (int j = 0; j < E; ++j) {
    const int i = lane * E + j;
    if (i < D) row[i] = v[j];
  }
}

constexpr int kAlWarps = 8;

// ComputeAutoScaledPenalty (augmented_lagrangian.h:312-318, 451-476) on outer iteration 1.
template <class Obj>
__global__ void __launch_bounds__(kAlWarps * 32)
al_autoscale_kernel(const Obj obj, const AlView<typename Obj::Scalar> v, const long long batch,
                    const AlParams<typename Obj::Scalar> p, AlArrays<typename Obj::Scalar> a) {
  using T = typename Obj::Scalar;
  constexpr int D = Obj::Dim;
  constexpr int E = Shape<D>::E;
  const int lane = threadIdx.x & 31;
  const long long b = (long long)blockIdx.x * kAlWarps + (threadIdx.x >> 5);
  if (b >= batch) return;
  if (!(p.auto_scale_initial_penalty && a.penalty[b] == T(0))) return;
  const EvalCtx ctx{lane, b, nullptr};
  T x[E], gc[E];
  al_load<T, D>(a.x + b * D, lane, x);
  T om = cabs(obj(ctx, x, nullptr));
  om = smax(om, T(1));
  T srs = T(0);
#pragma unroll 1
  for (int i = 0; i < v.n_eq; ++i) {
    const T c = al_con_eval<T, D>(v, b, i, lane, x, gc);
    srs += T(0.5) * c * c;
  }
#pragma unroll 1
  for (int j = 0; j < v.n_ineq; ++j) {
    const T c = al_con_eval<T, D>(v, b, v.n_eq + j, lane, x, gc);
    if (uni(c < T(0))) srs += T(0.5) * c * c;
  }
  const T denom = smax(srs, T(1));
  const T rho = p.penalty_auto_objective_scale * om / denom;
  if (lane == 0) {
    a.penalty[b] = sclamp(rho, p.penalty_auto_min, p.penalty_auto_max);
    a.nfev[b] += 1;  // function.objective(x)
  }
}

// The rest of OptimizationStep after the inner solve (augmented_lagrangian.h:356-433) and
// Progress::Update's constrained branch (progress.h:162-252).
template <class Obj>
__global__ void __launch_bounds__(kAlWarps * 32)
al_outer_step_kernel(const Obj obj, const AlView<typename Obj::Scalar> v, const long long batch,
                     const AlParams<typename Obj::Scalar> p, AlArrays<typename Obj::Scalar> a) {
  using T = typename Obj::Scalar;
  constexpr int D = Obj::Dim;
  constexpr int E = Shape<D>::E;
  __shared__ T prev_mult[kAlWarps][2 * kAlMaxCon];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const long long b = (long long)blockIdx.x * kAlWarps + warp;
  if (b >= batch) return;
  {
    const int s = a.status[b];
    if (!((s == CNO_STATUS_CONTINUE) | (s == CNO_STATUS_NOT_STARTED))) return;
  }
  const EvalCtx ctx{lane, b, nullptr};
  const AugLagFn<Obj> composite{obj, v};
  T* const lam = a.lambda + b * v.n_eq;
  T* const mu = a.mu + b * v.n_ineq;
  T* const prev_lam = prev_mult[warp];
  T* const prev_mu = prev_mult[warp] + kAlMaxCon;

  T x[E], xp[E], gc[E];
  al_load<T, D>(a.x_work + b * D, lane, x);   // the inner solver's solution (:354)
  al_load<T, D>(a.x + b * D, lane, xp);       // previous outer iterate
  const T penalty = a.penalty[b];             // (auto-scaled on iteration 1)
  const T prev_max_violation = a.max_violation[b];

  // ---- multiplier updates + residuals (:356-387); lane i owns multiplier i ----
  T my_lam = (lane < v.n_eq) ? lam[lane] : T(0);
  T my_mu = (lane < v.n_ineq) ? mu[lane] : T(0);
  prev_lam[lane] = my_lam;
  prev_mu[lane] = my_mu;
  T max_violation = T(0);
#pragma unroll 1
  for (int i = 0; i < v.n_eq; ++i) {
    const T cv = al_con_eval<T, D>(v, b, i, lane, x, gc);
    max_violation = smax(max_violation, cabs(cv));
    if (lane == i) {
      const T cand = my_lam + penalty * cv;
      my_lam = cfinite(cand) ? sclamp(cand, -p.multiplier_max, p.multiplier_max) : T(0);
    }
  }
#pragma unroll 1
  for (int j = 0; j < v.n_ineq; ++j) {
    const T cv = al_con_eval<T, D>(v, b, v.n_eq + j, lane, x, gc);
    const T violation = smax(T(0), -cv);
    max_violation = smax(max_violation, violation);
    if (lane == j) {
      const T cand = smax(T(0), my_mu - penalty * cv);
      my_mu = cfinite(cand) ? sclamp(cand, T(0), p.multiplier_max) : T(0);
    }
  }
  if (lane < v.n_eq) lam[lane] = my_lam;
  if (lane < v.n_ineq) mu[lane] = my_mu;
  __syncwarp();

  // ---- ComputeLagrangianGradientKktNorm (:501-527): raw sup-norm (plain Lbfgs inner solver) ----
  T sum_grad[E];
  const T objective = obj(ctx, x, &sum_grad);
#pragma unroll 1
  for (int i = 0; i < v.n_eq; ++i) {
    al_con_eval<T, D>(v, b, i, lane, x, gc);
    const T l = __shfl_sync(kFullMask, my_lam, i);
#pragma unroll
    for (int k = 0; k < E; ++k) sum_grad[k] = sum_grad[k] + l * gc[k];
  }
#pragma unroll 1
  for (int j = 0; j < v.n_ineq; ++j) {
    al_con_eval<T, D>(v, b, v.n_eq + j, lane, x, gc);
    const T m = __shfl_sync(kFullMask, my_mu, j);
#pragma unroll
    for (int k = 0; k < E; ++k) sum_grad[k] = sum_grad[k] - m * gc[k];
  }
  const T max_lagr = warp_maxabs<T, E>(sum_grad);

  // ---- UpdateBestIterateInPlace (:546-594); its objective(x) = the value just computed ----
  {
    bool finite = cfinite(objective) & cfinite(max_violation);
    bool x_finite = true;
#pragma unroll
    for (int k = 0; k < E; ++k) x_finite = x_finite & cfinite(x[k]);
    finite = finite & (__all_sync(kFullMask, x_finite) != 0);
    bool record = false;
    if (finite) {
      const T tol = T(1e-5);
      if (!a.best_recorded[b]) {
        record = true;
      } else {
        const T bv = a.best_violation[b], bo = a.best_objective[b];
        const bool cand_feasible = max_violation <= tol, best_feasible = bv <= tol;
        if (cand_feasible & !best_feasible) record = true;
        else if (!cand_feasible & best_feasible) record = false;
        else if (cand_feasible & best_feasible) record = objective < bo;
        else record = (max_violation < bv) | ((max_violation == bv) & (objective < bo));
      }
    }
    if (uni(record)) {  // RecordBestIterate (:595-604): penalty before growth, multipliers after the update
      al_store<T, D>(a.best_x + b * D, lane, x);
      if (lane < v.n_eq) a.best_lambda[b * v.n_eq + lane] = my_lam;
      if (lane < v.n_ineq) a.best_mu[b * v.n_ineq + lane] = my_mu;
      if (lane == 0) {
        a.best_recorded[b] = 1;
        a.best_penalty[b] = penalty;
        a.best_objective[b] = objective;
        a.best_violation[b] = max_violation;
        a.best_kkt[b] = max_lagr;
      }
    }
  }

  // ---- penalty growth (:426-433) ----
  const bool shrank = max_violation <= p.violation_shrink_ratio * prev_max_violation;
  const T new_penalty = shrank ? penalty : penalty * p.penalty_growth_factor;

  // ---- Progress::Update, constrained branch (progress.h:162-252) ----
  __syncwarp();
  T cg[E];
  const T pv = composite.eval_with(ctx, xp, nullptr, prev_lam, prev_mu, a.prev_penalty[b]);
  const T cv2 = composite.eval_with(ctx, x, &cg, lam, mu, new_penalty);
  T dx[E];
#pragma unroll
  for (int k = 0; k < E; ++k) dx[k] = x[k] - xp[k];
  const T x_delta = warp_maxabs<T, E>(dx);
  const T gnorm = warp_maxabs<T, E>(cg);
  const unsigned long long it = (unsigned long long)a.num_iterations[b] + 1ULL;
  int status;
  if ((p.num_iterations > 0) && (it > p.num_iterations)) {
    status = CNO_STATUS_ITERATION_LIMIT;
  } else if (!cfinite(max_violation) | !cfinite(max_lagr)) {
    status = CNO_STATUS_ITERATION_LIMIT;
  } else {
    const bool primal_feasible = cabs(max_violation) <= p.constraint_threshold;
    const bool kkt_stationary = (p.kkt_stationarity_threshold <= 0) | (max_lagr <= (T)p.kkt_stationarity_threshold);
    status = (primal_feasible & kkt_stationary) ? CNO_STATUS_FINISHED : CNO_STATUS_CONTINUE;
  }

  // ---- commit ----
  al_store<T, D>(a.x + b * D, lane, x);
  if (lane == 0) {
    a.penalty[b] = new_penalty;
    a.prev_penalty[b] = new_penalty;
    a.max_violation[b] = max_violation;
    a.max_lagrangian_gradient[b] = max_lagr;
    a.num_iterations[b] = (uint32_t)it;
    a.status[b] = (int8_t)status;
    // inner composite evaluations + KKT + best-iterate + the two Progress composites
    a.nfev[b] += a.inner_nfev[b] + 4u;
    if (a.x_delta) a.x_delta[b] = x_delta;
    if (a.f_delta) a.f_delta[b] = cabs(cv2 - pv);
    if (a.gradient_norm) a.gradient_norm[b] = gnorm;
    if (status == CNO_STATUS_CONTINUE) atomicAdd(a.remaining, 1);
  }
}

// AugmentedLagrangian::Minimize epilogue (:436-449): the best iterate replaces the last one.
template <class T, int D>
__global__ void al_finalize_kernel(const long long batch, const int n_eq, const int n_ineq, AlArrays<T> a) {
  const int lane = threadIdx.x & 31;
  const long long b = (long long)blockIdx.x * kAlWarps + (threadIdx.x >> 5);
  if (b >= batch) return;
  if (!a.best_recorded[b]) return;
  T x[Shape<D>::E];
  al_load<T, D>(a.best_x + b * D, lane, x);
  al_store<T, D>(a.x + b * D, lane, x);
  if (lane < n_eq) a.lambda[b * n_eq + lane] = a.best_lambda[b * n_eq + lane];
  if (lane < n_ineq) a.mu[b * n_ineq + lane] = a.best_mu[b * n_ineq + lane];
  if (lane == 0) {
    a.penalty[b] = a.best_penalty[b];
    a.max_violation[b] = a.best_violation[b];
    a.max_lagrangian_gradient[b] = a.best_kkt[b];
  }
}

}  // namespace cno

#endif  // CNO_AUGLAG_CUH_
