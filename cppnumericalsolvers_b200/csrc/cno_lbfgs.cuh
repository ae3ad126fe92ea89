// cno_lbfgs.cuh -- batched Lbfgs<F, m>::Minimize, one warp per instance, the
// whole Solver::Minimize loop fused into ONE persistent kernel (sm_90a).
//
// Reference path (include/cppoptlib/...):
//   solver/solver.h:181-224   Solver::Minimize driver loop
//   solver/lbfgs.h:72-87      InitializeSolver
//   solver/lbfgs.h:89-303     OptimizationStep (two-loop recursion, descent
//                             test / fallback, pair + gamma update)
//   linesearch/more_thuente.h MoreThuente::Search / cvsrch / cstep
//   solver/progress.h:153-327 Progress::Update
//
// Design: grid = #SMs persistent CTAs; each warp pulls instance ids from
// a global atomic queue (instances run 20..10000 iterations, so retire +
// refill is what keeps all warps busy through the tail).  The m-deep (s, y)
// history of the instance a warp is working on stays ON CHIP for the instance's
// whole lifetime, in the warp's private slice of shared memory (at d = 128 fp64
// that is 20 KB per instance: 11 resident warps per SM); x, g, the
// search direction and the trial point live in registers.  HBM is touched twice
// per instance: one coalesced vectorised read of x0 and one write of the result.
// Inner products: in-lane tree, then the cross-lane sum on the FP64 tensor core
// (fp64: 2 DMMA + 1 DADD) or a shuffle butterfly (fp32) -- the arithmetic
// specification in cno_device.cuh; s_i.y_i is cached per slot when the pair is
// stored (the reference recomputes the same dot twice per pair per iteration,
// lbfgs.h:163-164,187-188 -- same operands, same order, same bits).
#ifndef CNO_LBFGS_CUH_
#define CNO_LBFGS_CUH_

#include "cno_device.cuh"
#include "cno_linesearch.cuh"
#include "cno_kernel_params.h"

namespace cno {

template <class T, int D, int M, int kStage = 0, int kScratchPerLane = 0, int kMaxW = 16, int kHelpers = 0>
struct LbfgsSmem {
  static constexpr int E = Shape<D>::E;
  static constexpr int kVec = 32 * E;                        // elements per stored vector
  static constexpr int kScalars = 2 * M + CNO_MAX_PAST + 32 * kScratchPerLane;  // rho[M], alpha[M], f ring, policy scratch
  static constexpr int kHistElems = 2 * M * kVec + ((kScalars + 3) / 4) * 4;  // S, Y + scalars
  static constexpr int kWarpElems = kHistElems + kStage;     // + the functor's staged block
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  // warps per CTA: as many as fit in 227 KB, at most 16 (register budget).
  static constexpr int kMaxSmem = 227 * 1024;
  static constexpr int kWarpsFit = (int)(kMaxSmem / kWarpBytes);
  static constexpr int kMaxWarps = kMaxW;  // register budget: 65536 / (32 * warps) per thread (FnPreferredWarps)
  static constexpr int kWarps = kWarpsFit > kMaxWarps ? kMaxWarps : (kWarpsFit < 1 ? 1 : kWarpsFit);
  // Functors with a helper warp per instance (FnHelperWarps): solver warps 0 .. kWarps-1, the helper of solver warp t is
  // warp kHelperBase + t.
  static constexpr int kHelperBase = kWarps;
  static constexpr int kThreads = 32 * (kHelpers > 0 ? 2 * kWarps : kWarps);
};

// y-history accessor: the warp's shared-memory slice (chunk-interleaved).  A load is issued before the reduction it
// overlaps and consumed after it (issue / wait).
template <class T, int E>
struct YHist {
  T* base;
  int lane;
  struct Pending {};
  __device__ __forceinline__ void store(int slot, const T (&v)[E]) const { SmemVec<T, E>::store(base + slot * 32 * E, lane, v); }
  __device__ __forceinline__ void issue(int slot, T (&v)[E], Pending&) const { SmemVec<T, E>::load(base + slot * 32 * E, lane, v); }
  __device__ __forceinline__ void wait(T (&)[E], Pending&) const {}
  __device__ __forceinline__ void fence_store() const {}
};

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

template <class T>
__device__ __forceinline__ void progress_update(ProgressState<T>& p, const StopParams<T>& stop,
                                                T* __restrict__ ring, const int lane,
                                                T prev_value, T cur_value, T x_delta,
                                                T gradient_norm, T x_inf) {
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
  if (status == CNO_STATUS_CONTINUE && stop.gradient_norm > 0) {  // :299-317
    const T scale = stop.gradient_norm_relative ? smax(T(1), x_inf) : T(1);
    if (p.gradient_norm < stop.gradient_norm * scale) status = CNO_STATUS_GRADIENT_NORM_VIOLATION;
  }
  p.status = status;
}

// Record of one parked instance (stepwise solves): S slots, Y slots (lane-major),
// then scalars.  What Lbfgs keeps as members between OptimizationStep calls
// (lbfgs.h:305-323) plus the Progress counters (progress.h:87-140).
template <class T, int E, int M>
struct ResumeLayout {
  static constexpr int kVec = 32 * E;
  static constexpr size_t kS = 0;
  static constexpr size_t kY = kS + (size_t)M * kVec * sizeof(T);
  static constexpr size_t kScal = kY + (size_t)M * kVec * sizeof(T);  // rho[M], ring[MAX_PAST], gamma, xx
  static constexpr int kNumScal = M + CNO_MAX_PAST + 2;
  static constexpr size_t kInts = kScal + (size_t)kNumScal * sizeof(T);
  static constexpr int kNumInts = 9;
  static constexpr size_t kBytes = ((kInts + kNumInts * sizeof(int) + 15) / 16) * 16;
};

// The shared-memory / warp plan of lbfgs_minimize_kernel<Fn, M, kResume, LS>.  The functor's preferred warp
// count applies to the plain kernel only (MoreThuente, First mode, fused): the other variants carry more live
// state per thread and keep the 128-register budget.
template <class Fn, int M, bool kResume = false, class LS = LsMoreThuente>
struct LbfgsPlan {
  static constexpr bool kPlain = std::is_same<LS, LsMoreThuente>::value && !IsSecondMode<Fn>::value && !kResume;
  using SM = LbfgsSmem<typename Fn::Scalar, Fn::Dim, M, StageElems<Fn>::value,
                       PolicyScratch<typename PolicyOf<Fn>::type>::kElemsPerLane,
                       kPlain ? FnPreferredWarps<Fn>::value : 16, FnHelperWarps<Fn>::value>;
};

template <class Fn, int M, bool kResume = false, class LS = LsMoreThuente>
__global__ void __launch_bounds__(LbfgsPlan<Fn, M, kResume, LS>::SM::kThreads, 1)
lbfgs_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0,
                      const long long batch, const StopParams<typename Fn::Scalar> stop,
                      const BatchOut<typename Fn::Scalar> out,
                      unsigned long long* __restrict__ queue, const ResumeArgs ra = ResumeArgs{}) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  constexpr int E = Shape<D>::E;
  constexpr int kStage = StageElems<Fn>::value;
  using P = typename PolicyOf<Fn>::type;
  constexpr bool kSecond = IsSecondMode<Fn>::value;  // lbfgs.h:116-118 has_diagonal_preconditioner
  using SM = typename LbfgsPlan<Fn, M, kResume, LS>::SM;
  using SV = SmemVec<T, E>;
  constexpr T eps = Num<T>::eps;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  constexpr int kHelpers = FnHelperWarps<Fn>::value;
  // the instance slot this warp works for: its own, or (helper warps) the one of its solver warp
  const int slot = (kHelpers > 0 && warp >= SM::kHelperBase) ? warp - SM::kHelperBase : warp;
  T* const S = reinterpret_cast<T*>(smem_raw) + (size_t)slot * SM::kWarpElems;
  T* const rho_s = S + 2 * M * SM::kVec;  // 1 / (s_i . y_i) per slot
  const YHist<T, E> Y{S + M * SM::kVec, lane};
  typename YHist<T, E>::Pending ypend;
  T* const alpha = rho_s + M;
  T* const ring = alpha + M;
  // policy scratch (PolicyEigenSSE2): 16-byte aligned tail of the scalar block; handed to
  // functors through EvalCtx::stage when they stage nothing themselves
  T* const red_scratch = (PolicyScratch<P>::kElemsPerLane > 0) ? (ring + CNO_MAX_PAST) : nullptr;
  const RedCtx<T> rc{red_scratch, lane};
  void* const stage_ptr = (kStage > 0) ? static_cast<void*>(S + SM::kHistElems) : static_cast<void*>(red_scratch);
  uint32_t stage_parity = 0;
  bool solver_warp = true;
  if constexpr (kHelpers > 0) {
    solver_warp = uni(warp < SM::kWarps);
    if (uni(warp >= SM::kHelperBase)) fn.helper(EvalCtx{lane, 0, stage_ptr, slot});  // until its solver warp releases it
  }
  if constexpr (kStage > 0) {
    if (solver_warp) fn.init_stage(EvalCtx{lane, 0, stage_ptr, slot});
  }

  for (; solver_warp;) {
    // ---- retire + refill: next instance from the global queue ----
    unsigned long long b = 0;
    if (lane == 0) b = atomicAdd(queue, 1ULL);
    b = __shfl_sync(kFullMask, b, 0);
    if (uni(b >= (unsigned long long)batch)) break;
    if constexpr (FnSkipsInstances<Fn>::value) {  // e.g. AugLagFn: the instance's outer loop has finished
      if (uni(!fn.active((long long)b))) continue;
    }
    const EvalCtx ctx{lane, (long long)b, stage_ptr, slot};
    if constexpr (kStage > 0) fn.stage(ctx, stage_parity);  // per-instance data -> shared memory (TMA)

    T x[E], g[E];
    T f;
    uint32_t nfev;
    int mem_count, mem_pos;
    unsigned valid;  // bit idx set <=> !(|s_idx . y_idx| < eps)  (lbfgs.h:165,189)
    T gamma;
    T xx;            // ||x||^2 carried across iterations (the dot the reference recomputes at lbfgs.h:95)
    ProgressState<T> prog;
    prog.x_delta = prog.f_delta = prog.gradient_norm = T(0);
    bool resumed = false;
    using RL = ResumeLayout<T, E, M>;
    if constexpr (kResume) {
      if (uni(!ra.first)) {
        if (uni(out.status[b] != CNO_STATUS_CONTINUE)) continue;  // finished in an earlier call
        // ---- un-park: state saved by the previous call + its outputs (x, g, f) ----
        unsigned char* rec = ra.state + (size_t)b * ra.stride;
        load_row<T, D, false>(out.x + b * D, lane, x);
        load_row<T, D, false>(out.gradient + b * D, lane, g);
        f = out.value[b];
        const T* sc = reinterpret_cast<const T*>(rec + RL::kScal);
        const int* in = reinterpret_cast<const int*>(rec + RL::kInts);
        __syncwarp();
        if (lane < M) rho_s[lane] = sc[lane];
        if (lane < CNO_MAX_PAST) ring[lane] = sc[M + lane];
        gamma = sc[M + CNO_MAX_PAST];
        xx = sc[M + CNO_MAX_PAST + 1];
        mem_count = in[0];
        mem_pos = in[1];
        valid = (unsigned)in[2];
        prog.num_iterations = (uint32_t)in[3];
        prog.x_delta_violations = in[4];
        prog.f_delta_violations = in[5];
        prog.ring_size = in[6];
        prog.ring_pos = in[7];
        nfev = (uint32_t)in[8];
        prog.status = CNO_STATUS_CONTINUE;
#pragma unroll 1
        for (int slot = 0; slot < M; ++slot) {
          T v[E];
          load_row<T, 32 * E, false>(reinterpret_cast<const T*>(rec + RL::kS) + slot * 32 * E, lane, v);
          SV::store(S + slot * SM::kVec, lane, v);
          load_row<T, 32 * E, false>(reinterpret_cast<const T*>(rec + RL::kY) + slot * 32 * E, lane, v);
          Y.store(slot, v);
        }
        Y.fence_store();
        __syncwarp();
        resumed = true;
      }
    }
    if (!kResume || uni(!resumed)) {
      // ---- solver.h:189-192: evaluate once at the start point ----
      load_row<T, D>(x0 + b * D, lane, x);
      f = fn(ctx, x, &g);
      nfev = 1;
      // ---- lbfgs.h:72-87 InitializeSolver ----
      mem_count = 0;
      mem_pos = 0;
      valid = 0;
      gamma = T(1);
      prog.num_iterations = 0;
      prog.x_delta_violations = 0;
      prog.f_delta_violations = 0;
      prog.ring_size = 0;
      prog.ring_pos = 0;
      prog.status = CNO_STATUS_NOT_STARTED;
      xx = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(x, x), rc);
    }
    int local_it = 0;

    do {  // solver.h:196-220
      // ================= Lbfgs::OptimizationStep (lbfgs.h:89-303) =========
      // relative_eps = eps * max(1, ||x||) (:93-95) enters ONE comparison, the descent test below; it is formed there,
      // and only when a square-root-free bound does not already decide the comparison.

      // Second mode (:129-135): M^-1 = 1 / (|diag H| + eps); the gradient the reference
      // re-evaluates there is the state's gradient (same function, same x, same bits).
      T precond[E];
      if constexpr (kSecond) {
        fn.hess_diag(ctx, x, precond);
        nfev++;  // function(current.x, &gradient, &hessian)
#pragma unroll
        for (int j = 0; j < E; ++j) precond[j] = T(1) / (cabs(precond[j]) + eps);
      }
      T q[E];  // search_direction
#pragma unroll
      for (int j = 0; j < E; ++j) q[j] = g[j];  // :145
      const int k = mem_count;

      // ================= two-loop recursion (:157-196) =====================
      // chronological i -> slot (mem_pos + i) mod M; mem_pos stays 0 until the
      // buffer is full, so this is the reference's index map (:162).  In both
      // loops the loads of the next pair are issued before the current reduction
      // (the reduction is the critical path; LDS latency hides under it).
      if (uni(k == M && valid == ((1u << M) - 1u))) {
        // ---- steady state (full history, every pair usable): both loops fully
        //      unrolled, alpha_i in registers, no per-pair control flow ----
        int idx = mem_pos + M - 1;
        idx = (idx >= M) ? idx - M : idx;
        T sv[E], yv[E];
        SV::load(S + idx * SM::kVec, lane, sv);
#pragma unroll
        for (int i = M - 1; i >= 0; --i) {  // first loop (:157-171): newest pair first
          const int idx_next = (idx == 0) ? M - 1 : idx - 1;
          const auto part = lane_dot_p<P, T, E>(sv, q);
          const T r = rho_s[idx];
          Y.issue(idx, yv, ypend);
          if (i > 0) SV::load(S + idx_next * SM::kVec, lane, sv);
          const T a = r * warp_sum_p<P, T, E>(part, rc);
          if (lane == 0) alpha[i] = a;
          Y.wait(yv, ypend);
#pragma unroll
          for (int j = 0; j < E; ++j) q[j] = q[j] - a * yv[j];
          idx = idx_next;
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < E; ++j) q[j] = kSecond ? (precond[j] * q[j]) : (q[j] * gamma);  // H0 (:177-182)
        idx = mem_pos;
        // (yv still holds y of the oldest pair: the last pair of loop 1 is the first of loop 2)
#pragma unroll
        for (int i = 0; i < M; ++i) {  // second loop (:185-196): oldest pair first
          const int idx_next = (idx + 1 == M) ? 0 : idx + 1;
          const auto part = lane_dot_p<P, T, E>(yv, q);
          const T r = rho_s[idx];
          const T al = alpha[i];
          SV::load(S + idx * SM::kVec, lane, sv);
          if (i + 1 < M) Y.issue(idx_next, yv, ypend);
          const T beta = r * warp_sum_p<P, T, E>(part, rc);
          const T coef = al - beta;
#pragma unroll
          for (int j = 0; j < E; ++j) q[j] = q[j] + sv[j] * coef;
          if (i + 1 < M) Y.wait(yv, ypend);
          idx = idx_next;
        }
      } else {
        // ---- warm-up (k < M) or a skipped pair: generic rolled loops ----
        // ---- first loop (:157-171): newest pair first ----
        // chronological i -> slot (mem_pos + i) mod M; mem_pos stays 0 until the
        // buffer is full, so this is the reference's index map (:162).  The loads
        // of the next pair are issued before the current reduction (software
        // pipelining: the butterfly is the critical path, LDS latency hides under it).
        if (uni(k > 0)) {
          int idx = mem_pos + k - 1;
          idx = (idx >= M) ? idx - M : idx;
          T sv[E];
          SV::load(S + idx * SM::kVec, lane, sv);
  #pragma unroll 1
          for (int i = k - 1; uni(i >= 0); --i) {
            const int idx_next = (idx == 0) ? M - 1 : idx - 1;
            const auto part = lane_dot_p<P, T, E>(sv, q);
            T yv[E];
            Y.issue(idx, yv, ypend);
            SV::load(S + idx_next * SM::kVec, lane, sv);  // prefetch (harmless at i == 0)
            const T a = rho_s[idx] * warp_sum_p<P, T, E>(part, rc);
            Y.wait(yv, ypend);
            if (uni((valid >> idx) & 1u)) {  // lbfgs.h:165 skip
              if (lane == 0) alpha[i] = a;
  #pragma unroll
              for (int j = 0; j < E; ++j) q[j] = q[j] - a * yv[j];
            }
            idx = idx_next;
          }
        }
        __syncwarp();
        // ---- H0 scaling (:177-182) ----
  #pragma unroll
        for (int j = 0; j < E; ++j) q[j] = kSecond ? (precond[j] * q[j]) : (q[j] * gamma);
        // ---- second loop (:185-196): oldest pair first ----
        if (uni(k > 0)) {
          int idx = mem_pos;
          T yv[E];
          Y.issue(idx, yv, ypend);
          Y.wait(yv, ypend);
  #pragma unroll 1
          for (int i = 0; uni(i < k); ++i) {
            const int idx_next = (idx + 1 == M) ? 0 : idx + 1;
            const auto part = lane_dot_p<P, T, E>(yv, q);
            T sv[E];
            SV::load(S + idx * SM::kVec, lane, sv);
            Y.issue(idx_next, yv, ypend);  // prefetch (harmless past the end: a valid slot)
            const T beta = rho_s[idx] * warp_sum_p<P, T, E>(part, rc);
            Y.wait(yv, ypend);
            if (uni((valid >> idx) & 1u)) {  // lbfgs.h:189 skip
              const T coef = alpha[i] - beta;
  #pragma unroll
              for (int j = 0; j < E; ++j) q[j] = q[j] + sv[j] * coef;
            }
            idx = idx_next;
          }
        }
      }

      // ---- descent test, alpha_init, fallback (:199-224) ----
      T alpha_init = T(1);
      T gq;
      if (uni(mem_count == 0)) {  // :208-213 (||q|| only matters without history)
        T qq;
        warp_sum2_p<P, T, E>(lane_dot_p<P, T, E>(g, q), lane_dot_p<P, T, E>(q, q), rc, gq, qq);
        const T qn = csqrt(qq);
        alpha_init = (qn > eps) ? T(1) / qn : T(1);
      } else {
        gq = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(g, q), rc);
      }
      const T descent_direction = -gq;
      T dginit = descent_direction;  // = g.(-q), bit for bit
      // The search runs along -q (the line search negates inside its products, cno_linesearch.cuh
      // kNeg), so no negated copy of q is ever made.
      // descent_direction > -eps * relative_eps?  |eps * relative_eps| <= eps^2 max(1, ||x||) (1 + 2^-50) and
      // sqrt(t) <= max(1, t), so a finite direction below -2 eps^2 max(1, x.x) is below the exact threshold whatever
      // its rounding: the comparison is false and neither the square root nor the products are needed.  Anything else
      // (a non-finite operand, a direction that close to zero) takes the specification's expression.
      bool fallback;
      if (cfinite(descent_direction) && cfinite(xx) && descent_direction < -(T(2) * eps * eps) * smax(T(1), xx)) {
        fallback = false;
      } else {
        const T relative_eps = eps * smax(T(1.0), csqrt(xx));  // :93-95
        fallback = !cfinite(descent_direction) || descent_direction > -eps * relative_eps;
      }
      if (uni(fallback)) {
        // fallback: search_direction = -g, and the reference then searches
        // along -search_direction = +g (SURVEY.md 7.2a): dginit = g.g >= 0.
#pragma unroll
        for (int j = 0; j < E; ++j) q[j] = -g[j];
        mem_count = 0;
        mem_pos = 0;
        valid = 0;
        const T gg = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(g, g), rc);  // :221 (rare path)
        const T gn = csqrt(gg);
        alpha_init = (gn > eps) ? T(1) / gn : T(1);
        dginit = gg;
      }

      // ---- MoreThuente::Search (:231-232) ----
      T xn[E], gn[E];
      T fn_val;
      if (uni(dginit >= T(0))) {  // the search's own early return (more_thuente.h:152-156): state untouched
#pragma unroll
        for (int j = 0; j < E; ++j) { xn[j] = x[j]; gn[j] = g[j]; }
        fn_val = f;
      } else {
        nfev += LS::template search<Fn, T, E, true, std::is_same<LS, LsMoreThuente>::value>(
            fn, ctx, rc, x, f, g, xn, fn_val, gn, alpha_init, q, dginit);
      }

      const T prev_value = f;
      T x_delta, gnorm_inf, x_inf;
      if (uni(!cfinite(fn_val))) {
        // :239-241 return current: x, g, f unchanged; x_delta = |x - x|_inf (progress.h:190) is 0,
        // or NaN when x itself holds a non-finite component (rare path, computed as written).
        gnorm_inf = warp_maxabs<T, E>(g);
        x_inf = warp_maxabs<T, E>(x);
        T zd[E];
#pragma unroll
        for (int j = 0; j < E; ++j) zd[j] = x[j] - x[j];
        x_delta = warp_maxabs<T, E>(zd);
      } else {
        // ---- pair + gamma update (:248-298) ----
        T sd[E], yd[E];
#pragma unroll
        for (int j = 0; j < E; ++j) { sd[j] = xn[j] - x[j]; yd[j] = gn[j] - g[j]; }
        // s.y, s.s, y.y (:265-266) and the next step's ||x||^2 (:95), reduced together
        T sy, ss, yy, xx_next;
        warp_sum4_p<P, T, E>(lane_dot_p<P, T, E>(sd, yd), lane_dot_p<P, T, E>(sd, sd),
                             lane_dot_p<P, T, E>(yd, yd), lane_dot_p<P, T, E>(xn, xn), rc, sy, ss, yy, xx_next);
        // s.y > eps ||s|| ||y|| (:266), decided without the two square roots whenever a rigorous bound allows
        const bool curvature_ok = curvature_above_eps<T>(sy, ss, yy);
        if (uni(curvature_ok)) {
          int slot;
          if (mem_count < M) {
            slot = mem_count;
            mem_count++;
          } else {
            slot = mem_pos;
            mem_pos = (mem_pos + 1 == M) ? 0 : mem_pos + 1;
          }
          SV::store(S + slot * SM::kVec, lane, sd);
          Y.store(slot, yd);
          Y.fence_store();
          // s.y is exactly the dot the reference recomputes per use; cache 1/(s.y)
          __syncwarp();  // all lanes are done reading rho_s in this iteration's loops
          if (lane == 0) rho_s[slot] = T(1) / sy;
          valid = (cabs(sy) < eps) ? (valid & ~(1u << slot)) : (valid | (1u << slot));
        }
        if (yy > eps) {
          const T temp_scaling = sy / yy;
          if (cfinite(temp_scaling) && cabs(temp_scaling) <= T(1e7)) gamma = smax(temp_scaling, eps);
        }
        // next state + the norms Progress::Update and the next step need
        x_delta = warp_maxabs<T, E>(sd);
#pragma unroll
        for (int j = 0; j < E; ++j) { x[j] = xn[j]; g[j] = gn[j]; }
        f = fn_val;
        gnorm_inf = warp_maxabs<T, E>(g);
        x_inf = warp_maxabs<T, E>(x);
        xx = xx_next;
        __syncwarp();
      }

      // ================= Progress::Update (progress.h:153-327) ============
      if constexpr (kSecond) nfev++;  // its Hessian evaluation (progress.h:206-207; value unused, DESIGN.md)
      progress_update<T>(prog, stop, ring, lane, prev_value, f, x_delta, gnorm_inf, x_inf);
      local_it++;
    } while (uni(prog.status == CNO_STATUS_CONTINUE && (!kResume || local_it < ra.max_iterations)));

    if constexpr (kResume) {
      if (uni(prog.status == CNO_STATUS_CONTINUE)) {
        // ---- park: the members Lbfgs keeps between OptimizationStep calls ----
        unsigned char* rec = ra.state + (size_t)b * ra.stride;
        T* sc = reinterpret_cast<T*>(rec + RL::kScal);
        int* in = reinterpret_cast<int*>(rec + RL::kInts);
        __syncwarp();
        if (lane < M) sc[lane] = rho_s[lane];
        if (lane < CNO_MAX_PAST) sc[M + lane] = ring[lane];
        if (lane == 0) {
          sc[M + CNO_MAX_PAST] = gamma;
          sc[M + CNO_MAX_PAST + 1] = xx;
          in[0] = mem_count;
          in[1] = mem_pos;
          in[2] = (int)valid;
          in[3] = (int)prog.num_iterations;
          in[4] = prog.x_delta_violations;
          in[5] = prog.f_delta_violations;
          in[6] = prog.ring_size;
          in[7] = prog.ring_pos;
          in[8] = (int)nfev;
        }
#pragma unroll 1
        for (int slot = 0; slot < M; ++slot) {
          T v[E];
          SV::load(S + slot * SM::kVec, lane, v);
          store_row<T, 32 * E>(reinterpret_cast<T*>(rec + RL::kS) + slot * 32 * E, lane, v);
          Y.issue(slot, v, ypend);
          Y.wait(v, ypend);
          store_row<T, 32 * E>(reinterpret_cast<T*>(rec + RL::kY) + slot * 32 * E, lane, v);
        }
      }
    }

    // ---- write the returned FunctionState + Progress ----
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
  if constexpr (kHelpers > 0) {
    if (solver_warp) fn.release_helper(EvalCtx{lane, 0, stage_ptr, slot});
  }
}

}  // namespace cno

#endif  // CNO_LBFGS_CUH_
