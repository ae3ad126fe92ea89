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
// whole lifetime, its newest pairs in registers and the rest in the warp's private slice of shared memory
// (LbfgsPlan; at d = 128 fp64, m = 10: one pair in registers, 18 KB per instance, 12 resident warps per SM); x, g, the
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
#include "cno_progress.cuh"

// Compile-time cap on the warps per CTA of every L-BFGS plan (default: none).  tools/lbfgs_warp_sweep.py builds
// copies of the library with -DCNO_LBFGS_MAX_WARPS=w to measure throughput against resident warps.
#ifndef CNO_LBFGS_MAX_WARPS
#define CNO_LBFGS_MAX_WARPS 32
#endif

namespace cno {

// Phase clock probe of lbfgs_minimize_kernel.  tools/lbfgs_phase_clocks.py builds a copy of the library with
// -DCNO_LBFGS_PHASE_CLOCKS; without it every member below is empty and the kernel compiles to the same code.  Lane 0
// of each warp reads clock64() at the phase boundaries of each steady-state iteration (full history, every pair
// usable, a line search run), adds the phase's cycles to per-warp counters and, when the warp exits, adds those into
// cno_lbfgs_phase_clocks: the cycles of each phase, then the iterations counted, the evaluations past each search's
// first trial, and the loop-backs counted (the loop-back phase runs from the end of one counted iteration to the
// start of the next).
enum LbfgsPhase {
  kPhRecursion, kPhDirection, kPhFirstTrial, kPhMoreTrials, kPhPairUpdate, kPhProgress, kPhLoopBack,
  kPhIterations, kPhExtraEvals, kPhLoopBacks, kPhSlots
};
#ifdef CNO_LBFGS_PHASE_CLOCKS
__device__ unsigned long long cno_lbfgs_phase_clocks[kPhSlots];
struct LbfgsPhaseProbe {
  unsigned long long acc[kPhSlots];
  long long t, cur[kPhLoopBack];
  bool steady, counted;
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int i = 0; i < kPhSlots; ++i) acc[i] = 0;
    counted = false;
  }
  __device__ __forceinline__ void top() {  // start of an iteration
    const long long n = clock64();
    if (counted) {
      acc[kPhLoopBack] += n - t;
      acc[kPhLoopBacks]++;
    }
    t = n;
    steady = false;
    counted = false;
  }
  __device__ __forceinline__ void set_steady() { steady = true; }
  __device__ __forceinline__ void mark(const int phase) {  // end of `phase`
    const long long n = clock64();
    cur[phase] = n - t;
    t = n;
  }
  __device__ __forceinline__ void search(const bool searched, const uint32_t evals) {  // end of the line search
    const long long n = clock64(), first = cno_ls_first_trial_clock[threadIdx.x >> 5];
    cur[kPhFirstTrial] = first - t;
    cur[kPhMoreTrials] = n - first;
    t = n;
    steady = steady && searched;
    if (steady) acc[kPhExtraEvals] += evals - 1;
  }
  __device__ __forceinline__ void end() {  // end of the iteration (Progress::Update done)
    mark(kPhProgress);
    if (steady) {
#pragma unroll
      for (int i = 0; i < kPhLoopBack; ++i) acc[i] += cur[i];
      acc[kPhIterations]++;
    }
    counted = steady;
  }
  __device__ __forceinline__ void stop() { counted = false; }  // the instance is done: no loop-back
  __device__ __forceinline__ void flush(const int lane) {
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < kPhSlots; ++i) atomicAdd(&cno_lbfgs_phase_clocks[i], acc[i]);
    }
  }
};
#else
struct LbfgsPhaseProbe {
  __device__ __forceinline__ void init() {}
  __device__ __forceinline__ void top() {}
  __device__ __forceinline__ void set_steady() {}
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void search(bool, uint32_t) {}
  __device__ __forceinline__ void end() {}
  __device__ __forceinline__ void stop() {}
  __device__ __forceinline__ void flush(int) {}
};
#endif

// The warp's shared-memory slice when the kRegPairs newest (s, y) pairs are held in registers and the older
// M - kRegPairs in shared memory.
template <class T, int D, int M, int kStage = 0, int kScratchPerLane = 0, int kMaxW = 16, int kHelpers = 0,
          int kRegPairs_ = 0>
struct LbfgsSmem {
  static constexpr int E = Shape<D>::E;
  static constexpr int kVec = 32 * E;                        // elements per stored vector
  static constexpr int kRegPairs = kRegPairs_;
  static constexpr int kSmemPairs = M - kRegPairs;           // slots of the shared ring
  static_assert(kRegPairs >= 0 && kSmemPairs >= 1, "at least one pair lives in shared memory");
  // rho and alpha of the shared pairs, f ring, policy scratch
  static constexpr int kScalars = 2 * kSmemPairs + CNO_MAX_PAST + 32 * kScratchPerLane;
  static constexpr int kHistElems = 2 * kSmemPairs * kVec + ((kScalars + 3) / 4) * 4;  // S, Y + scalars
  static constexpr int kWarpElems = kHistElems + kStage;     // + the functor's staged block
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  // warps per CTA: as many as fit in 227 KB, at most kMaxW (register budget).
  static constexpr int kMaxSmem = 227 * 1024;
  static constexpr int kWarpsFit = (int)(kMaxSmem / kWarpBytes);
  static constexpr int kMaxWarps = kMaxW < CNO_LBFGS_MAX_WARPS ? kMaxW : CNO_LBFGS_MAX_WARPS;
  static constexpr int kWarps = kWarpsFit > kMaxWarps ? kMaxWarps : (kWarpsFit < 1 ? 1 : kWarpsFit);
  // Functors with a helper warp per instance (FnHelperWarps): solver warps 0 .. kWarps-1, the helper of solver warp t is
  // warp kHelperBase + t.
  static constexpr int kHelperBase = kWarps;
  static constexpr int kThreads = 32 * (kHelpers > 0 ? 2 * kWarps : kWarps);
  static constexpr size_t kBytes = kWarpBytes * kWarps;
};

// ---- the steps of Lbfgs::OptimizationStep shared by lbfgs_minimize_kernel and the group kernel
//      (cno_lbfgs_group.cuh); RC is the reduction context, RedCtx<T> or GroupCtx<T, W> ----

// Which (s, y) pairs the history holds: mem_count pairs, chronological i = 0 (oldest) .. mem_count - 1.  Pair i lives in
// register slot mem_count - 1 - i if that is below R (the newest), else in slot (mem_pos + i) mod MS of the shared ring;
// mem_pos stays 0 until the ring is full.  At R = 0 this is the reference's index map (lbfgs.h:162).
template <int M, int R = 0>
struct LbfgsHistory {
  static constexpr int MS = M - R;  // slots of the shared ring
  int mem_count, mem_pos;
  unsigned valid;  // bit i set <=> !(|s_i . y_i| < eps), i chronological  (lbfgs.h:165,189)
  __device__ __forceinline__ void clear() {
    mem_count = 0;
    mem_pos = 0;
    valid = 0;
  }
  __device__ __forceinline__ bool pair_usable(int i) const { return (valid >> i) & 1u; }
  // The ring slot of the pair that enters the shared ring (mem_count >= R): the oldest register pair, or (R = 0) the
  // new one; when the ring is full it replaces the oldest pair there, which leaves the history.
  __device__ __forceinline__ int ring_slot() {
    int slot = mem_count - R;
    if (slot == MS) {
      slot = mem_pos;
      mem_pos = (mem_pos + 1 == MS) ? 0 : mem_pos + 1;
    }
    return slot;
  }
  // a new pair with s.y = sy joins the history (lbfgs.h:269-279) with its bit of `valid`
  template <class T>
  __device__ __forceinline__ void record(T sy) {
    const unsigned usable = (cabs(sy) < Num<T>::eps) ? 0u : 1u;
    if (mem_count < M) {
      valid |= usable << mem_count;
      mem_count++;
    } else {
      valid = (valid >> 1) | (usable << (M - 1));
    }
  }
};

// Descent test, alpha_init and fallback (lbfgs.h:199-224) on the two-loop direction q.  Returns dginit = g.(-q): the
// search runs along -q (the line search negates inside its products, cno_linesearch.cuh kNeg), so no negated copy of q
// is ever made.  The fallback sets q = -g and empties the history (register pairs included).
template <class P, class T, int E, int M, int R, class RC>
__device__ __forceinline__ T lbfgs_direction(const RC& rc, const T (&g)[E], T (&q)[E], const T xx,
                                             LbfgsHistory<M, R>& h, T& alpha_init) {
  constexpr T eps = Num<T>::eps;
  alpha_init = T(1);
  T gq;
  if (uni(h.mem_count == 0)) {  // :208-213 (||q|| only matters without history)
    T qq;
    warp_sum2_p<P, T, E>(lane_dot_p<P, T, E>(g, q), lane_dot_p<P, T, E>(q, q), rc, gq, qq);
    const T qn = csqrt(qq);
    alpha_init = (qn > eps) ? T(1) / qn : T(1);
  } else {
    gq = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(g, q), rc);
  }
  const T descent_direction = -gq;
  T dginit = descent_direction;  // = g.(-q), bit for bit
  // descent_direction > -eps * relative_eps, relative_eps = eps * max(1, ||x||) (:93-95)?  |eps * relative_eps| <=
  // eps^2 max(1, ||x||) (1 + 2^-50) and sqrt(t) <= max(1, t), so a finite direction below -2 eps^2 max(1, x.x) is below
  // the exact threshold whatever its rounding: the comparison is false and neither the square root nor the products
  // are needed.  Anything else (a non-finite operand, a direction that close to zero) takes the specification's
  // expression.
  bool fallback;
  if (cfinite(descent_direction) && cfinite(xx) && descent_direction < -(T(2) * eps * eps) * smax(T(1), xx)) {
    fallback = false;
  } else {
    const T relative_eps = eps * smax(T(1.0), csqrt(xx));
    fallback = !cfinite(descent_direction) || descent_direction > -eps * relative_eps;
  }
  if (uni(fallback)) {
    // search_direction = -g, and the reference then searches along -search_direction = +g (SURVEY.md 7.2a):
    // dginit = g.g >= 0.
#pragma unroll
    for (int j = 0; j < E; ++j) q[j] = -g[j];
    h.clear();
    const T gg = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(g, g), rc);  // :221 (rare path)
    const T gn = csqrt(gg);
    alpha_init = (gn > eps) ? T(1) / gn : T(1);
    dginit = gg;
  }
  return dginit;
}

// MoreThuente::Search / HagerZhang (lbfgs.h:231-232) along -q, its evaluations added to nfev, or the search's own
// early return for dginit >= 0 (more_thuente.h:152-156): the state untouched.
template <class LS, class Fn, class T, int E, class Ctx, class RC>
__device__ __forceinline__ void lbfgs_search(const Fn& fn, const Ctx& ctx, const RC& rc, const T (&x)[E],
                                             const T f, const T (&g)[E], T (&xn)[E], T& fn_val, T (&gn)[E],
                                             const T alpha_init, const T (&q)[E], const T dginit, uint32_t& nfev) {
  if (uni(dginit >= T(0))) {
#pragma unroll
    for (int j = 0; j < E; ++j) { xn[j] = x[j]; gn[j] = g[j]; }
    fn_val = f;
  } else {
    nfev += LS::template search<Fn, T, E, true, std::is_same<LS, LsMoreThuente>::value>(fn, ctx, rc, x, f, g, xn,
                                                                                        fn_val, gn, alpha_init, q,
                                                                                        dginit);
  }
}

// s.y, s.s, y.y (:265-266) and the next step's ||x||^2 (:95), reduced together.  Returns s.y > eps ||s|| ||y|| (:266),
// decided without the two square roots whenever a rigorous bound allows.
template <class P, class T, int E, class RC>
__device__ __forceinline__ bool lbfgs_pair_sums(const RC& rc, const T (&sd)[E], const T (&yd)[E], const T (&xn)[E],
                                                T& sy, T& yy, T& xx_next) {
  T ss;
  warp_sum4_p<P, T, E>(lane_dot_p<P, T, E>(sd, yd), lane_dot_p<P, T, E>(sd, sd), lane_dot_p<P, T, E>(yd, yd),
                       lane_dot_p<P, T, E>(xn, xn), rc, sy, ss, yy, xx_next);
  return curvature_above_eps<T>(sy, ss, yy);
}

// gamma = s.y / y.y when that is usable (lbfgs.h:289-298)
template <class T>
__device__ __forceinline__ void lbfgs_update_gamma(T& gamma, const T sy, const T yy) {
  constexpr T eps = Num<T>::eps;
  if (yy > eps) {
    const T temp_scaling = sy / yy;
    if (cfinite(temp_scaling) && cabs(temp_scaling) <= T(1e7)) gamma = smax(temp_scaling, eps);
  }
}

// lpNorm<Infinity> of three vectors of one warp (the GroupCtx overload is in cno_lbfgs_group.cuh).
template <class T, int E>
__device__ __forceinline__ void maxabs3(const RedCtx<T>&, const T (&a)[E], const T (&b)[E], const T (&c)[E], T& ra,
                                        T& rb, T& rc_out) {
  ra = warp_maxabs<T, E>(a);
  rb = warp_maxabs<T, E>(b);
  rc_out = warp_maxabs<T, E>(c);
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

// Most warps per CTA (one CTA per SM) whose per-thread register budget holds `regs`.  The warps are spread over the
// SM's 4 sub-partitions, each with its own 16384-register file, and registers are allocated in units of 8 per
// thread: the budget is 16384 / (32 ceil(W / 4)) rounded down to a multiple of 8 -- 168 up to 12 warps, 128 up to 16,
// 96 up to 20 -- and ptxas's cap is 255.
constexpr int lbfgs_register_warps(int regs) {
  int w = 32;
  while (w > 1 && ((16384 / (32 * ((w + 3) / 4))) & ~7) < regs) --w;
  return regs > 255 ? 1 : w;
}

// The shared-memory / register / warp plan of lbfgs_minimize_kernel<Fn, M, kResume, LS>.  Shared memory holds the
// history of one instance per warp; registers hold the functor's plain-kernel state (FnRegsPerThread) plus,
// per pair kept in registers, 2 E values per lane.  Where shared memory limits the warp count, pairs held in the
// registers the SM has spare make room for more warps: the plan takes the fewest register pairs (at most 2: each one
// is unrolled code in both loops of the recursion) that reach the most warps, counting only warps that keep the
// per-thread register budget of the kernel without register pairs (measured at d = 128 fp64, m = 10 on an H100:
// 1 pair and 12 warps at 168 registers beat 2 pairs and 14 warps at 128, where the kernel spills).  Only the plain
// kernel (MoreThuente, First mode, fused, no helper warp) does so: the other variants carry more live state per
// thread and keep the 128-register budget and the whole history in shared memory (the stepwise record layout,
// ResumeLayout, assumes it).
template <class Fn, int M, bool kResume = false, class LS = LsMoreThuente>
struct LbfgsPlan {
  using T = typename Fn::Scalar;
  static constexpr bool kPlain = std::is_same<LS, LsMoreThuente>::value && !IsSecondMode<Fn>::value && !kResume &&
                                 FnHelperWarps<Fn>::value == 0;
  static constexpr int kRegs = kPlain ? FnRegsPerThread<Fn>::value : 128;
  static constexpr int kPairRegs = 2 * Shape<Fn::Dim>::E * (int)(sizeof(T) / 4);
  template <int R, int kCap>
  using Smem = LbfgsSmem<T, Fn::Dim, M, StageElems<Fn>::value, PolicyScratch<typename PolicyOf<Fn>::type>::kElemsPerLane,
                         kCap, FnHelperWarps<Fn>::value, R>;
  static constexpr int kW0 = Smem<0, lbfgs_register_warps(kRegs)>::kWarps;
  static constexpr int kSameBudget = 4 * ((kW0 + 3) / 4);  // most warps with the register budget of kW0 warps
  template <int R>
  using WithPairs = Smem<R, R == 0 ? lbfgs_register_warps(kRegs)
                                   : (lbfgs_register_warps(kRegs + R * kPairRegs) < kSameBudget
                                          ? lbfgs_register_warps(kRegs + R * kPairRegs) : kSameBudget)>;
  static constexpr int kW1 = (kPlain && M > 1) ? WithPairs<(M > 1 ? 1 : 0)>::kWarps : 0;
  static constexpr int kW2 = (kPlain && M > 2) ? WithPairs<(M > 2 ? 2 : 0)>::kWarps : 0;
  static constexpr int kRegPairs = (kW2 > kW1 && kW2 > kW0) ? 2 : (kW1 > kW0 ? 1 : 0);
  using SM = WithPairs<kRegPairs>;
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
  // History split: the R newest pairs in registers, the MS = M - R older ones in the shared ring.
  constexpr int R = SM::kRegPairs;
  constexpr int MS = SM::kSmemPairs;
  constexpr int RA = R > 0 ? R : 1;  // (extent of the register arrays)
  static_assert(!kResume || R == 0, "the stepwise record holds the whole history in shared-memory slot order");

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  constexpr int kHelpers = FnHelperWarps<Fn>::value;
  // the instance slot this warp works for: its own, or (helper warps) the one of its solver warp
  const int slot = (kHelpers > 0 && warp >= SM::kHelperBase) ? warp - SM::kHelperBase : warp;
  T* const S = reinterpret_cast<T*>(smem_raw) + (size_t)slot * SM::kWarpElems;
  T* const Y = S + MS * SM::kVec;
  T* const rho_s = S + 2 * MS * SM::kVec;  // 1 / (s_i . y_i) per slot
  T* const alpha = rho_s + MS;
  T* const ring = alpha + MS;
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

  LbfgsPhaseProbe probe;
  probe.init();
  for (; solver_warp;) {
    // ---- retire + refill: next instance from the global queue ----
    const unsigned long long b = claim_instance(queue, lane);
    if (uni(b >= (unsigned long long)batch)) break;
    if constexpr (FnSkipsInstances<Fn>::value) {  // e.g. AugLagFn: the instance's outer loop has finished
      if (uni(!fn.active((long long)b))) continue;
    }
    const EvalCtx ctx{lane, (long long)b, stage_ptr, slot};
    if constexpr (kStage > 0) fn.stage(ctx, stage_parity);  // per-instance data -> shared memory (TMA)

    T x[E], g[E];
    T f;
    uint32_t nfev;
    LbfgsHistory<M, R> hist;
    T rs[RA][E], ry[RA][E], rrho[RA];  // the register pairs, [0] the newest
    T gamma;
    T xx;            // ||x||^2 carried across iterations (the dot the reference recomputes at lbfgs.h:95)
    ProgressState<T> prog;
    progress_start(prog);
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
        hist.mem_count = in[0];
        hist.mem_pos = in[1];
        hist.valid = (unsigned)in[2];
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
          SV::store(Y + slot * SM::kVec, lane, v);
        }
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
      hist.clear();
      gamma = T(1);
      xx = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(x, x), rc);
    }
    int local_it = 0;
    const auto max_local_it = ra.max_iterations;  // (`ra` is shadowed inside the loop)

    for (;;) {  // solver.h:196-220
      probe.top();
      // ================= Lbfgs::OptimizationStep (lbfgs.h:89-303) =========
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
      const int k = hist.mem_count;

      // ================= two-loop recursion (:157-196) =====================
      // Pairs in chronological order (see LbfgsHistory): loop 1 takes the register pairs, then the shared ones;
      // loop 2 the reverse.  In both loops the loads of the next shared pair are issued before the current
      // reduction (the reduction is the critical path; LDS latency hides under it).
      T ra[RA];  // alpha of the register pairs
      const bool full = uni(k == M && hist.valid == ((1u << M) - 1u));
      if (full) {
        // ---- steady state (full history, every pair usable): both loops fully
        //      unrolled, alpha_i in registers, no per-pair control flow ----
        probe.set_steady();
        int idx = hist.mem_pos + MS - 1;
        idx = (idx >= MS) ? idx - MS : idx;
        T sv[E], yv[E];
        if (R == 0) SV::load(S + idx * SM::kVec, lane, sv);
#pragma unroll
        for (int j = 0; j < R; ++j) {  // first loop (:157-171), register pairs: newest first
          const auto part = lane_dot_p<P, T, E>(rs[j], q);
          if (j + 1 == R) SV::load(S + idx * SM::kVec, lane, sv);
          ra[j] = rrho[j] * warp_sum_p<P, T, E>(part, rc);
#pragma unroll
          for (int e = 0; e < E; ++e) q[e] = q[e] - ra[j] * ry[j][e];
        }
#pragma unroll
        for (int i = MS - 1; i >= 0; --i) {  // first loop, shared pairs
          const int idx_next = (idx == 0) ? MS - 1 : idx - 1;
          const auto part = lane_dot_p<P, T, E>(sv, q);
          const T r = rho_s[idx];
          SV::load(Y + idx * SM::kVec, lane, yv);
          if (i > 0) SV::load(S + idx_next * SM::kVec, lane, sv);
          const T a = r * warp_sum_p<P, T, E>(part, rc);
          if (lane == 0) alpha[i] = a;
#pragma unroll
          for (int j = 0; j < E; ++j) q[j] = q[j] - a * yv[j];
          idx = idx_next;
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < E; ++j) q[j] = kSecond ? (precond[j] * q[j]) : (q[j] * gamma);  // H0 (:177-182)
        idx = hist.mem_pos;
        // (yv still holds y of the oldest pair: the last pair of loop 1 is the first of loop 2)
#pragma unroll
        for (int i = 0; i < MS; ++i) {  // second loop (:185-196), shared pairs: oldest first
          const int idx_next = (idx + 1 == MS) ? 0 : idx + 1;
          const auto part = lane_dot_p<P, T, E>(yv, q);
          const T r = rho_s[idx];
          const T al = alpha[i];
          SV::load(S + idx * SM::kVec, lane, sv);
          if (i + 1 < MS) SV::load(Y + idx_next * SM::kVec, lane, yv);
          const T beta = r * warp_sum_p<P, T, E>(part, rc);
          const T coef = al - beta;
#pragma unroll
          for (int j = 0; j < E; ++j) q[j] = q[j] + sv[j] * coef;
          idx = idx_next;
        }
#pragma unroll
        for (int j = R - 1; j >= 0; --j) {  // second loop, register pairs
          const auto part = lane_dot_p<P, T, E>(ry[j], q);
          const T beta = rrho[j] * warp_sum_p<P, T, E>(part, rc);
          const T coef = ra[j] - beta;
#pragma unroll
          for (int e = 0; e < E; ++e) q[e] = q[e] + rs[j][e] * coef;
        }
      } else {
        // ---- warm-up (k < M) or a skipped pair: the register pairs unrolled, the shared ones in rolled loops ----
        const int kr = k < R ? k : R;  // pairs in registers
        const int ks = k - kr;         // pairs in shared memory
        // ---- first loop (:157-171): newest pair first ----
#pragma unroll
        for (int j = 0; j < R; ++j) {
          if (uni(j < kr)) {
            const auto part = lane_dot_p<P, T, E>(rs[j], q);
            const T a = rrho[j] * warp_sum_p<P, T, E>(part, rc);
            if (uni(hist.pair_usable(k - 1 - j))) {  // lbfgs.h:165 skip
              ra[j] = a;
#pragma unroll
              for (int e = 0; e < E; ++e) q[e] = q[e] - a * ry[j][e];
            }
          }
        }
        if (uni(ks > 0)) {
          int idx = hist.mem_pos + ks - 1;
          idx = (idx >= MS) ? idx - MS : idx;
          T sv[E];
          SV::load(S + idx * SM::kVec, lane, sv);
  #pragma unroll 1
          for (int i = ks - 1; uni(i >= 0); --i) {
            const int idx_next = (idx == 0) ? MS - 1 : idx - 1;
            const auto part = lane_dot_p<P, T, E>(sv, q);
            T yv[E];
            SV::load(Y + idx * SM::kVec, lane, yv);
            SV::load(S + idx_next * SM::kVec, lane, sv);  // prefetch (harmless at i == 0)
            const T a = rho_s[idx] * warp_sum_p<P, T, E>(part, rc);
            if (uni(hist.pair_usable(i))) {  // lbfgs.h:165 skip
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
        if (uni(ks > 0)) {
          int idx = hist.mem_pos;
          T yv[E];
          SV::load(Y + idx * SM::kVec, lane, yv);
  #pragma unroll 1
          for (int i = 0; uni(i < ks); ++i) {
            const int idx_next = (idx + 1 == MS) ? 0 : idx + 1;
            const auto part = lane_dot_p<P, T, E>(yv, q);
            T sv[E];
            SV::load(S + idx * SM::kVec, lane, sv);
            SV::load(Y + idx_next * SM::kVec, lane, yv);  // prefetch (harmless past the end: a valid slot)
            const T beta = rho_s[idx] * warp_sum_p<P, T, E>(part, rc);
            if (uni(hist.pair_usable(i))) {  // lbfgs.h:189 skip
              const T coef = alpha[i] - beta;
  #pragma unroll
              for (int j = 0; j < E; ++j) q[j] = q[j] + sv[j] * coef;
            }
            idx = idx_next;
          }
        }
#pragma unroll
        for (int j = R - 1; j >= 0; --j) {
          if (uni(j < kr)) {
            const auto part = lane_dot_p<P, T, E>(ry[j], q);
            const T beta = rrho[j] * warp_sum_p<P, T, E>(part, rc);
            if (uni(hist.pair_usable(k - 1 - j))) {  // lbfgs.h:189 skip
              const T coef = ra[j] - beta;
#pragma unroll
              for (int e = 0; e < E; ++e) q[e] = q[e] + rs[j][e] * coef;
            }
          }
        }
      }

      probe.mark(kPhRecursion);
      T alpha_init;
      const T dginit = lbfgs_direction<P>(rc, g, q, xx, hist, alpha_init);
      probe.mark(kPhDirection);
      T xn[E], gn[E];
      T fn_val;
      const uint32_t nfev_before = nfev;
      lbfgs_search<LS>(fn, ctx, rc, x, f, g, xn, fn_val, gn, alpha_init, q, dginit, nfev);
      probe.search(!(dginit >= T(0)), nfev - nfev_before);

      const T prev_value = f;
      T x_delta, gnorm_inf, x_inf;
      if constexpr (LbfgsPlan<Fn, M, kResume, LS>::kPlain) {
        // ---- steady-state tail: the pair update and Progress::Update as one straight block behind ONE vote ----
        // The pair sums, the three norms and the stopping tests read only the line search's result, so they are
        // formed together, the norms' REDUX and the tests overlapping the sums' DMMA chain.  The block runs when the
        // history was full and usable, the trial value is finite, the curvature bound accepts the pair outright, the
        // plateau test (stop.past > 0) has its ring filled and either does not compare yet or its division-free bound
        // says it does not fire, and no other stopping test fires; then it makes exactly the effects of the general
        // path below, in the same order.  Otherwise it has made none and the general path runs.
        T sd[E], yd[E];
#pragma unroll
        for (int j = 0; j < E; ++j) { sd[j] = xn[j] - x[j]; yd[j] = gn[j] - g[j]; }
        T sy, ss, yy, xx_next;
        warp_sum4_p<P, T, E>(lane_dot_p<P, T, E>(sd, yd), lane_dot_p<P, T, E>(sd, sd), lane_dot_p<P, T, E>(yd, yd),
                             lane_dot_p<P, T, E>(xn, xn), rc, sy, ss, yy, xx_next);
        maxabs3(rc, sd, gn, xn, x_delta, gnorm_inf, x_inf);
        ProgressState<T> next = prog;
        const int status =
            progress_gradient_test(progress_update_head(next, stop, prev_value, fn_val, x_delta, gnorm_inf), next,
                                   stop, x_inf);
        // progress.h:280-298 (cno_progress.cuh): the plateau test's first bound, "does not fire"
        const T past_f = ring[prog.ring_pos];
        const T diff = cabs(past_f - fn_val), bound = stop.past_delta * smax(T(1), cabs(fn_val));
        const bool past_quiet =
            !(stop.past > 0) ||
            (prog.ring_size == stop.past &&
             ((int)next.num_iterations <= stop.past ||
              (cfinite(diff) && cfinite(bound) && bound > T(0) && diff > T(2) * bound)));
        if (uni(full && cfinite(fn_val) && curvature_surely_above_eps(sy, ss, yy) && past_quiet &&
                status == CNO_STATUS_CONTINUE)) {
          const T rho_new = T(1) / sy;
          const int slot = hist.ring_slot();  // mem_count = M >= R
          if constexpr (R > 0) {
            SV::store(S + slot * SM::kVec, lane, rs[R - 1]);
            SV::store(Y + slot * SM::kVec, lane, ry[R - 1]);
          } else {
            SV::store(S + slot * SM::kVec, lane, sd);
            SV::store(Y + slot * SM::kVec, lane, yd);
          }
          __syncwarp();  // all lanes are done reading rho_s in this iteration's loops
          if (lane == 0) rho_s[slot] = (R > 0) ? rrho[RA - 1] : rho_new;
#pragma unroll
          for (int j = R - 1; j > 0; --j) {
#pragma unroll
            for (int e = 0; e < E; ++e) { rs[j][e] = rs[j - 1][e]; ry[j][e] = ry[j - 1][e]; }
            rrho[j] = rrho[j - 1];
          }
          if constexpr (R > 0) {
#pragma unroll
            for (int e = 0; e < E; ++e) { rs[0][e] = sd[e]; ry[0][e] = yd[e]; }
            rrho[0] = rho_new;
          }
          hist.record(sy);
          lbfgs_update_gamma(gamma, sy, yy);
#pragma unroll
          for (int j = 0; j < E; ++j) { x[j] = xn[j]; g[j] = gn[j]; }
          f = fn_val;
          xx = xx_next;
          __syncwarp();
          if (stop.past > 0) {
            if (lane == 0) ring[next.ring_pos] = fn_val;
            next.ring_pos = (next.ring_pos + 1 == stop.past) ? 0 : next.ring_pos + 1;
            __syncwarp();
          }
          prog = next;
          prog.status = status;
          local_it++;
          probe.mark(kPhPairUpdate);
          probe.end();
          continue;
        }
      }
      if (uni(!cfinite(fn_val))) {
        // :239-241 return current: x, g, f unchanged; x_delta = |x - x|_inf (progress.h:190) is 0,
        // or NaN when x itself holds a non-finite component (rare path, computed as written).
        T zd[E];
#pragma unroll
        for (int j = 0; j < E; ++j) zd[j] = x[j] - x[j];
        maxabs3(rc, zd, g, x, x_delta, gnorm_inf, x_inf);
      } else {
        // ---- pair + gamma update (:248-298) ----
        T sd[E], yd[E];
#pragma unroll
        for (int j = 0; j < E; ++j) { sd[j] = xn[j] - x[j]; yd[j] = gn[j] - g[j]; }
        T sy, yy, xx_next;
        if (uni(lbfgs_pair_sums<P>(rc, sd, yd, xn, sy, yy, xx_next))) {
          // s.y is exactly the dot the reference recomputes per use; cache 1/(s.y)
          const T rho_new = T(1) / sy;
          if (uni(hist.mem_count >= R)) {
            const int slot = hist.ring_slot();
            if constexpr (R > 0) {
              SV::store(S + slot * SM::kVec, lane, rs[R - 1]);
              SV::store(Y + slot * SM::kVec, lane, ry[R - 1]);
            } else {
              SV::store(S + slot * SM::kVec, lane, sd);
              SV::store(Y + slot * SM::kVec, lane, yd);
            }
            __syncwarp();  // all lanes are done reading rho_s in this iteration's loops
            if (lane == 0) rho_s[slot] = (R > 0) ? rrho[RA - 1] : rho_new;
          }
#pragma unroll
          for (int j = R - 1; j > 0; --j) {  // register moves, newest pair into slot 0
#pragma unroll
            for (int e = 0; e < E; ++e) { rs[j][e] = rs[j - 1][e]; ry[j][e] = ry[j - 1][e]; }
            rrho[j] = rrho[j - 1];
          }
          if constexpr (R > 0) {
#pragma unroll
            for (int e = 0; e < E; ++e) { rs[0][e] = sd[e]; ry[0][e] = yd[e]; }
            rrho[0] = rho_new;
          }
          hist.record(sy);
        }
        lbfgs_update_gamma(gamma, sy, yy);
        probe.mark(kPhPairUpdate);
        // the norms Progress::Update and the next step need, then the next state
        maxabs3(rc, sd, gn, xn, x_delta, gnorm_inf, x_inf);
#pragma unroll
        for (int j = 0; j < E; ++j) { x[j] = xn[j]; g[j] = gn[j]; }
        f = fn_val;
        xx = xx_next;
        __syncwarp();
      }

      // ================= Progress::Update (progress.h:153-327) ============
      if constexpr (kSecond) nfev++;  // its Hessian evaluation (progress.h:206-207; value unused, DESIGN.md)
      progress_update<T>(prog, stop, ring, lane, prev_value, f, x_delta, gnorm_inf, x_inf);
      local_it++;
      probe.end();
      if (!uni(prog.status == CNO_STATUS_CONTINUE && (!kResume || local_it < max_local_it))) break;
    }
    probe.stop();

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
          in[0] = hist.mem_count;
          in[1] = hist.mem_pos;
          in[2] = (int)hist.valid;
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
          SV::load(Y + slot * SM::kVec, lane, v);
          store_row<T, 32 * E>(reinterpret_cast<T*>(rec + RL::kY) + slot * 32 * E, lane, v);
        }
      }
    }

    store_result<T, D>(out, b, lane, x, g, f, prog, nfev);
  }
  probe.flush(lane);
  if constexpr (kHelpers > 0) {
    if (solver_warp) fn.release_helper(EvalCtx{lane, 0, stage_ptr, slot});
  }
}

}  // namespace cno

#endif  // CNO_LBFGS_CUH_
