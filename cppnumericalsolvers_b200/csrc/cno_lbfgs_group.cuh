// cno_lbfgs_group.cuh -- batched Lbfgs<F, m>::Minimize for d = 256 .. 1024: one GROUP of W = d / 128 warps owns one
// instance, the whole Solver::Minimize loop fused into one persistent kernel (sm_90a).
//
// The one-warp kernel (cno_lbfgs.cuh) keeps E = d / 32 elements per lane in registers and the whole (s, y) history of
// an instance in one warp's slice of shared memory; past d = 128 both run out.  Here thread (w, l) of a group holds the
// 4 elements l E + 4 w .. l E + 4 w + 3 (E = d / 32), and the group's history (2 m d values, 160 KB at d = 1024) sits
// in shared memory that the group alone uses.  Each thread reads and writes only its own elements of the history, so
// the history needs no barrier.
//
// Reduction order (DESIGN.md 2.10): the same specification as the one-warp kernels, distributed.  The in-thread tree
// over a thread's 4 elements is exactly the first two levels of lane l's in-lane tree; the levels with stride 4, 8,
// 16 combine the W sub-partials of lane l in warp order -- (0,1), (2,3), ..., then (0,2), (4,6), ..., then (0,4) --
// which is lane_tree over the W values; the result is the specification's lane partial p[l], fed to the same two
// mma.sync.m8n8k4.f64.  Every warp of the group combines the sub-partials of its lanes itself and runs the two DMMAs,
// so all warps hold identical bits without a second broadcast; every scalar is replicated in every warp and every
// branch is uniform across the group.  The oracle (reduce_dmma_tree) is the same function of the same terms.
//
// The iteration runs the one-warp kernel's steps (cno_lbfgs.cuh: LbfgsHistory, lbfgs_direction, lbfgs_search,
// lbfgs_pair_sums, lbfgs_update_gamma, maxabs3) on a GroupCtx, with the whole history in shared memory (R = 0); the two
// loops of the recursion and the pair store are the group's own.
//
// Functors: the built-in GroupRosenbrockFn, and any fp64 functor with the group form of the functor concept
// (cno_functors.cuh; GroupEvalCtx, group_sum_terms, group_neighbours below).  CNO_INSTANTIATE_FUNCTION routes Lbfgs on
// such a functor here at d = 1024 (include/cppoptlib_b200/device.cuh: user_minimize).
//
// Not covered: register-held pairs, the stepwise (parked) form, Second mode, HagerZhang, staged functors (kStageElems).
#ifndef CNO_LBFGS_GROUP_CUH_
#define CNO_LBFGS_GROUP_CUH_

#include "cno_lbfgs.cuh"

namespace cno {

// Named barrier `id` of `threads` threads (one group): orders the group's shared-memory traffic.
__device__ __forceinline__ void group_bar(int id, int threads) {
#ifdef CNO_WARP_EMULATION
  (void)id;
  (void)threads;
  emu::team_sync();
#else
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
#endif
}

// The reduction context of a group (the counterpart of RedCtx<T>; the line search and the L-BFGS steps take either).
// scratch holds two buffers of kMaxSums x W x 32 sub-partials.  Consecutive collectives alternate between them (`phase`): a warp can only
// write a buffer again after passing the barrier of the collective in between, which every other warp reaches only
// after it has read that buffer, so one barrier per collective suffices.
template <class T, int W>
struct GroupCtx {
  static constexpr int kMaxSums = 4;  // sums reduced together (warp_sum4_p)
  static constexpr int kBufElems = kMaxSums * W * 32;
  T* scratch;
  int lane, warp, bar;
  mutable int phase;
};

// v[k] (this thread's sub-partial of sum k) -> the specification's lane partial p[lane] of sum k.
template <int K, class T, int W>
__device__ __forceinline__ void group_lane_partials(const GroupCtx<T, W>& rc, T (&v)[K]) {
  T* const buf = rc.scratch + rc.phase * GroupCtx<T, W>::kBufElems;
  rc.phase ^= 1;
#pragma unroll
  for (int k = 0; k < K; ++k) buf[(k * W + rc.warp) * 32 + rc.lane] = v[k];
  group_bar(rc.bar, 32 * W);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    T p[W];
#pragma unroll
    for (int w = 0; w < W; ++w) p[w] = buf[(k * W + w) * 32 + rc.lane];
    v[k] = lane_tree<T, W>(p);  // strides 4, 8, 16 of the lane's in-lane tree
  }
}

template <class P, class T, int E, int W>
__device__ __forceinline__ T warp_sum_p(const typename LanePartial<P, T, E>::type& part, const GroupCtx<T, W>& rc) {
  static_assert(std::is_same<P, PolicyFast>::value && E == 4, "group sums: default policy, 4 elements per thread");
  T v[1] = {part};
  group_lane_partials<1>(rc, v);
  return warp_sum(v[0]);
}
template <class P, class T, int E, int W>
__device__ __forceinline__ void warp_sum2_p(const typename LanePartial<P, T, E>::type& a,
                                            const typename LanePartial<P, T, E>::type& b, const GroupCtx<T, W>& rc,
                                            T& ra, T& rb) {
  static_assert(std::is_same<P, PolicyFast>::value && E == 4, "group sums: default policy, 4 elements per thread");
  T v[2] = {a, b};
  group_lane_partials<2>(rc, v);
  ra = v[0];
  rb = v[1];
  warp_sum2(ra, rb);
}
template <class P, class T, int E, int W>
__device__ __forceinline__ void warp_sum4_p(const typename LanePartial<P, T, E>::type& a,
                                            const typename LanePartial<P, T, E>::type& b,
                                            const typename LanePartial<P, T, E>::type& c,
                                            const typename LanePartial<P, T, E>::type& d, const GroupCtx<T, W>& rc,
                                            T& ra, T& rb, T& rc_out, T& rd) {
  static_assert(std::is_same<P, PolicyFast>::value && E == 4, "group sums: default policy, 4 elements per thread");
  T v[4] = {a, b, c, d};
  group_lane_partials<4>(rc, v);
  ra = v[0];
  rb = v[1];
  rc_out = v[2];
  rd = v[3];
  warp_sum4(ra, rb, rc_out, rd);
}

// ---- the group form of the functor concept (cno_functors.cuh): what a functor needs, so that it never writes a barrier
// The first of thread t's 4 elements in a group of W warps (d = 128 W): lane l's run of d / 32 elements starts at
// l d / 32, and warp w holds its 4 elements from 4 w on.
template <int W>
__device__ __forceinline__ int group_first_elem(int t) { return (t & 31) * (4 * W) + 4 * (t >> 5); }

// The sum over the group of the functor's terms (4 per thread), in the order of the reduction specification (DESIGN.md
// 3): the same bits as warp_sum(lane_tree<T, d / 32>(terms)) of the one-warp form.  Every thread gets the sum.  The sum
// ends with a barrier of the whole group, and it flips the kernel's own double buffer (c.rc).
template <int W>
__device__ __forceinline__ double group_sum_terms(const GroupEvalCtx<W>& c, const double (&terms)[4]) {
  double t[4] = {terms[0], terms[1], terms[2], terms[3]};
  return warp_sum_p<PolicyFast, double, 4>(lane_tree<double, 4>(t), *c.rc);
}

// x_{first - 1} and x_{first + 4}, the neighbours of a thread's 4 elements, through the group's exchange block.  They
// come from (w -+ 1, l), or at the ends of a lane's run from (W - 1, l - 1) and (0, l + 1).  At the ends of the vector
// (x_{-1}, x_d) the thread gets its own x[3] and x[0]; those values are not elements and must not be used.
// Barrier rule: an evaluation that calls this must be followed by a group sum (group_sum_terms, or the kernel's sum of
// a partial) before the exchange block is written again -- every thread has then read its neighbours.  A functor that
// returns group_sum_terms keeps the rule, so composites with several such leaves do too.
template <int W, class T>
__device__ __forceinline__ void group_neighbours(const GroupEvalCtx<W>& c, const T (&x)[4], T& x_prev, T& x_next) {
  constexpr int NT = 32 * W;
  const int t = c.lane, w = t >> 5, l = t & 31;
  T* const xch = static_cast<T*>(c.stage);
  xch[t] = x[0];
  xch[NT + t] = x[3];
  group_bar(c.team, NT);
  const int tn = (w + 1 < W) ? t + 32 : (l + 1 < 32 ? l + 1 : t);        // owner of element first + 4
  const int tp = (w > 0) ? t - 32 : (l > 0 ? 32 * (W - 1) + l - 1 : t);  // owner of element first - 1
  x_next = xch[tn];
  x_prev = xch[NT + tp];
}

// lpNorm<Infinity> of three group-distributed vectors in one barrier (warp_maxabs's specification: the largest IEEE bit
// pattern of |v_i| read as an unsigned integer; order free): each warp's maximum, then the maximum over the W warps as
// 64-bit patterns.
template <class T, int W>
__device__ __forceinline__ void maxabs3(const GroupCtx<T, W>& rc, const T (&a)[4], const T (&b)[4], const T (&c)[4],
                                        T& ra, T& rb, T& rc_out) {
  static_assert(sizeof(T) == 8, "group maxabs: fp64");
  T* const buf = rc.scratch + rc.phase * GroupCtx<T, W>::kBufElems;
  rc.phase ^= 1;
  const T m[3] = {warp_maxabs<T, 4>(a), warp_maxabs<T, 4>(b), warp_maxabs<T, 4>(c)};
  if (rc.lane == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) buf[k * W * 32 + rc.warp] = m[k];
  }
  group_bar(rc.bar, 32 * W);
  T r[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    unsigned hi = 0u, lo = 0u;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const T v = buf[k * W * 32 + w];
      const unsigned h = (unsigned)__double2hiint(v), l = (unsigned)__double2loint(v);
      const bool above = (h > hi) || (h == hi && l > lo);
      hi = above ? h : hi;
      lo = above ? l : lo;
    }
    r[k] = __hiloint2double((int)hi, (int)lo);
  }
  ra = r[0];
  rb = r[1];
  rc_out = r[2];
}

// One vector of the group's history in shared memory: chunk c (CE elements) of thread t at element (c * 32 W + t) CE,
// so every warp access is one conflict-free contiguous run of 32 packs.
template <class T, int W>
struct GroupVec {
  using LP = LanePack<T, 4>;
  __device__ __forceinline__ static void load(const T* base, int t, T (&v)[4]) {
    const typename LP::P::type* p = reinterpret_cast<const typename LP::P::type*>(base);
#pragma unroll
    for (int c = 0; c < LP::NC; ++c) LP::P::get(p[c * 32 * W + t], &v[c * LP::CE]);
  }
  __device__ __forceinline__ static void store(T* base, int t, const T (&v)[4]) {
    typename LP::P::type* p = reinterpret_cast<typename LP::P::type*>(base);
#pragma unroll
    for (int c = 0; c < LP::NC; ++c) p[c * 32 * W + t] = LP::P::make(&v[c * LP::CE]);
  }
};

// A thread's 4 contiguous elements of a row-major [B, D] row (16-byte aligned: the offset is a multiple of 4).
template <class T, bool kReadOnly>
__device__ __forceinline__ void load_quad(const T* __restrict__ p, T (&v)[4]) {
  using LP = LanePack<T, 4>;
  const typename LP::P::type* q = reinterpret_cast<const typename LP::P::type*>(p);
#pragma unroll
  for (int c = 0; c < LP::NC; ++c) {
    typename LP::P::type u;
    if constexpr (kReadOnly) u = __ldg(q + c); else u = q[c];
    LP::P::get(u, &v[c * LP::CE]);
  }
}
template <class T>
__device__ __forceinline__ void store_quad(T* __restrict__ p, const T (&v)[4]) {
  using LP = LanePack<T, 4>;
  typename LP::P::type* q = reinterpret_cast<typename LP::P::type*>(p);
#pragma unroll
  for (int c = 0; c < LP::NC; ++c) q[c] = LP::P::make(&v[c * LP::CE]);
}

// Chained Rosenbrock for a group (same operation order as RosenbrockFn and the oracle's eval_rosenbrock).  x_{i+1} of a
// thread's last element and x_{i-1} of its first come from group_neighbours; B_{i-1} = 200 (x_i - x_{i-1}^2) is then
// formed in the thread that needs it (the same operands in the same order as in the thread that owns element i - 1).
// partial() leaves the sum to its caller, which keeps group_neighbours' barrier rule by summing it.
template <class T, int D>
struct GroupRosenbrockFn {
  static_assert(D % 128 == 0 && (D / 128 & (D / 128 - 1)) == 0 && D / 128 >= 2 && D / 128 <= 8,
                "group Rosenbrock: d = 256, 512 or 1024");
  using Scalar = T;
  using Policy = PolicyFast;
  static constexpr int Dim = D;
  static constexpr int Mode = 1;
  static constexpr int kGroupWarps = D / 128;
  static constexpr int E = 4;  // elements per thread
  static constexpr bool kHasPartial = true;
  static constexpr int kXchElems = 2 * 32 * kGroupWarps;

  // the first of thread t's 4 elements
  __device__ __forceinline__ static int first_elem(int t) { return group_first_elem<kGroupWarps>(t); }

  __device__ __forceinline__ T partial(const GroupEvalCtx<kGroupWarps>& c, const T (&x)[4], T (*grad)[4]) const {
    T x_prev, x_next;
    group_neighbours(c, x, x_prev, x_next);
    const int i0 = c.first;
    T term[4], A[4], Bv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = i0 + j;
      const T xi = x[j];
      const T xn = (j + 1 < 4) ? x[(j + 1 < 4) ? j + 1 : 0] : x_next;
      const T t1 = (1 - xi);
      const T t2 = (xn - xi * xi);
      const bool live = (i + 1 < D);
      term[j] = live ? (t1 * t1 + 100 * t2 * t2) : T(0);
      A[j] = -2 * (1 - xi) + 200 * (xn - xi * xi) * (-2 * xi);
      Bv[j] = 200 * (xn - xi * xi);
    }
    if (grad) {
      const T b_prev = 200 * (x[0] - x_prev * x_prev);  // B_{i0-1}
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = i0 + j;
        const T bprev = (j > 0) ? Bv[(j > 0) ? j - 1 : 0] : b_prev;
        T gi;
        if (i == 0) gi = A[j];
        else if (i == D - 1) gi = bprev;
        else gi = bprev + A[j];
        (*grad)[j] = gi;
      }
    }
    return lane_tree<T, 4>(term);
  }
  // the group form of the functor concept: the value summed over the group (what the mirror's Rosenbrock forwards to)
  __device__ __forceinline__ T operator()(const GroupEvalCtx<kGroupWarps>& c, const T (&x)[4], T (*grad)[4]) const {
    return warp_sum_p<PolicyFast, T, 4>(partial(c, x, grad), *c.rc);
  }
};

// 0.5 * x.squaredNorm() for a group: HalfSquaredNormFn's arithmetic, summed over the group.
template <int D>
struct GroupHalfSquaredNormFn {
  __device__ __forceinline__ double operator()(const GroupEvalCtx<D / 128>& c, const double (&x)[4],
                                               double (*grad)[4]) const {
    double t[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (grad) (*grad)[j] = x[j];
      t[j] = x[j] * x[j];
    }
    return 0.5 * group_sum_terms(c, t);
  }
};

// Shared memory of one group, in elements: history S[M][D], Y[M][D]; the double-buffered reduction scratch; the
// functor's exchange block; the claimed instance id (16 bytes); then per warp rho[M], alpha[M] and the past-f ring.
// Groups per CTA: as many as fit in 227 KB (at most 15: named barriers 1..15); kFit = 0 when one group does not fit.
template <class T, int D, int M>
struct LbfgsGroupPlan {
  static constexpr int kGroupWarps = D / 128;
  static constexpr int kGroupThreads = 32 * kGroupWarps;
  static constexpr int kScratch = 2 * GroupCtx<T, kGroupWarps>::kBufElems;
  static constexpr int kXch = 2 * kGroupThreads;
  static constexpr int kClaim = 16 / (int)sizeof(T);
  static constexpr int kWarpScalars = ((2 * M + CNO_MAX_PAST + 1) / 2) * 2;
  static constexpr int kOffY = M * D;
  static constexpr int kOffScratch = 2 * M * D;
  static constexpr int kOffXch = kOffScratch + kScratch;
  static constexpr int kOffClaim = kOffXch + kXch;
  static constexpr int kOffWarp = kOffClaim + kClaim;
  static constexpr int kGroupElems = kOffWarp + kGroupWarps * kWarpScalars;
  static constexpr size_t kGroupBytes = (size_t)kGroupElems * sizeof(T);
  static constexpr int kMaxSmem = 227 * 1024;
  static constexpr int kFit = (int)(kMaxSmem / kGroupBytes);
  static constexpr int kGroups = kFit > 15 ? 15 : (kFit < 1 ? 1 : kFit);
  // launch_persistent's plan: kWarps = resident instances per CTA (one per group), kThreads = the block
  static constexpr int kWarps = kGroups;
  static constexpr int kThreads = kGroups * kGroupThreads;
  static constexpr size_t kBytes = kGroupBytes * kGroups;
};

// Lbfgs<Fn, M>::Minimize with MoreThuente, First mode, on a group functor: GroupRosenbrockFn (its unreduced partial,
// reduced with ||x||^2 and the slopes) or a functor with the group form (it reduces its own value).
template <class Fn, int M>
__global__ void __launch_bounds__(LbfgsGroupPlan<typename Fn::Scalar, Fn::Dim, M>::kThreads, 1)
lbfgs_group_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0, const long long batch,
                            const StopParams<typename Fn::Scalar> stop, const BatchOut<typename Fn::Scalar> out,
                            unsigned long long* __restrict__ queue) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  using PL = LbfgsGroupPlan<T, D, M>;
  static_assert(PL::kFit >= 1, "one group's history does not fit in shared memory");
  constexpr int W = PL::kGroupWarps;
  constexpr int NT = PL::kGroupThreads;
  constexpr int E = 4;
  using P = PolicyFast;
  using GV = GroupVec<T, W>;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int group = (int)threadIdx.x / NT;
  const int t = (int)threadIdx.x % NT;
  const int warp = t >> 5, lane = t & 31;
  T* const G = reinterpret_cast<T*>(smem_raw) + (size_t)group * PL::kGroupElems;
  T* const S = G;
  T* const Yh = G + PL::kOffY;
  unsigned long long* const claim = reinterpret_cast<unsigned long long*>(G + PL::kOffClaim);
  T* const rho_s = G + PL::kOffWarp + warp * PL::kWarpScalars;  // 1 / (s_i . y_i) per slot (this warp's copy)
  T* const alpha = rho_s + M;
  T* const ring = alpha + M;
  const GroupCtx<T, W> rc{G + PL::kOffScratch, lane, warp, 1 + group, 0};
  const int e0 = group_first_elem<W>(t);

  for (;;) {
    // ---- retire + refill: one thread of the group claims the next instance ----
    if (t == 0) *claim = atomicAdd(queue, 1ULL);
    group_bar(rc.bar, NT);
    const unsigned long long b = *claim;
    if (uni(b >= (unsigned long long)batch)) break;
    const GroupEvalCtx<W> ctx{t, (long long)b, G + PL::kOffXch, rc.bar, e0, &rc};

    T x[E], g[E];
    T f;
    uint32_t nfev;
    LbfgsHistory<M> hist;
    hist.clear();
    T gamma = T(1);
    T xx;
    ProgressState<T> prog;
    progress_start(prog);
    // ---- solver.h:189-192: evaluate once at the start point; ||x||^2 of lbfgs.h:95 in the same round ----
    load_quad<T, true>(x0 + b * D + e0, x);
    if constexpr (FnHasPartial<Fn>::value) {
      warp_sum2_p<P, T, E>(fn.partial(ctx, x, &g), lane_dot_p<P, T, E>(x, x), rc, f, xx);
    } else {
      f = fn(ctx, x, &g);
      xx = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(x, x), rc);
    }
    nfev = 1;

    do {  // solver.h:196-220
      // ================= Lbfgs::OptimizationStep (lbfgs.h:89-303) =========
      T q[E];
#pragma unroll
      for (int j = 0; j < E; ++j) q[j] = g[j];  // :145
      const int k = hist.mem_count;
      // ---- first loop (:157-171): newest pair first ----
      if (uni(k > 0)) {
        int idx = hist.mem_pos + k - 1;
        idx = (idx >= M) ? idx - M : idx;
#pragma unroll 1
        for (int i = k - 1; uni(i >= 0); --i) {
          T sv[E], yv[E];
          GV::load(S + idx * D, t, sv);
          GV::load(Yh + idx * D, t, yv);
          const T a = rho_s[idx] * warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(sv, q), rc);
          if (uni(hist.pair_usable(i))) {  // lbfgs.h:165 skip
            if (lane == 0) alpha[i] = a;
#pragma unroll
            for (int j = 0; j < E; ++j) q[j] = q[j] - a * yv[j];
          }
          idx = (idx == 0) ? M - 1 : idx - 1;
        }
      }
      __syncwarp();
#pragma unroll
      for (int j = 0; j < E; ++j) q[j] = q[j] * gamma;  // H0 (:177-182)
      // ---- second loop (:185-196): oldest pair first ----
      if (uni(k > 0)) {
        int idx = hist.mem_pos;
#pragma unroll 1
        for (int i = 0; uni(i < k); ++i) {
          T sv[E], yv[E];
          GV::load(Yh + idx * D, t, yv);
          GV::load(S + idx * D, t, sv);
          const T beta = rho_s[idx] * warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(yv, q), rc);
          if (uni(hist.pair_usable(i))) {  // lbfgs.h:189 skip
            const T coef = alpha[i] - beta;
#pragma unroll
            for (int j = 0; j < E; ++j) q[j] = q[j] + sv[j] * coef;
          }
          idx = (idx + 1 == M) ? 0 : idx + 1;
        }
      }

      T alpha_init;
      const T dginit = lbfgs_direction<P>(rc, g, q, xx, hist, alpha_init);
      T xn[E], gn[E];
      T fn_val;
      lbfgs_search<LsMoreThuente>(fn, ctx, rc, x, f, g, xn, fn_val, gn, alpha_init, q, dginit, nfev);

      const T prev_value = f;
      T x_delta, gnorm_inf, x_inf;
      if (uni(!cfinite(fn_val))) {
        // :239-241 return current; x_delta = |x - x|_inf (0, or NaN for a non-finite x)
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
          const T rho_new = T(1) / sy;
          const int slot = hist.ring_slot();
          GV::store(S + slot * D, t, sd);
          GV::store(Yh + slot * D, t, yd);
          __syncwarp();  // all lanes are done reading rho_s in this iteration's loops
          if (lane == 0) rho_s[slot] = rho_new;
          hist.record(sy);
        }
        lbfgs_update_gamma(gamma, sy, yy);
        maxabs3(rc, sd, gn, xn, x_delta, gnorm_inf, x_inf);
#pragma unroll
        for (int j = 0; j < E; ++j) { x[j] = xn[j]; g[j] = gn[j]; }
        f = fn_val;
        xx = xx_next;
        __syncwarp();
      }

      // ================= Progress::Update (progress.h:153-327) ============
      progress_update<T>(prog, stop, ring, lane, prev_value, f, x_delta, gnorm_inf, x_inf);
    } while (uni(prog.status == CNO_STATUS_CONTINUE));

    if (out.x) store_quad<T>(out.x + b * D + e0, x);
    if (out.gradient) store_quad<T>(out.gradient + b * D + e0, g);
    if (t == 0) store_result_scalars<T>(out, b, f, prog, nfev);
    __syncwarp();
  }
}

}  // namespace cno

#endif  // CNO_LBFGS_GROUP_CUH_
