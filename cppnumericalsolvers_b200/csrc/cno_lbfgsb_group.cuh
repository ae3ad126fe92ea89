// cno_lbfgsb_group.cuh -- batched Lbfgsb<F, m = 5>::Minimize for d = 256, 512 and 1024: one GROUP of W = d / 128 warps
// owns one instance, the whole overridden Minimize loop in one persistent kernel (sm_90a).
//
// Reference path (include/cppoptlib/solver/lbfgsb.h): the same as the one-warp kernel (cno_lbfgsb.cuh), which past
// d = 128 runs out of registers and of its warp's slice of shared memory.  Outputs and arithmetic are those of
// lbfgsb_minimize_kernel (DESIGN.md 3, "Lbfgsb"); what differs is where the data lives and how sums are distributed.
//
// Layout (DESIGN.md 2.11).
//   * Per thread: thread (w, l) of the group holds the 4 elements from group_first_elem<W>(t) = l d / 32 + 4 w on, as
//     the group L-BFGS kernel does: x, g, the box, the Cauchy direction and breakpoints, the Cauchy point, r, du, the
//     trial point and its gradient.
//   * Per group, in shared memory: the m (y, s) pairs.  Unlike the group L-BFGS kernel, other threads read them (row b
//     of W in the breakpoint loop, any row in the compacted sums), so every element goes through one map,
//     lbfgsb_hist_index, and a group barrier lies between a pair store and the next read of that row by another thread:
//     the S'Y / S'S sums that follow every store provide it.  Also per group: the reduction scratch of GroupCtx, the
//     functor's exchange block, and r with the compaction map of the subspace step.
//   * Replicated in every warp (each warp its own copy, all holding the same bits): the 2k-vectors p, c, w_b, v (entry i
//     in lane i), the S'Y / S'S caches, the LU factors of MM and NN with their pivots, theta and the past-f ring.  Every
//     branch is therefore uniform across the group, as in the group L-BFGS kernel (DESIGN.md 2.10).
//
// Sums.  Full-length sums (W'd, d.d, s.y, y.y, the S'Y / S'S entries) are GroupCtx sums, up to four per barrier, each
// in its own specified order.  Sums over the free variables follow the specification on the COMPACTED vector of length
// n = nfree: lane l holds positions l E' .. l E' + E' - 1, E' = ceil(n / 32); thread (w, l) takes positions 4 w .. 4 w + 3
// of that run, strides 1 and 2 of the in-lane tree run in the thread, strides 4, 8 and 16 across the warps, all under the
// tree's own mask j + s < E' (group_lane_partials_masked).  When n = d that is the ordinary group sum.
//
// Breakpoints: repeated selection of the smallest positive (t, index), one group barrier per visited breakpoint: each
// warp's winner publishes (t, index) with its d, g, x, lower and upper; after the barrier every warp takes the group
// minimum and has the coordinate's values.
//
// Not covered: m other than 5, fp32, the stepwise form, user functors (the dispatch refuses them).
#ifndef CNO_LBFGSB_GROUP_CUH_
#define CNO_LBFGSB_GROUP_CUH_

#include "cno_lbfgs_group.cuh"
#include "cno_lbfgsb.cuh"

namespace cno {

// Address of element i of one history vector (the layout of GroupVec<double, W>: 2-element chunk c of thread t at
// element (c * 32 W + t) * 2): the one map from element index to shared memory for the reads of other threads' rows.
template <int W>
__device__ __forceinline__ int lbfgsb_hist_index(int i) {
  const int l = i / (4 * W), r = i - l * (4 * W);
  const int t = 32 * (r >> 2) + l, j = r & 3;
  return ((j >> 1) * 32 * W + t) * 2 + (j & 1);
}

// The buffer of the next collective of the group (GroupCtx's double buffer; one barrier per collective suffices).
template <class T, int W>
__device__ __forceinline__ T* group_next_buf(const GroupCtx<T, W>& rc) {
  T* const buf = rc.scratch + rc.phase * GroupCtx<T, W>::kBufElems;
  rc.phase ^= 1;
  return buf;
}

// Any thread of the group: one barrier.
template <class T, int W>
__device__ __forceinline__ bool group_any(const GroupCtx<T, W>& rc, bool c) {
  T* const buf = group_next_buf(rc);
  const bool any = __any_sync(kFullMask, c);
  if (rc.lane == 0) buf[rc.warp] = any ? T(1) : T(0);
  group_bar(rc.bar, 32 * W);
  bool r = false;
#pragma unroll
  for (int w = 0; w < W; ++w) r = r || (buf[w] != T(0));
  return r;
}

// The minimum over the group of per-warp values (warp order; a NaN never wins a comparison): one barrier.
template <class T, int W>
__device__ __forceinline__ T group_min_of_warps(const GroupCtx<T, W>& rc, T v) {
  T* const buf = group_next_buf(rc);
  if (rc.lane == 0) buf[rc.warp] = v;
  group_bar(rc.bar, 32 * W);
  T m = buf[0];
#pragma unroll
  for (int w = 1; w < W; ++w) {
    const T o = buf[w];
    m = (o < m) ? o : m;
  }
  return m;
}

// lpNorm<Infinity> of K group-distributed vectors from their per-warp maxima (warp_maxabs): the largest IEEE bit
// pattern over the W warps (maxabs3's specification), one barrier for all K.
template <int K, int W>
__device__ __forceinline__ void group_max_bits(const GroupCtx<double, W>& rc, double (&m)[K]) {
  double* const buf = group_next_buf(rc);
  if (rc.lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) buf[k * W + rc.warp] = m[k];
  }
  group_bar(rc.bar, 32 * W);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    unsigned hi = 0u, lo = 0u;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const double v = buf[k * W + w];
      const unsigned h = (unsigned)__double2hiint(v), l = (unsigned)__double2loint(v);
      const bool above = (h > hi) || (h == hi && l > lo);
      hi = above ? h : hi;
      lo = above ? l : lo;
    }
    m[k] = __hiloint2double((int)hi, (int)lo);
  }
}

// K compacted sums: v[k][c] = the term at position 4 w + c of lane l's run of E' = ep positions (zero at positions
// >= n inside the run).  Returns the specification's lane partial p[l] of each sum: the in-lane tree over the E'
// positions, with v[j] += v[j + s] only where j + s < E' (absent positions are skipped, not added as zeros).
template <int K, class T, int W>
__device__ __forceinline__ void group_lane_partials_masked(const GroupCtx<T, W>& rc, const T (&v)[K][4], int ep,
                                                           T (&part)[K]) {
  const int j0 = 4 * rc.warp;
  T* const buf = group_next_buf(rc);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    T a = v[k][0], b = v[k][2];
    if (j0 + 1 < ep) a = a + v[k][1];  // stride 1
    if (j0 + 3 < ep) b = b + v[k][3];
    if (j0 + 2 < ep) a = a + b;        // stride 2
    buf[(k * W + rc.warp) * 32 + rc.lane] = a;
  }
  group_bar(rc.bar, 32 * W);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    T p[W];
#pragma unroll
    for (int w = 0; w < W; ++w) p[w] = buf[(k * W + w) * 32 + rc.lane];
#pragma unroll
    for (int s = 1; s < W; s <<= 1) {  // strides 4 s = 4, 8, 16
#pragma unroll
      for (int w = 0; w + s < W; w += 2 * s)
        if (4 * (w + s) < ep) p[w] = p[w] + p[w + s];
    }
    part[k] = p[0];
  }
}

// Shared memory of one group, in elements: history Y[M][D], S[M][D]; the double-buffered reduction scratch; the
// functor's exchange block; the claimed instance id (16 bytes); r and the compaction map (ints) of the subspace step;
// then per warp MM, NN (LU factors, column-major, leading dimension 2M), S'Y, S'S, the past-f ring and the pivots.
// Groups per CTA: as many as fit in 227 KB and in the registers of 256 threads (named barriers 1..15).
template <class T, int D, int M>
struct LbfgsbGroupPlan {
  static_assert(sizeof(T) == 8 && D % 128 == 0, "group Lbfgsb: fp64, d a multiple of 128");
  static constexpr int kGroupWarps = D / 128;
  static constexpr int kGroupThreads = 32 * kGroupWarps;
  static constexpr int L2 = 2 * M;
  static constexpr int kScratch = 2 * GroupCtx<T, kGroupWarps>::kBufElems;
  static constexpr int kXch = 2 * kGroupThreads;
  static constexpr int kClaim = 16 / (int)sizeof(T);
  static constexpr int kMap = (D * (int)sizeof(int) + (int)sizeof(T) - 1) / (int)sizeof(T);
  static constexpr int kPivElems = (2 * L2 * (int)sizeof(int) + (int)sizeof(T) - 1) / (int)sizeof(T);
  static constexpr int kWarpSmall = ((2 * L2 * L2 + 2 * M * M + CNO_MAX_PAST + kPivElems + 1) / 2) * 2;
  static constexpr int kOffY = 0;
  static constexpr int kOffS = M * D;
  static constexpr int kOffScratch = 2 * M * D;
  static constexpr int kOffXch = kOffScratch + kScratch;
  static constexpr int kOffClaim = kOffXch + kXch;
  static constexpr int kOffR = kOffClaim + kClaim;
  static constexpr int kOffMap = kOffR + D;
  static constexpr int kOffWarp = ((kOffMap + kMap + 1) / 2) * 2;
  static constexpr int kGroupElems = kOffWarp + kGroupWarps * kWarpSmall;
  static constexpr size_t kGroupBytes = (size_t)kGroupElems * sizeof(T);
  static constexpr int kMaxSmem = 227 * 1024;
  static constexpr int kFit = (int)(kMaxSmem / kGroupBytes);
  // Registers bound the CTA before shared memory does: the iteration needs about 210 registers per thread, so a CTA of
  // at most 256 threads (255 registers each) runs without spills.  That is 4, 2 and 1 groups at d = 256, 512, 1024.
  static constexpr int kMaxThreads = 256;
  static constexpr int kRegFit = kMaxThreads / kGroupThreads;
  static constexpr int kGroups0 = kFit < kRegFit ? kFit : kRegFit;
  static constexpr int kGroups = kGroups0 > 15 ? 15 : (kGroups0 < 1 ? 1 : kGroups0);
  // launch_persistent's plan: kWarps = resident instances per CTA (one per group), kThreads = the block
  static constexpr int kWarps = kGroups;
  static constexpr int kThreads = kGroups * kGroupThreads;
  static constexpr size_t kBytes = kGroupBytes * kGroups;
};

// Lbfgsb<Fn, M>::Minimize with MoreThuente on a group functor (GroupRosenbrockFn).
template <class Fn, int M = 5>
__global__ void __launch_bounds__(LbfgsbGroupPlan<typename Fn::Scalar, Fn::Dim, M>::kThreads, 1)
lbfgsb_group_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0, const long long batch,
                             const StopParams<typename Fn::Scalar> stop, const BatchOut<typename Fn::Scalar> out,
                             unsigned long long* __restrict__ queue, const BoundsArgs<typename Fn::Scalar> bounds) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  using PL = LbfgsbGroupPlan<T, D, M>;
  static_assert(PL::kFit >= 1, "one group's state does not fit in shared memory");
  constexpr int W = PL::kGroupWarps;
  constexpr int NT = PL::kGroupThreads;
  constexpr int E = 4;
  constexpr int L2 = PL::L2;
  using P = PolicyFast;
  using GV = GroupVec<T, W>;
  constexpr T kMaxValue = (T)1.7976931348623157e308;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int group = (int)threadIdx.x / NT;
  const int t = (int)threadIdx.x % NT;
  const int warp = t >> 5, lane = t & 31;
  T* const G = reinterpret_cast<T*>(smem_raw) + (size_t)group * PL::kGroupElems;
  T* const Ys = G + PL::kOffY;
  T* const Ss = G + PL::kOffS;
  unsigned long long* const claim = reinterpret_cast<unsigned long long*>(G + PL::kOffClaim);
  T* const rstage = G + PL::kOffR;                                 // r at compacted position q
  int* const cmap = reinterpret_cast<int*>(G + PL::kOffMap);       // element at compacted position q
  T* const MM = G + PL::kOffWarp + warp * PL::kWarpSmall;          // this warp's copy of the small state
  T* const NN = MM + L2 * L2;
  T* const SY = NN + L2 * L2;     // SY[pi + pj*M] = s_pi . y_pj  (physical slots)
  T* const SSc = SY + M * M;      // SSc[pi + pj*M] = s_pi . s_pj
  T* const ring = SSc + M * M;
  int* const piv = reinterpret_cast<int*>(ring + CNO_MAX_PAST);
  int* const pivN = piv + L2;
  const GroupCtx<T, W> rc{G + PL::kOffScratch, lane, warp, 1 + group, 0};
  const int e0 = group_first_elem<W>(t);

  for (;;) {
    // ---- retire + refill: one thread of the group claims the next instance ----
    if (t == 0) *claim = atomicAdd(queue, 1ULL);
    group_bar(rc.bar, NT);
    const unsigned long long b = *claim;
    if (uni(b >= (unsigned long long)batch)) break;
    const GroupEvalCtx<W> ctx{t, (long long)b, G + PL::kOffXch, rc.bar, e0, &rc};

    // ---- the box (:88-92; defaults of InitializeSolver :122-128) ----
    T lo[E], hi[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      lo[e] = bounds.lower ? bounds.lower[b * bounds.stride + e0 + e] : -kMaxValue;
      hi[e] = bounds.upper ? bounds.upper[b * bounds.stride + e0 + e] : kMaxValue;
    }
    auto clip = [&](const T (&v)[E], T (&o)[E]) -> bool {  // cwiseMin(upper).cwiseMax(lower); true if it changed v
      bool changed = false;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const T a = (hi[e] < v[e]) ? hi[e] : v[e];
        o[e] = (a < lo[e]) ? lo[e] : a;
        changed = changed || (o[e] != v[e]);
      }
      return group_any(rc, changed);
    };

    T x[E], g[E];
    load_quad<T, true>(x0 + b * D + e0, x);
    T f = fn(ctx, x, &g);  // :246
    uint32_t nfev = 1;

    // ---- InitializeSolver (:118-136) ----
    T theta = T(1);
    int kp = 0;    // pairs stored
    int base = 0;  // physical slot of the oldest pair
    bool have_lu = false;
    auto slot = [&](int i) -> int { const int s2 = base + i; return s2 >= M ? s2 - M : s2; };

    ProgressState<T> prog;
    progress_start(prog);
    StopParams<T> stop_nograd = stop;  // :254-256: the base class's full-gradient test is suppressed
    stop_nograd.gradient_norm = T(0);
    const T pg_tol = stop.gradient_norm;

    do {  // :260-278
      // =================== OptimizationStep (:138-229) ===================
      const int n2 = 2 * kp;
      // W = [Y, theta S]: entry (element i, column c) for c < 2k, and the same for one of this thread's elements
      auto w_at = [&](int i, int c) -> T {
        const int a = lbfgsb_hist_index<W>(i);
        return (c < kp) ? Ys[slot(c) * D + a] : (theta * Ss[slot(c - kp) * D + a]);
      };
      auto w_own = [&](int e, int c) -> T { return w_at(e0 + e, c); };
      auto solveM = [&](T r) -> T { return (have_lu && n2 > 0) ? lu_solve_warp<L2>(MM, piv, n2, r, lane) : r; };

      // ---- :145-150 project the iterate; re-evaluate if it moved ----
      const T prev_value_state = f;
      T xprev[E];
#pragma unroll
      for (int e = 0; e < E; ++e) xprev[e] = x[e];
      {
        T xcur[E];
        if (clip(x, xcur)) {
#pragma unroll
          for (int e = 0; e < E; ++e) x[e] = xcur[e];
          f = fn(ctx, x, &g);
          nfev++;
        }
      }
      // ---- :162-163 projected-gradient norm (this warp's part; the group maximum is taken with Progress's norms) ----
      T pg_warp;
      {
        T pgv[E];
#pragma unroll
        for (int e = 0; e < E; ++e) {
          T gj = g[e];
          if (x[e] <= lo[e] && gj > T(0)) gj = T(0);
          if (x[e] >= hi[e] && gj < T(0)) gj = T(0);
          const T a = cabs(gj);
          pgv[e] = (a != a) ? T(0) : a;
        }
        pg_warp = warp_maxabs<T, E>(pgv);
      }

      // =================== GetGeneralizedCauchyPoint (:322-446) ===================
      T dvec[E], tbp[E], xc[E];
      bool done[E];  // sorted order = ascending t, ties by index; `done` = positions before the current one
      int cnt_own = 0;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        dvec[e] = -g[e];
        T tj;
        if (g[e] == T(0)) {
          tj = kMaxValue;
        } else {
          tj = (g[e] < T(0)) ? ((x[e] - hi[e]) / g[e]) : ((x[e] - lo[e]) / g[e]);
          if (tj == T(0)) dvec[e] = T(0);
        }
        tbp[e] = tj;
        xc[e] = x[e];
        done[e] = !(tbp[e] > T(0));
        cnt_own += done[e] ? 1 : 0;
      }
      // p = W'd (:354, entry i in lane i), d.d (:358) and the number of non-positive t: up to four sums per round
      T pvec = T(0), dd = T(0);
      int cnt_np = 0;
#pragma unroll 1
      for (int i0 = 0; i0 < n2 + 2; i0 += 4) {
        T v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int i = i0 + k;
          if (i < n2) {
            T wcol[E];
#pragma unroll
            for (int e = 0; e < E; ++e) wcol[e] = w_own(e, i);
            v[k] = lane_dot<T, E>(wcol, dvec);
          } else if (i == n2) {
            v[k] = lane_dot<T, E>(dvec, dvec);
          } else {
            v[k] = (i == n2 + 1) ? T(cnt_own) : T(0);  // a count: exact in any order
          }
        }
        group_lane_partials<4>(rc, v);
        warp_sum4(v[0], v[1], v[2], v[3]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int i = i0 + k;
          if (i < n2 && lane == i) pvec = v[k];
          if (i == n2) dd = v[k];
          if (i == n2 + 1) cnt_np = (int)v[k];
        }
      }
      T cvec = T(0);
      T f_prime = -dd;                                                        // :358
      T f_dp = (-theta) * f_prime - warp_sum(pvec * solveM(pvec));            // :362-363
      f_dp = smax(T(1e-12), f_dp);                                            // :364
      const T f_dp_orig = f_dp;
      T dt_min = -f_prime / f_dp;
      T t_old = T(0);
      int ipos, bidx;
      T tcur, db, gb, xb, ub, lb;  // the current breakpoint: t, and d, g, x, upper, lower of its coordinate
      // publish this warp's candidate (t, index) with its coordinate's values; after the barrier every warp folds the
      // W candidates with `better` in warp order.  The owner of a warp's candidate writes it; a warp without one
      // writes index -1.
      auto publish_fold = [&](int iw, T tw, auto better) {
        T* const buf = group_next_buf(rc);
        T* const mine = buf + warp * 8;
        const bool own = (iw >= e0) && (iw < e0 + E);
        if (own) {
          const int e = iw - e0;
          T vd = T(0), vg = T(0), vx = T(0), vu = T(0), vl = T(0);
#pragma unroll
          for (int j = 0; j < E; ++j)
            if (j == e) { vd = dvec[j]; vg = g[j]; vx = x[j]; vu = hi[j]; vl = lo[j]; }
          mine[0] = tw; mine[1] = T(iw); mine[2] = vd; mine[3] = vg; mine[4] = vx; mine[5] = vu; mine[6] = vl;
        } else if (iw < 0 && lane == 0) {
          mine[1] = T(-1);
        }
        group_bar(rc.bar, NT);
        int wb = -1;
        T tb = T(0);
        int ib = -1;
#pragma unroll
        for (int w = 0; w < W; ++w) {
          const int iv = (int)buf[w * 8 + 1];
          const T tv = buf[w * 8];
          if (iv >= 0 && (ib < 0 || better(tv, iv, tb, ib))) { tb = tv; ib = iv; wb = w; }
        }
        const T* const win = buf + wb * 8;
        tcur = tb;
        bidx = ib;
        db = win[2]; gb = win[3]; xb = win[4]; ub = win[5]; lb = win[6];
      };
      auto next_breakpoint = [&]() {  // smallest (t, index) among the positions not yet visited: one barrier
        T best = kMaxValue;
        int bi = 0x7fffffff;
        bool has = false;
#pragma unroll
        for (int e = 0; e < E; ++e)
          if (!done[e] && (!has || tbp[e] < best)) { best = tbp[e]; bi = e0 + e; has = true; }
        T tw;
        const int iw = warp_argmin_pos(best, bi, has, tw);
        publish_fold(iw, tw, [](T tv, int iv, T tb, int ib) { return tv < tb || (tv == tb && iv < ib); });
      };
      if (uni(cnt_np < D)) {
        ipos = cnt_np;
        next_breakpoint();
      } else {
        // no positive t at all: the loop at :371-374 leaves i = dim - 1, the LAST element of the sorted order
        ipos = D - 1;
        T best = -kMaxValue;
        int bi = -1;
#pragma unroll
        for (int e = 0; e < E; ++e)
          if (bi < 0 || tbp[e] >= best) { best = tbp[e]; bi = e0 + e; }
        // lexicographic maximum (t, index): values are <= 0 here; compare as reals
        T vmax = best;
        int imax = bi;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
          const T ov = __shfl_xor_sync(kFullMask, vmax, off);
          const int oi = __shfl_xor_sync(kFullMask, imax, off);
          if (oi >= 0 && (imax < 0 || ov > vmax || (ov == vmax && oi > imax))) { vmax = ov; imax = oi; }
        }
        publish_fold(imax, vmax, [](T tv, int iv, T tb, int ib) { return tv > tb || (tv == tb && iv > ib); });
#pragma unroll
        for (int e = 0; e < E; ++e) done[e] = (e0 + e != bidx);
      }
      T dt = tcur;
      // ---- examination of subsequent segments (:383-416) ----
      while (uni((dt_min >= dt) && (ipos < D))) {
        T xcb = xb;
        if (db > T(0)) xcb = ub;
        else if (db < T(0)) xcb = lb;
        const T zb = xcb - xb;
        cvec = cvec + dt * pvec;                                            // :391
        const T wbt = (lane < n2) ? w_at(bidx, lane) : T(0);                // :393 W_.row(b)
        const T Mc = solveM(cvec), Mp = solveM(pvec), Mw = solveM(wbt);
        f_prime = f_prime + (((dt * f_dp + gb * gb) + (theta * gb) * zb) - warp_sum((gb * wbt) * Mc));          // :397-398
        f_dp = f_dp + (((((T(-1.0) * theta) * gb) * gb) - T(2.0) * (gb * warp_sum(wbt * Mp))) -
                       warp_sum(((gb * gb) * wbt) * Mw));                                                      // :399-401
        f_dp = smax(T(1e-12) * f_dp_orig, f_dp);
        pvec = pvec + gb * wbt;                                              // :403
#pragma unroll
        for (int e = 0; e < E; ++e)
          if (e0 + e == bidx) { dvec[e] = T(0); xc[e] = xcb; done[e] = true; }
        dt_min = -f_prime / f_dp;
        t_old = tcur;
        ++ipos;
        if (uni(ipos < D)) {
          next_breakpoint();
          dt = tcur - t_old;
        }
      }
      dt_min = smax(dt_min, T(0));
      t_old = t_old + dt_min;
#pragma unroll
      for (int e = 0; e < E; ++e)
        if (!done[e]) xc[e] = x[e] + t_old * dvec[e];                        // :429-432
      cvec = cvec + dt_min * pvec;                                           // :434

      // =================== SubspaceMinimization (:477-525) ===================
      bool freev[E];
      int fc = 0;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        freev[e] = (xc[e] != hi[e]) && (xc[e] != lo[e]);
        fc += freev[e] ? 1 : 0;
      }
      // compacted positions: a prefix count in element order (lane l's run, then warp, then element) -- one barrier
      int pos0, nfree;
      {
        T* const buf = group_next_buf(rc);
        buf[lane * W + warp] = T(fc);
        group_bar(rc.bar, NT);
        int run = 0, before = 0;
#pragma unroll
        for (int w = 0; w < W; ++w) {
          const int c = (int)buf[lane * W + w];
          run += c;
          before += (w < warp) ? c : 0;
        }
        int incl = run;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const int o = __shfl_up_sync(kFullMask, incl, off);
          if (lane >= off) incl += o;
        }
        nfree = __shfl_sync(kFullMask, incl, 31);
        pos0 = incl - run + before;
      }
      T xn[E], gn[E];
      T fn_val;
      if (uni(nfree == 0)) {
        // :485-487 the Cauchy point is the minimiser on the active face: evaluate there (:181-183)
#pragma unroll
        for (int e = 0; e < E; ++e) xn[e] = xc[e];
        fn_val = fn(ctx, xn, &gn);
        nfev++;
      } else {
        const T theta_inv = T(1) / theta;
        // rr = g + theta (xc - x) - W (M c)   (:491); r = rr(free)
        const T Mc2 = solveM(cvec);
        T rr[E];
#pragma unroll
        for (int e = 0; e < E; ++e) {
          T acc = T(0);
#pragma unroll 1
          for (int j = 0; j < n2; ++j) {
            const T mj = __shfl_sync(kFullMask, Mc2, j);
            const T pr = w_own(e, j) * mj;
            acc = (j == 0) ? pr : (acc + pr);
          }
          rr[e] = (g[e] + theta * (xc[e] - x[e])) - acc;
        }
        // the compacted vector: all elements (n = d: the ordinary group sum over this thread's own elements), or r and
        // the map staged in the group's shared memory, read back at this thread's compacted positions
        const bool full = uni(nfree == D);
        const int ep = (nfree + 31) / 32;
        int qel[E];  // element at this thread's compacted positions; -1 = a zero term (or an absent position)
        if (full) {
#pragma unroll
          for (int e = 0; e < E; ++e) qel[e] = e0 + e;
        } else {
          int run = pos0;
#pragma unroll
          for (int e = 0; e < E; ++e)
            if (freev[e]) { rstage[run] = rr[e]; cmap[run] = e0 + e; ++run; }
          group_bar(rc.bar, NT);
#pragma unroll
          for (int c = 0; c < E; ++c) {
            const int j = 4 * warp + c, q = lane * ep + j;
            qel[c] = (j < ep && q < nfree) ? cmap[q] : -1;
          }
        }
        T rq[E];
#pragma unroll
        for (int c = 0; c < E; ++c) {
          if (full) rq[c] = rr[c];
          else rq[c] = (qel[c] >= 0) ? rstage[lane * ep + 4 * warp + c] : T(0);
        }
        // (W'Z) r (n2 sums, :496) and (1/theta) W'Z (W'Z)' (n2 x n2 sums, :498): four per round.  Entry (i, j) of the
        // second goes to NN[i + j L2] (lane 0 of each warp), v_i to lane i.
        T vv = T(0);
        const int nsum = n2 + n2 * n2;
#pragma unroll 1
        for (int s0 = 0; s0 < nsum; s0 += 4) {
          T terms[4][E];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int s = s0 + k;
            const int ci = (s < n2) ? s : (s - n2) % (n2 > 0 ? n2 : 1);
            const int cj = (s < n2) ? -1 : (s - n2) / (n2 > 0 ? n2 : 1);
#pragma unroll
            for (int c = 0; c < E; ++c) {
              T tv = T(0);
              if (s < nsum && qel[c] >= 0) {
                const T wi = w_at(qel[c], ci);
                tv = (cj < 0) ? (wi * rq[c]) : ((theta_inv * wi) * w_at(qel[c], cj));
              }
              terms[k][c] = tv;
            }
          }
          T v[4];
          if (full) {
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = lane_tree<T, E>(terms[k]);
            group_lane_partials<4>(rc, v);
          } else {
            group_lane_partials_masked<4>(rc, terms, ep, v);
          }
          warp_sum4(v[0], v[1], v[2], v[3]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int s = s0 + k;
            if (s < n2) {
              if (lane == s) vv = v[k];
            } else if (s < nsum && lane == 0) {
              NN[(s - n2) % n2 + ((s - n2) / n2) * L2] = v[k];
            }
          }
        }
        vv = solveM(vv);
        if (uni(n2 > 0)) {
          // N = I - M N column by column (:500-506), v = N^{-1} v (:509-511)
          __syncwarp();
#pragma unroll 1
          for (int j = 0; j < n2; ++j) {
            const T ncol = (lane < n2) ? NN[lane + j * L2] : T(0);
            const T mn = solveM(ncol);
            __syncwarp();
            if (lane < n2) NN[lane + j * L2] = ((lane == j) ? T(1) : T(0)) - mn;
          }
          lu_factor_warp<L2>(NN, pivN, n2, lane);
          vv = lu_solve_warp<L2>(NN, pivN, n2, vv, lane);
        }
        // du = -(1/theta) r - (1/theta)^2 (W'Z)' v   (:515-516); alpha* (:451-475); subspace_min (:520-524)
        T du[E];
        T amin = T(1);
        const T ti2 = theta_inv * theta_inv;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          T acc = T(0);
#pragma unroll 1
          for (int j = 0; j < n2; ++j) {
            const T vj = __shfl_sync(kFullMask, vv, j);
            const T pr = (ti2 * w_own(e, j)) * vj;
            acc = (j == 0) ? pr : (acc + pr);
          }
          du[e] = ((-theta_inv) * rr[e]) - acc;
          if (freev[e]) {
            const T ad = cabs(du[e]);
            if (!(ad < 1e-7)) {
              const T cand = (du[e] > T(0)) ? ((hi[e] - xc[e]) / du[e]) : ((lo[e] - xc[e]) / du[e]);
              amin = (cand < amin) ? cand : amin;
            }
          }
        }
        // min over lanes, then over warps (a NaN candidate never wins a comparison, in any order)
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
          const T o = __shfl_xor_sync(kFullMask, amin, off);
          amin = (o < amin) ? o : amin;
        }
        amin = group_min_of_warps(rc, amin);
        T dirv[E];
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const T sm = freev[e] ? (xc[e] + amin * du[e]) : xc[e];
          dirv[e] = sm - x[e];   // :174 direction = subspace_min - x
        }
        // ---- LineSearch::Search (:175-176), alpha_init = 1; dginit = g.s (more_thuente.h:151) ----
        const T dginit = warp_sum_p<P, T, E>(lane_dot_p<P, T, E>(g, dirv), rc);
        nfev += LsMoreThuente::template search<Fn, T, E>(fn, ctx, rc, x, f, g, xn, fn_val, gn, T(1), dirv, dginit);
      }
      // ---- :189-193 project the new point; re-evaluate if it moved ----
      {
        T xcl[E];
        if (clip(xn, xcl)) {
#pragma unroll
          for (int e = 0; e < E; ++e) xn[e] = xcl[e];
          fn_val = fn(ctx, xn, &gn);
          nfev++;
        }
      }
      // ---- pair update (:196-228) ----
      T ny[E], ns[E];
#pragma unroll
      for (int e = 0; e < E; ++e) { ny[e] = gn[e] - g[e]; ns[e] = xn[e] - x[e]; }
      T sTy, yy;
      warp_sum2_p<P, T, E>(lane_dot_p<P, T, E>(ns, ny), lane_dot_p<P, T, E>(ny, ny), rc, sTy, yy);
      if (uni(sTy > 1e-7 * yy)) {
        int ps;  // physical slot of the new pair
        if (kp < M) {
          ps = slot(kp);
          kp++;
        } else {
          ps = base;
          base = (base + 1 == M) ? 0 : base + 1;
        }
        GV::store(Ys + ps * D, t, ny);
        GV::store(Ss + ps * D, t, ns);
        theta = yy / sTy;  // :215-216
        // S'Y and S'S entries that involve the new pair, one group round per stored pair.  The barrier of the first
        // round also orders this store before the next read of the new rows by other threads (breakpoints, compacted
        // sums); every such read of the old rows lies before this iteration's line search, whose sums order it before
        // the store.
#pragma unroll 1
        for (int i = 0; i < kp; ++i) {
          const int pi = slot(i);
          T sv[E], yv[E];
          GV::load(Ss + pi * D, t, sv);
          GV::load(Ys + pi * D, t, yv);
          T v[3] = {lane_dot<T, E>(sv, ny), lane_dot<T, E>(ns, yv), lane_dot<T, E>(sv, ns)};
          group_lane_partials<3>(rc, v);
          warp_sum3(v[0], v[1], v[2]);
          if (lane == 0) {
            SY[pi + ps * M] = v[0];   // s_i . y_new
            SY[ps + pi * M] = v[1];   // s_new . y_i
            SSc[pi + ps * M] = v[2];  // s_i . s_new = s_new . s_i (products commute bit for bit)
            SSc[ps + pi * M] = v[2];
          }
        }
        __syncwarp();
        mm_assemble_warp<M>(MM, SY, SSc, theta, kp, base, lane);
        lu_factor_warp<L2>(MM, piv, 2 * kp, lane);
        have_lu = true;
      }

      // =================== Progress::Update + the projected-gradient test (:266-277) ===================
      T sdx[E];
#pragma unroll
      for (int e = 0; e < E; ++e) sdx[e] = xn[e] - xprev[e];
#pragma unroll
      for (int e = 0; e < E; ++e) { x[e] = xn[e]; g[e] = gn[e]; }
      f = fn_val;
      T norms[4] = {warp_maxabs<T, E>(sdx), warp_maxabs<T, E>(g), warp_maxabs<T, E>(x), pg_warp};
      group_max_bits<4>(rc, norms);
      progress_update<T>(prog, stop_nograd, ring, lane, prev_value_state, f, norms[0], norms[1], norms[2]);
      if ((pg_tol > T(0)) && (norms[3] < pg_tol)) prog.status = CNO_STATUS_GRADIENT_NORM_VIOLATION;
    } while (uni(prog.status == CNO_STATUS_CONTINUE));

    if (out.x) store_quad<T>(out.x + b * D + e0, x);
    if (out.gradient) store_quad<T>(out.gradient + b * D + e0, g);
    if (t == 0) store_result_scalars<T>(out, b, f, prog, nfev);
    __syncwarp();
  }
}

}  // namespace cno

#endif  // CNO_LBFGSB_GROUP_CUH_
