// cno_lbfgsb.cuh -- batched Lbfgsb<F, m = 5>::Minimize (box constraints l <= x <= u), one warp per instance, the
// whole overridden Minimize loop in one persistent kernel (sm_90a).
//
// Reference path (include/cppoptlib/solver/lbfgsb.h):
//   :78-81    Lbfgsb() preset (default + f_delta = 2.22e-9 relative)      -> cno_lbfgsb_default_stop
//   :88-92    SetBounds                                                   -> cno_bounds_t
//   :104-116  ProjectedGradientInfNorm
//   :118-136  InitializeSolver (theta = 1, empty W / histories)
//   :138-229  OptimizationStep: clip, Cauchy point, subspace minimisation, line search (MoreThuente), clip,
//             pair update + theta + W + MM = [[-D, L'], [L, theta S'S]] and its LU
//   :238-286  the overridden Minimize loop: projected-gradient stop test on top of Progress::Update
//   :322-446  GetGeneralizedCauchyPoint      :451-475 FindAlpha      :477-525 SubspaceMinimization
//
// Design.  x, g, the Cauchy point and the search direction live in registers (E = ceil(d/32) elements per
// lane); the m-deep (y, s) history (2 x 5 x d) and a compaction buffer live in the warp's shared-memory slice;
// the 2k-vectors of the compact representation (p, c, w_b, v: 2k <= 10 entries) are ONE register per lane (entry i
// in lane i), so their inner products are ordinary warp sums and the (2k x 2k) solves with the LU factors of MM
// run as lane-parallel substitutions (one shuffle broadcast per pivot step).  S'Y and S'S are cached per slot pair
// (the reference recomputes all k^2 dots every update: same operands, same order, same bits).
//
// Arithmetic specification (what oracle/_ref = the reference's own header on the Eigen-API shim computes):
//   * every inner product whose length is d or the number of free variables -- W'd, d.d, S'Y, S'S, (W'Z)r,
//     (W'Z)(W'Z)', y.y, s.y -- follows the reduction specification (lane-blocked partials + tensor-core tree),
//     over the COMPACTED free-variable order where the reference indexes with free_variables_index;
//   * products with a 2k-long inner index (W M c, (W'Z)' v) sum that index ascending from the first product;
//   * the 2k x 2k systems: unblocked partial-pivot LU (first maximal |a_ik|), explicit row swaps, forward and back
//     substitution column by column;
//   * breakpoints are visited in ascending t with ties by ascending index (std::sort leaves the order of exact
//     ties unspecified; see DESIGN.md).
#ifndef CNO_LBFGSB_CUH_
#define CNO_LBFGSB_CUH_

#include "cno_device.cuh"
#include "cno_kernel_params.h"
#include "cno_lbfgs.cuh"  // ProgressState / progress_update
#include "cno_linesearch.cuh"

namespace cno {

template <class T>
struct BoundsArgs {
  const T* lower;    // [d] or [B, d]; nullptr = unbounded below
  const T* upper;    // nullptr = unbounded above
  long long stride;  // 0 = one box for the whole batch, d = per instance
};

template <class T, int D, int M>
struct LbfgsbSmem {
  static constexpr int E = Shape<D>::E;
  static_assert(E <= 4, "Lbfgsb: d <= 128");
  static constexpr int kVec = 32 * E;
  static constexpr int L2 = 2 * M;
  // Y[M][kVec] | S[M][kVec] | scratch[kVec] | MM[L2*L2] | NN[L2*L2] | SY[M*M] | SS[M*M] | ring[MAX_PAST] | piv (ints)
  static constexpr int kSmall = 2 * L2 * L2 + 2 * M * M + CNO_MAX_PAST;
  static constexpr int kPivElems = (2 * L2 * (int)sizeof(int) + (int)sizeof(T) - 1) / (int)sizeof(T);
  static constexpr int kWarpElems = (((2 * M + 1) * kVec + kSmall + kPivElems + 3) / 4) * 4;
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  static constexpr int kFit = (int)((size_t)(227 * 1024) / kWarpBytes);
  static constexpr int kWarps = kFit > 12 ? 12 : (kFit < 1 ? 1 : kFit);
};

// warp minimum of POSITIVE values by (value, index): returns the index of the smallest value, ties to the smaller
// index; `has` = this lane's candidate is valid.  (The bit pattern of a positive double is monotone.)
__device__ __forceinline__ int warp_argmin_pos(double v, int idx, bool has, double& vmin) {
  const unsigned hi = has ? (unsigned)__double2hiint(v) : 0xffffffffu;
  const unsigned H = __reduce_min_sync(kFullMask, hi);
  const unsigned lo = (has && hi == H) ? (unsigned)__double2loint(v) : 0xffffffffu;
  const unsigned Lw = __reduce_min_sync(kFullMask, lo);
  const bool win = has && hi == H && lo == Lw;
  const int I = (int)__reduce_min_sync(kFullMask, win ? (unsigned)idx : 0xffffffffu);
  vmin = __hiloint2double((int)H, (int)Lw);
  return I;
}
__device__ __forceinline__ int warp_argmin_pos(float v, int idx, bool has, float& vmin) {
  const unsigned u = has ? __float_as_uint(v) : 0xffffffffu;
  const unsigned U = __reduce_min_sync(kFullMask, u);
  const int I = (int)__reduce_min_sync(kFullMask, (has && u == U) ? (unsigned)idx : 0xffffffffu);
  vmin = __uint_as_float(U);
  return I;
}

template <class Fn, int M = 5, class LS = LsMoreThuente>
__global__ void __launch_bounds__(LbfgsbSmem<typename Fn::Scalar, Fn::Dim, M>::kWarps * 32, 1)
lbfgsb_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0, const long long batch,
                       const StopParams<typename Fn::Scalar> stop, const BatchOut<typename Fn::Scalar> out,
                       unsigned long long* __restrict__ queue, const BoundsArgs<typename Fn::Scalar> bounds) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  constexpr int E = Shape<D>::E;
  using SM = LbfgsbSmem<T, D, M>;
  constexpr int L2 = SM::L2;
  constexpr int kVec = SM::kVec;
  constexpr T kMaxValue = sizeof(T) == 8 ? (T)1.7976931348623157e308 : (T)3.4028234663852886e38f;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T* const Ys = reinterpret_cast<T*>(smem_raw) + (size_t)warp * SM::kWarpElems;
  T* const Ss = Ys + M * kVec;
  T* const scratch = Ss + M * kVec;
  T* const MM = scratch + kVec;   // LU factors of MM, column-major, leading dimension L2
  T* const NN = MM + L2 * L2;
  T* const SY = NN + L2 * L2;     // SY[pi + pj*M] = s_pi . y_pj  (physical slots)
  T* const SSc = SY + M * M;      // SSc[pi + pj*M] = s_pi . s_pj
  T* const ring = SSc + M * M;
  int* const piv = reinterpret_cast<int*>(ring + CNO_MAX_PAST);  // row exchanged with k at step k: MM, then NN
  int* const pivN = piv + L2;
  const RedCtx<T> rc{nullptr, lane};

  // ---- lane-blocked vectors in shared memory (element i at index i) ----
  auto ld_vec = [&](const T* base, T (&v)[E]) {
#pragma unroll
    for (int e = 0; e < E; ++e) v[e] = base[lane * E + e];
  };
  auto st_vec = [&](T* base, const T (&v)[E]) {
#pragma unroll
    for (int e = 0; e < E; ++e) base[lane * E + e] = v[e];
  };
  auto wdot = [&](const T (&a)[E], const T (&b)[E]) -> T { return warp_sum(lane_dot<T, E>(a, b)); };

  // ---- (n x n) LU of a column-major matrix in shared memory: the shim's / Eigen's partial-pivot elimination ----
  auto lu_factor = [&](T* A, int* pv, int n) {
#pragma unroll 1
    for (int k = 0; k < n; ++k) {
      __syncwarp();
      T best = cabs(A[k + k * L2]);
      int p = k;
#pragma unroll 1
      for (int i = k + 1; i < n; ++i) {  // first maximal |a_ik| (uniform scan: n <= 10)
        const T v = cabs(A[i + k * L2]);
        if (uni(v > best)) { best = v; p = i; }
      }
      if (lane == 0) pv[k] = p;
      if (uni(p != k)) {
        if (lane < n) {
          const T a = A[k + lane * L2], b2 = A[p + lane * L2];
          A[k + lane * L2] = b2;
          A[p + lane * L2] = a;
        }
        __syncwarp();
      }
      const T pivot = A[k + k * L2];
      const bool below = (lane > k) && (lane < n);
      T lik = T(0);
      if (below) {
        lik = A[lane + k * L2] / pivot;
        A[lane + k * L2] = lik;
      }
#pragma unroll 1
      for (int j = k + 1; j < n; ++j) {
        const T akj = A[k + j * L2];
        if (below) A[lane + j * L2] = A[lane + j * L2] - lik * akj;
      }
    }
    __syncwarp();
  };
  // solve with the factors: rhs entry i in lane i (i < n); returns the solution in the same convention
  auto lu_solve = [&](const T* A, const int* pv, int n, T r) -> T {
#pragma unroll 1
    for (int k = 0; k < n; ++k) {
      const int p = pv[k];
      if (uni(p != k)) {
        const int src = (lane == k) ? p : ((lane == p) ? k : lane);
        r = __shfl_sync(kFullMask, r, src);
      }
    }
#pragma unroll 1
    for (int k = 0; k < n; ++k) {
      const T bk = __shfl_sync(kFullMask, r, k);
      if (lane > k && lane < n) r = r - A[lane + k * L2] * bk;
    }
#pragma unroll 1
    for (int k = n - 1; k >= 0; --k) {
      const T akk = A[k + k * L2];
      if (lane == k) r = r / akk;
      const T xk = __shfl_sync(kFullMask, r, k);
      if (lane < k) r = r - A[lane + k * L2] * xk;
    }
    return (lane < n) ? r : T(0);
  };

  for (;;) {
    unsigned long long b = 0;
    if (lane == 0) b = atomicAdd(queue, 1ULL);
    b = __shfl_sync(kFullMask, b, 0);
    if (uni(b >= (unsigned long long)batch)) break;
    const EvalCtx ctx{lane, (long long)b, nullptr};

    // ---- the box (:88-92; defaults of InitializeSolver :122-128) ----
    T lo[E], hi[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int i = lane * E + e;
      lo[e] = (bounds.lower && i < D) ? bounds.lower[b * bounds.stride + i] : -kMaxValue;
      hi[e] = (bounds.upper && i < D) ? bounds.upper[b * bounds.stride + i] : kMaxValue;
    }
    auto clip = [&](const T (&v)[E], T (&o)[E]) -> bool {  // cwiseMin(upper).cwiseMax(lower); true if it changed v
      bool changed = false;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const T a = (hi[e] < v[e]) ? hi[e] : v[e];
        o[e] = (a < lo[e]) ? lo[e] : a;
        changed = changed || ((lane * E + e < D) && (o[e] != v[e]));
      }
      return uni(changed);
    };

    T x[E], g[E];
    load_row<T, D>(x0 + b * D, lane, x);
    T f = fn(ctx, x, &g);  // :246 StateType current_function_state(function, function_state.x)
    uint32_t nfev = 1;

    // ---- InitializeSolver (:118-136) ----
    T theta = T(1);
    int kp = 0;    // pairs stored
    int base = 0;  // physical slot of the oldest pair
    bool have_lu = false;
    auto slot = [&](int i) -> int { const int s2 = base + i; return s2 >= M ? s2 - M : s2; };

    ProgressState<T> prog;
    prog.num_iterations = 0;
    prog.x_delta_violations = 0;
    prog.f_delta_violations = 0;
    prog.x_delta = prog.f_delta = prog.gradient_norm = T(0);
    prog.ring_size = 0;
    prog.ring_pos = 0;
    prog.status = CNO_STATUS_NOT_STARTED;
    StopParams<T> stop_nograd = stop;  // :254-256: the base class's full-gradient test is suppressed
    stop_nograd.gradient_norm = T(0);
    const T pg_tol = stop.gradient_norm;

    do {  // :260-278
      // =================== OptimizationStep (:138-229) ===================
      // W = [Y, theta S]: entry (row, col i) for i < 2k
      const int n2 = 2 * kp;
      auto w_entry = [&](int row, int i) -> T {
        return (i < kp) ? Ys[slot(i) * kVec + row] : (theta * Ss[slot(i - kp) * kVec + row]);
      };
      auto solveM = [&](T r) -> T { return (have_lu && n2 > 0) ? lu_solve(MM, piv, n2, r) : r; };  // :311-316

      // ---- :145-150 project the iterate; re-evaluate if it moved ----
      T xcur[E];
      const T prev_value_state = f;
      T xprev[E];
#pragma unroll
      for (int e = 0; e < E; ++e) xprev[e] = x[e];
      if (clip(x, xcur)) {
#pragma unroll
        for (int e = 0; e < E; ++e) x[e] = xcur[e];
        f = fn(ctx, x, &g);
        nfev++;
      }
      // ---- :162-163 projected-gradient norm at the (projected) iterate; std::max drops a NaN ----
      T pgv[E];
#pragma unroll
      for (int e = 0; e < E; ++e) {
        T gj = g[e];
        if (x[e] <= lo[e] && gj > T(0)) gj = T(0);
        if (x[e] >= hi[e] && gj < T(0)) gj = T(0);
        const T a = cabs(gj);
        pgv[e] = (a != a) ? T(0) : a;
      }
      const T last_pg = warp_maxabs<T, E>(pgv);

      // =================== GetGeneralizedCauchyPoint (:322-446) ===================
      T dvec[E], tbp[E], xc[E];
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const int i = lane * E + e;
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
        if (i >= D) { dvec[e] = T(0); tbp[e] = kMaxValue; }
      }
      // p = W'd (:354), one entry per lane
      T pvec = T(0);
#pragma unroll 1
      for (int i = 0; i < n2; ++i) {
        T wcol[E];
#pragma unroll
        for (int e = 0; e < E; ++e) wcol[e] = w_entry(lane * E + e, i);
        const T v = wdot(wcol, dvec);
        if (lane == i) pvec = v;
      }
      T cvec = T(0);
      T f_prime = -wdot(dvec, dvec);                                          // :358
      T f_dp = (-theta) * f_prime - warp_sum(pvec * solveM(pvec));            // :362-363
      f_dp = smax(T(1e-12), f_dp);                                            // :364
      const T f_dp_orig = f_dp;
      T dt_min = -f_prime / f_dp;
      T t_old = T(0);
      // sorted order = ascending t, ties by index.  `done` = positions before the current one.
      bool done[E];
      int cnt_np = 0;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        done[e] = (lane * E + e < D) && !(tbp[e] > T(0));
        cnt_np += done[e] ? 1 : 0;
      }
      cnt_np = (int)__reduce_add_sync(kFullMask, (unsigned)cnt_np);
      int ipos, bidx;
      T tcur;
      auto next_breakpoint = [&](T& tval) -> int {  // smallest (t, index) among the positions not yet visited
        T best = kMaxValue;
        int bi = 0x7fffffff;
        bool has = false;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int i = lane * E + e;
          if (i < D && !done[e] && (!has || tbp[e] < best)) { best = tbp[e]; bi = i; has = true; }
        }
        return warp_argmin_pos(best, bi, has, tval);
      };
      if (uni(cnt_np < D)) {
        ipos = cnt_np;
        bidx = next_breakpoint(tcur);
      } else {
        // no positive t at all: the loop at :371-374 leaves i = dim - 1, the LAST element of the sorted order
        ipos = D - 1;
        T best = -kMaxValue;
        int bi = -1;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int i = lane * E + e;
          if (i < D && (bi < 0 || tbp[e] >= best)) { best = tbp[e]; bi = i; }
        }
        // lexicographic maximum (t, index) across lanes: values are <= 0 here; compare as reals
        T vmax = best;
        int imax = bi;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
          const T ov = __shfl_xor_sync(kFullMask, vmax, off);
          const int oi = __shfl_xor_sync(kFullMask, imax, off);
          if (oi >= 0 && (imax < 0 || ov > vmax || (ov == vmax && oi > imax))) { vmax = ov; imax = oi; }
        }
        bidx = imax;
        tcur = vmax;
#pragma unroll
        for (int e = 0; e < E; ++e) done[e] = (lane * E + e != bidx);
      }
      T dt = tcur;
      // ---- examination of subsequent segments (:383-416) ----
      while (uni((dt_min >= dt) && (ipos < D))) {
        const int bl = bidx / E, be = bidx % E;
        // values of coordinate b, broadcast from its owner
        T db = T(0), gb = T(0), xb = T(0), ub = T(0), lb = T(0);
#pragma unroll
        for (int e = 0; e < E; ++e)
          if (be == e) { db = dvec[e]; gb = g[e]; xb = x[e]; ub = hi[e]; lb = lo[e]; }
        db = __shfl_sync(kFullMask, db, bl);
        gb = __shfl_sync(kFullMask, gb, bl);
        xb = __shfl_sync(kFullMask, xb, bl);
        ub = __shfl_sync(kFullMask, ub, bl);
        lb = __shfl_sync(kFullMask, lb, bl);
        T xcb = xb;
        if (db > T(0)) xcb = ub;
        else if (db < T(0)) xcb = lb;
        const T zb = xcb - xb;
        cvec = cvec + dt * pvec;                                            // :391
        const T wbt = (lane < n2) ? w_entry(bidx, lane) : T(0);             // :393 W_.row(b)
        const T Mc = solveM(cvec), Mp = solveM(pvec), Mw = solveM(wbt);
        f_prime = f_prime + (((dt * f_dp + gb * gb) + (theta * gb) * zb) - warp_sum((gb * wbt) * Mc));          // :397-398
        f_dp = f_dp + (((((T(-1.0) * theta) * gb) * gb) - T(2.0) * (gb * warp_sum(wbt * Mp))) -
                       warp_sum(((gb * gb) * wbt) * Mw));                                                      // :399-401
        f_dp = smax(T(1e-12) * f_dp_orig, f_dp);
        pvec = pvec + gb * wbt;                                              // :403
#pragma unroll
        for (int e = 0; e < E; ++e)
          if (lane * E + e == bidx) { dvec[e] = T(0); xc[e] = xcb; done[e] = true; }
        dt_min = -f_prime / f_dp;
        t_old = tcur;
        ++ipos;
        if (uni(ipos < D)) {
          bidx = next_breakpoint(tcur);
          dt = tcur - t_old;
        }
      }
      dt_min = smax(dt_min, T(0));
      t_old = t_old + dt_min;
#pragma unroll
      for (int e = 0; e < E; ++e)
        if (lane * E + e < D && !done[e]) xc[e] = x[e] + t_old * dvec[e];   // :429-432
      cvec = cvec + dt_min * pvec;                                           // :434

      // =================== SubspaceMinimization (:477-525) ===================
      bool freev[E];
      int fc = 0;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        freev[e] = (lane * E + e < D) && (xc[e] != hi[e]) && (xc[e] != lo[e]);
        fc += freev[e] ? 1 : 0;
      }
      int incl = fc;  // inclusive prefix sum over lanes
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(kFullMask, incl, off);
        if (lane >= off) incl += o;
      }
      const int nfree = __shfl_sync(kFullMask, incl, 31);
      int pos[E];
      {
        int run = incl - fc;
#pragma unroll
        for (int e = 0; e < E; ++e) { pos[e] = run; run += freev[e] ? 1 : 0; }
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
        // reduction over the free variables in their compacted order
        auto cred = [&](const T (&term)[E]) -> T {
          if (uni(nfree == D)) {
            T t2[E];
#pragma unroll
            for (int e = 0; e < E; ++e) t2[e] = term[e];
            return warp_sum(lane_tree<T, E>(t2));
          }
          __syncwarp();
#pragma unroll
          for (int e = 0; e < E; ++e)
            if (freev[e]) scratch[pos[e]] = term[e];
          __syncwarp();
          const int Ep = (nfree + 31) / 32;
          T v[E];
#pragma unroll
          for (int j = 0; j < E; ++j) {
            const int i = lane * Ep + j;
            v[j] = (j < Ep && i < nfree) ? scratch[i] : T(0);
          }
          T part = v[0];
          if constexpr (E >= 2) {
            if (Ep == 2) part = v[0] + v[1];
          }
          if constexpr (E >= 3) {
            if (Ep == 3) part = (v[0] + v[1]) + v[2];
          }
          if constexpr (E >= 4) {
            if (Ep == 4) part = (v[0] + v[1]) + (v[2] + v[3]);
          }
          return warp_sum(part);
        };
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
            const T pr = w_entry(lane * E + e, j) * mj;
            acc = (j == 0) ? pr : (acc + pr);
          }
          rr[e] = (g[e] + theta * (xc[e] - x[e])) - acc;
        }
        // v = M (W'Z r)   (:496)
        T vv = T(0);
#pragma unroll 1
        for (int i = 0; i < n2; ++i) {
          T term[E];
#pragma unroll
          for (int e = 0; e < E; ++e) term[e] = freev[e] ? (w_entry(lane * E + e, i) * rr[e]) : T(0);
          const T s2 = cred(term);
          if (lane == i) vv = s2;
        }
        vv = solveM(vv);
        if (uni(n2 > 0)) {
          // N = (1/theta) W'Z (W'Z)'  (:498), then N = I - M N column by column (:500-506), v = N^{-1} v (:509-511)
#pragma unroll 1
          for (int j = 0; j < n2; ++j) {
            T ncol = T(0);
#pragma unroll 1
            for (int i = 0; i < n2; ++i) {
              T term[E];
#pragma unroll
              for (int e = 0; e < E; ++e)
                term[e] = freev[e] ? ((theta_inv * w_entry(lane * E + e, i)) * w_entry(lane * E + e, j)) : T(0);
              const T s2 = cred(term);
              if (lane == i) ncol = s2;
            }
            const T mn = solveM(ncol);
            if (lane < n2) NN[lane + j * L2] = ((lane == j) ? T(1) : T(0)) - mn;
          }
          lu_factor(NN, pivN, n2);
          vv = lu_solve(NN, pivN, n2, vv);
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
            const T pr = (ti2 * w_entry(lane * E + e, j)) * vj;
            acc = (j == 0) ? pr : (acc + pr);
          }
          du[e] = ((-theta_inv) * rr[e]) - acc;
          if (freev[e]) {
            const T ad = cabs(du[e]);
            bool skip;
            if constexpr (sizeof(T) == 8) skip = ad < 1e-7; else skip = (double)ad < 1e-7;
            if (!skip) {
              const T cand = (du[e] > T(0)) ? ((hi[e] - xc[e]) / du[e]) : ((lo[e] - xc[e]) / du[e]);
              amin = (cand < amin) ? cand : amin;
            }
          }
        }
        // min over lanes (a NaN candidate never wins a comparison, in any order)
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
          const T o = __shfl_xor_sync(kFullMask, amin, off);
          amin = (o < amin) ? o : amin;
        }
        T dirv[E];
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const T sm = freev[e] ? (xc[e] + amin * du[e]) : xc[e];
          dirv[e] = (lane * E + e < D) ? (sm - x[e]) : T(0);   // :174 direction = subspace_min - x
        }
        // ---- LineSearch::Search (:175-176), alpha_init = 1; dginit = g.s (more_thuente.h:151) ----
        const T dginit = wdot(g, dirv);
        nfev += LS::template search<Fn, T, E>(fn, ctx, rc, x, f, g, xn, fn_val, gn, T(1), dirv, dginit);
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
      T sTy = lane_dot<T, E>(ns, ny), yy = lane_dot<T, E>(ny, ny);
      warp_sum2(sTy, yy);
      bool accept;
      if constexpr (sizeof(T) == 8) accept = sTy > 1e-7 * yy; else accept = (double)sTy > 1e-7 * (double)yy;
      if (uni(accept)) {
        int ps;  // physical slot of the new pair
        if (kp < M) {
          ps = slot(kp);
          kp++;
        } else {
          ps = base;
          base = (base + 1 == M) ? 0 : base + 1;
        }
        __syncwarp();
        st_vec(Ys + ps * kVec, ny);
        st_vec(Ss + ps * kVec, ns);
        __syncwarp();
        theta = yy / sTy;  // :215-216
        // S'Y and S'S entries that involve the new pair (the others are unchanged: same operands, same bits)
#pragma unroll 1
        for (int i = 0; i < kp; ++i) {
          const int pi = slot(i);
          T sv[E], yv[E];
          ld_vec(Ss + pi * kVec, sv);
          ld_vec(Ys + pi * kVec, yv);
          T a1 = lane_dot<T, E>(sv, ny), a2 = lane_dot<T, E>(ns, yv), a3 = lane_dot<T, E>(sv, ns);
          warp_sum3(a1, a2, a3);
          if (lane == 0) {
            SY[pi + ps * M] = a1;   // s_i . y_new
            SY[ps + pi * M] = a2;   // s_new . y_i
            SSc[pi + ps * M] = a3;  // s_i . s_new = s_new . s_i (products commute bit for bit)
            SSc[ps + pi * M] = a3;
          }
        }
        __syncwarp();
        // MM = [[D, L'], [L, theta S'S]], D = -1 * diag(S'Y) as a matrix (off-diagonal -0), L = strictly lower S'Y
        const int n = 2 * kp;
        if (lane < n) {
#pragma unroll 1
          for (int j = 0; j < n; ++j) {
            const int i = lane;
            T v;
            if (i < kp && j < kp) v = (i == j) ? (T(-1) * SY[slot(i) + slot(i) * M]) : (T(-1) * T(0));
            else if (i < kp) v = (j - kp > i) ? SY[slot(j - kp) + slot(i) * M] : T(0);            // L'(i, j-kp) = L(j-kp, i)
            else if (j < kp) v = (i - kp > j) ? SY[slot(i - kp) + slot(j) * M] : T(0);            // L(i-kp, j)
            else v = SSc[slot(i - kp) + slot(j - kp) * M] * theta;
            MM[i + j * L2] = v;
          }
        }
        lu_factor(MM, piv, n);
        have_lu = true;
      }

      // =================== Progress::Update + the projected-gradient test (:266-277) ===================
      T sdx[E];
#pragma unroll
      for (int e = 0; e < E; ++e) sdx[e] = xn[e] - xprev[e];
      const T x_delta = warp_maxabs<T, E>(sdx);
#pragma unroll
      for (int e = 0; e < E; ++e) { x[e] = xn[e]; g[e] = gn[e]; }
      f = fn_val;
      const T gnorm_inf = warp_maxabs<T, E>(g);
      const T x_inf = warp_maxabs<T, E>(x);
      progress_update<T>(prog, stop_nograd, ring, lane, prev_value_state, f, x_delta, gnorm_inf, x_inf);
      if ((pg_tol > T(0)) && (last_pg < pg_tol)) prog.status = CNO_STATUS_GRADIENT_NORM_VIOLATION;
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

#endif  // CNO_LBFGSB_CUH_
