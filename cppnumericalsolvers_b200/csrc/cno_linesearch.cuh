// cno_linesearch.cuh -- MoreThuente strong-Wolfe line search, one warp per
// instance, fused with the user's device functor (trial points never leave
// registers: 0 HBM bytes per trial).
//
// Mirrors linesearch/more_thuente.h of the reference:
//   cstep   :261-407  (scalar, warp-uniform: every lane computes the same bits)
//   cvsrch  :137-256
//   Search(State...) :120-135
// including the quirks that shape trajectories (SURVEY.md 7.2 c-f): evaluation
// at the returned step even on failure, info codes 6,5,4,3,2,1 assigned in that
// order, cstep's early "return -1" leaving infoc = 0, cstep receiving the
// loop-local stmin/stmax.
#ifndef CNO_LINESEARCH_CUH_
#define CNO_LINESEARCH_CUH_

#include "cno_device.cuh"

namespace cno {

#ifdef CNO_LBFGS_PHASE_CLOCKS
// Phase probe of lbfgs_minimize_kernel (cno_lbfgs.cuh, measurement builds only): clock64() once the search's first
// trial has been decided, one slot per warp of the CTA, written by lane 0.
__shared__ long long cno_ls_first_trial_clock[32];
#define CNO_LS_FIRST_TRIAL_CLOCK(nfev) \
  if ((nfev) == 1 && (threadIdx.x & 31) == 0) cno_ls_first_trial_clock[threadIdx.x >> 5] = clock64()
#else
#define CNO_LS_FIRST_TRIAL_CLOCK(nfev)
#endif

template <class T>
__device__ __forceinline__ T max_abs3(T x, T y, T z) {  // more_thuente.h:409-411
  return smax(cabs(x), smax(cabs(y), cabs(z)));
}

// more_thuente.h:261-407
template <class T>
__device__ __forceinline__ int cstep(T& stx, T& fx, T& dx, T& sty, T& fy, T& dy,
                                  T& stp, T fp, T dp, bool& brackt, T stpmin,
                                  T stpmax, int& info) {
  info = 0;
  bool bound = false;

  if (uni((brackt && ((stp <= smin(stx, sty)) || (stp >= smax(stx, sty)))) ||
          (dx * (stp - stx) >= T(0)) || (stpmax < stpmin))) {
    return -1;
  }

  const T sgnd = dp * (dx / cabs(dx));

  T stpf = 0, stpc = 0, stpq = 0;

  if (uni(fp > fx)) {
    info = 1;
    bound = true;
    const T theta = T(3) * (fx - fp) / (stp - stx) + dx + dp;
    const T s = max_abs3(theta, dx, dp);
    T gamma = s * csqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
    if (stp < stx) gamma = -gamma;
    const T p = (gamma - dx) + theta;
    const T q = ((gamma - dx) + gamma) + dp;
    const T r = p / q;
    stpc = stx + r * (stp - stx);
    stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / T(2)) * (stp - stx);
    stpf = (cabs(stpc - stx) < cabs(stpq - stx)) ? stpc : (stpc + (stpq - stpc) / 2);
    brackt = true;
  } else if (uni(sgnd < T(0))) {
    info = 2;
    bound = false;
    const T theta = 3 * (fx - fp) / (stp - stx) + dx + dp;
    const T s = max_abs3(theta, dx, dp);
    T gamma = s * csqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
    if (stp > stx) gamma = -gamma;
    const T p = (gamma - dp) + theta;
    const T q = ((gamma - dp) + gamma) + dx;
    const T r = p / q;
    stpc = stp + r * (stx - stp);
    stpq = stp + (dp / (dp - dx)) * (stx - stp);
    stpf = (cabs(stpc - stp) > cabs(stpq - stp)) ? stpc : stpq;
    brackt = true;
  } else if (uni(cabs(dp) < cabs(dx))) {
    info = 3;
    bound = true;
    const T theta = 3 * (fx - fp) / (stp - stx) + dx + dp;
    const T s = max_abs3(theta, dx, dp);
    T gamma = s * csqrt(smax(T(0.), (theta / s) * (theta / s) - (dx / s) * (dp / s)));
    if (stp > stx) gamma = -gamma;
    const T p = (gamma - dp) + theta;
    const T q = (gamma + (dx - dp)) + gamma;
    const T r = p / q;
    stpc = ((r < T(0)) & (gamma != T(0))) ? (stp + r * (stx - stp))
                                          : ((stp > stx) ? stpmax : stpmin);
    stpq = stp + (dp / (dp - dx)) * (stx - stp);
    if (brackt) {
      stpf = (cabs(stp - stpc) < cabs(stp - stpq)) ? stpc : stpq;
    } else {
      stpf = (cabs(stp - stpc) > cabs(stp - stpq)) ? stpc : stpq;
    }
  } else {
    info = 4;
    bound = false;
    if (uni(brackt)) {
      const T theta = 3 * (fp - fy) / (sty - stp) + dy + dp;
      const T s = max_abs3(theta, dy, dp);
      T gamma = s * csqrt((theta / s) * (theta / s) - (dy / s) * (dp / s));
      if (stp > sty) gamma = -gamma;
      const T p = (gamma - dp) + theta;
      const T q = ((gamma - dp) + gamma) + dy;
      const T r = p / q;
      stpc = stp + r * (sty - stp);
      stpf = stpc;
    } else {
      stpf = (stp > stx) ? stpmax : stpmin;
    }
  }

  {  // :377-391 as selects (no control flow)
    const bool up = fp > fx;
    const bool flip = !up && (sgnd < T(0));
    const T nsty = up ? stp : (flip ? stx : sty);
    const T nfy = up ? fp : (flip ? fx : fy);
    const T ndy = up ? dp : (flip ? dx : dy);
    stx = up ? stx : stp;
    fx = up ? fx : fp;
    dx = up ? dx : dp;
    sty = nsty;
    fy = nfy;
    dy = ndy;
  }

  stpf = sclamp(stpf, stpmin, stpmax);
  stp = stpf;

  if (brackt & bound) {
    const T lim = stx + T(0.66) * (sty - stx);
    stp = (sty > stx) ? smin(lim, stp) : smax(lim, stp);
  }
  return 0;
}

// more_thuente.h:137-256 fused with Search(State...) :120-135.
// x0/g0/f0 = the start state (the reference's `wa` and the copies made at
// :125-129), s = the direction, dginit = g0.s (the caller already has it: for
// L-BFGS it equals the descent-test value bit for bit because negation commutes
// with rounding).  On exit x/g/f hold the last evaluated point exactly as in the
// reference; when dginit >= 0 the search returns at once (:152-156) and
// x/g/f = x0/g0/f0.  Returns the number of objective evaluations.
// kNeg: the search direction is -s (the caller passes q of an L-BFGS step instead of a materialised
// -q): x = x0 - stp*s and g.(-s) with the negation folded into the products -- the same bits as a
// search along a stored -s, without the negation pass and its registers.  kChecked: the caller has
// already taken the dginit >= 0 early return (so the start state is not copied speculatively).
template <class P, bool kNeg, class T, int E>
__device__ __forceinline__ typename LanePartial<P, T, E>::type ls_dir_dot(const T (&g)[E], const T (&s)[E]) {
  if constexpr (kNeg) return lane_dot_neg_p<P, T, E>(g, s);
  else return lane_dot_p<P, T, E>(g, s);
}
// f(x0 +- stp*s) and g.(+-s): the trial point of every line search (more_thuente.h:198-201,
// hager_zhang.h:152-159), f and the slope reduced together when the functor exposes its partial.
// RC: the reduction context -- RedCtx<T> of the one-warp kernels, or the group context of a kernel in which several
// warps share one instance (cno_lbfgs_group.cuh); warp_sum_p / warp_sum2_p are overloaded on it.  Ctx: the context
// the functor is called with -- EvalCtx, or GroupEvalCtx<W> in the group kernel.
template <bool kNeg, class Fn, class T, int E, class Ctx, class RC>
__device__ __forceinline__ void ls_eval(const Fn& fn, const Ctx& ctx, const RC& rc, const T (&x0)[E],
                                        const T stp, const T (&s)[E], T (&x)[E], T& f, T (&g)[E], T& dg) {
  using P = typename PolicyOf<Fn>::type;
#pragma unroll
  for (int j = 0; j < E; ++j) x[j] = kNeg ? (x0[j] - stp * s[j]) : (x0[j] + stp * s[j]);
  if constexpr (FnHasPartial<Fn>::value) {
    const auto pf = fn.partial(ctx, x, &g);
    warp_sum2_p<P, T, E>(pf, ls_dir_dot<P, kNeg, T, E>(g, s), rc, f, dg);
  } else {
    f = fn(ctx, x, &g);
    dg = warp_sum_p<P, T, E>(ls_dir_dot<P, kNeg, T, E>(g, s), rc);
  }
}

template <class Fn, class T, int E, bool kNeg = false, bool kChecked = false, class Ctx, class RC>
__device__ __forceinline__ int cvsrch(const Fn& fn, const Ctx& ctx, const RC& rc, const T (&x0)[E],
                                      const T f0, const T (&g0)[E], T (&x)[E], T& f,
                                      T (&g)[E], T stp, const T (&s)[E], const T dginit) {
  int info = 0;
  int infoc = 1;
  const T xtol = T(1e-15);
  const T ftol = T(1e-4);
  const T gtol = T(0.9);
  const T stpmin = T(1e-15);
  const T stpmax = T(1e15);
  const T xtrapf = T(4);
  const int maxfev = 20;
  int nfev = 0;

  if constexpr (!kChecked) {
    if (uni(dginit >= T(0))) {  // :152-156 (state untouched)
#pragma unroll
      for (int j = 0; j < E; ++j) { x[j] = x0[j]; g[j] = g0[j]; }
      f = f0;
      return 0;
    }
  }

  bool brackt = false;
  bool stage1 = true;

  const T finit = f0;
  const T dgtest = ftol * dginit;
  T width = stpmax - stpmin;
  T width1 = T(2) * width;

  T stx = T(0), fx = finit, dgx = dginit;
  T sty = T(0), fy = finit, dgy = dginit;

  for (;;) {
    T stmin, stmax;
    if (brackt) {
      stmin = smin(stx, sty);
      stmax = smax(stx, sty);
    } else {
      stmin = stx;
      stmax = stp + xtrapf * (stp - stx);
    }
    stp = sclamp(stp, stpmin, stpmax);
    if ((brackt && ((stp <= stmin) || (stp >= stmax))) || (nfev >= maxfev - 1) ||
        (infoc == 0) || (brackt && ((stmax - stmin) <= (xtol * stmax)))) {
      stp = stx;
    }

    T dg;
    ls_eval<kNeg, Fn, T, E>(fn, ctx, rc, x0, stp, s, x, f, g, dg);  // :198-201
    nfev++;
    const T ftest1 = finit + stp * dgtest;

    if ((brackt & ((stp <= stmin) | (stp >= stmax))) | (infoc == 0)) info = 6;
    if ((stp == stpmax) & (f <= ftest1) & (dg <= dgtest)) info = 5;
    if ((stp == stpmin) & ((f > ftest1) | (dg >= dgtest))) info = 4;
    if (nfev >= maxfev) info = 3;
    if (brackt & (stmax - stmin <= xtol * stmax)) info = 2;
    if ((f <= ftest1) & (cabs(dg) <= gtol * (-dginit))) info = 1;

    CNO_LS_FIRST_TRIAL_CLOCK(nfev);
    if (uni(info != 0)) return nfev;  // :219

    if (stage1 & (f <= ftest1) & (dg >= smin(ftol, gtol) * dginit)) stage1 = false;

    // :225-244 with ONE cstep call site: the modified-function values are formed
    // and undone by selects (x - 0 and x + 0 are exact, but selects keep even
    // the sign of zero identical to the reference's two branches).
    const bool mod = stage1 & (f <= fx) & (f > ftest1);
    T a_fx = mod ? (fx - stx * dgtest) : fx;
    T a_fy = mod ? (fy - sty * dgtest) : fy;
    T a_dx = mod ? (dgx - dgtest) : dgx;
    T a_dy = mod ? (dgy - dgtest) : dgy;
    const T a_fp = mod ? (f - stp * dgtest) : f;
    const T a_dp = mod ? (dg - dgtest) : dg;
    cstep<T>(stx, a_fx, a_dx, sty, a_fy, a_dy, stp, a_fp, a_dp, brackt, stmin, stmax, infoc);
    fx = mod ? (a_fx + stx * dgtest) : a_fx;
    fy = mod ? (a_fy + sty * dgtest) : a_fy;
    dgx = mod ? (a_dx + dgtest) : a_dx;
    dgy = mod ? (a_dy + dgtest) : a_dy;

    if (brackt) {
      if (cabs(sty - stx) >= T(0.66) * width1) stp = stx + T(0.5) * (sty - stx);
      width1 = width;
      width = cabs(sty - stx);
    }
  }
}

// ---- HagerZhang (linesearch/hager_zhang.h:54-552), the alternative LineSearch policy ----
//
// The reference keeps every sample (alpha, phi, dphi) in a std::vector and passes
// indices around.  Only three samples are ever live -- the bracket ends a, b and the
// newest one -- plus, during the bracket phase, "the most recent earlier sample with
// phi <= phi_lim" (what the backward scan at :366-371 finds).  They are kept here as
// value tuples in registers, each carrying the index it would have in the reference's
// vector so that the index comparisons of Secant2 (:253-254) stay exact.  Control flow
// is warp-uniform (every lane holds the same scalars) and voted through uni().
// State: the last evaluated point (xa, gx) and the best-sample copy (best_x, best_g)
// of :318-329, E registers per lane each.
template <class T>
struct HzSample {
  T alpha, phi, dphi;
  int id;
};

template <class Fn, class T, int E, bool kNeg = false>
struct HzSearch {
  using P = typename PolicyOf<Fn>::type;
  const Fn& fn;
  const EvalCtx& ctx;
  const RedCtx<T>& rc;
  const T (&x0)[E];
  const T (&s)[E];
  T (&xa)[E];  // last evaluated point
  T (&gx)[E];  // its gradient
  T phi_0, dphi_0, phi_lim, delta, sigma;
  int n;     // history.size()
  int nfev;

  // PhiDphi (:152-159) + history.push_back
  __device__ __forceinline__ HzSample<T> eval(T alpha) {
    HzSample<T> r;
    r.alpha = alpha;
    ls_eval<kNeg, Fn, T, E>(fn, ctx, rc, x0, alpha, s, xa, r.phi, gx, r.dphi);
    r.id = -1;
    nfev++;
    return r;
  }
  __device__ __forceinline__ void push(HzSample<T>& r) { r.id = n++; }

  // SatisfiesWolfe (:137-146)
  __device__ __forceinline__ bool wolfe(const HzSample<T>& r) const {
    const bool w1 = (delta * dphi_0 >= (r.phi - phi_0) / r.alpha) & (r.dphi >= sigma * dphi_0);
    const bool w2 = ((T(2) * delta - T(1)) * dphi_0 >= r.dphi) & (r.dphi >= sigma * dphi_0) & (r.phi <= phi_lim);
    return w1 | w2;
  }
  __device__ __forceinline__ static T secant(T a, T b, T da, T db) {  // :148-151
    return (a * db - b * da) / (db - da);
  }

  // Bisect (:189-218): returns wolfe_hit; A / B updated like the returned indices
  __device__ __forceinline__ bool bisect(HzSample<T>& A, HzSample<T>& B) {
    T a = A.alpha, b = B.alpha;
    while (uni(b - a > Num<T>::eps * b)) {
      const T dd = (a + b) / T(2);
      HzSample<T> r = eval(dd);
      push(r);
      if (uni(wolfe(r))) { B = r; return true; }
      if (uni(r.dphi >= T(0))) { B = r; return false; }
      if (uni(r.phi <= phi_lim)) { a = dd; A = r; }
      else { b = dd; B = r; }
    }
    return false;
  }

  // Update (:165-187) with the new sample C
  __device__ __forceinline__ bool update(HzSample<T>& A, HzSample<T>& B, const HzSample<T>& C) {
    if (uni((C.alpha < A.alpha) | (C.alpha > B.alpha))) return false;  // U0
    if (uni(C.dphi >= T(0))) { B = C; return false; }                   // U1
    if (uni(C.phi <= phi_lim)) { A = C; return false; }                 // U2
    B = C;                                                              // U3
    return bisect(A, B);
  }

  // Secant2 (:222-283): returns wolfe_hit with the accepted sample in A (= B); else the new bracket
  __device__ __forceinline__ bool secant2(HzSample<T>& A, HzSample<T>& B) {
    const HzSample<T> a0 = A, b0 = B;
    T cc = secant(a0.alpha, b0.alpha, a0.dphi, b0.dphi);  // S1
    if (uni(!cfinite(cc))) cc = (a0.alpha + b0.alpha) / T(2);
    HzSample<T> c1 = eval(cc);
    push(c1);
    if (uni(wolfe(c1))) { A = B = c1; return true; }
    if (update(A, B, c1)) { A = B; return true; }  // S2
    T c2 = cc;  // S3
    const bool moved_b = (B.id == c1.id), moved_a = (A.id == c1.id);
    if (uni(moved_b)) c2 = secant(b0.alpha, B.alpha, b0.dphi, B.dphi);
    else if (uni(moved_a)) c2 = secant(a0.alpha, A.alpha, a0.dphi, A.dphi);
    if (uni((moved_a | moved_b) & (A.alpha <= c2) & (c2 <= B.alpha))) {
      HzSample<T> r2 = eval(c2);
      push(r2);
      if (uni(wolfe(r2))) { A = B = r2; return true; }
      if (update(A, B, r2)) { A = B; return true; }  // S4
    }
    return false;
  }
};

// hzls (:290-548).  Same contract as cvsrch: returns the number of evaluations; (x, f, g)
// is the accepted state, or the start state when the search fails (return -1 there).
// stp_out / ok = the reference's `*stp` on return and `return value == 0`: GradientDescent rebuilds
// its next point from the step width alone (gradient_descent.h:72), which differs from the
// returned state exactly when the search failed.
template <class Fn, class T, int E, bool kNeg = false>
__device__ __forceinline__ int hzls(const Fn& fn, const EvalCtx& ctx, const RedCtx<T>& rc, const T (&x0)[E],
                                 const T f0, const T (&g0)[E], T (&x)[E], T& f, T (&g)[E], T stp,
                                 const T (&s)[E], const T dginit, T& stp_out, bool& ok) {
  const T epsilon_k = T(1e-6), gamma = T(0.66), rho = T(5), psi3 = T(0.1);
  const int maxlinesearch = 50, iterfinitemax = 60;
  // x / g double as the PhiDphi workspaces (xa, gx); they hold the start state until the
  // first evaluation and the accepted state on success
#pragma unroll
  for (int j = 0; j < E; ++j) { x[j] = x0[j]; g[j] = g0[j]; }
  f = f0;
  stp_out = stp;
  ok = false;
  if (uni(dginit >= T(0))) return 0;  // :316 (the step is left at its initial value)

  HzSearch<Fn, T, E, kNeg> z{fn, ctx, rc, x0, s, x, g, f0, dginit, T(0), T(1) / T(10), T(9) / T(10), 1, 0};
  z.phi_lim = f0 + epsilon_k * cabs(f0);
  const HzSample<T> origin{T(0), f0, dginit, 0};
  T best_alpha = T(0), best_phi = f0;
  T best_x[E], best_g[E];
#pragma unroll
  for (int j = 0; j < E; ++j) { best_x[j] = x0[j]; best_g[j] = g0[j]; }

  // the three ways out (:338-341 etc.)
  auto update_best = [&](const HzSample<T>& r) {
    if (uni((r.alpha > T(0)) & (r.phi < best_phi))) {
      best_alpha = r.alpha;
      best_phi = r.phi;
#pragma unroll
      for (int j = 0; j < E; ++j) { best_x[j] = x[j]; best_g[j] = g[j]; }
    }
  };
  auto fail = [&]() {  // state untouched, *stp = 0
#pragma unroll
    for (int j = 0; j < E; ++j) { x[j] = x0[j]; g[j] = g0[j]; }
    f = f0;
    stp_out = T(0);
    ok = false;
  };
  auto accept = [&](const T phi, const T alpha) {  // (x, g) already hold the accepted point
    f = phi;
    stp_out = alpha;
    ok = true;
  };
  auto best_or_fail = [&]() {
    if (uni(best_alpha > T(0))) {
#pragma unroll
      for (int j = 0; j < E; ++j) { x[j] = best_x[j]; g[j] = best_g[j]; }
      accept(best_phi, best_alpha);
    } else {
      fail();
    }
  };

  T cc = stp;  // :330
  if (uni(!(cc > T(0)))) cc = T(1);
  HzSample<T> ec = z.eval(cc);
  int iterfinite = 0;
  while (uni(!(cfinite(ec.phi) & cfinite(ec.dphi)) & (iterfinite < iterfinitemax))) {
    cc *= psi3;
    ec = z.eval(cc);
    ++iterfinite;
  }
  if (uni(!(cfinite(ec.phi) & cfinite(ec.dphi)))) { fail(); return z.nfev; }
  z.push(ec);
  update_best(ec);
  if (uni(z.wolfe(ec))) { accept(ec.phi, cc); return z.nfev; }

  bool bracketed = false;
  HzSample<T> A = origin, B = ec;
  HzSample<T> last = ec;      // history.back()
  HzSample<T> cand = origin;  // most recent sample before `last` with phi <= phi_lim (else the origin: ia stays 0)
  int iter = 1;
  while (uni(!bracketed & (iter < maxlinesearch))) {  // bracket phase, :361-437
    if (uni(last.dphi >= T(0))) {
      B = last;
      A = cand;
      bracketed = true;
    } else if (uni(last.phi > z.phi_lim)) {
      B = last;
      A = origin;
      if (z.bisect(A, B)) { accept(B.phi, B.alpha); return z.nfev; }
      bracketed = true;
    } else {
      cc *= rho;
      ec = z.eval(cc);
      iterfinite = 0;
      while (uni(!(cfinite(ec.phi) & cfinite(ec.dphi)) & (iterfinite < iterfinitemax))) {
        cc = (last.alpha + cc) / T(2);
        ec = z.eval(cc);
        ++iterfinite;
      }
      if (uni(!(cfinite(ec.phi) & cfinite(ec.dphi)))) { best_or_fail(); return z.nfev; }
      if (uni(last.phi <= z.phi_lim)) cand = last;
      z.push(ec);
      last = ec;
      update_best(ec);
      if (uni(z.wolfe(ec))) { accept(ec.phi, cc); return z.nfev; }
    }
    ++iter;
  }
  if (uni(!bracketed)) { best_or_fail(); return z.nfev; }

  while (uni(iter < maxlinesearch)) {  // secant phase, :449-538
    const T a = A.alpha, b = B.alpha;
    if (uni(b - a <= Num<T>::eps * b)) {
      if (uni(a > T(0))) {
        ec = z.eval(a);
        accept(ec.phi, a);
        return z.nfev;
      }
      best_or_fail();
      return z.nfev;
    }
    HzSample<T> nA = A, nB = B;
    if (z.secant2(nA, nB)) { accept(nA.phi, nA.alpha); return z.nfev; }
    if (uni(nB.alpha - nA.alpha < gamma * (b - a))) {
      A = nA;
      B = nB;
    } else {
      const T cm = (nA.alpha + nB.alpha) / T(2);
      HzSample<T> rm = z.eval(cm);
      z.push(rm);
      update_best(rm);
      if (uni(z.wolfe(rm))) { accept(rm.phi, cm); return z.nfev; }
      if (z.update(nA, nB, rm)) { accept(nB.phi, nB.alpha); return z.nfev; }
      A = nA;
      B = nB;
    }
    ++iter;
  }
  best_or_fail();
  return z.nfev;
}

// The LineSearch template parameter of the solvers (lbfgs.h:41, bfgs.h:40, gradient_descent.h:38).
struct LsMoreThuente {
  // cvsrch always evaluates at the step it returns: the returned state IS x0 + stp * s
  static constexpr bool kStateMayDifferFromStep = false;
  template <class Fn, class T, int E, bool kNeg = false, bool kChecked = false, class Ctx, class RC>
  __device__ __forceinline__ static int search(const Fn& fn, const Ctx& ctx, const RC& rc,
                                               const T (&x0)[E], const T f0, const T (&g0)[E], T (&x)[E],
                                               T& f, T (&g)[E], T stp, const T (&s)[E], const T dginit) {
    return cvsrch<Fn, T, E, kNeg, kChecked>(fn, ctx, rc, x0, f0, g0, x, f, g, stp, s, dginit);
  }
};
struct LsHagerZhang {
  // a failed hzls leaves the state at the start point and the step at 0 (or at its initial value)
  static constexpr bool kStateMayDifferFromStep = true;
  template <class Fn, class T, int E, bool kNeg = false, bool kChecked = false>
  __device__ __forceinline__ static int search(const Fn& fn, const EvalCtx& ctx, const RedCtx<T>& rc,
                                               const T (&x0)[E], const T f0, const T (&g0)[E], T (&x)[E],
                                               T& f, T (&g)[E], T stp, const T (&s)[E], const T dginit) {
    T stp_out;
    bool ok;
    return hzls<Fn, T, E, kNeg>(fn, ctx, rc, x0, f0, g0, x, f, g, stp, s, dginit, stp_out, ok);
  }
  template <class Fn, class T, int E>
  __device__ __forceinline__ static int search_with_step(const Fn& fn, const EvalCtx& ctx, const RedCtx<T>& rc,
                                                         const T (&x0)[E], const T f0, const T (&g0)[E],
                                                         T (&x)[E], T& f, T (&g)[E], T stp, const T (&s)[E],
                                                         const T dginit, T& stp_out, bool& ok) {
    return hzls<Fn, T, E>(fn, ctx, rc, x0, f0, g0, x, f, g, stp, s, dginit, stp_out, ok);
  }
};

}  // namespace cno

#endif  // CNO_LINESEARCH_CUH_
