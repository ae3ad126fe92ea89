// cno_bfgs.cuh -- batched Bfgs<F>::Minimize (dense inverse Hessian), one warp
// per instance, whole Solver::Minimize loop in one persistent kernel (sm_90a).
//
// Reference path (include/cppoptlib/...):
//   solver/solver.h:181-224   Solver::Minimize driver loop
//   solver/bfgs.h:65-71       InitializeSolver (H = I, fresh = true)
//   solver/bfgs.h:73-137      OptimizationStep: d = -H g, reset test, alpha_init,
//                             MoreThuente::Search, rank-2 update (N&W 6.17)
//   solver/progress.h:153-327 Progress::Update
//
// Design (D <= 32): lane i keeps ROW i of the inverse Hessian in registers
// (D doubles; the update keeps H bitwise symmetric, so row i == column i) for
// the instance's whole lifetime -- H never touches HBM, and not even shared
// memory.  Vectors (x, g, d, s, y, Hy) are one element per lane.  The two GEMVs
// and the rank-2 update read the broadcast operand (g, y, s, Hy) from a 256-byte
// warp-private shared-memory vector with LDS.128 broadcasts (1 wavefront each)
// instead of 2 SHFL per element.  Arithmetic spec (DESIGN.md 3):
// (Hv)_i = sum_j H_ij v_j, j ascending from the first product; update
// H_ij = (H_ij - rho (s_i Hy_j + Hy_i s_j)) + c2 (s_i s_j), element-wise.
#ifndef CNO_BFGS_CUH_
#define CNO_BFGS_CUH_

#include "cno_device.cuh"
#include "cno_kernel_params.h"
#include "cno_lbfgs.cuh"  // ProgressState / progress_update
#include "cno_linesearch.cuh"

namespace cno {

template <class T, int D>
struct BfgsSmem {
  static_assert(D <= 32, "register-resident BFGS supports D <= 32");
  static constexpr int kVecs = 2;                      // two broadcast vectors
  static constexpr int kWarpElems = kVecs * 32 + CNO_MAX_PAST;
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  // register-limited: H row = D scalars per thread (64 regs at D=32 fp64)
  static constexpr int kWarps = (D * (int)sizeof(T) > 128) ? 10 : 12;
};

// out_i = sum_j Hrow[j] * v_j with v broadcast from shared memory (v_s[j]).
template <class T, int D>
__device__ __forceinline__ T gemv_row(const T (&Hrow)[D], const T* __restrict__ v_s) {
  T acc = Hrow[0] * v_s[0];
#pragma unroll
  for (int j = 1; j < D; ++j) acc = acc + Hrow[j] * v_s[j];
  return acc;
}

template <class Fn, class LS = LsMoreThuente>
__global__ void __launch_bounds__(BfgsSmem<typename Fn::Scalar, Fn::Dim>::kWarps * 32, 1)
bfgs_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0,
                     const long long batch, const StopParams<typename Fn::Scalar> stop,
                     const BatchOut<typename Fn::Scalar> out,
                     unsigned long long* __restrict__ queue) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  static_assert(Shape<D>::E == 1, "one element per lane");
  using SMB = BfgsSmem<T, D>;
  constexpr T eps = Num<T>::eps;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T* const va = reinterpret_cast<T*>(smem_raw) + (size_t)warp * SMB::kWarpElems;  // broadcast vec A
  T* const vb = va + 32;                                                          // broadcast vec B
  T* const ring = vb + 32;

  for (;;) {
    unsigned long long b = 0;
    if (lane == 0) b = atomicAdd(queue, 1ULL);
    b = __shfl_sync(kFullMask, b, 0);
    if (uni(b >= (unsigned long long)batch)) break;
    const EvalCtx ctx{lane, (long long)b, nullptr};

    // solver.h:189-192
    T x[1], g[1];
    load_row<T, D>(x0 + b * D, lane, x);
    T f = fn(ctx, x, &g);
    uint32_t nfev = 1;

    // bfgs.h:65-71
    T Hrow[D];
#pragma unroll
    for (int j = 0; j < D; ++j) Hrow[j] = (j == lane) ? T(1) : T(0);
    bool fresh = true;

    ProgressState<T> prog;
    prog.num_iterations = 0;
    prog.x_delta_violations = 0;
    prog.f_delta_violations = 0;
    prog.x_delta = prog.f_delta = prog.gradient_norm = T(0);
    prog.ring_size = 0;
    prog.ring_pos = 0;
    prog.status = CNO_STATUS_NOT_STARTED;

    do {  // solver.h:196-220
      // ---- d = -H g (bfgs.h:81) ----
      __syncwarp();
      va[lane] = g[0];
      __syncwarp();
      T dir[1];
      dir[0] = (lane < D) ? -gemv_row<T, D>(Hrow, va) : T(0);

      // ---- reset test (:87-92) ----
      T phi = warp_sum(lane_dot<T, 1>(g, dir));
      if (uni((phi > 0) || (phi != phi))) {
#pragma unroll
        for (int j = 0; j < D; ++j) Hrow[j] = (j == lane) ? T(1) : T(0);
        dir[0] = -g[0];
        fresh = true;
        phi = -warp_sum(lane_dot<T, 1>(g, g));  // = g.(-g), bit for bit
      }
      // ---- alpha_init (:100-106) ----
      T alpha_init = T(1);
      if (uni(fresh)) {
        const T dn = csqrt(warp_sum(lane_dot<T, 1>(dir, dir)));
        alpha_init = (dn > eps) ? T(1) / dn : T(1);
      }
      // ---- MoreThuente::Search (:111-112); dginit = g.d = phi ----
      T xn[1], gn[1];
      T fn_val;
      nfev += LS::template search<Fn, T, 1>(fn, ctx, RedCtx<T>{nullptr, lane}, x, f, g, xn, fn_val, gn, alpha_init, dir, phi);

      // ---- rank-2 update (:122-133) ----
      T s[1], y[1];
      s[0] = xn[0] - x[0];
      y[0] = gn[0] - g[0];
      T ys = lane_dot<T, 1>(y, s), ss = lane_dot<T, 1>(s, s), yy = lane_dot<T, 1>(y, y);
      warp_sum3(ys, ss, yy);
      if (uni(curvature_above_eps<T>(ys, ss, yy))) {  // ys > eps ||s|| ||y|| (bfgs.h:125)
        const T rho = T(1) / ys;
        __syncwarp();
        va[lane] = y[0];
        __syncwarp();
        T Hy[1];
        Hy[0] = (lane < D) ? gemv_row<T, D>(Hrow, va) : T(0);
        const T yHy = warp_sum(lane_dot<T, 1>(y, Hy));
        const T c2 = rho * (rho * yHy + T(1));
        __syncwarp();
        va[lane] = s[0];
        vb[lane] = Hy[0];
        __syncwarp();
        const T si = s[0], hyi = Hy[0];
#pragma unroll
        for (int j = 0; j < D; ++j) {
          const T sj = va[j], hyj = vb[j];
          Hrow[j] = (Hrow[j] - rho * (si * hyj + hyi * sj)) + c2 * (si * sj);
        }
        fresh = false;
      }

      // ---- Progress::Update ----
      const T prev_value = f;
      const T x_delta = warp_maxabs<T, 1>(s);
      x[0] = xn[0];
      g[0] = gn[0];
      f = fn_val;
      const T gnorm_inf = warp_maxabs<T, 1>(g);
      const T x_inf = warp_maxabs<T, 1>(x);
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

// ---- D > 32: the inverse Hessian in the warp's shared-memory slice -----------------------------------
// bfgs.h:65-137 is dimension-agnostic; above 32 a row no longer fits a lane's registers, so H (D x D,
// bitwise symmetric, column-major with 32*E padded rows per column) lives in shared memory: lane l owns
// rows l*E .. l*E+E-1 of every column (one conflict-free vector access per column and warp), vectors are
// E elements per lane.  Same arithmetic specification as the register-resident kernel: (Hv)_i = sum_j H_ij
// v_j, j ascending from the first product; H_ij = (H_ij - rho (s_i Hy_j + Hy_i s_j)) + c2 (s_i s_j).
// One instance needs 8 D^2 bytes (32 KB at d = 64 fp64: 6 resident warps per SM; 128 KB at d = 128: one).
template <class T, int D>
struct BfgsBigSmem {
  static constexpr int E = Shape<D>::E;
  static constexpr int kRows = 32 * E;  // padded rows of a column
  static constexpr int kH = D * kRows;
  static constexpr int kWarpElems = ((kH + 2 * kRows + CNO_MAX_PAST + 3) / 4) * 4;
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  static constexpr int kFit = (int)((size_t)(227 * 1024) / kWarpBytes);
  static_assert(kFit >= 1, "BFGS: the inverse Hessian does not fit one SM's shared memory");
  static constexpr int kWarps = kFit > 8 ? 8 : kFit;
};

template <class Fn, class LS = LsMoreThuente>
__global__ void __launch_bounds__(BfgsBigSmem<typename Fn::Scalar, Fn::Dim>::kWarps * 32, 1)
bfgs_smem_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0, const long long batch,
                          const StopParams<typename Fn::Scalar> stop, const BatchOut<typename Fn::Scalar> out,
                          unsigned long long* __restrict__ queue) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  constexpr int E = Shape<D>::E;
  using SMB = BfgsBigSmem<T, D>;
  constexpr T eps = Num<T>::eps;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T* const H = reinterpret_cast<T*>(smem_raw) + (size_t)warp * SMB::kWarpElems;
  T* const va = H + SMB::kH;
  T* const vb = va + SMB::kRows;
  T* const ring = vb + SMB::kRows;
  using LP = LanePack<T, E>;
  // this lane's rows of column j  <->  registers
  auto load_col = [&](int j, T (&c)[E]) {
    const typename LP::P::type* p = reinterpret_cast<const typename LP::P::type*>(H + (size_t)j * SMB::kRows + lane * E);
#pragma unroll
    for (int k = 0; k < LP::NC; ++k) LP::P::get(p[k], &c[k * LP::CE]);
  };
  auto store_col = [&](int j, const T (&c)[E]) {
    typename LP::P::type* p = reinterpret_cast<typename LP::P::type*>(H + (size_t)j * SMB::kRows + lane * E);
#pragma unroll
    for (int k = 0; k < LP::NC; ++k) p[k] = LP::P::make(&c[k * LP::CE]);
  };
  auto store_vec = [&](T* dst, const T (&v)[E]) {
#pragma unroll
    for (int e = 0; e < E; ++e) dst[lane * E + e] = v[e];
  };
  auto set_identity = [&]() {
#pragma unroll 1
    for (int j = 0; j < D; ++j) {
      T c[E];
#pragma unroll
      for (int e = 0; e < E; ++e) c[e] = (lane * E + e == j) ? T(1) : T(0);
      store_col(j, c);
    }
  };
  // out_i = sum_j H_ij v_j, v broadcast from shared memory
  auto gemv = [&](const T* v, T (&o)[E]) {
    T c[E];
    load_col(0, c);
    const T v0 = v[0];
#pragma unroll
    for (int e = 0; e < E; ++e) o[e] = c[e] * v0;
#pragma unroll 4
    for (int j = 1; j < D; ++j) {
      load_col(j, c);
      const T vj = v[j];
#pragma unroll
      for (int e = 0; e < E; ++e) o[e] = o[e] + c[e] * vj;
    }
  };

  for (;;) {
    unsigned long long b = 0;
    if (lane == 0) b = atomicAdd(queue, 1ULL);
    b = __shfl_sync(kFullMask, b, 0);
    if (uni(b >= (unsigned long long)batch)) break;
    const EvalCtx ctx{lane, (long long)b, nullptr};

    T x[E], g[E];
    load_row<T, D>(x0 + b * D, lane, x);
    T f = fn(ctx, x, &g);  // solver.h:189-192
    uint32_t nfev = 1;
    __syncwarp();
    set_identity();  // bfgs.h:65-71
    bool fresh = true;

    ProgressState<T> prog;
    prog.num_iterations = 0;
    prog.x_delta_violations = 0;
    prog.f_delta_violations = 0;
    prog.x_delta = prog.f_delta = prog.gradient_norm = T(0);
    prog.ring_size = 0;
    prog.ring_pos = 0;
    prog.status = CNO_STATUS_NOT_STARTED;

    do {  // solver.h:196-220
      // ---- d = -H g (bfgs.h:81) ----
      __syncwarp();
      store_vec(va, g);
      __syncwarp();
      T dir[E];
      gemv(va, dir);
#pragma unroll
      for (int e = 0; e < E; ++e) dir[e] = (lane * E + e < D) ? -dir[e] : T(0);
      // ---- reset test (:87-92) ----
      T phi = warp_sum(lane_dot<T, E>(g, dir));
      if (uni((phi > 0) || (phi != phi))) {
        __syncwarp();
        set_identity();
#pragma unroll
        for (int e = 0; e < E; ++e) dir[e] = -g[e];
        fresh = true;
        phi = -warp_sum(lane_dot<T, E>(g, g));  // = g.(-g), bit for bit
      }
      // ---- alpha_init (:100-106) ----
      T alpha_init = T(1);
      if (uni(fresh)) {
        const T dn = csqrt(warp_sum(lane_dot<T, E>(dir, dir)));
        alpha_init = (dn > eps) ? T(1) / dn : T(1);
      }
      // ---- LineSearch::Search (:111-112); dginit = g.d = phi ----
      T xn[E], gn[E];
      T fn_val;
      nfev += LS::template search<Fn, T, E>(fn, ctx, RedCtx<T>{nullptr, lane}, x, f, g, xn, fn_val, gn, alpha_init, dir, phi);

      // ---- rank-2 update (:122-133) ----
      T s[E], y[E];
#pragma unroll
      for (int e = 0; e < E; ++e) { s[e] = xn[e] - x[e]; y[e] = gn[e] - g[e]; }
      T ys = lane_dot<T, E>(y, s), ss = lane_dot<T, E>(s, s), yy = lane_dot<T, E>(y, y);
      warp_sum3(ys, ss, yy);
      if (uni(curvature_above_eps<T>(ys, ss, yy))) {  // ys > eps ||s|| ||y|| (bfgs.h:125)
        const T rho = T(1) / ys;
        __syncwarp();
        store_vec(va, y);
        __syncwarp();
        T Hy[E];
        gemv(va, Hy);
#pragma unroll
        for (int e = 0; e < E; ++e) Hy[e] = (lane * E + e < D) ? Hy[e] : T(0);
        const T yHy = warp_sum(lane_dot<T, E>(y, Hy));
        const T c2 = rho * (rho * yHy + T(1));
        __syncwarp();
        store_vec(va, s);
        store_vec(vb, Hy);
        __syncwarp();
#pragma unroll 2
        for (int j = 0; j < D; ++j) {
          T c[E];
          load_col(j, c);
          const T sj = va[j], hyj = vb[j];
#pragma unroll
          for (int e = 0; e < E; ++e)
            c[e] = (lane * E + e < D) ? ((c[e] - rho * (s[e] * hyj + Hy[e] * sj)) + c2 * (s[e] * sj)) : T(0);
          store_col(j, c);
        }
        fresh = false;
      }

      // ---- Progress::Update ----
      const T prev_value = f;
      const T x_delta = warp_maxabs<T, E>(s);
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

#endif  // CNO_BFGS_CUH_
