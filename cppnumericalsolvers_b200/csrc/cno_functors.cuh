// cno_functors.cuh -- device objective functors compiled into libcno.so.
//
// Device functor concept (the warp-cooperative form of the reference's
// FunctionCRTP::operator()(x, grad, hess), function_base.h:96-126):
//
//   struct F {
//     using Scalar = double|float;
//     static constexpr int Dim = D;           // compile-time dimension
//     static constexpr int Mode = 1|2;        // DifferentiabilityMode First/Second
//     // every lane passes its E = ceil(D/32) elements of x; returns f(x)
//     // (identical in all lanes) and, if grad != nullptr, this lane's slice
//     // of the gradient.
//     __device__ Scalar operator()(const cno::EvalCtx&, const Scalar (&x)[E],
//                                  Scalar (*grad)[E]) const;
//   };
//
// Optional members the solver kernels look for (traits in cno_device.cuh):
//   kStageElems + init_stage()/stage()  per-instance data staged into the warp's shared-memory slice (StageElems)
//   kRegsPerThread                      registers per thread the plain L-BFGS kernel needs (FnRegsPerThread)
//   active(instance)                    instances the kernel skips (FnSkipsInstances; AugLagFn)
//   kHelperWarps = 1 + helper()/release_helper()   a second warp per instance that the functor drives through a
//                                       named barrier (FnHelperWarps; LogisticFn, built-in functors only)
//
// Group form (fp64, First mode; HasGroupForm): a second operator() for the group L-BFGS kernel (cno_lbfgs_group.cuh),
// in which W = d / 128 warps own one instance:
//     __device__ double operator()(const cno::GroupEvalCtx<W>& c, const double (&x)[4], double (*grad)[4]) const;
//   thread t = 32 w + l of the group holds elements c.first .. c.first + 3 (c.first = group_first_elem<W>(t): lane l's
//   run of d / 32 elements, warp w's 4 of them); returns f(x) in every thread and, if grad != nullptr, the thread's 4
//   gradient elements.  The functor never writes a barrier: group_sum_terms(c, terms) sums 4 terms per thread over the
//   group with the bits of warp_sum(lane_tree<T, d / 32>(terms)) in the one-warp form; group_neighbours(c, x, x_prev,
//   x_next) gives x_{first-1} and x_{first+4} through the group's exchange block.  Barrier rule: an evaluation that
//   uses the exchange block is followed by a group sum before the block is written again (a functor that returns
//   group_sum_terms keeps it, and so does every composite of such functors).  CNO_INSTANTIATE_FUNCTION runs Lbfgs
//   (MoreThuente, default policy, nothing staged) on this form at d = 1024.
//
// The operation order of each functor below is restated one-for-one by the
// CPU oracle (oracle/cno_oracle_impl.inc: eval_*), so values and gradients
// agree bit for bit.
#ifndef CNO_FUNCTORS_CUH_
#define CNO_FUNCTORS_CUH_

#include "cno_device.cuh"

namespace cno {

// Chained Rosenbrock: f = sum_{i<d-1} (1-x_i)^2 + 100 (x_{i+1}-x_i^2)^2.
// At D = 2 the expressions are exactly src/test/verify.cc:58-69.
template <class T, int D, class P = PolicyFast>
struct RosenbrockFn {
  using Scalar = T;
  using Policy = P;
  static constexpr int Dim = D;
  static constexpr int Mode = 1;
  static constexpr int E = Shape<D>::E;

  static constexpr bool kHasPartial = true;
  // fp64, 4 elements per lane, default policy: 96 registers (20 warps where shared memory has room, as at m = 5).
  // The kernel then spills a little (at m = 5: 88 bytes stored, 164 loaded per thread), and was measured faster on an
  // H100 than 16 warps at 128 registers without spills (DESIGN.md 2.1).
  static constexpr int kRegsPerThread = (sizeof(T) == 8 && E == 4 && std::is_same<P, PolicyFast>::value) ? 96 : 128;
  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[E],
                                          T (*grad)[E]) const {
    return warp_sum_p<P, T, E>(partial(c, x, grad), RedCtx<T>{static_cast<T*>(c.stage), c.lane});
  }
  // the lane's share of sum_i term_i (unreduced) and, if grad != nullptr, its slice of the gradient
  __device__ __forceinline__ typename LanePartial<P, T, E>::type partial(const EvalCtx& c, const T (&x)[E],
                                                                         T (*grad)[E]) const {
    const int lane = c.lane;
    // x_{i+1} of this lane's last element lives in lane+1, slot 0.
    const T x_next_lane = __shfl_down_sync(kFullMask, x[0], 1);
    T term[E], A[E], Bv[E];
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int i = lane * E + j;
      const T xi = x[j];
      const T xn = (j + 1 < E) ? x[(j + 1 < E) ? j + 1 : 0] : x_next_lane;
      const T t1 = (1 - xi);
      const T t2 = (xn - xi * xi);
      const bool live = (i + 1 < D);
      term[j] = live ? (t1 * t1 + 100 * t2 * t2) : T(0);
      A[j] = -2 * (1 - xi) + 200 * (xn - xi * xi) * (-2 * xi);
      Bv[j] = 200 * (xn - xi * xi);
    }
    if (grad) {
      // g_i = B_{i-1} + A_i ; g_0 = A_0 ; g_{D-1} = B_{D-2}
      const T b_prev_lane = __shfl_up_sync(kFullMask, Bv[E - 1], 1);
#pragma unroll
      for (int j = 0; j < E; ++j) {
        const int i = lane * E + j;
        const T bprev = (j > 0) ? Bv[(j > 0) ? j - 1 : 0] : b_prev_lane;
        T gi;
        if (D == 1) gi = T(0);
        else if (i == 0) gi = A[j];
        else if (i == D - 1) gi = bprev;
        else gi = bprev + A[j];
        (*grad)[j] = (i < D) ? gi : T(0);
      }
    }
    return lane_terms_p<P, T, E>(term);
  }

  // Diagonal of the Hessian (Second mode; at D = 2 src/test/verify.cc:93-97 incl. the
  // reference's "+ 1"): H_ii = [1200 x_i^2 - 400 x_{i+1} + 1]_{i<D-1} (+) [200]_{i>0}.
  __device__ __forceinline__ void hess_diag(const EvalCtx& c, const T (&x)[E], T (&h)[E]) const {
    const T x_next_lane = __shfl_down_sync(kFullMask, x[0], 1);
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int i = c.lane * E + j;
      const T xi = x[j];
      const T xn = (j + 1 < E) ? x[(j + 1 < E) ? j + 1 : 0] : x_next_lane;
      const T hii = 1200 * xi * xi - 400 * xn + 1;
      T v;
      if (i == 0) v = hii;
      else if (i == D - 1) v = T(200);
      else v = T(200) + hii;
      h[j] = (i < D) ? v : T(1);
    }
  }

  // Column j of the (symmetric, tridiagonal) Hessian, this lane's rows: H_jj as in hess_diag,
  // H_{j+1,j} = H_{j,j+1} = -400 x_j (src/test/verify.cc:93-97 at D = 2).
  __device__ __forceinline__ void hess_col(const EvalCtx& c, const T (&x)[E], int j, bool, T (&col)[E]) const {
    const T xj = lane_bcast<T, E>(x, j);
    const T xjn = lane_bcast<T, E>(x, (j + 1 < D) ? j + 1 : j);
    const T hii = 1200 * xj * xj - 400 * xjn + 1;
    T djj;
    if (j == 0) djj = hii;
    else if (j == D - 1) djj = T(200);
    else djj = T(200) + hii;
    if (D == 1) djj = T(0);
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int r = c.lane * E + e;
      T v = T(0);
      if (r == j) v = djj;
      else if (r == j + 1) v = -400 * xj;       // below the diagonal
      else if (r + 1 == j) v = -400 * x[e];     // above it: -400 x_{j-1} = -400 x_r
      col[e] = (r < D) ? v : T(0);
    }
  }
};

// Dockerfile.test:21-29: 5 x0^2 + 100 x1^2 + 5 (D = 2).
template <class T>
struct DiagQuadraticFn {
  using Scalar = T;
  static constexpr int Dim = 2;
  static constexpr int Mode = 1;
  static constexpr int E = 1;
  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[1],
                                          T (*grad)[1]) const {
    const T x0 = __shfl_sync(kFullMask, x[0], 0);
    const T x1 = __shfl_sync(kFullMask, x[0], 1);
    if (grad) (*grad)[0] = (c.lane == 0) ? (10 * x0) : ((c.lane == 1) ? (200 * x1) : T(0));
    return 5 * x0 * x0 + 100 * x1 * x1 + 5;
  }
  __device__ __forceinline__ void hess_diag(const EvalCtx& c, const T (&)[1], T (&h)[1]) const {
    h[0] = (c.lane == 0) ? T(10) : ((c.lane == 1) ? T(200) : T(0));
  }
  __device__ __forceinline__ void hess_col(const EvalCtx& c, const T (&)[1], int j, bool, T (&col)[1]) const {
    col[0] = (c.lane == j) ? ((j == 0) ? T(10) : T(200)) : T(0);
  }
};

// src/test/augmented_lagrangian_test.cc:123-130: 0.5 * x.squaredNorm().
template <class T, int D>
struct HalfSquaredNormFn {
  using Scalar = T;
  static constexpr int Dim = D;
  static constexpr int Mode = 1;
  static constexpr int E = Shape<D>::E;
  __device__ __forceinline__ T operator()(const EvalCtx&, const T (&x)[E],
                                          T (*grad)[E]) const {
    if (grad) {
#pragma unroll
      for (int j = 0; j < E; ++j) (*grad)[j] = x[j];
    }
    return T(0.5) * warp_dot<T, E>(x, x);
  }
  __device__ __forceinline__ void hess_diag(const EvalCtx& c, const T (&)[E], T (&h)[E]) const {
#pragma unroll
    for (int e = 0; e < E; ++e) h[e] = (c.lane * E + e < D) ? T(1) : T(0);
  }
  __device__ __forceinline__ void hess_col(const EvalCtx& c, const T (&)[E], int j, bool, T (&col)[E]) const {
#pragma unroll
    for (int e = 0; e < E; ++e) col[e] = (c.lane * E + e == j) ? T(1) : T(0);
  }
};

// 0.5 x'Ax - b'x with per-instance [A (d x d col-major) | b] read from global memory (L2) at every
// evaluation: the First-mode counterpart of DenseQuadraticFn (cno_newton.cuh), for the solvers that keep
// no matrix on chip (Lbfgs, and AugmentedLagrangian's batched "QP with affine constraints" use).
// Reference analogue: src/examples/debug.cc:43-65; src/test/augmented_lagrangian_test.cc:78-176
// (QuadraticAt12 / QuadraticAt20).  (Ax)_i = sum_j A_ij x_j, j ascending from the first product;
// x_j is broadcast from its owner lane.  Parity: tests/test_al_gpu.py (GPU) and the CPU warp emulation
// (tests/test_device_emulated.py), both bit for bit against the oracle.
template <class T, int D>
struct DenseQuadraticGlobalFn {
  using Scalar = T;
  static constexpr int Dim = D;
  static constexpr int Mode = 1;
  static constexpr int E = Shape<D>::E;
  const T* data;     // [B, stride]
  long long stride;  // scalars per instance (>= D*D + D)

  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E]) const {
    const T* A = data + c.instance * stride;
    T Ax[E], bb[E];
#pragma unroll
    for (int e = 0; e < E; ++e) Ax[e] = T(0);
#pragma unroll 1
    for (int jl = 0; jl * E < D; ++jl) {
#pragma unroll
      for (int ej = 0; ej < E; ++ej) {
        const int j = jl * E + ej;
        const T xj = __shfl_sync(kFullMask, x[ej], jl);  // x_j lives in lane j / E, slot j % E
        if (j < D) {
#pragma unroll
          for (int e = 0; e < E; ++e) {
            const int i = c.lane * E + e;
            if (i < D) {
              const T a = __ldg(A + i + (long long)j * D);
              Ax[e] = (j == 0) ? (a * xj) : (Ax[e] + a * xj);
            }
          }
        }
      }
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int i = c.lane * E + e;
      bb[e] = (i < D) ? __ldg(A + D * D + i) : T(0);
    }
    if (grad) {
#pragma unroll
      for (int e = 0; e < E; ++e) (*grad)[e] = (c.lane * E + e < D) ? (Ax[e] - bb[e]) : T(0);
    }
    T p1 = lane_dot<T, E>(x, Ax), p2 = lane_dot<T, E>(bb, x);
    warp_sum2(p1, p2);
    return T(0.5) * p1 - p2;
  }
};

}  // namespace cno

#endif  // CNO_FUNCTORS_CUH_
