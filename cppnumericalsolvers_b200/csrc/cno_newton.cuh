// cno_newton.cuh -- batched NewtonDescent<F>::Minimize, one warp per instance,
// whole Solver::Minimize loop in one persistent kernel (sm_90a).
//
// Reference path (include/cppoptlib/...):
//   solver/solver.h:181-224          Minimize loop (incl. the re-evaluation of a
//                                    gradient-less state, :210-216)
//   solver/newton_descent.h:61-81    H += 1e-5 I;  delta = H.lu().solve(-g);
//                                    Armijo<F,2>::Search;  x + rate * delta
//   linesearch/armijo.h:82-101       Armijo<F,2> (unshifted H in the slope, no
//                                    lower bound on alpha)
//   solver/progress.h:153-327        Progress::Update
//
// Design: the per-instance Hessian block ([A | b] of the dense-quadratic
// family: 32.5 KB at d=64 fp64) is staged into the warp's shared-memory slice by
// ONE TMA bulk copy (cp.async.bulk + mbarrier complete_tx), twice per iteration:
// once as the LU workspace, once (unshifted) for the Armijo slope and the trial
// evaluations.  LU = unblocked right-looking elimination with partial pivoting,
// done in place in shared memory with IMPLICIT row exchanges (a virtual-position
// register per row instead of 32-way-conflicting physical swaps); the right-hand
// side rides along as column D.  Every floating-point operation and its order
// equal the oracle's lu_solve (oracle/cno_oracle_impl.inc), so the result is
// bit-identical; only the storage position of a row differs.
//
// What the device path reuses instead of recomputing (same function, same x,
// therefore the same bits): the step's and Armijo's f(x), g(x) are the state's
// cached value/gradient; the re-evaluation at x + rate*delta (solver.h:210-216)
// is the last Armijo trial.  nfev still counts every evaluation the reference
// makes.  Progress::condition_hessian (progress.h:203-210) is output-only under
// every preset (threshold 0) and is not computed; a non-zero threshold is
// rejected with CNO_ERR_UNSUPPORTED.
#ifndef CNO_NEWTON_CUH_
#define CNO_NEWTON_CUH_

#include "cno_device.cuh"
#include "cno_kernel_params.h"
#include "cno_lbfgs.cuh"  // ProgressState / progress_update

namespace cno {

// ---- TMA bulk copy + mbarrier (one barrier per warp) ---------------------------
#ifdef CNO_WARP_EMULATION  // tests/emu: the bulk copy is a memcpy by the issuing lane; the vote in mbar_wait is the barrier
__device__ __forceinline__ void mbar_init(uint64_t*, int) {}
__device__ __forceinline__ void mbar_expect_tx(uint64_t*, uint32_t) {}
__device__ __forceinline__ void mbar_wait(uint64_t*, uint32_t) { (void)uni(true); }
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t*) {
  std::memcpy(dst_smem, src_gmem, bytes);
}
__device__ __forceinline__ void fence_proxy_async() {}
#else
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!uni(mbar_try_wait(bar, parity))) {
  }
}
// global -> shared bulk copy (bytes % 16 == 0, both 16-byte aligned), completion
// signalled on `bar` (SASS: UBLKCP).
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

#endif  // CNO_WARP_EMULATION

// ---- plain-layout shared-memory vectors/columns (element i at index i) ----------
// Lane l owns elements l*E .. l*E+E-1 (a contiguous chunk, so an access by the
// whole warp is one contiguous conflict-free vector access when D % 32 == 0).
template <class T, int D>
struct SmemRowVec {
  static constexpr int E = Shape<D>::E;
  using LP = LanePack<T, E>;
  __device__ __forceinline__ static void load(const T* base, int lane, T (&v)[E]) {
    if constexpr (D % 32 == 0) {
      const typename LP::P::type* p = reinterpret_cast<const typename LP::P::type*>(base + lane * E);
#pragma unroll
      for (int c = 0; c < LP::NC; ++c) {
        const typename LP::P::type u = p[c];
        LP::P::get(u, &v[c * LP::CE]);
      }
    } else {
#pragma unroll
      for (int e = 0; e < E; ++e) v[e] = (lane * E + e < D) ? base[lane * E + e] : T(0);
    }
  }
  __device__ __forceinline__ static void store(T* base, int lane, const T (&v)[E]) {
    if constexpr (D % 32 == 0) {
      typename LP::P::type* p = reinterpret_cast<typename LP::P::type*>(base + lane * E);
#pragma unroll
      for (int c = 0; c < LP::NC; ++c) p[c] = LP::P::make(&v[c * LP::CE]);
    } else {
#pragma unroll
      for (int e = 0; e < E; ++e)
        if (lane * E + e < D) base[lane * E + e] = v[e];
    }
  }
  // out_i = sum_j H[i + j*D] * vec[j], j ascending from the first product.
  __device__ __forceinline__ static void gemv(const T* H, const T* vec, int lane, T (&out)[E]) {
    T col[E];
    load(H, lane, col);
    const T v0 = vec[0];
#pragma unroll
    for (int e = 0; e < E; ++e) out[e] = col[e] * v0;
#pragma unroll 4
    for (int j = 1; j < D; ++j) {
      load(H + j * D, lane, col);
      const T vj = vec[j];
#pragma unroll
      for (int e = 0; e < E; ++e) out[e] = out[e] + col[e] * vj;
    }
  }
};

// ---- the augmented matrix [H | rhs] in the warp's shared-memory slice ----
// Column-major, lane l owns rows l*E .. l*E+E-1 of every column.  For D = 64 fp64
// the matrix alone is 32 KB per instance: 6 resident warps per SM.
template <class T, int D>
struct AugStore {
  static constexpr int E = Shape<D>::E;
  using RV = SmemRowVec<T, D>;
  T* sm;        // [D matrix columns | rhs], each D rows
  int lane;

  __device__ __forceinline__ T* rhs() const { return sm + D * D; }
  __device__ __forceinline__ T* smcol(int j) const { return sm + j * D; }
};

// ---- Second-mode device functors ------------------------------------------------
// Concept: Scalar, Dim, Mode = 2, kHessianConstant, plus
//   stage(ctx, x, A, bar, parity&)      stage H(x) (and per-instance data) into A
//   operator()(ctx, x, grad*, A, vec)   value (+ gradient) using the staged block

// out_i = sum_j H_ij v_j over the whole staged matrix, j ascending from the first
// product; v is read from the warp-private shared vector `vec`.
template <class T, int D>
__device__ __forceinline__ void aug_gemv(const AugStore<T, D>& A, const T* vec, T (&out)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
  using AS = AugStore<T, D>;
  T col[E];
  AS::RV::load(A.smcol(0), A.lane, col);
  const T v0 = vec[0];
#pragma unroll
  for (int e = 0; e < E; ++e) out[e] = col[e] * v0;
#pragma unroll 4
  for (int j = 1; j < D; ++j) {
    AS::RV::load(A.smcol(j), A.lane, col);
    const T vj = vec[j];
#pragma unroll
    for (int e = 0; e < E; ++e) out[e] = out[e] + col[e] * vj;
  }
}

// out_i = sum_j H_ij v_j with H (d x d col-major) streamed from GLOBAL memory (L2: the block was read a moment
// ago), j ascending from the first product; v is read from the warp-private shared vector `vec`.  kU columns are
// in flight per lane so the L2 latency is paid once per group, not once per column.
template <class T, int D>
__device__ __forceinline__ void gemv_global(const T* __restrict__ H, const T* vec, int lane, T (&out)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
  constexpr int kU = (E <= 2) ? 16 : 8;
#pragma unroll 1
  for (int j0 = 0; j0 < D; j0 += kU) {
    T c[kU][E];
#pragma unroll
    for (int t = 0; t < kU; ++t)
      if (j0 + t < D) load_row<T, D>(H + (size_t)(j0 + t) * D, lane, c[t]);
#pragma unroll
    for (int t = 0; t < kU; ++t) {
      if (j0 + t < D) {
        const T vj = vec[j0 + t];
#pragma unroll
        for (int e = 0; e < E; ++e) out[e] = (j0 + t == 0) ? (c[t][e] * vj) : (out[e] + c[t][e] * vj);
      }
    }
  }
}

// Two products with the SAME matrix in ONE pass over it: outa = H va, outb = H vb (each exactly as gemv_global
// computes it: j ascending from the first product).  The matrix is the instance's 32 KB block in L2: a constant
// Hessian is read once per iteration (Armijo's slope and the first trial evaluation together) instead of twice.
template <class T, int D>
__device__ __forceinline__ void gemv2_global(const T* __restrict__ H, const T* veca, const T* vecb, int lane,
                                             T (&outa)[Shape<D>::E], T (&outb)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
  constexpr int kU = (E <= 2) ? 16 : 8;
#pragma unroll 1
  for (int j0 = 0; j0 < D; j0 += kU) {
    T c[kU][E];
#pragma unroll
    for (int t = 0; t < kU; ++t)
      if (j0 + t < D) load_row<T, D>(H + (size_t)(j0 + t) * D, lane, c[t]);
#pragma unroll
    for (int t = 0; t < kU; ++t) {
      if (j0 + t < D) {
        const T va = veca[j0 + t], vb = vecb[j0 + t];
#pragma unroll
        for (int e = 0; e < E; ++e) {
          outa[e] = (j0 + t == 0) ? (c[t][e] * va) : (outa[e] + c[t][e] * va);
          outb[e] = (j0 + t == 0) ? (c[t][e] * vb) : (outb[e] + c[t][e] * vb);
        }
      }
    }
  }
}

// 0.5 x'Ax - b'x with per-instance [A (d x d col-major, bitwise symmetric) | b].
// Reference analogue: src/examples/debug.cc:43-65.  (Ax)_i = sum_j A_ij x_j,
// j ascending from the first product.  The Hessian is CONSTANT, so the solver factors H + 1e-5 I once per
// instance and keeps the factors in the warp's store; evaluations and the Armijo slope stream A from global
// memory (gemv_global) instead of restaging it over the factors.
template <class T, int D>
struct DenseQuadraticFn {
  using Scalar = T;
  static constexpr int Dim = D;
  static constexpr int Mode = 2;
  static constexpr int E = Shape<D>::E;
  using AS = AugStore<T, D>;
  static constexpr bool kHessianConstant = true;
  const T* data;        // [B, stride]
  long long stride;     // scalars per instance (>= D*D + D)

  // [A | b] -> the warp's store by TMA bulk copies (cp.async.bulk + mbarrier)
  __device__ __forceinline__ void stage(const EvalCtx& c, const T (&)[E], const AS& A, uint64_t* bar,
                                        uint32_t& parity) const {
    static_assert((D * D * sizeof(T)) % 16 == 0 && (D * sizeof(T)) % 16 == 0,
                  "bulk copy sizes must be multiples of 16 bytes");
    const T* src = data + c.instance * stride;
    __syncwarp();
    if (c.lane == 0) {
      fence_proxy_async();  // order prior generic-proxy accesses of the store before the async writes
      mbar_expect_tx(bar, (uint32_t)((D * D + D) * sizeof(T)));
      tma_bulk_g2s(A.sm, src, (uint32_t)(D * D * sizeof(T)), bar);
      tma_bulk_g2s(A.rhs(), src + D * D, (uint32_t)(D * sizeof(T)), bar);
    }
    mbar_wait(bar, parity);
    parity ^= 1u;
  }

  // The block of the instance this warp will solve NEXT, pulled into L2 while the current one is solved (the kernel
  // reads its work queue one instance ahead): staging and the evaluations then read L2 instead of waiting on DRAM.
  __device__ __forceinline__ void prefetch(long long instance, int lane) const {
#ifndef CNO_WARP_EMULATION
    const char* p = reinterpret_cast<const char*>(data + instance * stride);
    constexpr int kLines = (int)(((size_t)(D * D + D) * sizeof(T) + 127) / 128);
#pragma unroll
    for (int i = 0; i < (kLines + 31) / 32; ++i) {
      const int line = i * 32 + lane;
      if (line < kLines) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + (size_t)line * 128));
    }
#else
    (void)instance; (void)lane;
#endif
  }

  // H v (= v'H: A is bitwise symmetric) for the Armijo slope, A streamed from global memory
  __device__ __forceinline__ void hess_times(const EvalCtx& c, const T (&v)[E], T (&out)[E], T* vec) const {
    using SV = SmemRowVec<T, D>;
    __syncwarp();
    SV::store(vec, c.lane, v);
    __syncwarp();
    gemv_global<T, D>(data + c.instance * stride, vec, c.lane, out);
  }

  // hess_times(v) and operator()(x, grad) together, A read once (gemv2_global); vec and vec2: D scalars of
  // warp-private scratch each.  Same bits as the two separate calls.
  __device__ __forceinline__ T hess_times_and_eval(const EvalCtx& c, const T (&v)[E], T (&hv)[E], const T (&x)[E],
                                                   T (&grad)[E], T* vec, T* vec2) const {
    using SV = SmemRowVec<T, D>;
    const T* src = data + c.instance * stride;
    __syncwarp();
    SV::store(vec, c.lane, v);
    SV::store(vec2, c.lane, x);
    __syncwarp();
    T Ax[E], bb[E];
    gemv2_global<T, D>(src, vec, vec2, c.lane, hv, Ax);
    load_row<T, D>(src + D * D, c.lane, bb);
#pragma unroll
    for (int e = 0; e < E; ++e) grad[e] = (c.lane * E + e < D) ? (Ax[e] - bb[e]) : T(0);
    T p1 = lane_dot<T, E>(x, Ax), p2 = lane_dot<T, E>(bb, x);
    warp_sum2(p1, p2);
    return T(0.5) * p1 - p2;
  }

  // value/gradient with A and b read from global memory (the store holds the LU factors).
  // vec = D scalars of warp-private scratch for the broadcast operand.
  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E],
                                          const AS&, T* vec) const {
    using SV = SmemRowVec<T, D>;
    const T* src = data + c.instance * stride;
    __syncwarp();
    SV::store(vec, c.lane, x);
    __syncwarp();
    T Ax[E], bb[E];
    gemv_global<T, D>(src, vec, c.lane, Ax);
    load_row<T, D>(src + D * D, c.lane, bb);
    if (grad) {
#pragma unroll
      for (int e = 0; e < E; ++e) (*grad)[e] = (c.lane * E + e < D) ? (Ax[e] - bb[e]) : T(0);
    }
    T p1 = lane_dot<T, E>(x, Ax), p2 = lane_dot<T, E>(bb, x);
    warp_sum2(p1, p2);
    return T(0.5) * p1 - p2;
  }
};

// Chained Rosenbrock with Hessian; at D = 2 exactly src/test/verify.cc:81-99
// (including the reference's "+ 1" on H00).
template <class T, int D>
struct RosenbrockFullFn {
  using Scalar = T;
  static constexpr int Dim = D;
  static constexpr int Mode = 2;
  static constexpr int E = Shape<D>::E;
  using AS = AugStore<T, D>;
  static_assert(D <= 32, "dense Rosenbrock Hessian: D <= 32");
  static constexpr bool kHessianConstant = false;
  __device__ __forceinline__ void stage(const EvalCtx& c, const T (&x)[E], const AS& A, uint64_t*,
                                        uint32_t&) const {
    T* aug = A.sm;
    __syncwarp();
    const int i = c.lane;  // E == 1
    const T xi = x[0];
    const T xn = __shfl_down_sync(kFullMask, xi, 1);
    const T xp = __shfl_up_sync(kFullMask, xi, 1);
    if (i < D) {
#pragma unroll 1
      for (int j = 0; j < D; ++j) aug[i + j * D] = T(0);
      // H_ii = [1200 x_i^2 - 400 x_{i+1} + 1]_{i<D-1} (+) [200]_{i>0}
      T hii = T(0);
      if (i + 1 < D) hii = 1200 * xi * xi - 400 * xn + 1;
      if (i > 0) hii = (i + 1 < D) ? (T(200) + hii) : T(200);
      aug[i + i * D] = hii;
      if (i + 1 < D) aug[i + (i + 1) * D] = -400 * xi;
      if (i > 0) aug[i + (i - 1) * D] = -400 * xp;
    }
    __syncwarp();
  }
  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E],
                                          const AS&, T*) const {
    return RosenbrockFn<T, D>{}(c, x, grad);
  }
};

// ---- shared-memory layout + kernel ------------------------------------------------
template <class T, int D>
struct NewtonSmem {
  static constexpr int E = Shape<D>::E;
  using AS = AugStore<T, D>;
  static constexpr int kAug = D * (D + 1);                       // [matrix columns | rhs]
  static constexpr int kVecPad = ((D + 3) / 4) * 4;
  // + vec, ring, mbarrier (8 bytes); slice size kept a multiple of 16 bytes so every
  // warp's base stays aligned for 16-byte vector accesses and TMA bulk copies
  static constexpr int kWarpElems = ((kAug + kVecPad + CNO_MAX_PAST + 8 / (int)sizeof(T) + 3) / 4) * 4;
  static_assert((kAug * sizeof(T)) % 16 == 0 || D % 32 != 0, "columns must stay 16-byte aligned");
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  static constexpr int kMaxSmem = 227 * 1024;
  static constexpr int kWarpsFit = (int)(kMaxSmem / kWarpBytes);
  static constexpr int kCap = 8;
  static constexpr int kWarps = kWarpsFit > kCap ? kCap : (kWarpsFit < 1 ? 1 : kWarpsFit);
};

// One elimination step's trailing update over the SHARED-MEMORY columns [j0, j1).
template <class T, int D>
__device__ __forceinline__ void lu_update_smem(const AugStore<T, D>& A, int j0, int j1, int prow,
                                               const T (&l)[Shape<D>::E], const bool (&live)[Shape<D>::E],
                                               T* rhs_or_null) {
  constexpr int E = Shape<D>::E;
  using RV = SmemRowVec<T, D>;
  constexpr int kU = 8;
  const int lane = A.lane;
  int j = j0;
  // Columns are independent; kU of them are loaded before any is stored so the
  // LDS -> FP64 -> STS chains of different columns overlap.
#pragma unroll 1
  for (; j + kU <= j1; j += kU) {
    T u[kU], cj[kU][E];
#pragma unroll
    for (int t = 0; t < kU; ++t) {
      u[t] = A.smcol(j + t)[prow];  // broadcast
      RV::load(A.smcol(j + t), lane, cj[t]);
    }
    __syncwarp();  // every lane has read the pivot row's entries before its owner rewrites them
#pragma unroll
    for (int t = 0; t < kU; ++t) {
#pragma unroll
      for (int e = 0; e < E; ++e)
        if (live[e]) cj[t][e] = cj[t][e] - l[e] * u[t];
      RV::store(A.smcol(j + t), lane, cj[t]);
    }
  }
#pragma unroll 1
  for (; j < j1; ++j) {
    const T u = A.smcol(j)[prow];
    T cj[E];
    RV::load(A.smcol(j), lane, cj);
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (live[e]) cj[e] = cj[e] - l[e] * u;
    __syncwarp();
    RV::store(A.smcol(j), lane, cj);
  }
  if (rhs_or_null) {  // the right-hand side rides along as the last column
    const T u = rhs_or_null[prow];
    T cj[E];
    RV::load(rhs_or_null, lane, cj);
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (live[e]) cj[e] = cj[e] - l[e] * u;
    __syncwarp();
    RV::store(rhs_or_null, lane, cj);
  }
}

// this lane's rows of matrix column k
template <class T, int D>
__device__ __forceinline__ void aug_load_col(const AugStore<T, D>& A, int k, T (&col)[Shape<D>::E]) {
  AugStore<T, D>::RV::load(A.smcol(k), A.lane, col);
}
template <class T, int D>
__device__ __forceinline__ void aug_store_col(const AugStore<T, D>& A, int k, const T (&col)[Shape<D>::E]) {
  AugStore<T, D>::RV::store(A.smcol(k), A.lane, col);
}

// Any Second-mode functor (value/gradient through operator()(ctx, x, grad*), Hessian column by column
// through hess_col: cno_device.cuh) as a NewtonDescent objective -- user functors and the expression
// templates of include/cppoptlib_b200/expressions.h.  H(x) is written into the warp's store one column
// at a time; for the Armijo slope, whose d'H the kernel evaluates as a column sweep, the TRANSPOSE is
// staged, so a Hessian that is not bitwise symmetric (a product of functions) still gives the
// reference's sum_i d_i H_ij, i ascending.
template <class F>
struct SecondOrderAdapter {
  using Scalar = typename F::Scalar;
  using T = Scalar;
  static constexpr int Dim = F::Dim;
  static constexpr int Mode = 2;
  static constexpr int E = Shape<Dim>::E;
  using AS = AugStore<T, Dim>;
  static constexpr bool kHessianConstant = false;
  static constexpr bool kStageTakesTranspose = true;
  F f;
  __device__ __forceinline__ void stage(const EvalCtx& c, const T (&x)[E], const AS& A, uint64_t*, uint32_t&,
                                        bool transposed = false) const {
    __syncwarp();
    const auto st = hess_prepare(f, c, x);
#pragma unroll 1
    for (int j = 0; j < Dim; ++j) {
      T col[E];
      hess_col(f, c, x, st, j, transposed, col);
      aug_store_col<T, Dim>(A, j, col);
    }
    __syncwarp();
  }
  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E], const AS&, T*) const {
    return f(c, x, grad);
  }
};
template <class Fn, class = void>
struct FnPrefetches : std::false_type {};
template <class Fn>
struct FnPrefetches<Fn, std::void_t<decltype(&Fn::prefetch)>> : std::true_type {};
template <class Fn, class = void>
struct StageTakesTranspose : std::false_type {};
template <class Fn>
struct StageTakesTranspose<Fn, std::void_t<decltype(Fn::kStageTakesTranspose)>> : std::true_type {};

// delta = (H + shift I)^{-1} rhs by unblocked partial-pivot LU with implicit row
// exchanges.  A = [H | rhs] col-major, lane owns rows lane*E .. lane*E+E-1.  On
// return delta holds this lane's slice of the solution.
// Back substitution U x = y (pivot order), column oriented, on the factored store; vpos = the rows' final
// virtual positions, rv = this lane's rows of the right-hand side (kept in REGISTERS: a lane only ever updates its
// own rows, and the one value the others need per step -- x_k -- is broadcast from its owner).  On return delta
// holds this lane's slice of the solution.
template <class T, int D>
__device__ __forceinline__ void lu_back_substitute(const AugStore<T, D>& A, const int (&vpos)[Shape<D>::E],
                                                   T (&rv)[Shape<D>::E], T (&delta)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
  const int lane = A.lane;
  // The 64 quotients x_k = y_k / u_kk are the dependent chain of this loop.  Everything that does not depend on the
  // running right-hand side leaves it: column k-1 is loaded while step k computes, the owner of row k and the
  // reciprocal refinement of its divisor (div_rcp) are ready before y_k is, and the quotient is finished with
  // div_with's three operations.  Its range test is collected over the whole loop; when an operand fell outside
  // (rare: tiny / huge / non-finite), the loop is redone with the plain operator from the saved right-hand side.
  T rv0[E];
#pragma unroll
  for (int e = 0; e < E; ++e) rv0[e] = rv[e];
  bool all_ok = true;
  T col[E], nxt[E];
  aug_load_col<T, D>(A, D - 1, col);
#pragma unroll 1
  for (int k = D - 1; k >= 0; --k) {
    if (k > 0) aug_load_col<T, D>(A, k - 1, nxt);  // (uniform)
    T dv = T(1), nv = T(1);
    bool mine = false;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      if ((lane * E + e < D) && vpos[e] == k) {
        dv = col[e];
        nv = rv[e];
        mine = true;
      }
    }
    const unsigned owner = __ballot_sync(kFullMask, mine);
    bool ok;
    const T q = div_with(nv, dv, div_rcp(dv), ok);
    all_ok = all_ok && ok;
    const T xk = __shfl_sync(kFullMask, q, __ffs(owner) - 1);
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int row = lane * E + e;
      if ((row < D) && vpos[e] < k) rv[e] = rv[e] - col[e] * xk;
      if (row == k) delta[e] = xk;  // unknown k belongs to element k
    }
#pragma unroll
    for (int e = 0; e < E; ++e) col[e] = nxt[e];
  }
  if (uni(!all_ok)) {
#pragma unroll
    for (int e = 0; e < E; ++e) rv[e] = rv0[e];
#pragma unroll 1
    for (int k = D - 1; k >= 0; --k) {
      aug_load_col<T, D>(A, k, col);
      T xk_local = T(0);
      bool mine = false;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        if ((lane * E + e < D) && vpos[e] == k) {
          xk_local = rv[e] / col[e];
          mine = true;
        }
      }
      const unsigned owner = __ballot_sync(kFullMask, mine);
      const T xk = __shfl_sync(kFullMask, xk_local, __ffs(owner) - 1);
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const int row = lane * E + e;
        if ((row < D) && vpos[e] < k) rv[e] = rv[e] - col[e] * xk;
        if (row == k) delta[e] = xk;
      }
    }
  }
#pragma unroll
  for (int e = 0; e < E; ++e)
    if (lane * E + e >= D) delta[e] = T(0);
}

// Solve with the factors a previous lu_solve_inplace left in the store (a functor with a constant Hessian is
// factored once per instance): the right-hand side receives, in pivot order, exactly the updates it received while
// it rode along the elimination -- rhs_i -= l_ik * rhs_{pivot row k} for the rows not yet used as a pivot, l_ik
// being the multiplier stored in column k -- then the same back substitution.  Bit-identical to factoring again.
// rv = this lane's rows of the right-hand side, in registers.
template <class T, int D>
__device__ __forceinline__ void lu_resolve(const AugStore<T, D>& A, const int (&vpos)[Shape<D>::E],
                                           T (&rv)[Shape<D>::E], T (&delta)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
  const int lane = A.lane;
  T col[E], nxt[E];
  aug_load_col<T, D>(A, 0, col);
#pragma unroll 1
  for (int k = 0; k < D; ++k) {
    if (k + 1 < D) aug_load_col<T, D>(A, k + 1, nxt);  // (uniform) the next column is on its way during this step
    T u_local = T(0);
    bool mine = false;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      if ((lane * E + e < D) && vpos[e] == k) {
        u_local = rv[e];
        mine = true;
      }
    }
    const unsigned owner = __ballot_sync(kFullMask, mine);
    const T u = __shfl_sync(kFullMask, u_local, __ffs(owner) - 1);
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int row = lane * E + e;
      if ((row < D) && vpos[e] > k) rv[e] = rv[e] - col[e] * u;
    }
#pragma unroll
    for (int e = 0; e < E; ++e) col[e] = nxt[e];
  }
  lu_back_substitute<T, D>(A, vpos, rv, delta);
}

template <class T, int D>
__device__ __forceinline__ void lu_solve_inplace(const AugStore<T, D>& A, T (&delta)[Shape<D>::E],
                                                 int (&vpos)[Shape<D>::E]) {
  constexpr int E = Shape<D>::E;
  using AS = AugStore<T, D>;
  const int lane = A.lane;
  // vpos = virtual row position (what the reference's explicit swaps would give)
#pragma unroll
  for (int e = 0; e < E; ++e) vpos[e] = lane * E + e;

#pragma unroll 1
  for (int k = 0; k < D; ++k) {
    // ---- pivot: first maximal |a_ik| over virtual positions >= k ----
    T col[E];
    aug_load_col<T, D>(A, k, col);
    T best = T(-1);
    int bpos = 0x7fffffff;
    bool k_is_nan = false;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int row = lane * E + e;
      const T v = cabs(col[e]);
      const bool cand = (row < D) && (vpos[e] >= k);
      if (cand && (v > best || (v == best && vpos[e] < bpos))) { best = v; bpos = vpos[e]; }
      k_is_nan = k_is_nan || ((row < D) && (vpos[e] == k) && (v != v));
    }
    // warp arg-max: larger |v|, ties -> smaller virtual position.  A NaN at virtual position k stays the
    // pivot: the sequential scan of the specification starts from it and no comparison with a NaN is
    // true (oracle lu_solve); that also keeps the pivot position valid when every candidate is NaN.
    // Fast path (one REDUX + one vote): the high words (fp32: the whole pattern) of the lanes' best |v| decide when
    // exactly one lane holds the largest one; a NaN at position k makes its lane win outright.  Otherwise (ties, a
    // zero column, equal high words) the full comparison: low words, then the smallest position.
    unsigned hkey;
    if constexpr (sizeof(T) == 8) hkey = best < T(0) ? 0u : (unsigned)__double2hiint((double)best);
    else hkey = best < T(0) ? 0u : __float_as_uint((float)best);
    if (k_is_nan) hkey = 0xffffffffu;
    const unsigned hmax = __reduce_max_sync(kFullMask, hkey);
    const unsigned hset = __ballot_sync(kFullMask, hkey == hmax);
    int ppos;
    if (uni_likely((hset & (hset - 1u)) == 0u)) {
      ppos = __shfl_sync(kFullMask, k_is_nan ? k : bpos, __ffs(hset) - 1);
    } else {
      const T bmax = warp_max_nonneg(best < T(0) ? T(0) : best);
      const unsigned mypos = (best == bmax) ? (unsigned)bpos : 0xffffffffu;
      const int pmax = (int)__reduce_min_sync(kFullMask, mypos);
      ppos = uni(k_is_nan) ? k : pmax;
    }
    // the row at virtual position k and the pivot row exchange virtual positions
    T pivot_local = T(0);
    int prow_local = -1;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const bool is_p = (vpos[e] == ppos) && (lane * E + e < D);
      const bool is_k = (vpos[e] == k) && (lane * E + e < D);
      if (is_p) { pivot_local = col[e]; prow_local = lane * E + e; }
      vpos[e] = is_p ? k : (is_k ? ppos : vpos[e]);
    }
    const unsigned owner = __ballot_sync(kFullMask, prow_local >= 0);
    const int src = __ffs(owner) - 1;
    const T pivot = __shfl_sync(kFullMask, pivot_local, src);
    const int prow = __shfl_sync(kFullMask, prow_local, src);

    // ---- multipliers l_i = a_ik / pivot for rows not yet used as a pivot: the quotients of a lane share the pivot's
    //      reciprocal refinement and run side by side (div_rcp / div_with; the plain operator when the range test fails) ----
    T l[E];
    bool live[E];
    {
      const T rp = div_rcp(pivot);
      bool okall = true;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        live[e] = (lane * E + e < D) && (vpos[e] > k);
        bool ok;
        l[e] = div_with(live[e] ? col[e] : T(1), pivot, rp, ok);
        okall = okall && ok;
      }
      if (uni_unlikely(!okall)) {
#pragma unroll
        for (int e = 0; e < E; ++e) l[e] = col[e] / pivot;
      }
#pragma unroll
      for (int e = 0; e < E; ++e) {
        l[e] = live[e] ? l[e] : T(0);
        col[e] = live[e] ? l[e] : col[e];
      }
    }
    aug_store_col<T, D>(A, k, col);
    // ---- trailing update, columns k+1 .. D-1 and the right-hand side ----
    lu_update_smem<T, D>(A, k + 1, D, prow, l, live, A.rhs());  // (k = D - 1: the rhs only)
    __syncwarp();
  }
  T rv[E];
  AS::RV::load(A.rhs(), lane, rv);  // (the lu_update_smem calls above end with a warp sync)
  lu_back_substitute<T, D>(A, vpos, rv, delta);
}

template <class Fn>
__global__ void __launch_bounds__(NewtonSmem<typename Fn::Scalar, Fn::Dim>::kWarps * 32, 1)
newton_minimize_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x0,
                       const long long batch, const StopParams<typename Fn::Scalar> stop,
                       const BatchOut<typename Fn::Scalar> out,
                       unsigned long long* __restrict__ queue) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  constexpr int E = Shape<D>::E;
  using SMN = NewtonSmem<T, D>;
  using AS = AugStore<T, D>;
  using SV = SmemRowVec<T, D>;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T* const aug = reinterpret_cast<T*>(smem_raw) + (size_t)warp * SMN::kWarpElems;
  T* const vec = aug + SMN::kAug;
  T* const ring = vec + SMN::kVecPad;
  uint64_t* const bar = reinterpret_cast<uint64_t*>(ring + CNO_MAX_PAST);
  uint32_t parity = 0;
  const AS A{aug, lane};
  if (lane == 0) {
    mbar_init(bar, 1);
#ifndef CNO_WARP_EMULATION
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  }
  __syncwarp();

  // (the work queue is read one instance ahead, for the functors that prefetch their next block into L2)
  unsigned long long bnext = 0;
  if (lane == 0) bnext = atomicAdd(queue, 1ULL);
  bnext = __shfl_sync(kFullMask, bnext, 0);
  for (;;) {
    const unsigned long long b = bnext;
    if (uni(b >= (unsigned long long)batch)) break;
    if (lane == 0) bnext = atomicAdd(queue, 1ULL);
    bnext = __shfl_sync(kFullMask, bnext, 0);
    const EvalCtx ctx{lane, (long long)b, nullptr};

    T x[E], g[E];
    load_row<T, D>(x0 + b * D, lane, x);
    // A functor with a CONSTANT Hessian (kHessianConstant: the dense quadratic) is factored ONCE per instance:
    // the store keeps the LU factors of H + 1e-5 I, later iterations re-solve with them (lu_resolve: the same
    // arithmetic as factoring again), and evaluations / the Armijo slope read the matrix from global memory.
    fn.stage(ctx, x, A, bar, parity);
    T f = fn(ctx, x, &g, A, vec);  // solver.h:189-192
    uint32_t nfev = 1;
    bool factored = false;
    int vpos[E];
#pragma unroll
    for (int e = 0; e < E; ++e) vpos[e] = lane * E + e;

    ProgressState<T> prog;
    prog.num_iterations = 0;
    prog.x_delta_violations = 0;
    prog.f_delta_violations = 0;
    prog.x_delta = prog.f_delta = prog.gradient_norm = T(0);
    prog.ring_size = 0;
    prog.ring_pos = 0;
    prog.status = CNO_STATUS_NOT_STARTED;
    bool staged = true;  // the store currently holds the unshifted H(x)

    do {  // solver.h:196-220
      // ---- newton_descent.h:73-76 ----
      nfev++;  // function(current.x, &gradient, &hessian)
      T delta[E];
      if (uni(Fn::kHessianConstant && factored)) {
        T rv[E];
#pragma unroll
        for (int e = 0; e < E; ++e) rv[e] = -g[e];
        lu_resolve<T, D>(A, vpos, rv, delta);
      } else {
      if (!staged) fn.stage(ctx, x, A, bar, parity);
      // hessian += safe_guard * I ; rhs = -gradient
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const int row = lane * E + e;
        if (row < D) {
          A.rhs()[row] = -g[e];
          A.smcol(row)[row] += T(1e-5);
        }
      }
      __syncwarp();
      lu_solve_inplace<T, D>(A, delta, vpos);
      factored = true;
      }

      // ---- Armijo<F,2>::Search (armijo.h:82-101) ----
      nfev++;                            // f_in = function(x, &gradient, &hessian)
      const T cc = T(0.2), rho = T(0.9);
      T sd[E], r[E];
      const T half_cc = T(0.5) * cc * cc;
#pragma unroll
      for (int e = 0; e < E; ++e) sd[e] = half_cc * delta[e];
      T alpha = T(1.0);
      T xt[E], gt[E];
#pragma unroll
      for (int e = 0; e < E; ++e) xt[e] = x[e] + alpha * delta[e];
      T ft;
      if constexpr (Fn::kHessianConstant) {
        // ((0.5 c^2) d') H and the first trial evaluation in one pass over A (global memory / L2; the store keeps the
        // factors; the right-hand-side column of the store is free after the solve and serves as the second vector)
        ft = fn.hess_times_and_eval(ctx, sd, r, xt, gt, vec, A.rhs());
      } else {
        // unshifted H(x) again (its transpose where the functor tells them apart: the slope below is d'H)
        if constexpr (StageTakesTranspose<Fn>::value) fn.stage(ctx, x, A, bar, parity, true);
        else fn.stage(ctx, x, A, bar, parity);
        __syncwarp();
        SV::store(vec, lane, sd);
        __syncwarp();
        aug_gemv<T, D>(A, vec, r);  // ((0.5 c^2) d') H, H bitwise symmetric (or its staged transpose)
      }
      T p1 = lane_dot<T, E>(g, delta), p2 = lane_dot<T, E>(r, delta);
      warp_sum2(p1, p2);
      const T cache = cc * p1 + p2;
      if constexpr (!Fn::kHessianConstant) ft = fn(ctx, xt, &gt, A, vec);
      nfev++;
      while (uni(ft > f + alpha * cache)) {
        alpha *= rho;
#pragma unroll
        for (int e = 0; e < E; ++e) xt[e] = x[e] + alpha * delta[e];
        ft = fn(ctx, xt, &gt, A, vec);
        nfev++;
      }
      // ---- x + rate*delta (:80), re-evaluation (solver.h:210-216) = last trial ----
      nfev++;
      T sdx[E];
#pragma unroll
      for (int e = 0; e < E; ++e) sdx[e] = xt[e] - x[e];
      const T prev_value = f;
      const T x_delta = warp_maxabs<T, E>(sdx);
#pragma unroll
      for (int e = 0; e < E; ++e) { x[e] = xt[e]; g[e] = gt[e]; }
      f = ft;
      const T gnorm_inf = warp_maxabs<T, E>(g);
      const T x_inf = warp_maxabs<T, E>(x);
      nfev++;  // Progress::Update's Hessian evaluation (progress.h:206-207)
      staged = false;  // (a non-constant Hessian is staged again at the new x; a constant one stays factored)
      progress_update<T>(prog, stop, ring, lane, prev_value, f, x_delta, gnorm_inf, x_inf);
      if constexpr (FnPrefetches<Fn>::value) {
        // the next instance's block into L2, one iteration ahead (not for the whole solve: two blocks per warp in
        // flight all the time would fill the L2 and make the passes over the current block miss)
        if (uni(prog.num_iterations == 1 && bnext < (unsigned long long)batch)) fn.prefetch((long long)bnext, lane);
      }
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

// ---- Progress::condition_hessian on request (solver/progress.h:203-210) ------------------------------------------
// condition_hessian = hessian.norm() * hessian.inverse().norm() at the state's x, which the reference evaluates in
// every Progress::Update of a Second-mode function (one Hessian evaluation plus a full inverse: d solves) although no
// preset tests it.  The fused solve kernels do not carry it; this kernel computes it for a batch of points -- the
// final states of a solve, or the snapshots a callback sees -- one warp per point, with the store and the LU of
// NewtonDescent: H(x) staged, factored ONCE, column j of the inverse = the re-solve with e_j (the same bits as the
// d separate lu().solve(e_j) of the specification, oracle condition_hessian()).  Frobenius norms follow the policy's
// sum over the d*d squared coefficients in column-major order: lane l owns the d*d/32 consecutive coefficients
// l*E2 .. l*E2+E2-1 (in-lane binary tree), then the cross-lane policy sum.
//   D = 64: a lane's coefficients are two whole columns; a column's tree is the owner lanes' in-lane pairs followed by
//           an ASCENDING xor butterfly (1, 2, 4, 8, 16 = the binary tree over the column's 64 rows), so columns are
//           reduced where they live (shared memory or the registers of a solve) -- no d*d scratch;
//   else:   the inverse is written to a d*d shared-memory scratch and both matrices are read linearly.
template <class T, int D>
struct ConditionSmem {
  using NS = NewtonSmem<T, D>;
  static constexpr bool kColumnwise = (D == 64);
  static constexpr int kInv = kColumnwise ? 0 : ((D * D + 3) / 4) * 4;
  static constexpr int kWarpElems = NS::kWarpElems + kInv;
  static constexpr size_t kWarpBytes = (size_t)kWarpElems * sizeof(T);
  static constexpr int kWarpsFit = (int)(NS::kMaxSmem / kWarpBytes);
  static constexpr int kWarps = kWarpsFit > NS::kCap ? NS::kCap : (kWarpsFit < 1 ? 1 : kWarpsFit);
};

// binary tree over a column's D = 64 squared entries (lane l holds rows 2l, 2l+1), the result in every lane
template <class T>
__device__ __forceinline__ T column_tree64(const T (&c)[2]) {
  T p = c[0] * c[0] + c[1] * c[1];
#pragma unroll
  for (int off = 1; off <= 16; off <<= 1) p = p + __shfl_xor_sync(kFullMask, p, off);
  return p;
}

template <class Fn>
__global__ void __launch_bounds__(ConditionSmem<typename Fn::Scalar, Fn::Dim>::kWarps * 32, 1)
condition_hessian_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ xs, const long long batch,
                         typename Fn::Scalar* __restrict__ out, unsigned long long* __restrict__ queue) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  constexpr int E = Shape<D>::E;
  using SMN = NewtonSmem<T, D>;
  using CS = ConditionSmem<T, D>;
  using AS = AugStore<T, D>;

  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T* const aug = reinterpret_cast<T*>(smem_raw) + (size_t)warp * CS::kWarpElems;
  T* const vec = aug + SMN::kAug;
  T* const ring = vec + SMN::kVecPad;
  uint64_t* const bar = reinterpret_cast<uint64_t*>(ring + CNO_MAX_PAST);
  T* const inv = aug + SMN::kWarpElems;  // (kInv scalars; not used when kColumnwise)
  uint32_t parity = 0;
  const AS A{aug, lane};
  if (lane == 0) {
    mbar_init(bar, 1);
#ifndef CNO_WARP_EMULATION
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  }
  __syncwarp();

  for (;;) {
    unsigned long long b = 0;
    if (lane == 0) b = atomicAdd(queue, 1ULL);
    b = __shfl_sync(kFullMask, b, 0);
    if (uni(b >= (unsigned long long)batch)) break;
    const EvalCtx ctx{lane, (long long)b, nullptr};
    T x[E];
    load_row<T, D>(xs + b * D, lane, x);
    fn.stage(ctx, x, A, bar, parity);  // the store holds H(x)
    __syncwarp();

    // ---- sum of the squared coefficients of H, policy order ----
    T part_h = T(0), part_i = T(0);  // this lane's partials of the two sums
    if constexpr (CS::kColumnwise) {
#pragma unroll 1
      for (int j = 0; j < D; ++j) {
        T col[E];
        aug_load_col<T, D>(A, j, col);
        const T c = column_tree64<T>(col);
        if (lane == (j >> 1)) part_h = (j & 1) ? (part_h + c) : c;
      }
    } else {
      constexpr int E2 = (D * D + 31) / 32;
      T v[E2];
#pragma unroll
      for (int t = 0; t < E2; ++t) {
        const int i = lane * E2 + t;
        const T h = (i < D * D) ? aug[i] : T(0);
        v[t] = h * h;
      }
      part_h = lane_tree<T, E2>(v);
    }

    // ---- the inverse, column by column: factor once with e_0 riding along, then re-solve ----
    int vpos[E];
#pragma unroll 1
    for (int j = 0; j < D; ++j) {
      T delta[E];
      if (j == 0) {  // uniform
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int row = lane * E + e;
          if (row < D) A.rhs()[row] = (row == 0) ? T(1) : T(0);
        }
        __syncwarp();
        lu_solve_inplace<T, D>(A, delta, vpos);
      } else {
        T rv[E];
#pragma unroll
        for (int e = 0; e < E; ++e) rv[e] = (lane * E + e == j) ? T(1) : T(0);
        lu_resolve<T, D>(A, vpos, rv, delta);
      }
      if constexpr (CS::kColumnwise) {
        const T c = column_tree64<T>(delta);
        if (lane == (j >> 1)) part_i = (j & 1) ? (part_i + c) : c;
      } else {
#pragma unroll
        for (int e = 0; e < E; ++e)
          if (lane * E + e < D) inv[j * D + lane * E + e] = delta[e];
      }
    }
    if constexpr (!CS::kColumnwise) {
      constexpr int E2 = (D * D + 31) / 32;
      __syncwarp();
      T v[E2];
#pragma unroll
      for (int t = 0; t < E2; ++t) {
        const int i = lane * E2 + t;
        const T h = (i < D * D) ? inv[i] : T(0);
        v[t] = h * h;
      }
      part_i = lane_tree<T, E2>(v);
      __syncwarp();
    }
    warp_sum2(part_h, part_i);
    if (lane == 0) out[b] = csqrt(part_h) * csqrt(part_i);
    __syncwarp();
  }
}

}  // namespace cno

#endif  // CNO_NEWTON_CUH_
