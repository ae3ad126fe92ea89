// tests/cpp/al_user_problems.cuh -- the functor-constrained test problems of AugmentedLagrangian (tests/test_al_user.py,
// tests/test_al_user_gpu.py) as device functors.  The same source is compiled by nvcc into the GPU test library
// (al_user_functions.cu) and by g++ under the warp emulation (tests/emu/emu_al_user.cc).  Each problem has a twin in
// oracle/ref_al_user.cc (cno_ref_al_minimize_expr) built from the reference's own FunctionCRTP functors and operators.
//
// Problem ids (keep in step with oracle/ref_al_user.cc AL_P_* and tests/al_user_ref.py AL_P_*):
//   0  min -x0 x1  s.t.  48 - x0^2 - 2 x1^2 >= 0                       d = 2 f64  (augmented_lagrangian_test.cc Hs029)
//   1  (x0-1)^2 + (x1-2)^2, eq x0 - 0.5, ineq 2 - (x0 + x1)             d = 2 f64  (src/examples/constrained_simple.cc)
//   2  0.5 |x|^2, eq X0MinusTarget(1) - 0.5, ineq 0.5 - X0MinusTarget(1) d = 2 f64  (composites as constraints)
//   3  Rosenbrock + 0.5 HalfSquaredNorm, eq HalfSquaredNorm - 2, ineq 3 - Bowl(0.25)   d = 8, 128 f64; 37 f32
//   4  Rosenbrock, ineq r_b^2 - x.x >= 0, r_b = data[b] per instance     d = 37 f64
//   5  Rosenbrock, eq SqNormRow(0), ineq AffineRow(1) on [a | t] rows data (stride 0 = shared)   d = 8, 128 f64; 8 f32
//   6  Bowl(0.5), no constraints                                          d = 16 f64
//   7  DiagonalQuadratic2dSecond (Second mode), eq X0MinusTarget(1)       d = 2 f64
#ifndef CNO_TESTS_AL_USER_PROBLEMS_CUH_
#define CNO_TESTS_AL_USER_PROBLEMS_CUH_

#include "cno_device.cuh"
#include "cno_functors.cuh"
#include "cppoptlib_b200/constraint_list.h"
#include "cppoptlib_b200/expressions.h"
#include "cppoptlib_b200/modes.h"

namespace alu {

namespace fn = cppoptlib::function;
using cno::EvalCtx;
using fn::operator+;  // (the composite operators of expressions.h)
using fn::operator-;
using fn::operator*;

// the names of both vocabularies: the reference's (ScalarType, Dimension, Differentiability) and the device concept's
template <class T, int D, int M = 1>
struct Leaf {
  using ScalarType = T;
  static constexpr int Dimension = D;
  static constexpr fn::DifferentiabilityMode Differentiability = static_cast<fn::DifferentiabilityMode>(M);
  using Scalar = T;
  static constexpr int Dim = D;
  static constexpr int Mode = M;
  static constexpr int E = cno::Shape<D>::E;
};

// a built-in family as a leaf of composites
template <class Fn>
struct Builtin : Leaf<typename Fn::Scalar, Fn::Dim> {
  using T = typename Fn::Scalar;
  static constexpr int E = cno::Shape<Fn::Dim>::E;
  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E]) const { return Fn{}(c, x, grad); }
};
template <class T, int D>
using Rosenbrock = Builtin<cno::RosenbrockFn<T, D>>;
template <class T, int D>
using HalfSquaredNorm = Builtin<cno::HalfSquaredNormFn<T, D>>;

// d = 2: x0 in lane 0, x1 in lane 1 (E = 1)
__device__ __forceinline__ double x0_of(const double (&x)[1]) { return __shfl_sync(cno::kFullMask, x[0], 0); }
__device__ __forceinline__ double x1_of(const double (&x)[1]) { return __shfl_sync(cno::kFullMask, x[0], 1); }
__device__ __forceinline__ void grad2(const EvalCtx& c, double (*grad)[1], double g0, double g1) {
  if (grad) (*grad)[0] = (c.lane == 0) ? g0 : ((c.lane == 1) ? g1 : 0.0);
}

// augmented_lagrangian_test.cc: ProductObjective3D, f = -x0 x1
struct NegProduct : Leaf<double, 2> {
  __device__ double operator()(const EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    const double x0 = x0_of(x), x1 = x1_of(x);
    grad2(c, grad, -x1, -x0);
    return -x0 * x1;
  }
};
// augmented_lagrangian_test.cc: Hs029Ellipse, c = 48 - x0^2 - 2 x1^2 >= 0
struct Ellipse : Leaf<double, 2> {
  __device__ double operator()(const EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    const double x0 = x0_of(x), x1 = x1_of(x);
    grad2(c, grad, -2.0 * x0, -4.0 * x1);
    return 48.0 - x0 * x0 - 2.0 * x1 * x1;
  }
};
// constrained_simple.cc: QuadraticObjective2, f = (x0-1)^2 + (x1-2)^2
struct QuadraticAt12 : Leaf<double, 2> {
  __device__ double operator()(const EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    const double x0 = x0_of(x), x1 = x1_of(x);
    grad2(c, grad, 2 * (x0 - 1), 2 * (x1 - 2));
    return (x0 - 1) * (x0 - 1) + (x1 - 2) * (x1 - 2);
  }
};
// constrained_simple.cc: InequalityConstraint3, c = 2 - (x0 + x1) >= 0
struct SumUpperBound : Leaf<double, 2> {
  __device__ double operator()(const EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    const double x0 = x0_of(x), x1 = x1_of(x);
    grad2(c, grad, -1.0, -1.0);
    return 2 - (x0 + x1);
  }
};
// augmented_lagrangian_test.cc: X0MinusTarget, c = x0 - target (constrained_simple.cc's equality is target 0.5)
struct X0MinusTarget : Leaf<double, 2> {
  double target;
  __device__ double operator()(const EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    grad2(c, grad, 1.0, 0.0);
    return x0_of(x) - target;
  }
};
// augmented_lagrangian_test.cc: DiagonalQuadratic2dSecond, f = 2 x0^2 + x1^2 (Second mode)
struct DiagonalQuadratic2dSecond : Leaf<double, 2, 2> {
  __device__ double operator()(const EvalCtx& c, const double (&x)[1], double (*grad)[1]) const {
    const double x0 = x0_of(x), x1 = x1_of(x);
    grad2(c, grad, 4.0 * x0, 2.0 * x1);
    return 2 * x0 * x0 + x1 * x1;
  }
  __device__ void hess_diag(const EvalCtx& c, const double (&)[1], double (&h)[1]) const {
    h[0] = (c.lane == 0) ? 4.0 : ((c.lane == 1) ? 2.0 : 0.0);
  }
  __device__ void hess_col(const EvalCtx& c, const double (&)[1], int j, bool, double (&col)[1]) const {
    col[0] = (c.lane == j) ? ((j == 0) ? 4.0 : 2.0) : 0.0;
  }
};
// f = sum_i a_i (x_i - c)^2, a_i = 1 + i/8 (tests/cpp/user_functions.cu: Bowl)
template <class T, int D>
struct Bowl : Leaf<T, D> {
  static constexpr int E = cno::Shape<D>::E;
  T c;
  __device__ T operator()(const EvalCtx& ctx, const T (&x)[E], T (*grad)[E]) const {
    T t[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int i = ctx.lane * E + e;
      const T a = T(1.0) + T(0.125) * i;
      const T r = x[e] - c;
      t[e] = (i < D) ? a * r * r : T(0);
      if (grad) (*grad)[e] = (i < D) ? T(2.0) * a * r : T(0);
    }
    return cno::warp_sum(cno::lane_tree<T, E>(t));
  }
};
// c = r_b^2 - x.x >= 0 with the radius of instance b read through ctx.instance
template <class T, int D>
struct BallOfInstance : Leaf<T, D> {
  static constexpr int E = cno::Shape<D>::E;
  const T* radius;  // [B]
  __device__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E]) const {
    const T r = radius[c.instance];
    if (grad) {
#pragma unroll
      for (int e = 0; e < E; ++e) (*grad)[e] = T(-2) * x[e];
    }
    return r * r - cno::warp_sum(cno::lane_dot<T, E>(x, x));
  }
};
// Row idx of [a | t] rows as cno_al_minimize reads it (csrc/cno_auglag.cuh: al_con_eval): a.x - t, and t - x.x
template <class T, int D>
struct AffineRow : Leaf<T, D> {
  static constexpr int E = cno::Shape<D>::E;
  const T* rows;
  long long stride;
  int idx;
  __device__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E]) const {
    const T* row = rows + c.instance * stride + (long long)idx * (D + 1);
    T a[E];
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int i = c.lane * E + j;
      a[j] = (i < D) ? __ldg(row + i) : T(0);
    }
    if (grad) {
#pragma unroll
      for (int j = 0; j < E; ++j) (*grad)[j] = a[j];
    }
    return cno::warp_sum(cno::lane_dot<T, E>(x, a)) - __ldg(row + D);
  }
};
template <class T, int D>
struct SqNormRow : Leaf<T, D> {
  static constexpr int E = cno::Shape<D>::E;
  const T* rows;
  long long stride;
  int idx;
  __device__ T operator()(const EvalCtx& c, const T (&x)[E], T (*grad)[E]) const {
    const T t = __ldg(rows + c.instance * stride + (long long)idx * (D + 1) + D);
    if (grad) {
#pragma unroll
      for (int j = 0; j < E; ++j) (*grad)[j] = T(-2) * x[j];
    }
    return t - cno::warp_sum(cno::lane_dot<T, E>(x, x));
  }
};

// ---- the problems: Obj, Eq, In, and make() from the test's data pointer / stride ----
template <class O, class Q, class I>
struct Parts {
  O objective;
  Q equality_constraints;
  I inequality_constraints;
};

struct P0 {
  using Obj = NegProduct;
  using Eq = fn::Equalities<>;
  using In = fn::Inequalities<Ellipse>;
  static Parts<Obj, Eq, In> make(const void*, long long) { return {Obj{}, Eq{}, In{Ellipse{}}}; }
};
struct P1 {
  using Obj = QuadraticAt12;
  using Eq = fn::Equalities<X0MinusTarget>;
  using In = fn::Inequalities<SumUpperBound>;
  static Parts<Obj, Eq, In> make(const void*, long long) {
    X0MinusTarget e;
    e.target = 0.5;
    return {Obj{}, Eq{e}, In{SumUpperBound{}}};
  }
};
struct P2 {
  using Obj = HalfSquaredNorm<double, 2>;
  using EqC = decltype(X0MinusTarget{} - 0.5);
  using InC = decltype(0.5 - X0MinusTarget{});
  using Eq = fn::Equalities<EqC>;
  using In = fn::Inequalities<InC>;
  static Parts<Obj, Eq, In> make(const void*, long long) {
    X0MinusTarget t;
    t.target = 1.0;
    return {Obj{}, Eq{t - 0.5}, In{0.5 - t}};
  }
};
template <class T, int D>
struct P3 {
  using Obj = decltype(Rosenbrock<T, D>{} + T(0.5) * HalfSquaredNorm<T, D>{});
  using EqC = decltype(HalfSquaredNorm<T, D>{} - T(2));
  using InC = decltype(T(3) - Bowl<T, D>{});
  using Eq = fn::Equalities<EqC>;
  using In = fn::Inequalities<InC>;
  static Parts<Obj, Eq, In> make(const void*, long long) {
    Bowl<T, D> bowl;
    bowl.c = T(0.25);
    return {Rosenbrock<T, D>{} + T(0.5) * HalfSquaredNorm<T, D>{}, Eq{HalfSquaredNorm<T, D>{} - T(2)}, In{T(3) - bowl}};
  }
};
struct P4 {
  using Obj = Rosenbrock<double, 37>;
  using Eq = fn::Equalities<>;
  using In = fn::Inequalities<BallOfInstance<double, 37>>;
  static Parts<Obj, Eq, In> make(const void* data, long long) {
    BallOfInstance<double, 37> ball;
    ball.radius = static_cast<const double*>(data);
    return {Obj{}, Eq{}, In{ball}};
  }
};
template <class T, int D>
struct P5 {
  using Obj = Rosenbrock<T, D>;
  using Eq = fn::Equalities<SqNormRow<T, D>>;
  using In = fn::Inequalities<AffineRow<T, D>>;
  static Parts<Obj, Eq, In> make(const void* data, long long stride) {
    const T* rows = static_cast<const T*>(data);
    SqNormRow<T, D> sphere;
    sphere.rows = rows;
    sphere.stride = stride;
    sphere.idx = 0;
    AffineRow<T, D> halfspace;
    halfspace.rows = rows;
    halfspace.stride = stride;
    halfspace.idx = 1;
    return {Obj{}, Eq{sphere}, In{halfspace}};
  }
};
struct P6 {
  using Obj = Bowl<double, 16>;
  using Eq = fn::Equalities<>;
  using In = fn::Inequalities<>;
  static Parts<Obj, Eq, In> make(const void*, long long) {
    Obj bowl;
    bowl.c = 0.5;
    return {bowl, Eq{}, In{}};
  }
};
struct P7 {
  using Obj = DiagonalQuadratic2dSecond;
  using Eq = fn::Equalities<X0MinusTarget>;
  using In = fn::Inequalities<>;
  static Parts<Obj, Eq, In> make(const void*, long long) {
    X0MinusTarget e;
    e.target = 1.0;
    return {Obj{}, Eq{e}, In{}};
  }
};

using P3d8 = P3<double, 8>;
using P3d128 = P3<double, 128>;
using P3f37 = P3<float, 37>;
using P5d8 = P5<double, 8>;
using P5d128 = P5<double, 128>;
using P5f8 = P5<float, 8>;

}  // namespace alu

// X(tag, id, dtype, d, Spec): every compiled (problem, dtype, d)
#define ALU_PROBLEMS(X)                                                                                          \
  X(alu_p0, 0, CNO_F64, 2, alu::P0) X(alu_p1, 1, CNO_F64, 2, alu::P1) X(alu_p2, 2, CNO_F64, 2, alu::P2)           \
  X(alu_p3d8, 3, CNO_F64, 8, alu::P3d8) X(alu_p3d128, 3, CNO_F64, 128, alu::P3d128)                              \
  X(alu_p3f37, 3, CNO_F32, 37, alu::P3f37) X(alu_p4, 4, CNO_F64, 37, alu::P4) X(alu_p5d8, 5, CNO_F64, 8, alu::P5d8) \
  X(alu_p5d128, 5, CNO_F64, 128, alu::P5d128) X(alu_p5f8, 5, CNO_F32, 8, alu::P5f8) X(alu_p6, 6, CNO_F64, 16, alu::P6) \
  X(alu_p7, 7, CNO_F64, 2, alu::P7)

#endif  // CNO_TESTS_AL_USER_PROBLEMS_CUH_
