// cppoptlib_b200/expressions.h -- function composition on the device: the expression templates of
// the reference (include/cppoptlib/function_expressions.h:45-518) as VALUE types over the
// warp-cooperative device-functor concept (cppnumericalsolvers_b200/csrc/cno_functors.cuh).
//
//   reference                                   here (namespace cppoptlib::function)
//   ------------------------------------------  -------------------------------------------------
//   :45-72   ConstExpression<T, Mode, Dim>      ConstExpression<T, Mode, Dim>
//   :74-90   MinDifferentiability[Mode]         MinDifferentiability / MinDifferentiabilityMode
//   :93-143  AddExpression<F, G>                AddExpression<F, G>
//   :146-196 SubExpression<F, G>                SubExpression<F, G>
//   :199-255 MulExpression<F>  (c == 0 short    MulExpression<F>   (same short cut: the source is
//            cut :219-227)                                          not evaluated at all)
//   :258-315 ProdExpression<F, G>               ProdExpression<F, G>
//   :318-399 MinZero / MaxZeroExpression<F>     MinZeroExpression / MaxZeroExpression<F>
//   :403-518 operator+ - * (function, scalar)   the same free operators
//   function_base.h:151-189 ModeDowngradeAdapter   ModeDowngrade<F, TargetMode>
//
// A node holds its operands BY VALUE and is trivially copyable, so a whole expression tree is one POD
// that travels to the kernel as a launch argument -- the reference's unique_ptr/clone() machinery and
// its per-evaluation temporaries (grad_f, grad_g, hess_f, hess_g: function_expressions.h:118-123) have
// no device counterpart.  What IS kept, node by node, is the reference's arithmetic: the same values
// are formed in the same order (e.g. Prod's gradient is gx*grad_f + fx*grad_g, element by element),
// so a composite built here and the same composite built from the reference's own operators on the
// CPU agree bit for bit (tests/test_expressions_gpu.py against oracle/_ref).
//
// Host translation units (g++) see the types, constructors and operators; the __device__ bodies are
// compiled by nvcc only.  Instantiate a composite for the device with
//   using H = decltype(f + 0.5 * g);
//   CNO_DECLARE_FUNCTION(h, H)  CNO_INSTANTIATE_FUNCTION(h, H)          (device.cuh)
//
// Second mode: a functor may also expose
//   void hess_diag(ctx, x, T (&h)[E]) const                     diagonal (Lbfgs's preconditioner branch)
//   HessState hess_prepare(ctx, x) const                         (optional) per-x values shared by all columns
//   void hess_col(ctx, x, [state,] int j, bool transposed, T (&col)[E]) const
//        this lane's rows of column j of the Hessian -- or of ROW j when `transposed` (NewtonDescent's
//        Armijo slope needs d'H, and a product's Hessian is not bitwise symmetric)
// and every node composes them the way the reference composes hess_f / hess_g.
//
// Group form (fp64, First mode; cno_functors.cuh): a node has
//   double operator()(const cno::GroupEvalCtx<W>&, const double (&x)[4], double (*grad)[4]) const
// when all its children have it, with the same arithmetic as its one-warp operator() (both are eval() below).  A
// composite of group-form leaves is then a group functor, which Lbfgs runs on the group kernel at d = 1024.  A node
// itself takes no sum and touches no shared memory, so the barrier rule of the group form (cno_lbfgs_group.cuh:
// group_neighbours) holds for a composite when it holds for each leaf.
#ifndef CPPOPTLIB_B200_EXPRESSIONS_H_
#define CPPOPTLIB_B200_EXPRESSIONS_H_

#include <type_traits>
#include <utility>

#include "modes.h"

#if defined(__CUDACC__) || defined(CNO_WARP_EMULATION)  // (tests/emu runs the same device bodies on the CPU)
#define CNO_DEVICE_CODE 1
#include "cno_device.cuh"
#define CNO_HD __host__ __device__ __forceinline__
#define CNO_D __device__ __forceinline__
#else
#define CNO_HD inline
#endif

namespace cppoptlib {
namespace function {

// function_expressions.h:74-90
template <DifferentiabilityMode A, DifferentiabilityMode B>
struct MinDifferentiabilityMode {
  static constexpr DifferentiabilityMode value = (static_cast<int>(A) < static_cast<int>(B) ? A : B);
};
template <class F, class G>
struct MinDifferentiability {
  static constexpr DifferentiabilityMode value =
      MinDifferentiabilityMode<F::Differentiability, G::Differentiability>::value;
};

namespace expr_detail {
template <int D> struct Elems { static constexpr int E = (D + 31) / 32; };

// The members every node shares (both vocabularies: the reference's and the device concept's).
template <class TScalar, DifferentiabilityMode TMode, int TDimension>
struct NodeBase {
  using ScalarType = TScalar;
  static constexpr int Dimension = TDimension;
  static constexpr DifferentiabilityMode Differentiability = TMode;
  using Scalar = TScalar;
  static constexpr int Dim = TDimension;
  static constexpr int Mode = static_cast<int>(TMode);
  static constexpr int E = Elems<TDimension>::E;
};

template <class F, class = void>
struct IsFunction : std::false_type {};
template <class F>
struct IsFunction<F, std::void_t<decltype(F::Differentiability), decltype(F::Dimension), typename F::ScalarType>>
    : std::true_type {};

#ifdef CNO_DEVICE_CODE
using cno::EvalCtx;

// elements past Dimension stay exactly zero (they take part in every lane-blocked sum)
template <int D, class T, int E>
CNO_D void mask_pad(int lane, T (&v)[E]) {
  if constexpr (D % 32 != 0) {
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (lane * E + e >= D) v[e] = T(0);
  }
}
template <class T, int E>
CNO_D void set_zero(T (&v)[E]) {
#pragma unroll
  for (int e = 0; e < E; ++e) v[e] = T(0);
}

using cno::HessStateOf;
using cno::hess_col;
using cno::hess_prepare;
template <class T, int E>
CNO_D T bcast_elem(const T (&v)[E], int j) { return cno::lane_bcast<T, E>(v, j); }

// every operand has the group form of W warps
template <int W, class... Fs>
struct AllGroupForm : std::bool_constant<(cno::HasGroupForm<Fs, W>::value && ...)> {};
#endif  // CNO_DEVICE_CODE
}  // namespace expr_detail

// ---- function_expressions.h:45-72 ------------------------------------------------------------
template <class TScalar, DifferentiabilityMode TMode = DifferentiabilityMode::Second, int TDimension = -1>
struct ConstExpression : expr_detail::NodeBase<TScalar, TMode, TDimension> {
  using Base = expr_detail::NodeBase<TScalar, TMode, TDimension>;
  TScalar c;
  CNO_HD explicit ConstExpression(TScalar c_ = TScalar(0)) : c(c_) {}
#ifdef CNO_DEVICE_CODE
  using T = TScalar;
  static constexpr int E = Base::E;
  CNO_D T operator()(const cno::EvalCtx& ctx, const T (&x)[E], T (*grad)[E]) const { return eval(ctx, x, grad); }
  template <int W>
  CNO_D T operator()(const cno::GroupEvalCtx<W>& ctx, const T (&x)[4], T (*grad)[4]) const { return eval(ctx, x, grad); }
  template <class Ctx, int N>
  CNO_D T eval(const Ctx&, const T (&)[N], T (*grad)[N]) const {
    if (grad) expr_detail::set_zero(*grad);
    return c;
  }
  CNO_D void hess_diag(const cno::EvalCtx&, const T (&)[E], T (&h)[E]) const { expr_detail::set_zero(h); }
  CNO_D void hess_col(const cno::EvalCtx&, const T (&)[E], int, bool, T (&col)[E]) const { expr_detail::set_zero(col); }
#endif
};

// ---- function_expressions.h:93-143 -----------------------------------------------------------
template <class F, class G, DifferentiabilityMode TMode = MinDifferentiability<F, G>::value>
struct AddExpression : expr_detail::NodeBase<typename F::ScalarType, TMode, F::Dimension> {
  static_assert(F::Dimension == G::Dimension, "Compile-time dimension mismatch: F and G must have the same dimension.");
  static_assert(std::is_same<typename F::ScalarType, typename G::ScalarType>::value,
                "Compile-time scalar-type mismatch: F and G must have the same scalar type.");
  using Base = expr_detail::NodeBase<typename F::ScalarType, TMode, F::Dimension>;
  F f;
  G g;
  CNO_HD AddExpression(const F& f_, const G& g_) : f(f_), g(g_) {}
#ifdef CNO_DEVICE_CODE
  using T = typename F::ScalarType;
  static constexpr int E = Base::E;
  CNO_D T operator()(const cno::EvalCtx& c, const T (&x)[E], T (*grad)[E]) const { return eval(c, x, grad); }
  template <int W, class F_ = F, class G_ = G, class = std::enable_if_t<expr_detail::AllGroupForm<W, F_, G_>::value>>
  CNO_D T operator()(const cno::GroupEvalCtx<W>& c, const T (&x)[4], T (*grad)[4]) const { return eval(c, x, grad); }
  template <class Ctx, int N>
  CNO_D T eval(const Ctx& c, const T (&x)[N], T (*grad)[N]) const {
    T gg[N];
    const T fx_f = f(c, x, grad);
    const T fx_g = g(c, x, grad ? &gg : nullptr);
    if (grad) {
#pragma unroll
      for (int e = 0; e < N; ++e) (*grad)[e] = (*grad)[e] + gg[e];  // :117, :130
    }
    return fx_f + fx_g;
  }
  CNO_D void hess_diag(const cno::EvalCtx& c, const T (&x)[E], T (&h)[E]) const {
    T hg[E];
    f.hess_diag(c, x, h);
    g.hess_diag(c, x, hg);
#pragma unroll
    for (int e = 0; e < E; ++e) h[e] = h[e] + hg[e];
  }
  struct HessState {
    typename expr_detail::HessStateOf<F>::type sf;
    typename expr_detail::HessStateOf<G>::type sg;
  };
  CNO_D HessState hess_prepare(const cno::EvalCtx& c, const T (&x)[E]) const {
    return HessState{expr_detail::hess_prepare(f, c, x), expr_detail::hess_prepare(g, c, x)};
  }
  CNO_D void hess_col(const cno::EvalCtx& c, const T (&x)[E], const HessState& st, int j, bool tr, T (&col)[E]) const {
    T cg[E];
    expr_detail::hess_col(f, c, x, st.sf, j, tr, col);
    expr_detail::hess_col(g, c, x, st.sg, j, tr, cg);
#pragma unroll
    for (int e = 0; e < E; ++e) col[e] = col[e] + cg[e];  // :133 hess_f + hess_g
  }
#endif
};

// ---- function_expressions.h:146-196 ----------------------------------------------------------
template <class F, class G, DifferentiabilityMode TMode = MinDifferentiability<F, G>::value>
struct SubExpression : expr_detail::NodeBase<typename F::ScalarType, TMode, F::Dimension> {
  static_assert(F::Dimension == G::Dimension, "Compile-time dimension mismatch: F and G must have the same dimension.");
  static_assert(std::is_same<typename F::ScalarType, typename G::ScalarType>::value,
                "Compile-time scalar-type mismatch: F and G must have the same scalar type.");
  using Base = expr_detail::NodeBase<typename F::ScalarType, TMode, F::Dimension>;
  F f;
  G g;
  CNO_HD SubExpression(const F& f_, const G& g_) : f(f_), g(g_) {}
#ifdef CNO_DEVICE_CODE
  using T = typename F::ScalarType;
  static constexpr int E = Base::E;
  CNO_D T operator()(const cno::EvalCtx& c, const T (&x)[E], T (*grad)[E]) const { return eval(c, x, grad); }
  template <int W, class F_ = F, class G_ = G, class = std::enable_if_t<expr_detail::AllGroupForm<W, F_, G_>::value>>
  CNO_D T operator()(const cno::GroupEvalCtx<W>& c, const T (&x)[4], T (*grad)[4]) const { return eval(c, x, grad); }
  template <class Ctx, int N>
  CNO_D T eval(const Ctx& c, const T (&x)[N], T (*grad)[N]) const {
    T gg[N];
    const T fx_f = f(c, x, grad);
    const T fx_g = g(c, x, grad ? &gg : nullptr);
    if (grad) {
#pragma unroll
      for (int e = 0; e < N; ++e) (*grad)[e] = (*grad)[e] - gg[e];  // :170, :183
    }
    return fx_f - fx_g;
  }
  CNO_D void hess_diag(const cno::EvalCtx& c, const T (&x)[E], T (&h)[E]) const {
    T hg[E];
    f.hess_diag(c, x, h);
    g.hess_diag(c, x, hg);
#pragma unroll
    for (int e = 0; e < E; ++e) h[e] = h[e] - hg[e];
  }
  struct HessState {
    typename expr_detail::HessStateOf<F>::type sf;
    typename expr_detail::HessStateOf<G>::type sg;
  };
  CNO_D HessState hess_prepare(const cno::EvalCtx& c, const T (&x)[E]) const {
    return HessState{expr_detail::hess_prepare(f, c, x), expr_detail::hess_prepare(g, c, x)};
  }
  CNO_D void hess_col(const cno::EvalCtx& c, const T (&x)[E], const HessState& st, int j, bool tr, T (&col)[E]) const {
    T cg[E];
    expr_detail::hess_col(f, c, x, st.sf, j, tr, col);
    expr_detail::hess_col(g, c, x, st.sg, j, tr, cg);
#pragma unroll
    for (int e = 0; e < E; ++e) col[e] = col[e] - cg[e];  // :186
  }
#endif
};

// ---- function_expressions.h:199-255 ----------------------------------------------------------
template <class F, class TScalar = typename F::ScalarType, DifferentiabilityMode TMode = F::Differentiability>
struct MulExpression : expr_detail::NodeBase<TScalar, TMode, F::Dimension> {
  static_assert(std::is_same<typename F::ScalarType, TScalar>::value,
                "Compile-time scalar-type mismatch: F and c must have the same scalar type.");
  using Base = expr_detail::NodeBase<TScalar, TMode, F::Dimension>;
  TScalar c;
  F f;
  CNO_HD MulExpression(const TScalar& c_, const F& f_) : c(c_), f(f_) {}
#ifdef CNO_DEVICE_CODE
  using T = TScalar;
  static constexpr int E = Base::E;
  CNO_D T operator()(const cno::EvalCtx& ctx, const T (&x)[E], T (*grad)[E]) const { return eval(ctx, x, grad); }
  template <int W, class F_ = F, class = std::enable_if_t<expr_detail::AllGroupForm<W, F_>::value>>
  CNO_D T operator()(const cno::GroupEvalCtx<W>& ctx, const T (&x)[4], T (*grad)[4]) const { return eval(ctx, x, grad); }
  template <class Ctx, int N>
  CNO_D T eval(const Ctx& ctx, const T (&x)[N], T (*grad)[N]) const {
    if (cno::uni(c == T(0))) {  // :219-227: the source is not evaluated (matters when it is not finite there)
      if (grad) expr_detail::set_zero(*grad);
      return T(0);
    }
    const T fx = f(ctx, x, grad);
    if (grad) {
#pragma unroll
      for (int e = 0; e < N; ++e) (*grad)[e] = c * (*grad)[e];  // :235, :244
      expr_detail::mask_pad<F::Dimension>(ctx.lane, *grad);
    }
    return c * fx;
  }
  CNO_D void hess_diag(const cno::EvalCtx& ctx, const T (&x)[E], T (&h)[E]) const {
    if (cno::uni(c == T(0))) { expr_detail::set_zero(h); return; }
    f.hess_diag(ctx, x, h);
#pragma unroll
    for (int e = 0; e < E; ++e) h[e] = c * h[e];
  }
  using HessState = typename expr_detail::HessStateOf<F>::type;
  CNO_D HessState hess_prepare(const cno::EvalCtx& ctx, const T (&x)[E]) const {
    if (cno::uni(c == T(0))) return HessState{};
    return expr_detail::hess_prepare(f, ctx, x);
  }
  CNO_D void hess_col(const cno::EvalCtx& ctx, const T (&x)[E], const HessState& st, int j, bool tr, T (&col)[E]) const {
    if (cno::uni(c == T(0))) { expr_detail::set_zero(col); return; }
    expr_detail::hess_col(f, ctx, x, st, j, tr, col);
#pragma unroll
    for (int e = 0; e < E; ++e) col[e] = c * col[e];  // :247
    expr_detail::mask_pad<F::Dimension>(ctx.lane, col);
  }
#endif
};

// ---- function_expressions.h:258-315 ----------------------------------------------------------
template <class F, class G, DifferentiabilityMode TMode = MinDifferentiability<F, G>::value>
struct ProdExpression : expr_detail::NodeBase<typename F::ScalarType, TMode, F::Dimension> {
  static_assert(F::Dimension == G::Dimension, "Compile-time dimension mismatch: F and G must have the same dimension.");
  static_assert(std::is_same<typename F::ScalarType, typename G::ScalarType>::value,
                "Compile-time scalar-type mismatch: F and G must have the same scalar type.");
  using Base = expr_detail::NodeBase<typename F::ScalarType, TMode, F::Dimension>;
  F f;
  G g;
  CNO_HD ProdExpression(const F& f_, const G& g_) : f(f_), g(g_) {}
#ifdef CNO_DEVICE_CODE
  using T = typename F::ScalarType;
  static constexpr int E = Base::E;
  CNO_D T operator()(const cno::EvalCtx& c, const T (&x)[E], T (*grad)[E]) const { return eval(c, x, grad); }
  template <int W, class F_ = F, class G_ = G, class = std::enable_if_t<expr_detail::AllGroupForm<W, F_, G_>::value>>
  CNO_D T operator()(const cno::GroupEvalCtx<W>& c, const T (&x)[4], T (*grad)[4]) const { return eval(c, x, grad); }
  template <class Ctx, int N>
  CNO_D T eval(const Ctx& c, const T (&x)[N], T (*grad)[N]) const {
    T gg[N];
    const T fx = f(c, x, grad);
    const T gx = g(c, x, grad ? &gg : nullptr);
    if (grad) {
#pragma unroll
      for (int e = 0; e < N; ++e) (*grad)[e] = gx * (*grad)[e] + fx * gg[e];  // :291, :300 product rule
      expr_detail::mask_pad<F::Dimension>(c.lane, *grad);
    }
    return fx * gx;
  }
  // values and gradients of both factors at x: what every Hessian column of f*g needs (:296-305)
  struct HessState {
    T fx, gx;
    T gf[E], gg[E];
    typename expr_detail::HessStateOf<F>::type sf;
    typename expr_detail::HessStateOf<G>::type sg;
  };
  CNO_D HessState hess_prepare(const cno::EvalCtx& c, const T (&x)[E]) const {
    HessState st;
    st.fx = f(c, x, &st.gf);
    st.gx = g(c, x, &st.gg);
    st.sf = expr_detail::hess_prepare(f, c, x);
    st.sg = expr_detail::hess_prepare(g, c, x);
    return st;
  }
  // H_rj = ((gx*Hf_rj + fx*Hg_rj) + gf_r*gg_j) + gg_r*gf_j (:304-305); transposed: element (j, r)
  CNO_D void hess_col(const cno::EvalCtx& c, const T (&x)[E], const HessState& st, int j, bool tr, T (&col)[E]) const {
    T cg[E];
    expr_detail::hess_col(f, c, x, st.sf, j, tr, col);
    expr_detail::hess_col(g, c, x, st.sg, j, tr, cg);
    const T gf_j = expr_detail::bcast_elem<T, E>(st.gf, j), gg_j = expr_detail::bcast_elem<T, E>(st.gg, j);
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const T base = st.gx * col[e] + st.fx * cg[e];
      col[e] = tr ? ((base + gf_j * st.gg[e]) + gg_j * st.gf[e]) : ((base + st.gf[e] * gg_j) + st.gg[e] * gf_j);
    }
    expr_detail::mask_pad<F::Dimension>(c.lane, col);
  }
  CNO_D void hess_diag(const cno::EvalCtx& c, const T (&x)[E], T (&h)[E]) const {
    T hg[E], gf[E], gg[E];
    const T fx = f(c, x, &gf);
    const T gx = g(c, x, &gg);
    f.hess_diag(c, x, h);
    g.hess_diag(c, x, hg);
#pragma unroll
    for (int e = 0; e < E; ++e) h[e] = ((gx * h[e] + fx * hg[e]) + gf[e] * gg[e]) + gg[e] * gf[e];
    expr_detail::mask_pad<F::Dimension>(c.lane, h);
  }
#endif
};

// ---- function_expressions.h:318-399: min{0, f} and max{0, f} -----------------------------------
template <class F, bool kMin>
struct ZeroClampExpression : expr_detail::NodeBase<typename F::ScalarType, F::Differentiability, F::Dimension> {
  using Base = expr_detail::NodeBase<typename F::ScalarType, F::Differentiability, F::Dimension>;
  F f;
  CNO_HD explicit ZeroClampExpression(const F& f_) : f(f_) {}
#ifdef CNO_DEVICE_CODE
  using T = typename F::ScalarType;
  static constexpr int E = Base::E;
  // inactive <=> val >= 0 (MinZero :343) or val <= 0 (MaxZero :388); a NaN value is "active" in both
  CNO_D static bool inactive(T val) { return kMin ? (val >= T(0)) : (val <= T(0)); }
  CNO_D T operator()(const cno::EvalCtx& c, const T (&x)[E], T (*grad)[E]) const { return eval(c, x, grad); }
  template <int W, class F_ = F, class = std::enable_if_t<expr_detail::AllGroupForm<W, F_>::value>>
  CNO_D T operator()(const cno::GroupEvalCtx<W>& c, const T (&x)[4], T (*grad)[4]) const { return eval(c, x, grad); }
  template <class Ctx, int N>
  CNO_D T eval(const Ctx& c, const T (&x)[N], T (*grad)[N]) const {
    const T val = f(c, x, grad);
    if (cno::uni(inactive(val))) {
      if (grad) expr_detail::set_zero(*grad);
      return T(0);
    }
    return val;
  }
  CNO_D void hess_diag(const cno::EvalCtx& c, const T (&x)[E], T (&h)[E]) const {
    const T val = f(c, x, nullptr);
    if (cno::uni(inactive(val))) { expr_detail::set_zero(h); return; }
    f.hess_diag(c, x, h);
  }
  struct HessState {
    bool off;
    typename expr_detail::HessStateOf<F>::type sf;
  };
  CNO_D HessState hess_prepare(const cno::EvalCtx& c, const T (&x)[E]) const {
    HessState st;
    st.off = cno::uni(inactive(f(c, x, nullptr)));
    if (!st.off) st.sf = expr_detail::hess_prepare(f, c, x);
    return st;
  }
  CNO_D void hess_col(const cno::EvalCtx& c, const T (&x)[E], const HessState& st, int j, bool tr, T (&col)[E]) const {
    if (st.off) { expr_detail::set_zero(col); return; }
    expr_detail::hess_col(f, c, x, st.sf, j, tr, col);
  }
#endif
};
template <class F> struct MinZeroExpression : ZeroClampExpression<F, true> {
  CNO_HD explicit MinZeroExpression(const F& f_) : ZeroClampExpression<F, true>(f_) {}
};
template <class F> struct MaxZeroExpression : ZeroClampExpression<F, false> {
  CNO_HD explicit MaxZeroExpression(const F& f_) : ZeroClampExpression<F, false>(f_) {}
};

// ---- function_base.h:151-189: use a stronger source where a weaker mode is expected ---------------
// (the FunctionExpr converting constructor wraps with this; the Hessian members are simply not there)
template <class F, DifferentiabilityMode TargetMode>
struct ModeDowngrade : expr_detail::NodeBase<typename F::ScalarType, TargetMode, F::Dimension> {
  static_assert(static_cast<int>(F::Differentiability) >= static_cast<int>(TargetMode),
                "ModeDowngrade only lowers the differentiability mode -- attempting to upgrade.");
  using Base = expr_detail::NodeBase<typename F::ScalarType, TargetMode, F::Dimension>;
  F source;
  CNO_HD explicit ModeDowngrade(const F& f) : source(f) {}
#ifdef CNO_DEVICE_CODE
  using T = typename F::ScalarType;
  static constexpr int E = Base::E;
  CNO_D T operator()(const cno::EvalCtx& c, const T (&x)[E], T (*grad)[E]) const {
    return source(c, x, TargetMode == DifferentiabilityMode::None ? nullptr : grad);
  }
  template <int W, class F_ = F, class = std::enable_if_t<expr_detail::AllGroupForm<W, F_>::value>>
  CNO_D T operator()(const cno::GroupEvalCtx<W>& c, const T (&x)[4], T (*grad)[4]) const {
    return source(c, x, TargetMode == DifferentiabilityMode::None ? nullptr : grad);
  }
#endif
};

// ---- function_expressions.h:403-518: the free operators ------------------------------------------
template <class F, class G, class = std::enable_if_t<expr_detail::IsFunction<F>::value && expr_detail::IsFunction<G>::value>>
CNO_HD auto operator+(const F& f, const G& g) {
  static_assert(std::is_same<typename F::ScalarType, typename G::ScalarType>::value, "ScalarType must match in addition.");
  static_assert(F::Dimension == G::Dimension, "Dimension mismatch: F and G must have the same compile-time dimension.");
  return AddExpression<F, G, MinDifferentiability<F, G>::value>(f, g);
}
template <class F, class G, class = std::enable_if_t<expr_detail::IsFunction<F>::value && expr_detail::IsFunction<G>::value>>
CNO_HD auto operator-(const F& f, const G& g) {
  static_assert(std::is_same<typename F::ScalarType, typename G::ScalarType>::value, "ScalarType must match in subtraction.");
  static_assert(F::Dimension == G::Dimension, "Dimension mismatch: F and G must have the same compile-time dimension.");
  return SubExpression<F, G, MinDifferentiability<F, G>::value>(f, g);
}
template <class F, class = std::enable_if_t<expr_detail::IsFunction<F>::value>>
CNO_HD auto operator*(const F& f, const typename F::ScalarType& c) {
  return MulExpression<F, typename F::ScalarType, F::Differentiability>(c, f);
}
template <class F, class = std::enable_if_t<expr_detail::IsFunction<F>::value>>
CNO_HD auto operator*(const typename F::ScalarType& c, const F& f) {
  return MulExpression<F, typename F::ScalarType, F::Differentiability>(c, f);
}
template <class F, class G, class = std::enable_if_t<expr_detail::IsFunction<F>::value && expr_detail::IsFunction<G>::value>>
CNO_HD auto operator*(const F& f, const G& g) {
  static_assert(std::is_same<typename F::ScalarType, typename G::ScalarType>::value, "ScalarType must match in a product.");
  static_assert(F::Dimension == G::Dimension, "Dimension mismatch: F and G must have the same compile-time dimension.");
  return ProdExpression<F, G, MinDifferentiability<F, G>::value>(f, g);
}
template <class F, class = std::enable_if_t<expr_detail::IsFunction<F>::value>>
CNO_HD auto operator-(const F& f) {  // :461-465 unary minus = (-1) * f
  return typename F::ScalarType(-1) * f;
}
template <class F, class = std::enable_if_t<expr_detail::IsFunction<F>::value>>
CNO_HD auto operator+(const F& f, const typename F::ScalarType& c) {  // :468-478
  using CE = ConstExpression<typename F::ScalarType, F::Differentiability, F::Dimension>;
  return AddExpression<F, CE, F::Differentiability>(f, CE(c));
}
template <class F, class = std::enable_if_t<expr_detail::IsFunction<F>::value>>
CNO_HD auto operator+(const typename F::ScalarType& c, const F& f) {  // :481-491
  using CE = ConstExpression<typename F::ScalarType, F::Differentiability, F::Dimension>;
  return AddExpression<CE, F, F::Differentiability>(CE(c), f);
}
template <class F, class = std::enable_if_t<expr_detail::IsFunction<F>::value>>
CNO_HD auto operator-(const F& f, const typename F::ScalarType& c) {  // :494-503
  using CE = ConstExpression<typename F::ScalarType, F::Differentiability, F::Dimension>;
  return SubExpression<F, CE, F::Differentiability>(f, CE(c));
}
template <class F, class = std::enable_if_t<expr_detail::IsFunction<F>::value>>
CNO_HD auto operator-(const typename F::ScalarType& c, const F& f) {  // :506-515
  using CE = ConstExpression<typename F::ScalarType, F::Differentiability, F::Dimension>;
  return SubExpression<CE, F, F::Differentiability>(CE(c), f);
}

}  // namespace function
}  // namespace cppoptlib

#endif  // CPPOPTLIB_B200_EXPRESSIONS_H_
