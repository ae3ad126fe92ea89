// tests/emu/emu_user_group.cc -- runs the DEVICE SOURCE of the group L-BFGS kernel (csrc/cno_lbfgs_group.cuh) on user
// objectives at d = 1024 -- a functor with the group form and composites of the group-form leaves
// (include/cppoptlib_b200/expressions.h) -- on the CPU under the warp emulation of warp_emu.h.  TEST INFRASTRUCTURE
// ONLY.  tests/test_user_group.py compiles it with the flags of tests/emu/Makefile into a temporary directory and
// compares it with the reference's own operators (oracle/ref_driver.cc: cno_ref_minimize_expr).
#include "emu_lbfgs_group.cc"  // run_group(): one group of W lock-step warps

#include "cppoptlib_b200/expressions.h"

namespace {

namespace fn = cppoptlib::function;
using fn::operator+;
using fn::operator-;
using fn::operator*;
constexpr int D = 1024;
constexpr int W = D / 128;
using Node = fn::expr_detail::NodeBase<double, fn::DifferentiabilityMode::First, D>;

// the group form of the mirror's Rosenbrock<double, 1024> and HalfSquaredNorm<double, 1024> (cppoptlib.h forwards to
// the same functors)
template <class G>
struct Leaf : Node {
  double operator()(const cno::GroupEvalCtx<W>& c, const double (&x)[4], double (*grad)[4]) const { return G{}(c, x, grad); }
};
using Rosen = Leaf<cno::GroupRosenbrockFn<double, D>>;
using Half = Leaf<cno::GroupHalfSquaredNormFn<D>>;

// f(x) = sum_i a_i (x_i - c)^2, a_i = 1 + i/8: the group form of tests/cpp/user_group_functions.cu GroupBowl
struct GroupBowl : Node {
  double c;
  double operator()(const cno::GroupEvalCtx<W>& ctx, const double (&x)[4], double (*grad)[4]) const {
    double t[4];
    for (int j = 0; j < 4; ++j) {
      const int i = ctx.first + j;
      const double a = 1.0 + 0.125 * i;
      const double r = x[j] - c;
      t[j] = a * r * r;
      if (grad) (*grad)[j] = 2.0 * a * r;
    }
    return cno::group_sum_terms(ctx, t);
  }
};

auto make_penalty() {  // as oracle/ref_driver.cc builds EXPR_PENALTY
  const Half h;
  const auto g1 = h - 2.0;
  const auto g2 = h - 0.125;
  const fn::MaxZeroExpression<std::decay_t<decltype(g1)>> p1(g1);
  const fn::MinZeroExpression<std::decay_t<decltype(g2)>> p2(g2);
  return (Rosen{} + 5.0 * (p1 * p1)) + 5.0 * (p2 * p2);
}

template <class Fn>
int run(const Fn& fn, long long B, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out) {
  static_assert(cno::HasGroupForm<Fn, W>::value, "a group functor");
  unsigned long long queue = 0;
  run_group(
      [&](int lane, int w) {
        blockIdx.x = 0;
        threadIdx.x = (unsigned)(32 * w + lane);
        cno::lbfgs_group_minimize_kernel<Fn, CNO_LBFGS_M>(fn, (const double*)x0, B, cno::make_stop<double>(*stop),
                                                          cno::make_out<double>(*out), &queue);
      },
      W);
  return 0;
}

}  // namespace

// Lbfgs (MoreThuente, m = CNO_LBFGS_M) at d = 1024 on composite `expr` (ids = oracle/ref_driver.cc EXPR_*: 0 Bowl(param),
// 1 Rosenbrock + 0.5 HalfSquaredNorm, 4 the penalty composite, 5 0 Rosenbrock + HalfSquaredNorm); 100 =
// (Rosenbrock + 1) (Rosenbrock + 1), two leaves that use the exchange block.  Host pointers.
extern "C" int emu_user_group(int expr, double param, long long batch, const void* x0, const cno_stop_t* stop,
                              const cno_batch_out_t* out) {
  switch (expr) {
    case 0: {
      GroupBowl b;
      b.c = param;
      return run(b, batch, x0, stop, out);
    }
    case 1: return run(Rosen{} + 0.5 * Half{}, batch, x0, stop, out);
    case 4: return run(make_penalty(), batch, x0, stop, out);
    case 5: return run(0.0 * Rosen{} + Half{}, batch, x0, stop, out);
    case 100: return run((Rosen{} + 1.0) * (Rosen{} + 1.0), batch, x0, stop, out);
  }
  return CNO_ERR_UNSUPPORTED;
}
