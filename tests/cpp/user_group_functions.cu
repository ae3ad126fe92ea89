// tests/cpp/user_group_functions.cu -- user objectives and composites at d = 512 and 1024 compiled for the device from
// the public headers with CNO_INSTANTIATE_FUNCTION, as a shared library for tests/test_user_group_gpu.py and
// tools/user_large_d_bench.py.  Lbfgs on a functor with the group form at d = 1024 runs the group kernel
// (csrc/cno_lbfgs_group.cuh); each tag also has an entry that runs the one-warp kernel on the same type
// (cno::user_lbfgs, E = 32 elements per lane), so the two can be compared bit for bit.  The composites other than
// ProdRosen have twins in oracle/ref_driver.cc (EXPR_*), built from the reference's own operators.
//
// The instantiations at d = 1024 are large, so the file is compiled in parts that build in parallel
// (-DCNO_USER_GROUP_PART=0 .. kParts - 1, each with -c), then linked into one library:
//   nvcc -shared part0.o ... -o <dir>/libcno_usergroup.so -lcno
//
//   int ug_<tag>(int path, int solver, int lbfgs_m, double param, int64_t batch, const double* x0,
//                const cno_stop_t* stop, const cno_batch_out_t* out, void* workspace, size_t workspace_bytes,
//                cno_launch_info_t* info)
//     path 0: cno_<tag>_minimize (what Lbfgs<F>::Minimize calls); path 1: the one-warp Lbfgs kernel
//   param: Bowl's centre c
#include <cstring>
#include <vector>

#include "cppoptlib_b200/device.cuh"

using cppoptlib::function::DifferentiabilityMode;
using cppoptlib::function::FunctionCRTP;
namespace fn = cppoptlib::function;

// f(x) = sum_i a_i (x_i - c)^2, a_i = 1 + i/8 (oracle/ref_driver.cc: Bowl), one-warp form only
template <int D>
struct PlainBowl : FunctionCRTP<PlainBowl<D>, double, DifferentiabilityMode::First, D> {
  static constexpr int E = cno::Shape<D>::E;
  double c;
  __device__ double operator()(const cno::EvalCtx& ctx, const double (&x)[E], double (*grad)[E]) const {
    double t[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int i = ctx.lane * E + e;
      const double a = 1.0 + 0.125 * i;
      const double r = x[e] - c;
      t[e] = (i < D) ? a * r * r : 0.0;
      if (grad) (*grad)[e] = (i < D) ? 2.0 * a * r : 0.0;
    }
    return cno::warp_sum(cno::lane_tree<double, E>(t));
  }
};
// the same objective with the group form as well (D = 128 W): thread t holds elements ctx.first .. + 3
template <int D>
struct GroupBowl : PlainBowl<D> {
  using PlainBowl<D>::operator();
  __device__ double operator()(const cno::GroupEvalCtx<D / 128>& ctx, const double (&x)[4], double (*grad)[4]) const {
    double t[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = ctx.first + j;
      const double a = 1.0 + 0.125 * i;
      const double r = x[j] - this->c;
      t[j] = a * r * r;
      if (grad) (*grad)[j] = 2.0 * a * r;
    }
    return cno::group_sum_terms(ctx, t);
  }
};

template <int D> using RosenPlusHalf = decltype(fn::Rosenbrock<double, D>{} + 0.5 * fn::HalfSquaredNorm<double, D>{});
template <int D> using ZeroMul = decltype(0.0 * fn::Rosenbrock<double, D>{} + fn::HalfSquaredNorm<double, D>{});
// Rosenbrock + 5 (MaxZero(h - 2))^2 + 5 (MinZero(h - 1/8))^2, h = HalfSquaredNorm, as oracle/ref_driver.cc builds it
template <int D>
auto make_penalty() {
  const fn::HalfSquaredNorm<double, D> h;
  const auto g1 = h - 2.0;
  const auto g2 = h - 0.125;
  const fn::MaxZeroExpression<std::decay_t<decltype(g1)>> p1(g1);
  const fn::MinZeroExpression<std::decay_t<decltype(g2)>> p2(g2);
  return (fn::Rosenbrock<double, D>{} + 5.0 * (p1 * p1)) + 5.0 * (p2 * p2);
}
template <int D> using Penalty = decltype(make_penalty<D>());
// two leaves that use the group's exchange block
template <int D> using ProdRosen = decltype((fn::Rosenbrock<double, D>{} + 1.0) * (fn::Rosenbrock<double, D>{} + 1.0));

using GroupBowl1024 = GroupBowl<1024>;
using PlainBowl1024 = PlainBowl<1024>;
using RosenPlusHalf1024 = RosenPlusHalf<1024>;
using ZeroMul1024 = ZeroMul<1024>;
using Penalty1024 = Penalty<1024>;
using ProdRosen1024 = ProdRosen<1024>;
using Rosen1024 = fn::Rosenbrock<double, 1024>;
using Rosen512 = fn::Rosenbrock<double, 512>;

static_assert(cno::HasGroupForm<GroupBowl1024, 8>::value && cno::HasGroupForm<RosenPlusHalf1024, 8>::value &&
                  cno::HasGroupForm<ZeroMul1024, 8>::value && cno::HasGroupForm<Penalty1024, 8>::value &&
                  cno::HasGroupForm<ProdRosen1024, 8>::value && cno::HasGroupForm<Rosen1024, 8>::value,
              "composites of group-form leaves have the group form");
static_assert(!cno::HasGroupForm<PlainBowl1024, 8>::value, "a functor without the group form");

// Lbfgs on the tag through the public symbol (path 0) or on the one-warp kernel (path 1)
#define UG_ENTRY(tag, F, make)                                                                                     \
  CNO_INSTANTIATE_FUNCTION(tag, F)                                                                                 \
  extern "C" int ug_##tag(int path, int solver, int lbfgs_m, double param, int64_t batch, const double* x0,       \
                          const cno_stop_t* stop, const cno_batch_out_t* out, void* workspace,                    \
                          size_t workspace_bytes, cno_launch_info_t* info) {                                      \
    (void)param;                                                                                                   \
    const F f__ = make;                                                                                            \
    if (path == 0)                                                                                                 \
      return cno_##tag##_minimize(solver, 1, lbfgs_m, &f__, batch, x0, stop, out, workspace, workspace_bytes,     \
                                  nullptr, info);                                                                  \
    if (solver != CNO_LBFGS) return CNO_ERR_UNSUPPORTED;                                                           \
    return cno::user_lbfgs<F, cno::LsMoreThuente, CNO_LBFGS_M>(f__, 1, lbfgs_m, batch, x0, stop, out, workspace,   \
                                                               workspace_bytes, nullptr, info);                    \
  }

template <class B>
B bowl(double c) {
  B b;
  b.c = c;
  return b;
}

#if CNO_USER_GROUP_PART == 0
UG_ENTRY(gbowl1024, GroupBowl1024, bowl<GroupBowl1024>(param))
UG_ENTRY(bowl1024, PlainBowl1024, bowl<PlainBowl1024>(param))
#elif CNO_USER_GROUP_PART == 1
UG_ENTRY(rph1024, RosenPlusHalf1024, RosenPlusHalf1024(Rosen1024{}, 0.5 * fn::HalfSquaredNorm<double, 1024>{}))
UG_ENTRY(zmul1024, ZeroMul1024, ZeroMul1024(0.0 * Rosen1024{}, fn::HalfSquaredNorm<double, 1024>{}))
#elif CNO_USER_GROUP_PART == 2
UG_ENTRY(pen1024, Penalty1024, make_penalty<1024>())
#elif CNO_USER_GROUP_PART == 3
UG_ENTRY(prodrosen1024, ProdRosen1024, (Rosen1024{} + 1.0) * (Rosen1024{} + 1.0))
#elif CNO_USER_GROUP_PART == 4
UG_ENTRY(rosen1024, Rosen1024, Rosen1024{})
UG_ENTRY(rosen512, Rosen512, Rosen512{})

// Lbfgs<RosenPlusHalf<1024>>::Minimize through the C++ mirror on host arrays x0 [B, 1024] -> x, value, iterations
// (the symbols of part 1).
CNO_DECLARE_FUNCTION(rph1024, RosenPlusHalf1024)
extern "C" int ug_mirror_lbfgs_rph1024(int64_t batch, const double* x0, double* x, double* value, uint32_t* iterations) {
  try {
    const RosenPlusHalf1024 f = Rosen1024{} + 0.5 * fn::HalfSquaredNorm<double, 1024>{};
    cppoptlib::solver::Lbfgs<RosenPlusHalf1024> solver;
    auto [solution, state] = solver.Minimize(
        f, fn::BatchedFunctionState<double, 1024>::FromHost(std::vector<double>(x0, x0 + batch * 1024), batch));
    const auto xs = solution.x.ToHost();
    const auto vs = solution.value.ToHost();
    const auto its = state.num_iterations.ToHost();
    std::memcpy(x, xs.data(), xs.size() * sizeof(double));
    std::memcpy(value, vs.data(), vs.size() * sizeof(double));
    for (size_t i = 0; i < its.size(); ++i) iterations[i] = (uint32_t)its[i];
    return 0;
  } catch (...) {
    return -1;
  }
}
#endif
