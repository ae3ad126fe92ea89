// tests/emu/emu_al_user.cc -- the DEVICE SOURCE of AugmentedLagrangian on functor constraints (csrc/cno_auglag.cuh:
// AugLagFn<Obj, AlFunctors<...>> and the AL kernels, on the problems of tests/cpp/al_user_problems.cuh) on the CPU
// under the warp emulation of warp_emu.h, driven by the same host logic as cno_<tag>_al_minimize
// (csrc/cno_auglag_host.h: al_outer_loop).  TEST INFRASTRUCTURE: tests/test_al_user.py compiles it with the flags of
// tests/emu/Makefile into a temporary directory.
#include <cstring>
#include <vector>

#include "cno_functors.cuh"
#include "cno_auglag.cuh"
#include "cno_auglag_host.h"
#include "cno_lbfgs.cuh"
#include "al_user_problems.cuh"

namespace {

template <class F>
void launch(long long batch, F&& body) {  // grid of ceil(batch / kAlWarps) blocks x kAlWarps warps
  const int blocks = (int)((batch + cno::kAlWarps - 1) / cno::kAlWarps);
  for (int blk = 0; blk < blocks; ++blk)
    for (int w = 0; w < cno::kAlWarps; ++w)
      emu::run_warp([&](int lane) {
        blockIdx.x = (unsigned)blk;
        threadIdx.x = (unsigned)(w * 32 + lane);
        body();
      });
}

// cno::al_outer_loop's backend with every kernel under emulation (the CUDA one is csrc/cno_auglag_launch.cuh)
template <class Obj, class Cons>
struct AlEmuBackend {
  using T = typename Obj::Scalar;
  Obj obj;
  Cons cons;
  long long B;
  cno::AlArrays<T> a;
  cno::AlView<T> view;
  cno::AlParams<T> p;
  int copy_or_zero(void* dst, const void* src, size_t bytes) {
    if (!bytes || src == dst) return 0;
    if (src) std::memcpy(dst, src, bytes); else std::memset(dst, 0, bytes);
    return 0;
  }
  int fill(void* dst, int byte, size_t bytes) { if (bytes) std::memset(dst, byte, bytes); return 0; }
  int autoscale() { launch(B, [&] { cno::al_autoscale_kernel<Obj, Cons>(obj, view, B, p, a, cons); }); return 0; }
  int inner(const cno_stop_t& stop) {
    using Fn = cno::AugLagFn<Obj, Cons>;
    const Fn fn(obj, view, cons);
    cno_batch_out_t o{};
    o.x = a.x_work;
    o.nfev = const_cast<uint32_t*>(a.inner_nfev);
    unsigned long long queue = 0;
    emu::run_warp([&](int lane) {
      blockIdx.x = 0;
      threadIdx.x = (unsigned)lane;
      cno::lbfgs_minimize_kernel<Fn, CNO_LBFGS_M>(fn, a.x, B, cno::make_stop<T>(stop), cno::make_out<T>(o), &queue,
                                                  cno::ResumeArgs{nullptr, 0, 0, 0});
    });
    return 0;
  }
  int outer_step(int* remaining) {
    *a.remaining = 0;
    launch(B, [&] { cno::al_outer_step_kernel<Obj, Cons>(obj, view, B, p, a, cons); });
    *remaining = *a.remaining;
    return 0;
  }
  int finalize() { launch(B, [&] { cno::al_finalize_kernel<T, Obj::Dim>(B, view.n_eq, view.n_ineq, a); }); return 0; }
};

template <class S>
int run_minimize(const void* data, long long stride, long long B, const void* x0, const void* eq0, const void* ineq0,
                 const void* penalty0, const cno_stop_t* inner_stop, const cno_al_stop_t* outer_stop,
                 const cno_al_config_t* config, const cno_al_out_t* out, int* launches) {
  using Cons = cno::AlFunctors<typename S::Eq, typename S::In>;
  using T = typename S::Obj::Scalar;
  const auto parts = S::make(data, stride);
  const cno_constraints_t k{Cons::kNumEq, Cons::kNumIneq, nullptr, nullptr, 0};
  const cno::AlLayout L((size_t)B, S::Obj::Dim, (size_t)k.n_eq, (size_t)k.n_ineq, sizeof(T));
  std::vector<unsigned char> storage(L.total + 256);
  unsigned char* ws = storage.data() + (256 - ((uintptr_t)storage.data() & 255)) % 256;
  AlEmuBackend<typename S::Obj, Cons> be{parts.objective, Cons{parts.equality_constraints, parts.inequality_constraints},
                                         B, cno::al_make_arrays<T>(*out, ws, L), {}, {}};
  be.view = cno::al_make_view<T>(k, be.a);
  be.p = cno::al_make_params<T>(*config, *outer_stop);
  return cno::al_outer_loop<T>(be, be.a, B, S::Obj::Dim, k.n_eq, k.n_ineq, x0, eq0, ineq0, penalty0, *inner_stop,
                               *config, launches);
}

// AugLagFn::operator() (the composite the inner solver minimises) at x under per-instance lambda [B, n_eq],
// mu [B, n_ineq] and penalty [B]
template <class S>
int run_composite(const void* data, long long stride, long long B, const void* x, const void* lambda, const void* mu,
                  const void* penalty, void* value, void* gradient) {
  using Cons = cno::AlFunctors<typename S::Eq, typename S::In>;
  using T = typename S::Obj::Scalar;
  constexpr int D = S::Obj::Dim;
  constexpr int E = cno::Shape<D>::E;
  const auto parts = S::make(data, stride);
  cno::AlView<T> v{};
  v.n_eq = Cons::kNumEq;
  v.n_ineq = Cons::kNumIneq;
  v.lambda = (const T*)lambda;
  v.mu = (const T*)mu;
  v.penalty = (const T*)penalty;
  const cno::AugLagFn<typename S::Obj, Cons> fn(parts.objective, v,
                                               Cons{parts.equality_constraints, parts.inequality_constraints});
  for (long long b = 0; b < B; ++b)
    emu::run_warp([&](int lane) {
      const cno::EvalCtx ctx{lane, b, nullptr};
      T xl[E], g[E];
      cno::al_load<T, D>((const T*)x + b * D, lane, xl);
      const T f = fn(ctx, xl, &g);
      cno::al_store<T, D>((T*)gradient + b * D, lane, g);
      if (lane == 0) ((T*)value)[b] = f;
    });
  return 0;
}

}  // namespace

// cno_<tag>_al_minimize's host logic and kernels under emulation for problem `problem` at (dtype, d).  Host pointers.
extern "C" int emu_al_user_minimize(int problem, int dtype, int d, const void* data, long long stride, long long batch,
                                    const void* x0, const void* eq0, const void* ineq0, const void* penalty0,
                                    const cno_stop_t* inner_stop, const cno_al_stop_t* outer_stop,
                                    const cno_al_config_t* config, const cno_al_out_t* out, int* launches) {
#define X(tag, id, dt, dim, S)                                                                                     \
  if (problem == id && dtype == dt && d == dim)                                                                    \
    return run_minimize<S>(data, stride, batch, x0, eq0, ineq0, penalty0, inner_stop, outer_stop, config, out, launches);
  ALU_PROBLEMS(X)
#undef X
  return CNO_ERR_UNSUPPORTED;
}

extern "C" int emu_al_user_composite(int problem, int dtype, int d, const void* data, long long stride, long long batch,
                                     const void* x, const void* lambda, const void* mu, const void* penalty, void* value,
                                     void* gradient) {
#define X(tag, id, dt, dim, S)                                                                                     \
  if (problem == id && dtype == dt && d == dim)                                                                    \
    return run_composite<S>(data, stride, batch, x, lambda, mu, penalty, value, gradient);
  ALU_PROBLEMS(X)
#undef X
  return CNO_ERR_UNSUPPORTED;
}
