// tests/emu/emu_lbfgs_group.cc -- runs the DEVICE SOURCE of the group L-BFGS kernel (csrc/cno_lbfgs_group.cuh: one group
// of d / 128 warps per instance, d = 256 / 512 / 1024) on the CPU under the warp emulation of warp_emu.h.  TEST
// INFRASTRUCTURE ONLY.  tests/test_lbfgs_group.py compiles it into a temporary directory:
//
//   g++ -std=c++20 -O1 -ffp-contract=off -fno-fast-math -fPIC -pthread -DCNO_WARP_EMULATION -shared \
//       -I tests/emu -I cppnumericalsolvers_b200/csrc -I include tests/emu/emu_lbfgs_group.cc -o <dir>/libcno_emu_group.so
#include <cstdlib>

#include "cno_functors.cuh"
#include "cno_lbfgs_group.cuh"

namespace {

// Runs f(lane, w) on 32 W lock-step threads = the W warps of one group, which share one named barrier
// (emu::team_sync(), what group_bar() calls under the emulation).  Shared memory is the kernel's function-static array.
void run_group(const std::function<void(int, int)>& f, int warps) {
  constexpr int kMaxWarps = 8;
  static emu::Warp w_storage[kMaxWarps];
  static emu::SpinBarrier group_bar;
  if (warps < 1 || warps > kMaxWarps) std::abort();
  new (&group_bar) emu::SpinBarrier();
  group_bar.total = 32 * warps;
  for (int w = 0; w < warps; ++w) {
    new (&w_storage[w]) emu::Warp();
    w_storage[w].team = &group_bar;
  }
  std::vector<std::thread> ts;
  for (int w = 0; w < warps; ++w)
    for (int l = 0; l < 32; ++l)
      ts.emplace_back([&, w, l] {
        emu::tl_lane = l;
        emu::tl_warp = &w_storage[w];
        f(l, w);
      });
  for (auto& t : ts) t.join();
}

// One group of the kernel's CTA draining the queue.  Host pointers.
template <int D>
int run_group_lbfgs(long long B, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out) {
  using Fn = cno::GroupRosenbrockFn<double, D>;
  unsigned long long queue = 0;
  run_group(
      [&](int lane, int w) {
        blockIdx.x = 0;
        threadIdx.x = (unsigned)(32 * w + lane);
        cno::lbfgs_group_minimize_kernel<Fn, CNO_LBFGS_M>(Fn{}, (const double*)x0, B, cno::make_stop<double>(*stop),
                                                          cno::make_out<double>(*out), &queue);
      },
      Fn::kGroupWarps);
  return 0;
}

// The group sum alone (warp_sum_p on a GroupCtx): sums[r] = the sum of terms[r, 0 .. d - 1] with thread t of the group
// contributing the in-thread tree of its 4 elements, as the group kernel forms every dot product.
template <int D>
void run_group_sum(long long rows, const double* terms, double* sums) {
  constexpr int W = D / 128;
  alignas(16) static double scratch[2 * cno::GroupCtx<double, W>::kBufElems];
  run_group(
      [&](int lane, int w) {
        const cno::GroupCtx<double, W> rc{scratch, lane, w, 1, 0};
        const int t = 32 * w + lane;
        for (long long r = 0; r < rows; ++r) {
          double v[4];
          for (int j = 0; j < 4; ++j) v[j] = terms[r * D + cno::GroupRosenbrockFn<double, D>::first_elem(t) + j];
          const double s = cno::warp_sum_p<cno::PolicyFast, double, 4>(cno::lane_tree<double, 4>(v), rc);
          if (t == 0) sums[r] = s;
        }
      },
      W);
}

}  // namespace

// Lbfgs on Rosenbrock fp64 at d = 256 / 512 / 1024 with MoreThuente, m = 10, the default policy.
extern "C" int emu_lbfgs_group(const cno_problem_t* p, long long batch, const void* x0, const cno_stop_t* stop,
                               const cno_batch_out_t* out) {
  if (p->family != CNO_FN_ROSENBROCK || p->dtype != CNO_F64 || p->mode == 2 || p->policy != CNO_POLICY_DMMA_TREE ||
      (p->lbfgs_m != 0 && p->lbfgs_m != CNO_LBFGS_M))
    return CNO_ERR_UNSUPPORTED;
  if (p->d == 256) return run_group_lbfgs<256>(batch, x0, stop, out);
  if (p->d == 512) return run_group_lbfgs<512>(batch, x0, stop, out);
  if (p->d == 1024) return run_group_lbfgs<1024>(batch, x0, stop, out);
  return CNO_ERR_UNSUPPORTED;
}

extern "C" int emu_group_sum(int d, long long rows, const double* terms, double* sums) {
  if (d == 256) run_group_sum<256>(rows, terms, sums);
  else if (d == 512) run_group_sum<512>(rows, terms, sums);
  else if (d == 1024) run_group_sum<1024>(rows, terms, sums);
  else return CNO_ERR_UNSUPPORTED;
  return 0;
}
