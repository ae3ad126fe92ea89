// tests/emu/emu_lbfgsb_group.cc -- runs the DEVICE SOURCE of the group Lbfgsb kernel (csrc/cno_lbfgsb_group.cuh: one
// group of d / 128 warps per instance, d = 256 / 512 / 1024) on the CPU under the warp emulation of warp_emu.h.  TEST
// INFRASTRUCTURE ONLY.  tests/test_lbfgsb_group.py compiles it into a temporary directory with the flags of
// tests/emu/Makefile:
//
//   g++ -std=c++20 -O1 -ffp-contract=off -fno-fast-math -fPIC -pthread -DCNO_WARP_EMULATION -shared \
//       -I tests/emu -I cppnumericalsolvers_b200/csrc -I include tests/emu/emu_lbfgsb_group.cc -o <dir>/libcno_emu_lbfgsb_group.so
#include <cstdlib>

#include "cno_functors.cuh"
#include "cno_lbfgsb_group.cuh"

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
int run_group_lbfgsb(long long B, const void* x0, const void* lower, const void* upper, long long stride,
                     const cno_stop_t* stop, const cno_batch_out_t* out) {
  using Fn = cno::GroupRosenbrockFn<double, D>;
  unsigned long long queue = 0;
  const cno::BoundsArgs<double> bd{static_cast<const double*>(lower), static_cast<const double*>(upper), stride};
  run_group(
      [&](int lane, int w) {
        blockIdx.x = 0;
        threadIdx.x = (unsigned)(32 * w + lane);
        cno::lbfgsb_group_minimize_kernel<Fn, 5>(Fn{}, (const double*)x0, B, cno::make_stop<double>(*stop),
                                                 cno::make_out<double>(*out), &queue, bd);
      },
      Fn::kGroupWarps);
  return 0;
}

// The compacted sum alone: sums[r] = the sum of terms[r, 0 .. n[r] - 1] (a compacted vector of length n[r] <= d) as the
// kernel forms (W'Z) r when n < d: thread (w, l) takes positions 4 w .. 4 w + 3 of lane l's run of ceil(n / 32),
// group_lane_partials_masked, then the warp sum.  Positions of a run at or past n take the value pad[r] (+0 in the
// kernel); absent positions (past the run) hold 1e300, which must never be added.
template <int D>
void run_compacted_sum(const int* ns, long long rows, const double* terms, const double* pad, double* sums) {
  constexpr int W = D / 128;
  alignas(16) static double scratch[2 * cno::GroupCtx<double, W>::kBufElems];
  run_group(
      [&](int lane, int w) {
        const cno::GroupCtx<double, W> rc{scratch, lane, w, 1, 0};
        for (long long r = 0; r < rows; ++r) {
          const int n = ns[r], ep = (n + 31) / 32;
          double v[1][4];
          for (int c = 0; c < 4; ++c) {
            const int j = 4 * w + c, q = lane * ep + j;
            v[0][c] = (j < ep && q < n) ? terms[r * D + q] : ((j < ep) ? pad[r] : 1e300);  // absent: never added
          }
          double part[1];
          cno::group_lane_partials_masked<1>(rc, v, ep, part);
          const double s = cno::warp_sum(part[0]);
          if (lane == 0 && w == 0) sums[r] = s;
        }
      },
      W);
}

}  // namespace

// Lbfgsb<Rosenbrock, 5> fp64 at d = 256 / 512 / 1024, the default policy.  lower / upper: [d] (stride 0) or [B, d]
// (stride d), or NULL.
extern "C" int emu_lbfgsb_group(const cno_problem_t* p, long long batch, const void* x0, const void* lower,
                                const void* upper, long long stride, const cno_stop_t* stop,
                                const cno_batch_out_t* out) {
  if (p->family != CNO_FN_ROSENBROCK || p->dtype != CNO_F64 || p->policy != CNO_POLICY_DMMA_TREE ||
      (p->lbfgs_m != 0 && p->lbfgs_m != 5))
    return CNO_ERR_UNSUPPORTED;
  if (p->d == 256) return run_group_lbfgsb<256>(batch, x0, lower, upper, stride, stop, out);
  if (p->d == 512) return run_group_lbfgsb<512>(batch, x0, lower, upper, stride, stop, out);
  if (p->d == 1024) return run_group_lbfgsb<1024>(batch, x0, lower, upper, stride, stop, out);
  return CNO_ERR_UNSUPPORTED;
}

// terms: [rows, d]; the first ns[r] entries of row r are its compacted vector.
extern "C" int emu_compacted_sum(int d, const int* ns, long long rows, const double* terms, const double* pad,
                                 double* sums) {
  for (long long r = 0; r < rows; ++r)
    if (ns[r] < 1 || ns[r] > d) return CNO_ERR_INVALID_ARGUMENT;
  if (d == 256) run_compacted_sum<256>(ns, rows, terms, pad, sums);
  else if (d == 512) run_compacted_sum<512>(ns, rows, terms, pad, sums);
  else if (d == 1024) run_compacted_sum<1024>(ns, rows, terms, pad, sums);
  else return CNO_ERR_UNSUPPORTED;
  return 0;
}
