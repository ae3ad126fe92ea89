// tests/emu/emu_bfgs.cc -- runs the DEVICE SOURCE of every Bfgs Rosenbrock kernel of cno_api.cu's dispatch table
// (csrc/cno_bfgs.cuh: bfgs_minimize_kernel for d <= 32, H in registers; bfgs_smem_minimize_kernel above, H in the warp's
// shared-memory slice) on the CPU under the warp emulation of warp_emu.h.  TEST INFRASTRUCTURE ONLY.
// tests/test_bfgs_rare_paths.py compiles it into a temporary directory with the flags of tests/emu/Makefile:
//
//   g++ -std=c++20 -O1 -ffp-contract=off -fno-fast-math -fPIC -pthread -DCNO_WARP_EMULATION -shared \
//       -I tests/emu -I cppnumericalsolvers_b200/csrc -I include tests/emu/emu_bfgs.cc -o <dir>/libcno_emu_bfgs.so
#include "cno_functors.cuh"
#include "cno_bfgs.cuh"

namespace {

// One warp draining the queue, as one warp of the kernel's CTA does.  Host pointers.
template <class Fn, class LS>
int run_bfgs(long long B, const void* x0, const cno_stop_t* stop, const cno_batch_out_t* out) {
  using T = typename Fn::Scalar;
  unsigned long long queue = 0;
  emu::run_warp([&](int lane) {
    blockIdx.x = 0;
    threadIdx.x = (unsigned)lane;
    const auto sp = cno::make_stop<T>(*stop);
    const auto bo = cno::make_out<T>(*out);
    if constexpr (Fn::Dim <= 32) cno::bfgs_minimize_kernel<Fn, LS>(Fn{}, (const T*)x0, B, sp, bo, &queue);
    else cno::bfgs_smem_minimize_kernel<Fn, LS>(Fn{}, (const T*)x0, B, sp, bo, &queue);
  });
  return 0;
}

}  // namespace

// Bfgs on Rosenbrock with the default policy of the dtype, at the shapes cno_api.cu compiles: MoreThuente at fp64
// d = 2, 8, 32, 37, 64 and 128 and fp32 d = 32 and 128; HagerZhang at fp64 d = 8, 32 and 64.
extern "C" int emu_bfgs(int hager_zhang, const cno_problem_t* p, long long batch, const void* x0, const cno_stop_t* stop,
                        const cno_batch_out_t* out) {
  if (p->family != CNO_FN_ROSENBROCK || p->mode == 2 || p->policy == CNO_POLICY_EIGEN_SSE2) return CNO_ERR_UNSUPPORTED;
#define BFGS_CASE(DT, TY, DIM, LS) \
  if (p->dtype == DT && p->d == DIM) return run_bfgs<cno::RosenbrockFn<TY, DIM>, cno::LS>(batch, x0, stop, out);
  if (hager_zhang) {
    BFGS_CASE(CNO_F64, double, 8, LsHagerZhang)
    BFGS_CASE(CNO_F64, double, 32, LsHagerZhang)
    BFGS_CASE(CNO_F64, double, 64, LsHagerZhang)
    return CNO_ERR_UNSUPPORTED;
  }
  BFGS_CASE(CNO_F64, double, 2, LsMoreThuente)
  BFGS_CASE(CNO_F64, double, 8, LsMoreThuente)
  BFGS_CASE(CNO_F64, double, 32, LsMoreThuente)
  BFGS_CASE(CNO_F64, double, 37, LsMoreThuente)
  BFGS_CASE(CNO_F64, double, 64, LsMoreThuente)
  BFGS_CASE(CNO_F64, double, 128, LsMoreThuente)
  BFGS_CASE(CNO_F32, float, 32, LsMoreThuente)
  BFGS_CASE(CNO_F32, float, 128, LsMoreThuente)
#undef BFGS_CASE
  return CNO_ERR_UNSUPPORTED;
}
