// tests/cpp/al_user_functions.cu -- AugmentedLagrangian on functor-constrained problems (al_user_problems.cuh),
// compiled for the device through CNO_INSTANTIATE_CONSTRAINED as a shared library for tests/test_al_user_gpu.py.
//
//   nvcc -shared ... tests/cpp/al_user_functions.cu -o libcno_al_user.so -lcno
#include <cstring>

#include "cppoptlib_b200/device.cuh"
#include "al_user_problems.cuh"

#define X(tag, id, dtype, d, S)                                                                               \
  using Problem_##tag = cppoptlib::function::ConstrainedOptimizationProblem<S::Obj, S::Eq, S::In>;            \
  CNO_DECLARE_CONSTRAINED(tag, Problem_##tag)                                                                 \
  CNO_INSTANTIATE_CONSTRAINED(tag, Problem_##tag)
ALU_PROBLEMS(X)
#undef X

// One entry point for the Python tests: builds problem `problem` at (dtype, d) from data / data_stride (problem 4:
// the radii [B]; problem 5: the [a | t] rows) and runs cno_<tag>_al_minimize, or (out == NULL) writes
// cno_<tag>_al_workspace_bytes into *bytes.
extern "C" int cno_test_al_user(int problem, int dtype, int d, const void* data, int64_t data_stride, int64_t batch,
                                const void* x0, const void* eq0, const void* ineq0, const void* penalty0,
                                const cno_stop_t* inner_stop, const cno_al_stop_t* outer_stop,
                                const cno_al_config_t* config, const cno_al_out_t* out, void* workspace,
                                size_t workspace_bytes, void* stream, cno_launch_info_t* info, size_t* bytes) {
#define X(tag, id, dt, dim, S)                                                                                 \
  if (problem == id && dtype == dt && d == dim) {                                                              \
    if (!out) return cno_##tag##_al_workspace_bytes(batch, bytes);                                             \
    const auto parts = S::make(data, (long long)data_stride);                                                  \
    const Problem_##tag p{parts.objective, parts.equality_constraints, parts.inequality_constraints};          \
    return cno_##tag##_al_minimize(&p, batch, x0, eq0, ineq0, penalty0, inner_stop, outer_stop, config, out,   \
                                   workspace, workspace_bytes, stream, info);                                  \
  }
  ALU_PROBLEMS(X)
#undef X
  return CNO_ERR_UNSUPPORTED;
}
