// tests/cpp/one_warp_rosenbrock.cu -- Rosenbrock fp64 at d = 256, 512 and 1024 as a USER functor compiled from the public
// headers: Lbfgs on it runs the one-warp kernel (csrc/cno_lbfgs.cuh, E = d / 32 elements per lane), while the built-in
// family at these d runs the group kernel (csrc/cno_lbfgs_group.cuh).  Both implement the same arithmetic
// specification, so tests/test_lbfgs_group_gpu.py and tools/lbfgs_large_d_bench.py require identical bits from the two.
// The launchers are cno::user_lbfgs, the Lbfgs path of CNO_INSTANTIATE_FUNCTION (whose Bfgs instantiation does not
// fit shared memory past d = 128).
//
//   nvcc -shared ... tests/cpp/one_warp_rosenbrock.cu -o <dir>/libcno_one_warp.so -lcno
//   int cno_one_warp_rosenbrock_minimize(int d, int64_t batch, const double* x0, const cno_stop_t* stop,
//                                        const cno_batch_out_t* out, void* workspace, size_t workspace_bytes,
//                                        void* stream, cno_launch_info_t* info)
#include <cstring>

#include "cppoptlib_b200/device.cuh"

extern "C" int cno_one_warp_rosenbrock_minimize(int d, int64_t batch, const double* x0, const cno_stop_t* stop,
                                                const cno_batch_out_t* out, void* workspace, size_t workspace_bytes,
                                                void* stream, cno_launch_info_t* info) {
#define ONE_WARP_CASE(D)                                                                                          \
  if (d == D)                                                                                                     \
    return cno::user_lbfgs<cppoptlib::function::Rosenbrock<double, D>, cno::LsMoreThuente, CNO_LBFGS_M>(          \
        {}, 1, 0, batch, x0, stop, out, workspace, workspace_bytes, stream, info);
  ONE_WARP_CASE(256)
  ONE_WARP_CASE(512)
  ONE_WARP_CASE(1024)
#undef ONE_WARP_CASE
  return CNO_ERR_UNSUPPORTED;
}
