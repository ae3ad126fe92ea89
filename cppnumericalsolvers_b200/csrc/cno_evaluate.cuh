// cno_evaluate.cuh -- batched F::operator()(x, &gradient) (function_base.h:103-120, and what
// FunctionExpr::operator() forwards to, :247-250): one warp per instance, value [B] and gradient [B, d]
// written back.  The evaluating FunctionState constructor (function_base.h:315-326) with a batch axis.
#ifndef CNO_EVALUATE_CUH_
#define CNO_EVALUATE_CUH_

#include "cno_device.cuh"
#include "cno_launch.cuh"
#include "../../include/cno.h"

namespace cno {

constexpr int kEvalWarps = 8;

template <class Fn>
__global__ void __launch_bounds__(kEvalWarps * 32)
evaluate_kernel(const Fn fn, const typename Fn::Scalar* __restrict__ x, const long long batch,
                typename Fn::Scalar* __restrict__ value, typename Fn::Scalar* __restrict__ gradient) {
  using T = typename Fn::Scalar;
  constexpr int D = Fn::Dim;
  constexpr int E = Shape<D>::E;
  static_assert(StageElems<Fn>::value == 0,
                "evaluate_kernel: functors that stage per-instance data are evaluated by their solver kernels only");
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * kEvalWarps;
  for (long long b = (long long)blockIdx.x * kEvalWarps + (threadIdx.x >> 5); b < batch; b += warps) {
    const EvalCtx ctx{lane, b, nullptr};
    T xv[E], g[E];
    load_row<T, D>(x + b * D, lane, xv);
    const T f = gradient ? fn(ctx, xv, &g) : fn(ctx, xv, nullptr);
    if (gradient) store_row<T, D>(gradient + b * D, lane, g);
    if (value && lane == 0) value[b] = f;
  }
}

#ifndef CNO_WARP_EMULATION
template <class Fn>
inline int launch_evaluate(const Fn& fn, int64_t batch, const void* x, void* value, void* gradient, void* stream) {
  using T = typename Fn::Scalar;
  if (batch < 0 || (!value && !gradient)) return CNO_ERR_INVALID_ARGUMENT;
  if (batch == 0) return CNO_OK;
  if (!x || ((uintptr_t)x & 15) || ((uintptr_t)gradient & 15)) return CNO_ERR_INVALID_ARGUMENT;
  cudaError_t last_error = cudaSuccess;
  int sms = 0;
  if (device_sm_count(&sms, last_error)) return CNO_ERR_NO_DEVICE;
  long long ctas = (batch + kEvalWarps - 1) / kEvalWarps;
  const long long cap = (long long)sms * 8;
  const int grid = (int)(ctas < cap ? ctas : cap);
  evaluate_kernel<Fn><<<grid, kEvalWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      fn, static_cast<const T*>(x), (long long)batch, static_cast<T*>(value), static_cast<T*>(gradient));
  return cudaGetLastError() == cudaSuccess ? CNO_OK : CNO_ERR_CUDA;
}
#endif

}  // namespace cno

#endif  // CNO_EVALUATE_CUH_
