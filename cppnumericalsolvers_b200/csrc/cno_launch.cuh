// cno_launch.cuh -- the host side of a persistent solver launch, shared by libcno.so (cno_api.cu) and the user-functor
// translation units (include/cppoptlib_b200/device.cuh).
//
// A persistent kernel runs at most one CTA per SM; each of its Plan::kWarps solver warps claims instances from an
// 8-byte queue counter until `batch` are taken.  Every plan struct (LbfgsSmem, BfgsSmem, ...) states its launch as
// kWarps (solver warps per CTA), kThreads (block size) and kBytes (dynamic shared memory per CTA).
// Errors: a failing SM-count query is CNO_ERR_NO_DEVICE, any other CUDA call CNO_ERR_CUDA; the cudaError_t goes to
// the caller's `last_error`.
#ifndef CNO_LAUNCH_CUH_
#define CNO_LAUNCH_CUH_

#ifndef CNO_WARP_EMULATION
#include <cuda_runtime.h>

#include "../../include/cno.h"

namespace cno {

inline int cuda_rc(cudaError_t e, cudaError_t& last_error) {
  if (e == cudaSuccess) return CNO_OK;
  last_error = e;
  return CNO_ERR_CUDA;
}

inline int device_sm_count(int* sms, cudaError_t& last_error) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) return CNO_OK;
  last_error = e;
  return CNO_ERR_NO_DEVICE;
}

// Zeroes the queue counter at `queue` on `stream`, launches kernel(args...) with grid = clamp(ceil(batch / kWarps), 1,
// SMs), and adds the launch to *info (kernel_launches += 1, the shape of this launch).
template <class Plan, class Kernel, class... Args>
inline int launch_persistent(Kernel kernel, long long batch, unsigned long long* queue, cudaStream_t stream,
                             cno_launch_info_t* info, cudaError_t& last_error, const Args&... args) {
  int rc = cuda_rc(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Plan::kBytes),
                   last_error);
  if (rc) return rc;
  int sms = 0;
  if ((rc = device_sm_count(&sms, last_error))) return rc;
  const long long ctas = (batch + Plan::kWarps - 1) / Plan::kWarps;
  const int grid = (int)(ctas < sms ? (ctas < 1 ? 1 : ctas) : sms);
  if ((rc = cuda_rc(cudaMemsetAsync(queue, 0, sizeof(unsigned long long), stream), last_error))) return rc;
  kernel<<<grid, Plan::kThreads, Plan::kBytes, stream>>>(args...);
  if ((rc = cuda_rc(cudaGetLastError(), last_error))) return rc;
  if (info) {
    info->kernel_launches += 1;
    info->grid = grid;
    info->block = Plan::kThreads;
    info->warps_per_cta = Plan::kWarps;
    info->dynamic_smem = (int64_t)Plan::kBytes;
  }
  return CNO_OK;
}

// Device time of what a call enqueues on `stream` between start() and stop(), into info->kernel_ms and
// info->total_ms; does nothing without info.  stop() synchronises on the stream.
class LaunchTimer {
 public:
  LaunchTimer(cudaStream_t stream, cno_launch_info_t* info) : s_(stream), info_(info) {}
  ~LaunchTimer() {
    if (e0_) cudaEventDestroy(e0_);
    if (e1_) cudaEventDestroy(e1_);
  }
  LaunchTimer(const LaunchTimer&) = delete;
  LaunchTimer& operator=(const LaunchTimer&) = delete;

  int start(cudaError_t& last_error) {
    if (!info_) return CNO_OK;
    int rc = cuda_rc(cudaEventCreate(&e0_), last_error);
    if (!rc) rc = cuda_rc(cudaEventCreate(&e1_), last_error);
    if (!rc) rc = cuda_rc(cudaEventRecord(e0_, s_), last_error);
    return rc;
  }
  int stop(cudaError_t& last_error) {
    if (!info_) return CNO_OK;
    int rc = cuda_rc(cudaEventRecord(e1_, s_), last_error);
    if (!rc) rc = cuda_rc(cudaEventSynchronize(e1_), last_error);
    if (!rc) rc = cuda_rc(cudaEventElapsedTime(&info_->kernel_ms, e0_, e1_), last_error);
    if (!rc) info_->total_ms = info_->kernel_ms;
    return rc;
  }

 private:
  cudaStream_t s_;
  cno_launch_info_t* info_;
  cudaEvent_t e0_ = nullptr, e1_ = nullptr;
};

}  // namespace cno

#endif  // CNO_WARP_EMULATION
#endif  // CNO_LAUNCH_CUH_
