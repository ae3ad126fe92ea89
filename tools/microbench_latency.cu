// tools/microbench_latency.cu -- dependent-issue latencies on the GPU that bound
// the one-warp-per-instance reduction chain (DADD, DMUL, SHFL.BFLY b32 pair, LDS).
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(double* out, long long* cyc, int n) {
  __shared__ double sm[64];
  double a = out[0] + threadIdx.x * 1e-3, b = out[1];
  sm[threadIdx.x & 63] = a;
  __syncthreads();
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) a = a + b;   // DADD chain
  long long t1 = clock64();
  for (int i = 0; i < n; ++i) a = a * b;   // DMUL chain
  long long t2 = clock64();
  for (int i = 0; i < n; ++i) a = __shfl_xor_sync(0xffffffffu, a, 1 + (i & 15));  // 2x SHFL chain
  long long t3 = clock64();
  for (int i = 0; i < n; ++i) a = a * 0.5 + __shfl_xor_sync(0xffffffffu, a, 1 + (i & 15));  // DMUL + butterfly stage
  long long t4 = clock64();
  int idx = threadIdx.x & 31;
  for (int i = 0; i < n; ++i) idx = (int)sm[idx & 63] & 63;  // LDS chain (+cvt)
  long long t5 = clock64();
  float fa = (float)a;
  for (int i = 0; i < n; ++i) fa = fa + 1.5f;
  long long t6 = clock64();
  if (threadIdx.x == 0) { cyc[0]=t1-t0; cyc[1]=t2-t1; cyc[2]=t3-t2; cyc[3]=t4-t3; cyc[4]=t5-t4; cyc[5]=t6-t5; }
  out[2 + threadIdx.x] = a + idx + fa;
}
int main() {
  double* d; long long* c; cudaMalloc(&d, 4096); cudaMalloc(&c, 64);
  double h[2] = {1.0, 1.0000001}; cudaMemcpy(d, h, 16, cudaMemcpyHostToDevice);
  const int n = 4096;
  for (int warps = 1; warps <= 16; warps *= 2) {
    k<<<1, 32 * warps>>>(d, c, n); cudaDeviceSynchronize();
    long long hc[6]; cudaMemcpy(hc, c, 48, cudaMemcpyDeviceToHost);
    printf("warps/SM=%2d  DADD %.1f  DMUL %.1f  SHFL64 %.1f  SHFL64+DADD %.1f  LDS+cvt %.1f  FADD %.1f cycles/op\n", warps,
           hc[0]/(double)n, hc[1]/(double)n, hc[2]/(double)n, hc[3]/(double)n, hc[4]/(double)n, hc[5]/(double)n);
  }
  return 0;
}
