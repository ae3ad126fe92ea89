// tests/emu/warp_emu.h -- HOST stand-ins for the CUDA warp intrinsics, so that device
// source (csrc/*.cuh functors and the one-warp-per-instance kernels, TMA copies as memcpy)
// can be executed on the CPU by 32 lock-step std::threads.
//
// TEST INFRASTRUCTURE ONLY (like oracle/): it is how device code whose first GPU run is
// still pending gets exercised against the oracle in the `-m "not gpu"` suite.  Nothing in
// the product includes this header (csrc/cno_device.cuh pulls it in only under
// CNO_WARP_EMULATION, which only tests/emu defines).
//
// Semantics: every collective is "publish my value -> barrier -> read -> barrier".  The
// FP64 tensor-core reduction (mma.sync.m8n8k4.f64 with A = ones) is restated with the
// arithmetic tools/dmma_probe.cu checks on the GPU: d = c; d = fma(1, b_k, d) = d + b_k.
#ifndef CNO_WARP_EMU_H_
#define CNO_WARP_EMU_H_

#include <atomic>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <functional>
#include <new>
#include <thread>
#include <vector>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __shared__ static
#define __restrict__ __restrict

// CUDA's built-in vector types, as far as csrc/cno_device.cuh uses them
struct alignas(16) double2 { double x, y; };
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
inline double2 make_double2(double x, double y) { return double2{x, y}; }
inline float2 make_float2(float x, float y) { return float2{x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }

namespace emu {
struct Dim3 { unsigned x = 0, y = 0, z = 0; };
// Sense-reversing spin barrier: the 32 lanes of an emulated warp meet thousands of times per solve, and a
// futex-based std::barrier spends most of that time in the kernel; spinning (the box has >= 32 cores) is
// several times faster.  Falls back to yielding when oversubscribed.
struct SpinBarrier {
  std::atomic<int> count{0};
  std::atomic<int> sense{0};
  int total = 32;
  void arrive_and_wait() {
    const int my = sense.load(std::memory_order_relaxed);
    if (count.fetch_add(1, std::memory_order_acq_rel) + 1 == total) {
      count.store(0, std::memory_order_relaxed);
      sense.store(my ^ 1, std::memory_order_release);
    } else {
      int spins = 0;
      while (sense.load(std::memory_order_acquire) == my) {
        if (++spins > 2000) { std::this_thread::yield(); spins = 0; }
        else __builtin_ia32_pause();
      }
    }
  }
};
struct Warp {
  SpinBarrier bar;
  uint64_t slot[32];
  double dslot[32];
  double dslot2[32];
  SpinBarrier* team = nullptr;  // named barrier of a leader + helper team (bar.sync id, 64)
};
inline thread_local int tl_lane = 0;
inline thread_local Warp* tl_warp = nullptr;
inline void sync() { tl_warp->bar.arrive_and_wait(); }

template <class T>
inline T exchange(T v, int src) {  // the value lane `src` published
  static_assert(sizeof(T) <= 8, "exchange: <= 64-bit values");
  uint64_t raw = 0;
  std::memcpy(&raw, &v, sizeof(T));
  tl_warp->slot[tl_lane] = raw;
  sync();
  const uint64_t got = tl_warp->slot[src & 31];
  sync();
  T out;
  std::memcpy(&out, &got, sizeof(T));
  return out;
}

// D = A*B + 0 with A = ones (8x4), B[k][n] from lane 4n+k; lane gets D[lane/4][2*(lane%4) + {0,1}]
inline void dmma_ones(double& d0, double& d1, double b) {
  tl_warp->dslot[tl_lane] = b;
  sync();
  const int j = tl_lane & 3;
  auto col = [&](int n) {
    double d = 0.0;
    for (int k = 0; k < 4; ++k) d = d + tl_warp->dslot[4 * n + k];
    return d;
  };
  d0 = col(2 * j);
  d1 = col(2 * j + 1);
  sync();
}

// General D = A*B + C (mma.sync.m8n8k4.f64): lane supplies A[lane/4][lane%4], B[lane%4][lane/4] and C[lane/4][2*(lane%4)
// + {0,1}]; every element is the FMA chain d = c; d = fma(A[m][k], B[k][n], d), k = 0..3 (tools/dmma_probe.cu).
inline void dmma(double& d0, double& d1, double a, double b, double c0, double c1) {
  tl_warp->dslot[tl_lane] = a;
  tl_warp->dslot2[tl_lane] = b;
  sync();
  const int mrow = tl_lane >> 2, j = tl_lane & 3;
  auto el = [&](int n, double c) {
    double d = c;
    for (int k = 0; k < 4; ++k) d = std::fma(tl_warp->dslot[4 * mrow + k], tl_warp->dslot2[4 * n + k], d);
    return d;
  };
  const double r0 = el(2 * j, c0), r1 = el(2 * j + 1, c1);
  sync();
  d0 = r0;
  d1 = r1;
}

// Runs f(lane) on 32 lock-step threads = one warp.
inline void run_warp(const std::function<void(int)>& f) {
  static Warp w_storage;  // (one emulated warp at a time; too large for the stack)
  Warp& w = w_storage;
  new (&w) Warp();
  std::vector<std::thread> ts;
  for (int l = 0; l < 32; ++l)
    ts.emplace_back([&, l] {
      tl_lane = l;
      tl_warp = &w;
      f(l);
    });
  for (auto& t : ts) t.join();
}
// bar.sync id, 64: the two warps of a team meet (all 64 threads arrive)
inline void team_sync() { tl_warp->team->arrive_and_wait(); }

// Runs f(lane, w) on 64 lock-step threads = a leader warp (w = 0) and its helper warp (w = 1), which share a named
// barrier; shared memory is the kernel's function-static array, as for one warp.
inline void run_team(const std::function<void(int, int)>& f) {
  static Warp w_storage[2];
  static SpinBarrier team_bar;
  new (&team_bar) SpinBarrier();
  team_bar.total = 64;
  for (int w = 0; w < 2; ++w) {
    new (&w_storage[w]) Warp();
    w_storage[w].team = &team_bar;
  }
  std::vector<std::thread> ts;
  for (int w = 0; w < 2; ++w)
    for (int l = 0; l < 32; ++l)
      ts.emplace_back([&, w, l] {
        tl_lane = l;
        tl_warp = &w_storage[w];
        f(l, w);
      });
  for (auto& t : ts) t.join();
}
}  // namespace emu

inline thread_local emu::Dim3 threadIdx, blockIdx, gridDim;

template <class T> inline T __shfl_sync(unsigned, T v, int src) { return emu::exchange(v, src); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m) { return emu::exchange(v, emu::tl_lane ^ m); }
template <class T> inline T __shfl_down_sync(unsigned, T v, int d) {
  const T got = emu::exchange(v, (emu::tl_lane + d) & 31);
  return (emu::tl_lane + d < 32) ? got : v;
}
template <class T> inline T __shfl_up_sync(unsigned, T v, int d) {
  const T got = emu::exchange(v, (emu::tl_lane - d) & 31);
  return (emu::tl_lane - d >= 0) ? got : v;
}
inline unsigned __ballot_sync(unsigned, int pred) {
  unsigned m = 0;
  emu::tl_warp->slot[emu::tl_lane] = pred ? 1u : 0u;
  emu::sync();
  for (int l = 0; l < 32; ++l) m |= (unsigned)(emu::tl_warp->slot[l] & 1u) << l;
  emu::sync();
  return m;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) == 0xffffffffu; }
inline unsigned __reduce_max_sync(unsigned, unsigned v) {
  emu::tl_warp->slot[emu::tl_lane] = v;
  emu::sync();
  unsigned m = 0;
  for (int l = 0; l < 32; ++l) m = std::max<unsigned>(m, (unsigned)emu::tl_warp->slot[l]);
  emu::sync();
  return m;
}
inline unsigned __reduce_min_sync(unsigned, unsigned v) {
  emu::tl_warp->slot[emu::tl_lane] = v;
  emu::sync();
  unsigned m = 0xffffffffu;
  for (int l = 0; l < 32; ++l) m = std::min<unsigned>(m, (unsigned)emu::tl_warp->slot[l]);
  emu::sync();
  return m;
}
inline unsigned __reduce_add_sync(unsigned, unsigned v) {
  emu::tl_warp->slot[emu::tl_lane] = v;
  emu::sync();
  unsigned m = 0;
  for (int l = 0; l < 32; ++l) m += (unsigned)emu::tl_warp->slot[l];
  emu::sync();
  return m;
}
inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::sync(); }
inline void __syncthreads() {}  // only reached from Tensor-Memory paths, which the emulation does not run
inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
template <class T> inline T __ldg(const T* p) { return *p; }
inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) {
  return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST);
}
inline int __double2loint(double d) { uint64_t u; std::memcpy(&u, &d, 8); return (int)(uint32_t)u; }
inline int __double2hiint(double d) { uint64_t u; std::memcpy(&u, &d, 8); return (int)(uint32_t)(u >> 32); }
inline double __hiloint2double(int hi, int lo) {
  const uint64_t u = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo;
  double d; std::memcpy(&d, &u, 8); return d;
}
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
using std::isfinite;

#endif  // CNO_WARP_EMU_H_
