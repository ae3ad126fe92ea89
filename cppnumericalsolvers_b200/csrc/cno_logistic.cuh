// cno_logistic.cuh -- batched logistic regression objective (BASELINE config 3:
// n = 256 samples, d = 64 features, fp32), a device functor with PER-INSTANCE
// DATA staged into shared memory by one TMA bulk copy per instance.
//
// Not in the reference (SURVEY.md 8(d) defines it).  Data block per instance:
//   [Xt (d x n, feature-major: Xt[i*n + j]) | y (n)]        66,560 B at fp32
// The block is read twice per evaluation (margins, gradient) and an instance
// needs ~40 evaluations, so it is staged ONCE per instance and stays ON CHIP:
// HBM traffic = one read of the block per instance instead of one per
// evaluation.  The block arrives in the instance's shared-memory slice by one TMA
// bulk copy (cp.async.bulk + mbarrier), in its global layout, and is evaluated by
// TWO WARPS per instance: the samples come in two chunks of 128; chunk 0 of every
// feature belongs to the solver warp, chunk 1 to the instance's helper warp.
//
// Lane ownership inside the functor: lane l owns samples 128c + 4l .. 4l+3 of
// its warp's chunk c, so every shared-memory access is a contiguous
// conflict-free LDS.128.  Arithmetic definition = oracle eval_logistic
// (oracle/cno_oracle_impl.inc), op for op, incl. the shared exp/log1p kernels
// (glibc's and CUDA's differ in ulps, SURVEY.md 7 hard part 6).
#ifndef CNO_LOGISTIC_CUH_
#define CNO_LOGISTIC_CUH_

#include "cno_device.cuh"
#include "cno_newton.cuh"  // TMA + mbarrier helpers

// Loop-size knobs of the functor: features per gradient round / per batch of margin loads
#ifndef CNO_LOGISTIC_ROUND_FEATURES
#define CNO_LOGISTIC_ROUND_FEATURES 16
#endif
#ifndef CNO_LOGISTIC_MARGIN_BATCH
#define CNO_LOGISTIC_MARGIN_BATCH 8
#endif

namespace cno {

// exp(x), x <= 0 in practice: 2^k * exp(r), degree-9 Taylor (no FMA).
__device__ __forceinline__ float cno_exp(float x) {
  if (x > 88.f) x = 88.f;
  if (x < -87.f) return 0.f;
  const float kf = rintf(x * 1.44269504088896341f);
  const float r = (x - kf * 0.693145751953125f) - kf * 1.42860682030941723212e-6f;
  float p = (float)(1.0 / 362880.0);
  p = p * r + (float)(1.0 / 40320.0);
  p = p * r + (float)(1.0 / 5040.0);
  p = p * r + (float)(1.0 / 720.0);
  p = p * r + (float)(1.0 / 120.0);
  p = p * r + (float)(1.0 / 24.0);
  p = p * r + (float)(1.0 / 6.0);
  p = p * r + 0.5f;
  p = p * r + 1.f;
  p = p * r + 1.f;
  // ldexpf(p, k) with k in [-126, 127] (x is clamped to [-87, 88]): 2^k is a normal float, so one IEEE multiplication
  // rounds the exact product p 2^k once, like ldexpf does -- without libdevice's ldexpf branches
  return p * __uint_as_float((uint32_t)((int)kf + 127) << 23);
}
__device__ __forceinline__ double cno_exp(double x) {
  if (x > 88.0) x = 88.0;
  if (x < -87.0) return 0.0;
  const double kf = rint(x * 1.44269504088896341);
  const double r = (x - kf * 0.693145751953125) - kf * 1.42860682030941723212e-6;
  double p = (1.0 / 362880.0);
  p = p * r + (1.0 / 40320.0);
  p = p * r + (1.0 / 5040.0);
  p = p * r + (1.0 / 720.0);
  p = p * r + (1.0 / 120.0);
  p = p * r + (1.0 / 24.0);
  p = p * r + (1.0 / 6.0);
  p = p * r + 0.5;
  p = p * r + 1.0;
  p = p * r + 1.0;
  return ldexp(p, (int)kf);
}
// log1p(u), u in [0, 1]: 2 atanh(u / (2 + u)).
template <class T>
__device__ __forceinline__ T cno_log1p01(T u) {
  const T z = u / (T(2) + u);
  const T z2 = z * z;
  T p = (T)(1.0 / 19.0);
  p = p * z2 + (T)(1.0 / 17.0);
  p = p * z2 + (T)(1.0 / 15.0);
  p = p * z2 + (T)(1.0 / 13.0);
  p = p * z2 + (T)(1.0 / 11.0);
  p = p * z2 + (T)(1.0 / 9.0);
  p = p * z2 + (T)(1.0 / 7.0);
  p = p * z2 + (T)(1.0 / 5.0);
  p = p * z2 + (T)(1.0 / 3.0);
  p = p * z2 + T(1);
  return (T(2) * z) * p;
}

template <class T, int D, int N>
struct LogisticFn {
  using Scalar = T;
  static constexpr int Dim = D;
  static constexpr int Mode = 1;
  static constexpr int E = Shape<D>::E;
  static_assert(sizeof(T) == 4, "LDS.128 = 4 samples; instantiate for float");
  static_assert(N == 256, "two chunks of 128 samples (32 lanes x 4): one per warp of the team");
  static_assert(D % 16 == 0, "the gradient is built in rounds of kRF features");
  static constexpr int kBlockElems = D * N + N;  // [Xt | y] in global memory
  static constexpr int kWvec = ((D + 3) / 4) * 4;
  // Features per gradient round (each warp owns kG = kRF / 2 of them: its butterflies in flight).  Code size matters
  // here: the solver and helper warps of several instances share a sub-partition's instruction cache (L0), so the four
  // samples' losses are a rolled loop (losses()) rather than straight-line code.
  static constexpr int kRF = CNO_LOGISTIC_ROUND_FEATURES;
  static constexpr int kG = kRF / 2;
  // A helper warp per instance (FnHelperWarps).  The split keeps every sum of the arithmetic definition in its order:
  //  * the margin of a sample is one serial chain over the features: each warp runs the chains of ITS chunk;
  //  * a gradient component is, per lane, (partial of chunk 0) + (partial of chunk 1), then the lane butterfly: each
  //    warp forms the partials of its chunk for kRF features per round, hands the other warp the partials of the
  //    features that warp owns (shared memory, double-buffered), adds what it received and runs the butterflies of
  //    its own features -- a + b is the same float whichever warp adds;
  //  * the loss is (lane partial of chunk 0) + (lane partial of chunk 1), then the lane butterfly: the helper hands over
  //    its lane partials.
  static constexpr int kHelperWarps = 1;
  static constexpr int kRounds = D / kRF;
  // shared-memory slice of the team (elements): Xt (feature i: chunk 0 | chunk 1) | y | broadcast copy of w |
  // mbarrier (8 bytes) | exchange area: partials for the solver warp [2 buffers][8][32], for the helper [2][8][32], the
  // helper's loss partials [32], its gradient sums [D/2], the command word
  static constexpr int kX = 0, kY = D * N, kW = kY + N, kBar = kW + kWvec;
  static constexpr int kXchgOff = ((kBar + 8 / (int)sizeof(T) + 3) / 4) * 4;
  static constexpr int kToL = 0, kToH = 2 * 8 * 32, kXLoss = 2 * kToH, kXGrad = kXLoss + 32, kXCmd = kXGrad + D / 2,
                       kXchgElems = kXCmd + 4;
  static constexpr int kCmdEval = 1, kCmdEvalGrad = 2, kCmdStage = 3, kCmdExit = 4;
  static constexpr int kStageElems = kXchgOff + kXchgElems;

  const T* data;
  long long stride;
  T lambda;

  using P4 = Pack<T, 4>;
  __device__ __forceinline__ static T* xchg(const EvalCtx& c) { return static_cast<T*>(c.stage) + kXchgOff; }
  __device__ __forceinline__ static volatile int* cmd_word(const EvalCtx& c) {
    return reinterpret_cast<volatile int*>(xchg(c) + kXCmd);
  }

  // once per instance: the block [Xt | y] -> shared memory, one TMA bulk copy issued by the solver warp; both warps of
  // the team wait for it on the mbarrier (the helper when it picks up kCmdStage)
  __device__ __forceinline__ void stage(const EvalCtx& c, uint32_t& parity) const {
    T* blk = static_cast<T*>(c.stage);
    uint64_t* bar = reinterpret_cast<uint64_t*>(blk + kBar);
    __syncwarp();
    fence_proxy_async();  // the previous instance's reads of the slice come before the copy overwrites it
    if (c.lane == 0) {
      cmd_word(c)[0] = kCmdStage;
      mbar_expect_tx(bar, (uint32_t)(kBlockElems * sizeof(T)));
      tma_bulk_g2s(blk + kX, data + c.instance * stride, (uint32_t)(kBlockElems * sizeof(T)), bar);
    }
    team_sync(c.team);  // the helper picks the command up (and every lane is past the expect_tx)
    mbar_wait(bar, parity);
    parity ^= 1u;
  }
  __device__ __forceinline__ void init_stage(const EvalCtx& c) const {
    T* blk = static_cast<T*>(c.stage);
    uint64_t* bar = reinterpret_cast<uint64_t*>(blk + kBar);
    if (c.lane == 0) {
      mbar_init(bar, 1);
#ifndef CNO_WARP_EMULATION
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
    }
    __syncwarp();
  }
  __device__ __forceinline__ void release_helper(const EvalCtx& c) const {
    __syncwarp();
    if (c.lane == 0) cmd_word(c)[0] = kCmdExit;
    team_sync(c.team);
  }

  // 4 values per lane of features i0 .. i0 + NF - 1 of this warp's chunk (solver warp: chunk 0, helper: chunk 1)
  template <bool kHelper, int NF>
  __device__ __forceinline__ void load_features(const EvalCtx& c, int i0, T (&x)[NF][4]) const {
    const T* X = static_cast<const T*>(c.stage) + kX + (kHelper ? 128 : 0) + 4 * c.lane;
#pragma unroll
    for (int q = 0; q < NF; ++q) P4::get(*reinterpret_cast<const typename P4::type*>(X + (i0 + q) * N), x[q]);
  }
  // margins z_j = sum_i Xt[i][j] w_i (i ascending) of the 4 samples this lane owns in its warp's chunk.  The chain
  // starts from -0: (-0) + p is p for every float p, the zeros with their signs included, so the first step leaves the
  // first product exactly as the definition has it and every batch runs the same code.
  template <bool kHelper>
  __device__ __forceinline__ void margins(const EvalCtx& c, T (&z)[4]) const {
    const T* wv = static_cast<const T*>(c.stage) + kW;
    constexpr int NF = CNO_LOGISTIC_MARGIN_BATCH;  // features per batch of loads
#pragma unroll
    for (int t = 0; t < 4; ++t) z[t] = -T(0);
#pragma unroll 1
    for (int i0 = 0; i0 < D; i0 += NF) {
      T x[NF][4];
      load_features<kHelper, NF>(c, i0, x);
#pragma unroll
      for (int q4 = 0; q4 < NF; q4 += 4) {
        T w4[4];
        P4::get(*reinterpret_cast<const typename P4::type*>(wv + i0 + q4), w4);
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int t = 0; t < 4; ++t) z[t] = z[t] + x[q4 + k][t] * w4[k];
      }
    }
  }
  // per-sample loss and coefficient of the chunk; returns the lane's loss partial of the chunk.  One sample per trip of a
  // ROLLED loop (the four samples rotate through one set of registers): the compiler serialises the samples anyway
  // (the exp early-out and the division slow paths are branches), so unrolled it is four times the code for nothing.
  template <bool kHelper>
  __device__ __forceinline__ T losses(const EvalCtx& c, const T (&z)[4], T (&coef)[4]) const {
    const T* y = static_cast<const T*>(c.stage) + kY;
    T yv[4], ls[4], zz[4];
    P4::get(*reinterpret_cast<const typename P4::type*>(y + (kHelper ? 128 : 0) + 4 * c.lane), yv);
#pragma unroll
    for (int t = 0; t < 4; ++t) { zz[t] = z[t]; ls[t] = coef[t] = T(0); }
#pragma unroll 1
    for (int t = 0; t < 4; ++t) {
      const T m = yv[0] * zz[0];
      const T e = cno_exp(-cabs(m));
      const T l1p = cno_log1p01<T>(e);
      const T l = (m < T(0)) ? (l1p - m) : l1p;
      const T sig = ((m < T(0)) ? T(1) : e) / (T(1) + e);  // 1 / (1 + e) or e / (1 + e): one division, the same operands
      const T cf = -(yv[0] * sig);
      // rotate: sample t+1 moves to the front, the results of sample t to the back
      yv[0] = yv[1]; yv[1] = yv[2]; yv[2] = yv[3];
      zz[0] = zz[1]; zz[1] = zz[2]; zz[2] = zz[3];
      ls[0] = ls[1]; ls[1] = ls[2]; ls[2] = ls[3]; ls[3] = l;
      coef[0] = coef[1]; coef[1] = coef[2]; coef[2] = coef[3]; coef[3] = cf;
    }
    return (ls[0] + ls[1]) + (ls[2] + ls[3]);
  }
  // One round of the gradient (features kRF r .. kRF r + kRF - 1; the solver warp owns the first kG, the helper the
  // last kG): the chunk's partials of all kRF, exchange of kG + kG, the complete sums of the features this warp owns in p.
  template <bool kHelper>
  __device__ __forceinline__ void gradient_round(const EvalCtx& c, int r, const T (&coef)[4], T (&p)[kG]) const {
    T* xc = xchg(c);
    const int lane = c.lane;
    T* mine_in = xc + (kHelper ? kToH : kToL) + (r & 1) * 256;    // what the other warp hands me
    T* other_in = xc + (kHelper ? kToL : kToH) + (r & 1) * 256;   // what I hand the other warp
    T x[kRF][4];
    load_features<kHelper, kRF>(c, kRF * r, x);
    T part[kRF];
#pragma unroll
    for (int q = 0; q < kRF; ++q) part[q] = (coef[0] * x[q][0] + coef[1] * x[q][1]) + (coef[2] * x[q][2] + coef[3] * x[q][3]);
#pragma unroll
    for (int q = 0; q < kG; ++q) other_in[q * 32 + lane] = part[kHelper ? q : kG + q];
    team_sync(c.team);
#pragma unroll
    for (int q = 0; q < kG; ++q) {
      const T got = mine_in[q * 32 + lane];
      p[q] = kHelper ? (got + part[kG + q]) : (part[q] + got);  // (chunk 0) + (chunk 1)
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
#pragma unroll
      for (int q = 0; q < kG; ++q) p[q] = p[q] + __shfl_xor_sync(kFullMask, p[q], off);
    }
  }

  // ---- the solver warp ----
  __device__ __forceinline__ T operator()(const EvalCtx& c, const T (&w)[E], T (*grad)[E]) const {
    T* wv = static_cast<T*>(c.stage) + kW;
    T* xc = xchg(c);
    const int lane = c.lane;
    // broadcast copy of w + the command
    __syncwarp();
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (lane * E + e < D) wv[lane * E + e] = w[e];
    if (lane == 0) cmd_word(c)[0] = grad ? kCmdEvalGrad : kCmdEval;
    team_sync(c.team);  // w and the command are visible to the helper
    T z[4], coef[4];
    margins<false>(c, z);
    const T part0 = losses<false>(c, z, coef);
    if (grad) {
#pragma unroll
      for (int e = 0; e < E; ++e) (*grad)[e] = T(0);
#pragma unroll 1
      for (int r = 0; r < kRounds; ++r) {
        T p[kG];
        gradient_round<false>(c, r, coef, p);
#pragma unroll
        for (int q = 0; q < kG; ++q) {
#pragma unroll
          for (int e = 0; e < E; ++e)
            if (lane * E + e == kRF * r + q) (*grad)[e] = p[q] + lambda * w[e];
        }
      }
    }
    team_sync(c.team);  // the helper's loss partials (and the sums of its features) are in the exchange area
    if (grad) {
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const int i = lane * E + e;
        if (i < D && (i & kG)) (*grad)[e] = xc[kXGrad + (i / kRF) * kG + (i & (kG - 1))] + lambda * w[e];
      }
    }
    const T lsum = part0 + xc[kXLoss + lane];
    const T data_loss = warp_sum(lsum);
    const T reg = (T(0.5) * lambda) * warp_dot<T, E>(w, w);
    return data_loss + reg;
  }

  // ---- the helper warp ----
  __device__ __noinline__ void helper(const EvalCtx& c) const {
    T* xc = xchg(c);
    const int lane = c.lane;
    uint64_t* bar = reinterpret_cast<uint64_t*>(static_cast<T*>(c.stage) + kBar);
    uint32_t parity = 0;
    for (;;) {
      team_sync(c.team);
      const int cmd = cmd_word(c)[0];
      if (cmd == kCmdExit) break;
      if (cmd == kCmdStage) {  // the next instance's block: wait until it has landed
        mbar_wait(bar, parity);
        parity ^= 1u;
        continue;
      }
      T z[4], coef[4];
      margins<true>(c, z);
      xc[kXLoss + lane] = losses<true>(c, z, coef);
      if (cmd == kCmdEvalGrad) {
#pragma unroll 1
        for (int r = 0; r < kRounds; ++r) {
          T p[kG];
          gradient_round<true>(c, r, coef, p);
          T mine = p[0];  // (every lane holds every sum after the butterfly)
#pragma unroll
          for (int q = 1; q < kG; ++q) mine = (lane == q) ? p[q] : mine;
          if (lane < kG) xc[kXGrad + kG * r + lane] = mine;
        }
      }
      team_sync(c.team);
    }
  }
};

}  // namespace cno

#endif  // CNO_LOGISTIC_CUH_
