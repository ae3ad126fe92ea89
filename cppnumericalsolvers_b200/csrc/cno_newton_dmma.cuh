// cno_newton_dmma.cuh -- NewtonDescent<F>::Minimize for d = 64 fp64 with the dense
// factorisation on the FP64 TENSOR CORE (policy CNO_POLICY_DMMA_LU), one warp per
// instance, whole Solver::Minimize loop in one persistent kernel (sm_90a).
//
// Reference path: solver/newton_descent.h:66-81 (H += 1e-5 I; delta = H.lu().solve(-g);
// Armijo<F,2>), linesearch/armijo.h:82-101, solver/solver.h:181-224, solver/progress.h:153-327.
//
// ARITHMETIC (CNO_POLICY_DMMA_LU, include/cno.h; oracle: lu_solve(..., fused = 1)): the
// reference's hessian.lu().solve(rhs) as right-looking partial-pivot LU in which every
// multiply-subtract a - l*u is ONE fused operation fma(-l, u, a); every other operation of the
// path follows the default fp64 specification.  An element of the trailing matrix receives
//   a = fma(-l_i0, u_0j, a); a = fma(-l_i1, u_1j, a); ...        (pivot index ascending)
// and mma.sync.m8n8k4.f64 evaluates exactly such a chain (d = c; d = fma(a_k, b_k, d), k = 0..3:
// tools/dmma_probe.cu checks this bit for bit on the GPU).  So the elimination is BLOCKED here -- panels
// of 4 pivots; per panel: (1) the 64 x 4 panel is factored in registers (pivot search, division,
// fused updates; the right-hand side rides along), (2) the row exchanges are applied to the matrix,
// (3) the 4 pivot rows of the trailing block are finished (U12: three fused steps inside each
// 4-lane group, directly in the B-fragment layout), (4) the trailing matrix takes its rank-4 update
// as one DMMA.8x8x4 per 8 x 8 tile with A = the NEGATED multipliers (that is how they are stored) --
// and the result equals the UNBLOCKED fused elimination of the oracle bit for bit.
//
// STORAGE (the factorisation is written against the store concept below):
//   SmemMat  the warp's shared-memory slice in TENSOR-CORE FRAGMENT ORDER: 64 tiles of 8 x 8 (tile (R, Cg) = rows 8R..,
//            columns 8Cg.. at (8R + Cg) * 512 bytes); inside a tile row a = i % 8 owns four 16-byte slots (column
//            pairs), slot 4a + (q ^ ((a >> 1) & 3)), halves exchanged in odd tile rows.  Lane 4a + q of a DMMA holds
//            C[a][2q], C[a][2q+1]: one conflict-free LDS.128 / STS.128 per tile and lane; the XORs spread the rows of one
//            COLUMN over the bank groups for the panel / substitution code (lane l owns rows 2l, 2l+1).  33.6 KB per
//            instance: 6 warps per SM (NewtonDmmaSmem).
// The right-hand side, the row permutation and the solution stay in registers.  DESIGN.md 2.3b.
#ifndef CNO_NEWTON_DMMA_CUH_
#define CNO_NEWTON_DMMA_CUH_

#include "cno_newton.cuh"

namespace cno {

// one fused multiply-add, explicitly (the translation unit is compiled with -fmad=false)
__device__ __forceinline__ double cfma(double a, double b, double c) {
#ifdef CNO_WARP_EMULATION
  return std::fma(a, b, c);
#else
  return __fma_rn(a, b, c);
#endif
}

// D = A*B + C on the FP64 tensor core.  Lane 4m+k supplies A[m][k] and B[k][n = lane/4 ... see below]:
// a = A[lane/4][lane%4], b = B[lane%4][lane/4]; c0, c1 / d0, d1 = C / D[lane/4][2*(lane%4) + {0,1}].
__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b, double c0, double c1) {
#ifdef CNO_WARP_EMULATION
  emu::dmma(d0, d1, a, b, c0, c1);
#else
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};"
      : "=d"(d0), "=d"(d1)
      : "d"(a), "d"(b), "d"(c0), "d"(c1));
#endif
}

__device__ __forceinline__ double2 ld2(const double* p) { return *reinterpret_cast<const double2*>(p); }
__device__ __forceinline__ void st2(double* p, double a, double b) { *reinterpret_cast<double2*>(p) = make_double2(a, b); }

// The 64 x 64 fp64 matrix in fragment order (see the header comment).
struct FragStore {
  static constexpr int kDim = 64;
  static constexpr int kElems = kDim * kDim;
  double* m;
  int lane;
  __device__ __forceinline__ static int swz(int a) { return (a >> 1) & 3; }
  // slot (0..31) of row a, column pair q inside a tile of tile row R: 4a + (q ^ swz(a)), with the two halves of the
  // tile exchanged in odd tile rows -- the lanes of a quarter warp that read one COLUMN of their rows 2l, 2l+1 sit in
  // two adjacent tile rows, which would otherwise share their banks
  __device__ __forceinline__ static int tslot(int R, int a, int q) {
    return ((a << 2) + (q ^ swz(a))) ^ ((R & 1) << 2);
  }
  // the 16-byte slot of row i that holds columns 8*cg + 2*q, 8*cg + 2*q + 1
  __device__ __forceinline__ static int slot(int i, int cg, int q) {
    const int R = i >> 3;
    return ((R << 3) + cg) * 64 + (tslot(R, i & 7, q) << 1);
  }
  __device__ __forceinline__ static int idx(int i, int j) { return slot(i, j >> 3, (j & 7) >> 1) + (j & 1); }
};

// ---- the matrix store, in shared memory ----------------------------------------------------------------
// Concept (lu_dmma_factor / _back / _forward are written against it):
//   stage(src, shift)            A (global, col-major, bitwise symmetric) + shift I -> the store
//   panel_load(kb, P)            P[e][c] = element (2 lane + e, kb + c)
//   swap_rows(k, p)              exchange two whole rows
//   panel_store(kb, vpos, P)     element (vpos[e], kb + c) = P[e][c] for the rows with vpos[e] >= kb
//   update<NCG>(kb)              steps (3) and (4) of a panel, see lu_dmma_factor
//   diag(kb, d)                  d[r][c] = element (kb + r, kb + c)   (valid after panel_load(kb, .))
struct SmemMat {
  double* m;  // fragment order, FragStore
  int lane;

  // A is bitwise symmetric, so COLUMN j read from global memory (lane l: rows 2l, 2l+1 -- one coalesced 16-byte
  // load) is ROW j, columns 2l, 2l+1: exactly one 16-byte slot of the fragment order.
  // xv (shared memory, 64 scalars) / ax: the product A xv is accumulated on the way -- the staged columns are exactly
  // what gemv_global would load, in the same order (j ascending from the first product): the first evaluation of an
  // instance costs no second pass over its block.
  __device__ __forceinline__ void stage(const double* __restrict__ src, double shift, const double* xv,
                                        double (&ax)[2]) const {
    __syncwarp();
#pragma unroll 1
    for (int j0 = 0; j0 < 64; j0 += 16) {  // 16 columns (8 KB per warp) in flight
      double v[16][2];
#pragma unroll
      for (int t = 0; t < 16; ++t) load_row<double, 64>(src + (j0 + t) * 64, lane, v[t]);
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        const int j = j0 + t;  // the diagonal element (j, j) is in the slot of lane j / 2
        const double xj = xv[j];
        ax[0] = (j == 0) ? (v[t][0] * xj) : (ax[0] + v[t][0] * xj);
        ax[1] = (j == 0) ? (v[t][1] * xj) : (ax[1] + v[t][1] * xj);
        if (lane == (j >> 1)) v[t][j & 1] = v[t][j & 1] + shift;
        st2(m + FragStore::slot(j, lane >> 2, lane & 3), v[t][0], v[t][1]);
      }
    }
    __syncwarp();
  }
  __device__ __forceinline__ void panel_load(int kb, double (&P)[2][4]) const {
    const int cgk = kb >> 3, q0 = (kb & 7) >> 1;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int row = 2 * lane + e;
      const double2 a = ld2(m + FragStore::slot(row, cgk, q0)), b = ld2(m + FragStore::slot(row, cgk, q0 + 1));
      P[e][0] = a.x; P[e][1] = a.y; P[e][2] = b.x; P[e][3] = b.y;
    }
  }
  // (lane = one 16-byte slot of each row)
  __device__ __forceinline__ void swap_rows(int k, int p) const {
    double* const pa = m + FragStore::slot(k, lane >> 2, lane & 3);
    double* const pb = m + FragStore::slot(p, lane >> 2, lane & 3);
    const double2 ra = ld2(pa), rb = ld2(pb);
    st2(pa, rb.x, rb.y);
    st2(pb, ra.x, ra.y);
  }
  // a finished panel column: elements (2 lane, j), (2 lane + 1, j) written where the rows currently are (the panel's
  // row exchanges are applied to whole rows afterwards and carry these entries along)
  __device__ __forceinline__ void panel_col_store(int j, double v0, double v1) const {
    m[FragStore::idx(2 * lane, j)] = v0;
    m[FragStore::idx(2 * lane + 1, j)] = v1;
  }
  __device__ __forceinline__ void panel_commit(int) const {}
  __device__ __forceinline__ void diag(int kb, double (&d)[4][4]) const {
    const int cgk = kb >> 3, q0 = (kb & 7) >> 1;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const double2 a = ld2(m + FragStore::slot(kb + r, cgk, q0)), b = ld2(m + FragStore::slot(kb + r, cgk, q0 + 1));
      d[r][0] = a.x; d[r][1] = a.y; d[r][2] = b.x; d[r][3] = b.y;
    }
  }
  // Steps (3) and (4) of a panel for NCG live column groups / tile rows (cg0 = 8 - NCG .. 7; the first one is partial --
  // columns / rows kb+4 .. kb+7 only -- when kb % 8 == 0).  Straight-line code: the NCG chains of step (3) and the
  // NCG x NCG load -> DMMA -> store chains of step (4) are independent and overlap.
  //   (3) U12: rows kb .. kb+3 of the columns right of the panel, in the B-fragment layout (lane = row kb + lane%4,
  //       column 8 cg + lane/4); the three fused steps run inside each 4-lane group.
  //   (4) C -= L21 * U12 as C + (-L21) * U12, one DMMA per 8 x 8 tile.
  template <int NCG>
  __device__ __forceinline__ void update(int kb) const {
    constexpr int cg0 = 8 - NCG;
    const int r4 = lane & 3, n8 = lane >> 2;
    const int cgk = kb >> 3, q0 = (kb & 7) >> 1;
    const bool part = (kb & 7) == 0;                   // the first live group / tile row is the panel's own
    const int prow = kb + r4;
    __syncwarp();
    const double2 l01 = ld2(m + FragStore::slot(prow, cgk, q0));
    const double nl2 = m[FragStore::slot(prow, cgk, q0 + 1)];
    const double nl0 = l01.x, nl1 = l01.y;
    const int base = lane & ~3;
    // element (prow, 8 cg + n8): tile (kb / 8, cg), row a = prow % 8, column pair n8 / 2, element n8 % 2
    const int uoff = (kb >> 3) * 512 + (FragStore::tslot(kb >> 3, prow & 7, n8 >> 1) << 1) + (n8 & 1);
    double bfrag[NCG];
#pragma unroll
    for (int t = 0; t < NCG; ++t) bfrag[t] = m[uoff + (cg0 + t) * 64];
    u12_solve<NCG>(bfrag, nl0, nl1, nl2, r4, base);
#pragma unroll
    for (int t = 0; t < NCG; ++t)  // (a column inside the panel is not part of U12)
      if (r4 > 0 && (t > 0 || !part || n8 >= 4)) m[uoff + (cg0 + t) * 64] = bfrag[t];
    __syncwarp();
#pragma unroll 2
    for (int tr = 0; tr < NCG; ++tr) {  // (rolled: eight variants of this body live in the instruction cache)
      const int R = cg0 + tr;
      // this lane's A-fragment element of tile row R, (8 R + n8, kb + r4), and its C-fragment slot (row n8, pair r4)
      const double afrag = m[R * 512 + cgk * 64 + (FragStore::tslot(R, n8, ((kb & 7) + r4) >> 1) << 1) + (r4 & 1)];
      double* const trow = m + R * 512 + (FragStore::tslot(R, n8, r4) << 1);
      const bool rvalid = tr > 0 || !part || n8 >= 4;
      double2 c[NCG];
#pragma unroll
      for (int t = 0; t < NCG; ++t) c[t] = ld2(trow + (cg0 + t) * 64);
#pragma unroll
      for (int t = 0; t < NCG; ++t) {
        double d0, d1;
        dmma(d0, d1, afrag, bfrag[t], c[t].x, c[t].y);
        if (rvalid && (t > 0 || !part || r4 >= 2)) st2(trow + (cg0 + t) * 64, d0, d1);
      }
    }
    __syncwarp();
  }
  // the three fused steps of U12 inside each 4-lane group (lane r4 of a group = row kb + r4 of one column)
  template <int NCG>
  __device__ __forceinline__ static void u12_solve(double (&b)[NCG], double nl0, double nl1, double nl2, int r4, int base) {
#pragma unroll
    for (int t = 0; t < NCG; ++t) {
      const double u0 = __shfl_sync(kFullMask, b[t], base);
      if (r4 > 0) b[t] = cfma(nl0, u0, b[t]);
    }
#pragma unroll
    for (int t = 0; t < NCG; ++t) {
      const double u1 = __shfl_sync(kFullMask, b[t], base + 1);
      if (r4 > 1) b[t] = cfma(nl1, u1, b[t]);
    }
#pragma unroll
    for (int t = 0; t < NCG; ++t) {
      const double u2 = __shfl_sync(kFullMask, b[t], base + 2);
      if (r4 > 2) b[t] = cfma(nl2, u2, b[t]);
    }
  }
};

// ---- factorisation -----------------------------------------------------------------
// In:  M = H + shift I; rv = this lane's rows (2 lane, 2 lane + 1) of the right-hand side.
// Out: M = the factors (NEGATED multipliers below the diagonal, U on and above it, rows in pivot order);
//      rv = L^{-1} P rhs in pivot order; src[e] = the original row now at position 2 lane + e (the permutation a
//      later lu_dmma_forward applies to a new right-hand side).  vec / permbuf: 64 doubles / 64 ints of warp-private
//      scratch.
template <class Mat>
__device__ __forceinline__ void lu_dmma_factor(const Mat& M, double (&rv)[2], int (&src)[2], double* vec,
                                               int* permbuf) {
  const int lane = M.lane;
  src[0] = 2 * lane;
  src[1] = 2 * lane + 1;

#pragma unroll 1
  for (int kb = 0; kb < 64; kb += 4) {
    // ---- (1) the panel: columns kb .. kb+3 of this lane's two rows, factored in registers with implicit row
    //          exchanges (vpos = the position the oracle's explicit swaps would give the row) ----
    double P[2][4];
    int vpos[2] = {2 * lane, 2 * lane + 1};
    M.panel_load(kb, P);
    unsigned ppos = 0;  // the four pivot positions, one byte each
    // The four pivot steps run as a LOOP (one copy of the step in the instruction cache): the panel is kept rotated so
    // that the column being eliminated is always P[.][0]; a finished column is stored at once, where the rows
    // currently are, and the row exchanges of the panel are applied to whole rows afterwards.
#pragma unroll 1
    for (int r = 0; r < 4; ++r) {
      const int k = kb + r;
      // pivot: first maximal |a_ik| over positions >= k; a NaN at position k stays (the oracle's sequential scan
      // starts from it and no comparison with a NaN is true)
      double best = -1.0;
      int bpos = 0x7fffffff;
      bool k_is_nan = false;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const double v = cabs(P[e][0]);
        const bool cand = vpos[e] >= k;
        if (cand && (v > best || (v == best && vpos[e] < bpos))) { best = v; bpos = vpos[e]; }
        k_is_nan = k_is_nan || ((vpos[e] == k) && (v != v));
      }
      // warp arg-max.  Fast path (one REDUX + one vote): the high words of the lanes' best |v| decide when exactly one
      // lane holds the largest one; a NaN at position k makes its lane win outright.  Otherwise (equal high words,
      // e.g. ties or a zero column) the full comparison: low words, then the smallest position.
      const unsigned hkey = k_is_nan ? 0xffffffffu : (best < 0.0 ? 0u : (unsigned)__double2hiint(best));
      const unsigned hmax = __reduce_max_sync(kFullMask, hkey);
      const unsigned hset = __ballot_sync(kFullMask, hkey == hmax);
      int pp, srcl;
      bool own1;  // in the owner lane: the pivot row is this lane's second row (other lanes' values are not read)
      if (uni_likely((hset & (hset - 1u)) == 0u)) {
        srcl = __ffs(hset) - 1;
        const int mine = k_is_nan ? k : bpos;
        own1 = vpos[1] == mine;  // (known before pp arrives: the value shuffles below do not wait for it)
        pp = __shfl_sync(kFullMask, mine, srcl);
      } else {
        const double bmax = warp_max_nonneg(best < 0.0 ? 0.0 : best);
        const unsigned mypos = (best == bmax) ? (unsigned)bpos : 0xffffffffu;
        const int pmax = (int)__reduce_min_sync(kFullMask, mypos);
        pp = uni(k_is_nan) ? k : pmax;
        const unsigned ob = __ballot_sync(kFullMask, (vpos[1] == pp) || (vpos[0] == pp));
        srcl = __ffs(ob) - 1;
        own1 = vpos[1] == pp;
      }
      ppos |= (unsigned)pp << (8 * r);
      // the pivot row's entries of the (rotated) panel and of the right-hand side, to every lane; the slots past the
      // panel's last column hold stale values that are never stored
      double u[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) u[c] = __shfl_sync(kFullMask, own1 ? P[1][c] : P[0][c], srcl);
      const double urhs = __shfl_sync(kFullMask, own1 ? rv[1] : rv[0], srcl);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool is_p = vpos[e] == pp, is_k = vpos[e] == k;
        vpos[e] = is_p ? k : (is_k ? pp : vpos[e]);
      }
      // multipliers (stored negated: (-a) / pivot) and the fused updates of the later panel columns and of the rhs.
      // The two quotients share the pivot's reciprocal refinement and run side by side, branch free.
      double nl[2];
      {
        const double rp = div_rcp(u[0]);
        bool ok0, ok1;  // (a row that is no longer live divides 1 instead: its entry may be an exact zero)
        nl[0] = div_with((vpos[0] > k) ? -P[0][0] : 1.0, u[0], rp, ok0);
        nl[1] = div_with((vpos[1] > k) ? -P[1][0] : 1.0, u[0], rp, ok1);
        if (uni_unlikely(!(ok0 && ok1))) {
          nl[0] = -P[0][0] / u[0];
          nl[1] = -P[1][0] / u[0];
        }
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (vpos[e] > k) {
          P[e][0] = nl[e];
#pragma unroll
          for (int c = 1; c < 4; ++c) P[e][c] = cfma(nl[e], u[c], P[e][c]);
          rv[e] = cfma(nl[e], urhs, rv[e]);
        }
      }
      M.panel_col_store(k, P[0][0], P[1][0]);
#pragma unroll
      for (int e = 0; e < 2; ++e) { P[e][0] = P[e][1]; P[e][1] = P[e][2]; P[e][2] = P[e][3]; }
    }
    // ---- (2) the four row exchanges on the stored matrix (whole rows: the panel's columns included), the riding
    //          vectors written to their rows' new positions ----
    __syncwarp();
#pragma unroll 1
    for (int r = 0; r < 4; ++r) {
      const int pp = (int)((ppos >> (8 * r)) & 0xffu);
      if (uni_unlikely(pp != kb + r)) M.swap_rows(kb + r, pp);
    }
    M.panel_commit(kb);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      vec[vpos[e]] = rv[e];
      permbuf[vpos[e]] = src[e];
    }
    __syncwarp();
    {
      const double2 t = ld2(vec + 2 * lane);
      rv[0] = t.x;
      rv[1] = t.y;
      src[0] = permbuf[2 * lane];
      src[1] = permbuf[2 * lane + 1];
    }
    if (kb == 60) break;

    // ---- (3) U12 and (4) the trailing update: straight-line code per number of (processed) column groups ----
    switch (8 - ((kb + 4) >> 3)) {
      case 8: M.template update<8>(kb); break;
      case 7: M.template update<7>(kb); break;
      case 6: M.template update<6>(kb); break;
      case 5: M.template update<5>(kb); break;
      case 4: M.template update<4>(kb); break;
      case 3: M.template update<3>(kb); break;
      case 2: M.template update<2>(kb); break;
      default: M.template update<1>(kb); break;
    }
  }
  __syncwarp();
}

// ---- substitutions, blocked by 4 (the 4 x 4 diagonal block is solved redundantly in every lane) ------
// U x = y, column oriented, pivot index descending; rv = this lane's rows of y.  delta = this lane's slice of x.
template <class Mat>
__device__ __forceinline__ void lu_dmma_back(const Mat& M, double (&rv)[2], double (&delta)[2]) {
  const int lane = M.lane;
#pragma unroll 1
  for (int kb = 60; kb >= 0; kb -= 4) {
    double P[2][4], d[4][4];
    M.panel_load(kb, P);
    M.diag(kb, d);
    const int l0 = kb >> 1;
    double y0 = __shfl_sync(kFullMask, rv[0], l0), y1 = __shfl_sync(kFullMask, rv[1], l0);
    double y2 = __shfl_sync(kFullMask, rv[0], l0 + 1), y3 = __shfl_sync(kFullMask, rv[1], l0 + 1);
    // the four divisors are known before their numerators: their reciprocal refinements run ahead of the chain
    const double i3 = div_rcp(d[3][3]), i2 = div_rcp(d[2][2]), i1 = div_rcp(d[1][1]), i0 = div_rcp(d[0][0]);
    const double y0s = y0, y1s = y1, y2s = y2, y3s = y3;
    bool k3, k2, k1, k0;
    double x3 = div_with(y3, d[3][3], i3, k3);
    y2 = cfma(-d[2][3], x3, y2);
    double x2 = div_with(y2, d[2][2], i2, k2);
    y1 = cfma(-d[1][3], x3, y1);
    y1 = cfma(-d[1][2], x2, y1);
    double x1 = div_with(y1, d[1][1], i1, k1);
    y0 = cfma(-d[0][3], x3, y0);
    y0 = cfma(-d[0][2], x2, y0);
    y0 = cfma(-d[0][1], x1, y0);
    double x0 = div_with(y0, d[0][0], i0, k0);
    if (uni_unlikely(!(k3 && k2 && k1 && k0))) {  // rare: an operand outside the short sequence's range
      y0 = y0s; y1 = y1s; y2 = y2s; y3 = y3s;
      x3 = y3 / d[3][3];
      y2 = cfma(-d[2][3], x3, y2);
      x2 = y2 / d[2][2];
      y1 = cfma(-d[1][3], x3, y1);
      y1 = cfma(-d[1][2], x2, y1);
      x1 = y1 / d[1][1];
      y0 = cfma(-d[0][3], x3, y0);
      y0 = cfma(-d[0][2], x2, y0);
      y0 = cfma(-d[0][1], x1, y0);
      x0 = y0 / d[0][0];
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if (2 * lane + e < kb) {
        rv[e] = cfma(-P[e][3], x3, rv[e]);
        rv[e] = cfma(-P[e][2], x2, rv[e]);
        rv[e] = cfma(-P[e][1], x1, rv[e]);
        rv[e] = cfma(-P[e][0], x0, rv[e]);
      }
    }
    if (lane == l0) { delta[0] = x0; delta[1] = x1; }
    if (lane == l0 + 1) { delta[0] = x2; delta[1] = x3; }
  }
  __syncwarp();
}

// L y = P b with the stored (negated) multipliers, pivot index ascending; rv = this lane's rows of P b on entry, of y
// on return: exactly the updates the right-hand side receives when it rides along lu_dmma_factor.
template <class Mat>
__device__ __forceinline__ void lu_dmma_forward(const Mat& M, double (&rv)[2]) {
  const int lane = M.lane;
#pragma unroll 1
  for (int kb = 0; kb < 64; kb += 4) {
    double P[2][4], d[4][4];
    M.panel_load(kb, P);
    M.diag(kb, d);
    const int l0 = kb >> 1;
    const double y0 = __shfl_sync(kFullMask, rv[0], l0);
    double y1 = __shfl_sync(kFullMask, rv[1], l0);
    double y2 = __shfl_sync(kFullMask, rv[0], l0 + 1), y3 = __shfl_sync(kFullMask, rv[1], l0 + 1);
    y1 = cfma(d[1][0], y0, y1);
    y2 = cfma(d[2][0], y0, y2);
    y2 = cfma(d[2][1], y1, y2);
    y3 = cfma(d[3][0], y0, y3);
    y3 = cfma(d[3][1], y1, y3);
    y3 = cfma(d[3][2], y2, y3);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if (2 * lane + e > kb + 3) {
        rv[e] = cfma(P[e][0], y0, rv[e]);
        rv[e] = cfma(P[e][1], y1, rv[e]);
        rv[e] = cfma(P[e][2], y2, rv[e]);
        rv[e] = cfma(P[e][3], y3, rv[e]);
      }
    }
    if (lane == l0) { rv[1] = y1; }
    if (lane == l0 + 1) { rv[0] = y2; rv[1] = y3; }
  }
  __syncwarp();
}

// 0.5 x'Ax - b'x, per-instance [A (64 x 64 col-major, bitwise symmetric) | b]: the functor of cno_newton.cuh
// (value / gradient / H v stream the block from global memory: the Hessian is constant, the store keeps its factors).
struct DenseQuadraticDmmaFn : DenseQuadraticFn<double, 64> {};

// Pulls an instance's [A | b] block (33 280 bytes = 260 lines of 128 bytes) into L2: issued for the instance a warp
// will solve NEXT, so that its staging and evaluations read L2 instead of waiting on DRAM.
__device__ __forceinline__ void prefetch_block_l2(const double* block, int lane) {
#ifndef CNO_WARP_EMULATION
  const char* p = reinterpret_cast<const char*>(block);
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int line = i * 32 + lane;
    if (line < 260) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + (size_t)line * 128));
  }
#else
  (void)block; (void)lane;
#endif
}

// The CTA: 6 warps, each with its matrix (33.6 KB) and vectors in its shared-memory slice.
struct NewtonDmmaSmem {
  static constexpr int kVecElems = 128 /*two vectors*/ + 32 /*64 ints*/ + CNO_MAX_PAST;
  static constexpr int kWarpElems = FragStore::kElems + kVecElems;
  static_assert(kWarpElems % 2 == 0, "warp slices stay 16-byte aligned");
  static constexpr int kWarps = 6;
  static constexpr int kThreads = kWarps * 32;
  static constexpr size_t kBytes = (size_t)kWarps * kWarpElems * sizeof(double);
  static_assert(kBytes <= 227 * 1024, "shared memory per CTA");
};

// One warp's work loop: instances from the queue, the whole Solver::Minimize loop per instance.
template <class Fn, class Mat>
__device__ __forceinline__ void newton_dmma_warp(const Fn& fn, const Mat& M, double* vec, int* permbuf, double* ring,
                                                 const double* __restrict__ x0, const long long batch,
                                                 const StopParams<double>& stop, const BatchOut<double>& out,
                                                 unsigned long long* __restrict__ queue) {
  using T = double;
  constexpr int D = 64;
  constexpr int E = 2;
  using AS = AugStore<T, D>;
  const int lane = M.lane;
  const AS none{nullptr, lane};  // (the functor's evaluations read global memory, not a staged block)

  // The work queue is read ONE INSTANCE AHEAD: while instance b is being solved, the block of the instance this warp
  // takes next is already on its way into L2.
  unsigned long long bnext = claim_instance(queue, lane);
  for (;;) {
    const unsigned long long b = bnext;
    if (uni(b >= (unsigned long long)batch)) break;
    bnext = claim_instance(queue, lane);
    // (the prefetch itself is issued after the first iteration, see below: with two 33 KB blocks per warp in flight for
    // the whole solve, 6 warps x 132 SMs come to about 52 MB -- the size of the 50 MB L2 -- and the second and third
    // pass over A would miss)
    const EvalCtx ctx{lane, (long long)b, nullptr};

    T x[E], g[E];
    load_row<T, D>(x0 + b * D, lane, x);
    // the store receives hessian + safe_guard * I (newton_descent.h:74; factored below), and the first evaluation
    // (solver.h:189-192) takes its A x from the same pass over the block
    T f;
    {
      const T* blk = fn.data + b * fn.stride;
      __syncwarp();
      st2(vec + 2 * lane, x[0], x[1]);
      __syncwarp();
      T Ax[E], bb[E];
      M.stage(blk, T(1e-5), vec, Ax);
      load_row<T, D>(blk + D * D, lane, bb);
#pragma unroll
      for (int e = 0; e < E; ++e) g[e] = Ax[e] - bb[e];
      T p1 = lane_dot<T, E>(x, Ax), p2 = lane_dot<T, E>(bb, x);
      warp_sum2(p1, p2);
      f = T(0.5) * p1 - p2;
    }
    uint32_t nfev = 1;
    bool factored = false;
    int src[E] = {2 * lane, 2 * lane + 1};

    ProgressState<T> prog;
    progress_start(prog);

    do {  // solver.h:196-220
      // ---- newton_descent.h:73-76: (H + 1e-5 I) delta = -g; the constant Hessian is factored once per instance ----
      nfev++;
      T rv[E], delta[E];
      if (uni(factored)) {
        __syncwarp();
        st2(vec + 2 * lane, -g[0], -g[1]);
        __syncwarp();
        rv[0] = vec[src[0]];
        rv[1] = vec[src[1]];
        lu_dmma_forward(M, rv);
      } else {
        rv[0] = -g[0];
        rv[1] = -g[1];
        lu_dmma_factor(M, rv, src, vec, permbuf);
        factored = true;
      }
      lu_dmma_back(M, rv, delta);

      // ---- Armijo<F,2>::Search (armijo.h:82-101) ----
      nfev++;  // f_in = function(x, &gradient, &hessian)
      const T cc = T(0.2), rho = T(0.9);
      T sd[E], r[E];
      const T half_cc = T(0.5) * cc * cc;
#pragma unroll
      for (int e = 0; e < E; ++e) sd[e] = half_cc * delta[e];
      T alpha = T(1.0);
      T xt[E], gt[E];
#pragma unroll
      for (int e = 0; e < E; ++e) xt[e] = x[e] + alpha * delta[e];
      // ((0.5 c^2) d') H and the first trial evaluation in ONE pass over A (global memory / L2)
      T ft = fn.hess_times_and_eval(ctx, sd, r, xt, gt, vec, vec + 64);
      T p1 = lane_dot<T, E>(g, delta), p2 = lane_dot<T, E>(r, delta);
      warp_sum2(p1, p2);
      const T cache = cc * p1 + p2;
      nfev++;
      while (uni(ft > f + alpha * cache)) {
        alpha *= rho;
#pragma unroll
        for (int e = 0; e < E; ++e) xt[e] = x[e] + alpha * delta[e];
        ft = fn(ctx, xt, &gt, none, vec);
        nfev++;
      }
      // ---- x + rate*delta (:80), re-evaluation (solver.h:210-216) = last trial ----
      nfev++;
      T sdx[E];
#pragma unroll
      for (int e = 0; e < E; ++e) sdx[e] = xt[e] - x[e];
      const T prev_value = f;
      const T x_delta = warp_maxabs<T, E>(sdx);
#pragma unroll
      for (int e = 0; e < E; ++e) { x[e] = xt[e]; g[e] = gt[e]; }
      f = ft;
      const T gnorm_inf = warp_maxabs<T, E>(g);
      const T x_inf = warp_maxabs<T, E>(x);
      nfev++;  // Progress::Update's Hessian evaluation (progress.h:206-207)
      progress_update<T>(prog, stop, ring, lane, prev_value, f, x_delta, gnorm_inf, x_inf);
      if (uni(prog.num_iterations == 1 && bnext < (unsigned long long)batch))
        prefetch_block_l2(fn.data + bnext * fn.stride, lane);  // the next instance's block, one iteration ahead
    } while (uni(prog.status == CNO_STATUS_CONTINUE));

    store_result<T, D>(out, b, lane, x, g, f, prog, nfev);
  }
}

template <class Fn>
__global__ void __launch_bounds__(NewtonDmmaSmem::kWarps * 32, 1)
newton_dmma_minimize_kernel(const Fn fn, const double* __restrict__ x0, const long long batch,
                            const StopParams<double> stop, const BatchOut<double> out,
                            unsigned long long* __restrict__ queue) {
  static_assert(Fn::Dim == 64 && sizeof(typename Fn::Scalar) == 8 && Fn::kHessianConstant,
                "the tensor-core factorisation is instantiated for constant 64 x 64 fp64 Hessians");
  using SMN = NewtonDmmaSmem;
  CNO_DYNAMIC_SMEM(smem_raw);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  double* const base = reinterpret_cast<double*>(smem_raw) + (size_t)warp * SMN::kWarpElems;
  double* const vec = base + FragStore::kElems;
  const SmemMat M{base, lane};
  newton_dmma_warp(fn, M, vec, reinterpret_cast<int*>(vec + 128), vec + 128 + 32, x0, batch, stop, out, queue);
}

}  // namespace cno

#endif  // CNO_NEWTON_DMMA_CUH_
