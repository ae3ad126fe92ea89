/*
 * cno_oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the reference's algorithm for the hot path
 * (cppoptlib solver::{Lbfgs,Bfgs,NewtonDescent}::Minimize).  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library; the product (libcno.so) never links or calls it.
 *
 * Pinning status: the restatement is checked (tests/test_oracle_pins.py)
 * against every golden vector the reference's own tests hold for this path
 * (7 cstep KATs, verify.cc Far/Near, Dockerfile.test quadratic, the AL-test
 * half-norm solve) AND, bit for bit, against oracle/_ref = the reference's own
 * headers compiled from /root/reference against an Eigen-API shim
 * (oracle/ref_shim).  Real Eigen is not available in this image, so the
 * reduction order of dot()/norm() is a specification of this repo
 * (DESIGN.md "Arithmetic specification"), not Eigen's: iteration-count parity
 * against a real Eigen build is therefore "parity unpinned".
 */
#ifndef CNO_ORACLE_H_
#define CNO_ORACLE_H_

#include "../include/cno.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Batched Minimize on the CPU.  Same argument meaning as cno_minimize_host;
 * all pointers are host pointers.  threads <= 0 = all cores (OpenMP, one
 * instance per task, schedule(dynamic)). Returns 0 or a cno_error_t. */
int cno_oracle_minimize(int solver, const cno_problem_t* problem, int64_t batch,
                        const void* x0, const cno_stop_t* stop,
                        const cno_batch_out_t* out, int threads);

/* The LineSearch template parameter of Lbfgs / Bfgs / GradientDescent (lbfgs.h:41,
 * bfgs.h:40, gradient_descent.h:38).  HagerZhang (linesearch/hager_zhang.h:54-552) is
 * SURVEY.md 8(f) rank 2: restated and pinned here, not on the device yet. */
typedef enum cno_oracle_linesearch { CNO_LS_MORE_THUENTE = 0, CNO_LS_HAGER_ZHANG = 1 } cno_oracle_linesearch_t;
int cno_oracle_minimize_ls(int solver, const cno_problem_t* problem, int64_t batch,
                           const void* x0, const cno_stop_t* stop,
                           const cno_batch_out_t* out, int threads, int linesearch);

/* Most pairs Lbfgs<F, m> may keep (cno_problem_t::lbfgs_m). */
#define CNO_ORACLE_MAX_M 32

/* How often one Lbfgs instance took the rare branches of OptimizationStep (lbfgs.h:89-303), so that tests can show
 * which paths an input reaches.  k = mem_count when the step begins. */
typedef struct cno_lbfgs_paths {
  /* pairs skipped by the first loop (|s_i . y_i| < eps, lbfgs.h:165): [k < m, k == m][position counted from the
   * newest pair: 0, 1, >= 2] */
  uint64_t skipped[2][3];
  /* pairs refused by the curvature test (lbfgs.h:267) while the history held at least one pair */
  uint64_t rejected;
  /* descent-test fallbacks (lbfgs.h:214-224), by k */
  uint64_t fallback[CNO_ORACLE_MAX_M + 1];
  /* non-finite line-search results (lbfgs.h:239-241), by k after the descent test */
  uint64_t nonfinite[CNO_ORACLE_MAX_M + 1];
} cno_lbfgs_paths_t;

/* cno_oracle_minimize(CNO_LBFGS, ...) with MoreThuente that also fills paths[batch]. */
int cno_oracle_lbfgs_paths(const cno_problem_t* problem, int64_t batch, const void* x0,
                           const cno_stop_t* stop, const cno_batch_out_t* out,
                           cno_lbfgs_paths_t* paths, int threads);

/* How often one Bfgs instance took the rare branches of OptimizationStep (bfgs.h:73-137), so that tests can show
 * which paths an input reaches.  Counting only reads the step's values; the arithmetic is the same with or without. */
typedef struct cno_bfgs_paths {
  /* resets of H to the identity (bfgs.h:88-92): phi > 0, phi NaN */
  uint64_t reset_positive, reset_nan;
  /* updates refused by the curvature test (bfgs.h:125) while H was the identity (fresh) / after an update */
  uint64_t refused_fresh, refused_updated;
  /* curvature tests that the device's square-root-free bound (s.y > 0, (s.y)^2 and (s.s)(y.y) finite, (s.y)^2
   * normal and (s.y)^2 > 2 eps^2 (s.s)(y.y); csrc/cno_device.cuh: curvature_above_eps) does not decide, so the
   * specification's expression does: by its outcome (false, true) */
  uint64_t curvature_fallback[2];
  /* line searches that returned a non-finite value */
  uint64_t nonfinite;
  /* fresh steps with ||d|| <= eps (alpha_init = 1, bfgs.h:100-106) */
  uint64_t small_direction;
} cno_bfgs_paths_t;

/* cno_oracle_minimize_ls(CNO_BFGS, ...) that also fills paths[batch]. */
int cno_oracle_bfgs_paths(const cno_problem_t* problem, int64_t batch, const void* x0, const cno_stop_t* stop,
                          const cno_batch_out_t* out, cno_bfgs_paths_t* paths, int threads, int linesearch);

/* HagerZhang<F,1>::Search on the 1-D quartic (((c4 v + c3) v + c2) v + c1) v + c0 of
 * src/test/hager_zhang_test.cc (Quadratic, Cubic, FlatQuartic) along s = +1 from x0. */
int cno_oracle_hz_search_poly(const double coef[5], double x0, double alpha_init,
                              double* alpha, double* f_out, double* x_out, int* nfev);

/* Objective evaluation only: f[B], g[B,d] (nullable), H[B,d,d] col-major
 * (nullable; Second-mode families only). */
int cno_oracle_evaluate(const cno_problem_t* problem, int64_t batch,
                        const void* x, void* f, void* g, void* H);

/* Progress::condition_hessian (solver/progress.h:203-210) = H(x).norm() * H(x).inverse().norm() at
 * x[b] (Second-mode families): out[B].  Oracle twin of cno_condition_hessian. */
int cno_oracle_condition_hessian(const cno_problem_t* problem, int64_t batch, const void* x, void* out);

/* Host twin of cno_fill_uniform (dst is a host pointer). */
int cno_oracle_fill_uniform(int dtype, void* dst, int64_t first, int64_t count,
                            uint64_t seed, double lo, double hi);

/* The reduction of the arithmetic spec, exposed for unit tests. */
double cno_oracle_reduce_sum_f64(const double* t, int d, int policy);
float cno_oracle_reduce_sum_f32(const float* t, int d, int policy);

/* MoreThuente::cstep (linesearch/more_thuente.h:261-407) on doubles; same io
 * layout as cno_device_cstep. */
int cno_oracle_cstep(double io[11], int* brackt, int* info, int* ret);

/* MoreThuente::cvsrch on one instance (f64): x[d], g[d] in/out, f in/out,
 * stp in/out, s[d] in. Returns nfev. */
int cno_oracle_cvsrch_f64(const cno_problem_t* problem, int64_t instance,
                          double* x, double* f, double* g, double* stp,
                          const double* s);

int cno_oracle_num_threads(void);

#ifdef __cplusplus
}
#endif
#endif /* CNO_ORACLE_H_ */
