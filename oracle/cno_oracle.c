/*
 * cno_oracle.c -- CPU ORACLE translation unit (TEST INFRASTRUCTURE ONLY, see
 * cno_oracle.h).  Instantiates cno_oracle_impl.inc for double and float and
 * provides the batched OpenMP driver used by tests and by bench.py's
 * cpu_baseline / --impl reference legs.
 *
 * Build: oracle/Makefile (gcc -O2 -ffp-contract=off -fopenmp).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "cno_al_oracle.h"
#include "cno_oracle.h"

static inline int problem_lbfgs_m(const cno_problem_t* p) {
  return (p->lbfgs_m > 0 && p->lbfgs_m <= CNO_ORACLE_MAX_M) ? p->lbfgs_m : CNO_LBFGS_M;
}

/* ---- double ---- */
#define REAL double
#define FN(name) name##_f64
#define R_EPS DBL_EPSILON
#define R_SQRT sqrt
#define R_FABS fabs
#define R_FMA fma
#define R_FMAX fmax
#define R_ISFINITE isfinite
#define R_IS_F32 0
#define R_MIN_NORMAL DBL_MIN
#include "cno_oracle_impl.inc"
#undef REAL
#undef FN
#undef R_EPS
#undef R_SQRT
#undef R_FABS
#undef R_FMA
#undef R_FMAX
#undef R_ISFINITE
#undef R_IS_F32
#undef R_MIN_NORMAL

/* ---- float ---- */
#define REAL float
#define FN(name) name##_f32
#define R_EPS FLT_EPSILON
#define R_SQRT sqrtf
#define R_FABS fabsf
#define R_FMA fmaf
#define R_FMAX fmaxf
#define R_ISFINITE isfinite
#define R_IS_F32 1
#define R_MIN_NORMAL FLT_MIN
#include "cno_oracle_impl.inc"
#undef REAL
#undef FN

/* solver/progress.h:353-431 */
static void oracle_default_stop(cno_stop_t* s) {
  memset(s, 0, sizeof(*s));
  s->num_iterations = 10000;
  s->x_delta = 1e-9;
  s->x_delta_violations = 1;
  s->f_delta = 0;
  s->f_delta_violations = 1;
  s->f_delta_relative = 0;
  s->gradient_norm = 1e-5;
  s->gradient_norm_relative = 1;
  s->condition_hessian = 0;
  s->past = 3;
  s->past_delta = 1e-6;
}

static int check_problem(int solver, const cno_problem_t* p) {
  if (!p || p->d <= 0 || p->d > CNO_MAX_D) return CNO_ERR_INVALID_ARGUMENT;
  if (solver < CNO_LBFGS || solver > CNO_CONJUGATED_GRADIENT_DESCENT) return CNO_ERR_INVALID_ARGUMENT;
  if (p->dtype != CNO_F64 && p->dtype != CNO_F32) return CNO_ERR_INVALID_ARGUMENT;
  switch (p->family) {
    case CNO_FN_ROSENBROCK:
    case CNO_FN_HALF_SQUARED_NORM:
      break;
    case CNO_FN_DIAG_QUADRATIC:
      if (p->d != 2) return CNO_ERR_INVALID_ARGUMENT;
      break;
    case CNO_FN_LOGISTIC:
      if (!p->data || p->n <= 0 || p->n > CNO_MAX_D || p->n % 128) return CNO_ERR_INVALID_ARGUMENT;
      if (solver == CNO_NEWTON) return CNO_ERR_UNSUPPORTED; /* First mode only */
      break;
    case CNO_FN_DENSE_QUADRATIC:
      if (!p->data) return CNO_ERR_INVALID_ARGUMENT;
      break;
    default:
      return CNO_ERR_INVALID_ARGUMENT;
  }
  return CNO_OK;
}

int cno_oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

int cno_oracle_minimize(int solver, const cno_problem_t* problem, int64_t batch,
                        const void* x0, const cno_stop_t* stop,
                        const cno_batch_out_t* out, int threads) {
  return cno_oracle_minimize_ls(solver, problem, batch, x0, stop, out, threads, CNO_LS_MORE_THUENTE);
}

static int minimize_batch(int solver, const cno_problem_t* problem, int64_t batch, const void* x0,
                          const cno_stop_t* stop, const cno_batch_out_t* out, int threads, int linesearch,
                          void* paths) {
  int rc = check_problem(solver, problem);
  if (linesearch != CNO_LS_MORE_THUENTE && linesearch != CNO_LS_HAGER_ZHANG) return CNO_ERR_INVALID_ARGUMENT;
  if (linesearch == CNO_LS_HAGER_ZHANG && solver != CNO_LBFGS && solver != CNO_BFGS &&
      solver != CNO_GRADIENT_DESCENT)
    return CNO_ERR_UNSUPPORTED; /* the solvers with a LineSearch template parameter */
  if (rc) return rc;
  if (batch < 0 || !x0 || !out) return CNO_ERR_INVALID_ARGUMENT;
  cno_stop_t dflt;
  if (!stop) {
    oracle_default_stop(&dflt);
    stop = &dflt;
  }
  if (stop->past > CNO_MAX_PAST) return CNO_ERR_INVALID_ARGUMENT;
  const int d = problem->d;
#ifdef _OPENMP
  if (threads <= 0) threads = omp_get_max_threads();
#else
  threads = 1;
#endif
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int64_t b = 0; b < batch; ++b) {
    void* const pb = !paths ? NULL
                     : solver == CNO_BFGS ? (void*)((cno_bfgs_paths_t*)paths + b)
                                          : (void*)((cno_lbfgs_paths_t*)paths + b);
    if (problem->dtype == CNO_F64) {
      minimize_one_f64(
          solver, problem, NULL, linesearch, b, (const double*)x0 + b * d, stop,
          out->x ? (double*)out->x + b * d : NULL,
          out->value ? (double*)out->value + b : NULL,
          out->gradient ? (double*)out->gradient + b * d : NULL,
          out->num_iterations ? out->num_iterations + b : NULL,
          out->status ? out->status + b : NULL, out->nfev ? out->nfev + b : NULL,
          out->x_delta ? (double*)out->x_delta + b : NULL,
          out->f_delta ? (double*)out->f_delta + b : NULL,
          out->gradient_norm ? (double*)out->gradient_norm + b : NULL, pb);
    } else {
      minimize_one_f32(
          solver, problem, NULL, linesearch, b, (const float*)x0 + b * d, stop,
          out->x ? (float*)out->x + b * d : NULL,
          out->value ? (float*)out->value + b : NULL,
          out->gradient ? (float*)out->gradient + b * d : NULL,
          out->num_iterations ? out->num_iterations + b : NULL,
          out->status ? out->status + b : NULL, out->nfev ? out->nfev + b : NULL,
          out->x_delta ? (float*)out->x_delta + b : NULL,
          out->f_delta ? (float*)out->f_delta + b : NULL,
          out->gradient_norm ? (float*)out->gradient_norm + b : NULL, pb);
    }
  }
  return CNO_OK;
}

int cno_oracle_minimize_ls(int solver, const cno_problem_t* problem, int64_t batch,
                           const void* x0, const cno_stop_t* stop,
                           const cno_batch_out_t* out, int threads, int linesearch) {
  return minimize_batch(solver, problem, batch, x0, stop, out, threads, linesearch, NULL);
}

int cno_oracle_lbfgs_paths(const cno_problem_t* problem, int64_t batch, const void* x0,
                           const cno_stop_t* stop, const cno_batch_out_t* out,
                           cno_lbfgs_paths_t* paths, int threads) {
  if (!paths) return CNO_ERR_INVALID_ARGUMENT;
  if (batch > 0) memset(paths, 0, sizeof(*paths) * (size_t)batch);
  return minimize_batch(CNO_LBFGS, problem, batch, x0, stop, out, threads, CNO_LS_MORE_THUENTE, paths);
}

int cno_oracle_bfgs_paths(const cno_problem_t* problem, int64_t batch, const void* x0, const cno_stop_t* stop,
                          const cno_batch_out_t* out, cno_bfgs_paths_t* paths, int threads, int linesearch) {
  if (!paths) return CNO_ERR_INVALID_ARGUMENT;
  if (batch > 0) memset(paths, 0, sizeof(*paths) * (size_t)batch);
  return minimize_batch(CNO_BFGS, problem, batch, x0, stop, out, threads, linesearch, paths);
}

int cno_oracle_evaluate(const cno_problem_t* problem, int64_t batch,
                        const void* x, void* f, void* g, void* H) {
  int rc = check_problem(CNO_LBFGS, problem);
  if (rc) return rc;
  const int d = problem->d;
  for (int64_t b = 0; b < batch; ++b) {
    if (problem->dtype == CNO_F64) {
      fnctx_t_f64 c = {problem, b, 0, NULL, 0};
      double v = eval_f64(&c, (const double*)x + b * d,
                          g ? (double*)g + b * d : NULL,
                          H ? (double*)H + b * d * d : NULL);
      if (f) ((double*)f)[b] = v;
    } else {
      fnctx_t_f32 c = {problem, b, 0, NULL, 0};
      float v = eval_f32(&c, (const float*)x + b * d,
                         g ? (float*)g + b * d : NULL,
                         H ? (float*)H + b * d * d : NULL);
      if (f) ((float*)f)[b] = v;
    }
  }
  return CNO_OK;
}

/* progress.condition_hessian (solver/progress.h:203-210) at x[b], Second-mode families only. */
int cno_oracle_condition_hessian(const cno_problem_t* problem, int64_t batch, const void* x, void* out) {
  int rc = check_problem(CNO_NEWTON, problem);
  if (rc) return rc;
  const int d = problem->d;
#pragma omp parallel for schedule(dynamic)
  for (int64_t b = 0; b < batch; ++b) {
    if (problem->dtype == CNO_F64)
      ((double*)out)[b] = condition_hessian_at_f64(problem, b, (const double*)x + b * d);
    else
      ((float*)out)[b] = condition_hessian_at_f32(problem, b, (const float*)x + b * d);
  }
  return CNO_OK;
}

/* splitmix64 finaliser; counter-based (SURVEY.md 8(d)). */
static inline uint64_t mix64(uint64_t z) {
  z ^= z >> 30;
  z *= 0xBF58476D1CE4E5B9ULL;
  z ^= z >> 27;
  z *= 0x94D049BB133111EBULL;
  z ^= z >> 31;
  return z;
}

int cno_oracle_fill_uniform(int dtype, void* dst, int64_t first, int64_t count,
                            uint64_t seed, double lo, double hi) {
  if (!dst || count < 0) return CNO_ERR_INVALID_ARGUMENT;
  for (int64_t k = 0; k < count; ++k) {
    const uint64_t n = (uint64_t)(first + k) + 1ULL;
    const uint64_t z = mix64(seed + n * 0x9E3779B97F4A7C15ULL);
    if (dtype == CNO_F64) {
      const double u = (double)(z >> 11) * 0x1.0p-53;
      ((double*)dst)[k] = lo + (hi - lo) * u;
    } else {
      const float u = (float)(z >> 40) * 0x1.0p-24f;
      ((float*)dst)[k] = (float)lo + ((float)hi - (float)lo) * u;
    }
  }
  return CNO_OK;
}

double cno_oracle_reduce_sum_f64(const double* t, int d, int policy) {
  return reduce_sum_f64(t, d, policy);
}
float cno_oracle_reduce_sum_f32(const float* t, int d, int policy) {
  return reduce_sum_f32(t, d, policy);
}

int cno_oracle_cstep(double io[11], int* brackt, int* info, int* ret) {
  *ret = cstep_f64(&io[0], &io[1], &io[2], &io[3], &io[4], &io[5], &io[6],
                   io[7], io[8], brackt, io[9], io[10], info);
  return CNO_OK;
}

int cno_oracle_cvsrch_f64(const cno_problem_t* problem, int64_t instance,
                          double* x, double* f, double* g, double* stp,
                          const double* s) {
  fnctx_t_f64 c = {problem, instance, 0, NULL, 0};
  cvsrch_f64(&c, x, f, g, stp, s);
  return (int)c.nfev;
}

/* HagerZhang<F,1>::Search(x, f0, g0, s, f, alpha_init, &x_out, &f_out, &g_out)
 * (hager_zhang.h:80-96) on the 1-D quartic of src/test/hager_zhang_test.cc with s = 1. */
int cno_oracle_hz_search_poly(const double coef[5], double x0, double alpha_init,
                              double* alpha, double* f_out, double* x_out, int* nfev) {
  cno_problem_t p;
  memset(&p, 0, sizeof(p));
  p.family = CNO_ORACLE_FN_POLY1D;
  p.dtype = CNO_F64;
  p.d = 1;
  p.data = coef;
  p.policy = CNO_POLICY_WARP_TREE;
  fnctx_t_f64 c = {&p, 0, 0, NULL, 1};
  double x = x0, g = 0, s = 1.0;
  double f = eval_f64(&c, &x, &g, NULL);
  double a = alpha_init;
  const uint32_t before = c.nfev;
  hzls_f64(&c, &x, &f, &g, &a, &s);
  if (alpha) *alpha = a;
  if (f_out) *f_out = f;
  if (x_out) *x_out = x;
  if (nfev) *nfev = (int)(c.nfev - before);
  return CNO_OK;
}

/* ---- AugmentedLagrangian (cno_al_oracle.h) ------------------------------- */
void cno_al_oracle_default_config(cno_al_config_t* c) { /* augmented_lagrangian.h:63-239 */
  memset(c, 0, sizeof(*c));
  c->penalty_growth_factor = 10;
  c->violation_shrink_ratio = 0.25;
  c->auto_scale_initial_penalty = 1;
  c->penalty_auto_objective_scale = 10;
  c->penalty_auto_min = 1e-8;
  c->penalty_auto_max = 1e8;
  c->warmup_max_inner_iterations = 10;
  c->warmup_inner_gradient_tolerance = 1e-2;
  c->multiplier_max = 1e20;
  c->kkt_gradient_tolerance = 1e-4;
}

void cno_al_oracle_default_stop(cno_al_stop_t* s) { /* progress.h:126, 353-431 */
  s->num_iterations = 10000;
  s->constraint_threshold = 1e-5;
  s->kkt_stationarity_threshold = 1e-4;
}

static int check_constraints(const cno_problem_t* p, const cno_constraints_t* k) {
  if (!k || k->n_eq < 0 || k->n_ineq < 0) return CNO_ERR_INVALID_ARGUMENT;
  if (k->n_eq > CNO_AL_MAX_CON || k->n_ineq > CNO_AL_MAX_CON) return CNO_ERR_UNSUPPORTED;
  if (k->n_eq + k->n_ineq > 0 && (!k->kinds || !k->data)) return CNO_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < k->n_eq + k->n_ineq; ++i)
    if (k->kinds[i] != CNO_CON_AFFINE && k->kinds[i] != CNO_CON_SQNORM) return CNO_ERR_INVALID_ARGUMENT;
  if (p->mode == 2) return CNO_ERR_UNSUPPORTED; /* First-mode composite only */
  return CNO_OK;
}

int cno_al_oracle_minimize(const cno_problem_t* objective, const cno_constraints_t* constraints,
                           int64_t batch, const void* x0, const void* eq0, const void* ineq0,
                           const void* penalty0, const cno_stop_t* inner_stop,
                           const cno_al_stop_t* outer_stop, const cno_al_config_t* config,
                           const cno_al_out_t* out, int threads) {
  int rc = check_problem(CNO_LBFGS, objective);
  if (rc) return rc;
  rc = check_constraints(objective, constraints);
  if (rc) return rc;
  if (batch < 0 || !x0 || !out) return CNO_ERR_INVALID_ARGUMENT;
  cno_stop_t idflt;
  if (!inner_stop) { oracle_default_stop(&idflt); inner_stop = &idflt; }
  if (inner_stop->past > CNO_MAX_PAST) return CNO_ERR_INVALID_ARGUMENT;
  cno_al_stop_t odflt;
  if (!outer_stop) { cno_al_oracle_default_stop(&odflt); outer_stop = &odflt; }
  cno_al_config_t cdflt;
  if (!config) { cno_al_oracle_default_config(&cdflt); config = &cdflt; }
  const int d = objective->d, ne = constraints->n_eq, ni = constraints->n_ineq;
#ifdef _OPENMP
  if (threads <= 0) threads = omp_get_max_threads();
#else
  threads = 1;
#endif
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int64_t b = 0; b < batch; ++b) {
#define CNO_AL_RUN(REAL_T, SUF)                                                                   \
  do {                                                                                            \
    alstate_t_##SUF* r = (alstate_t_##SUF*)malloc(sizeof(alstate_t_##SUF));                       \
    REAL_T xd = 0, fd = 0, gn = 0;                                                                \
    al_minimize_one_##SUF(objective, constraints, b, (const REAL_T*)x0 + b * d,                   \
                          eq0 ? (const REAL_T*)eq0 + b * ne : NULL,                               \
                          ineq0 ? (const REAL_T*)ineq0 + b * ni : NULL,                           \
                          penalty0 ? ((const REAL_T*)penalty0)[b] : (REAL_T)0, inner_stop,        \
                          outer_stop, config, r, out->num_iterations ? out->num_iterations + b : NULL, \
                          out->status ? out->status + b : NULL, out->nfev ? out->nfev + b : NULL, \
                          &xd, &fd, &gn);                                                         \
    if (out->x) memcpy((REAL_T*)out->x + b * d, r->x, sizeof(REAL_T) * d);                        \
    if (out->equality_multipliers)                                                                \
      memcpy((REAL_T*)out->equality_multipliers + b * ne, r->lambda, sizeof(REAL_T) * ne);        \
    if (out->inequality_multipliers)                                                              \
      memcpy((REAL_T*)out->inequality_multipliers + b * ni, r->mu, sizeof(REAL_T) * ni);          \
    if (out->penalty) ((REAL_T*)out->penalty)[b] = r->penalty;                                    \
    if (out->max_violation) ((REAL_T*)out->max_violation)[b] = r->max_violation;                  \
    if (out->max_lagrangian_gradient)                                                             \
      ((REAL_T*)out->max_lagrangian_gradient)[b] = r->max_lagrangian_gradient;                    \
    if (out->x_delta) ((REAL_T*)out->x_delta)[b] = xd;                                            \
    if (out->f_delta) ((REAL_T*)out->f_delta)[b] = fd;                                            \
    if (out->gradient_norm) ((REAL_T*)out->gradient_norm)[b] = gn;                                \
    free(r);                                                                                      \
  } while (0)
    if (objective->dtype == CNO_F64) CNO_AL_RUN(double, f64);
    else CNO_AL_RUN(float, f32);
#undef CNO_AL_RUN
  }
  return CNO_OK;
}

int cno_al_oracle_inner_minimize(const cno_problem_t* objective, const cno_constraints_t* constraints,
                                 int64_t batch, const void* x0, const void* eq, const void* ineq,
                                 const void* penalty, const cno_stop_t* inner_stop, void* x_out,
                                 uint32_t* nfev_out, int threads) {
  int rc = check_problem(CNO_LBFGS, objective);
  if (rc) return rc;
  rc = check_constraints(objective, constraints);
  if (rc) return rc;
  if (batch < 0 || !x0 || !penalty || !inner_stop || !x_out) return CNO_ERR_INVALID_ARGUMENT;
  const int d = objective->d, ne = constraints->n_eq, ni = constraints->n_ineq;
#ifdef _OPENMP
  if (threads <= 0) threads = omp_get_max_threads();
#else
  threads = 1;
#endif
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int64_t b = 0; b < batch; ++b) {
    if (objective->dtype == CNO_F64) {
      const alctx_t_f64 al = {constraints, eq ? (const double*)eq + b * ne : NULL,
                              ineq ? (const double*)ineq + b * ni : NULL, ((const double*)penalty)[b]};
      minimize_one_f64(CNO_LBFGS, objective, &al, 0, b, (const double*)x0 + b * d, inner_stop,
                       (double*)x_out + b * d, NULL, NULL, NULL, NULL, nfev_out ? nfev_out + b : NULL, NULL,
                       NULL, NULL, NULL);
    } else {
      const alctx_t_f32 al = {constraints, eq ? (const float*)eq + b * ne : NULL,
                              ineq ? (const float*)ineq + b * ni : NULL, ((const float*)penalty)[b]};
      minimize_one_f32(CNO_LBFGS, objective, &al, 0, b, (const float*)x0 + b * d, inner_stop,
                       (float*)x_out + b * d, NULL, NULL, NULL, NULL, nfev_out ? nfev_out + b : NULL, NULL,
                       NULL, NULL, NULL);
    }
  }
  return CNO_OK;
}

int cno_al_oracle_evaluate(const cno_problem_t* objective, const cno_constraints_t* constraints,
                           int64_t batch, const void* x, const void* eq, const void* ineq,
                           const void* penalty, void* value, void* grad) {
  int rc = check_problem(CNO_LBFGS, objective);
  if (rc) return rc;
  rc = check_constraints(objective, constraints);
  if (rc) return rc;
  if (batch < 0 || !x || !penalty) return CNO_ERR_INVALID_ARGUMENT;
  const int d = objective->d, ne = constraints->n_eq, ni = constraints->n_ineq;
  for (int64_t b = 0; b < batch; ++b) {
    if (objective->dtype == CNO_F64) {
      const alctx_t_f64 al = {constraints, eq ? (const double*)eq + b * ne : NULL,
                              ineq ? (const double*)ineq + b * ni : NULL, ((const double*)penalty)[b]};
      fnctx_t_f64 c = {objective, b, 0, &al, 0};
      const double v = eval_f64(&c, (const double*)x + b * d, grad ? (double*)grad + b * d : NULL, NULL);
      if (value) ((double*)value)[b] = v;
    } else {
      const alctx_t_f32 al = {constraints, eq ? (const float*)eq + b * ne : NULL,
                              ineq ? (const float*)ineq + b * ni : NULL, ((const float*)penalty)[b]};
      fnctx_t_f32 c = {objective, b, 0, &al, 0};
      const float v = eval_f32(&c, (const float*)x + b * d, grad ? (float*)grad + b * d : NULL, NULL);
      if (value) ((float*)value)[b] = v;
    }
  }
  return CNO_OK;
}
