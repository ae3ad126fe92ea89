/*
 * cno_al.h -- C ABI of the batched AugmentedLagrangian solver (SURVEY.md 8(f)
 * rank 1: the main in-tree caller of the hot path).
 *
 * Parity: the device path behind these entry points equals the pinned CPU oracle
 * (oracle/cno_al_oracle.h, tests/test_al_oracle.py) and the reference-headers
 * fixtures bit for bit on the GPU (tests/test_al_gpu.py).  DESIGN.md 8.
 *
 * Reference interfaces replaced (include/cppoptlib/...):
 *   solver/augmented_lagrangian.h:63-239    AugmentedLagrangianConfig   cno_al_config_t
 *   solver/augmented_lagrangian.h:241-276   AugmentedLagrangeState      x / multipliers / penalty /
 *                                                                       max_violation / max_lagrangian_gradient
 *                                                                       arrays of cno_al_out_t
 *   solver/augmented_lagrangian.h:278-449   AugmentedLagrangian<Problem, Lbfgs<FunctionExpr>>::Minimize
 *                                                                       cno_al_minimize()
 *   function_problem.h:38-60                ConstrainedOptimizationProblem: objective = cno_problem_t,
 *                                           constraints = cno_constraints_t
 *   function_penalty.h:97-250               ToAugmentedLagrangian: the composite the inner solver sees
 *   solver/progress.h:112-126,162-252       constraint_threshold / kkt_stationarity_threshold and the
 *                                           constrained branch of Progress::Update = cno_al_stop_t
 */
#ifndef CNO_AL_H_
#define CNO_AL_H_

#include "cno.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Constraint families.  A constraint row is d + 1 scalars [a (d) | t]. */
typedef enum cno_constraint_kind {
  CNO_CON_AFFINE = 0, /* c(x) = a.x - t,  grad = a   (a.x: products reduced under the policy) */
  CNO_CON_SQNORM = 1  /* c(x) = t - x.x,  grad = -2 x (a unused) */
} cno_constraint_kind_t;

/* function_problem.h:38-60: equality constraints c(x) == 0 first, then inequality
 * constraints c(x) >= 0. */
typedef struct cno_constraints {
  int32_t n_eq, n_ineq;
  const int32_t* kinds; /* [n_eq + n_ineq] */
  const void* data;     /* rows [a | t], (n_eq + n_ineq) rows per instance, dtype of the problem */
  int64_t data_stride;  /* scalars between instances; 0 = one set shared by the whole batch */
} cno_constraints_t;

/* solver/augmented_lagrangian.h:63-239 (AugmentedLagrangianConfig), same defaults. */
typedef struct cno_al_config {
  double penalty_growth_factor;           /* 10 */
  double violation_shrink_ratio;          /* 0.25 */
  int32_t auto_scale_initial_penalty;     /* 1 */
  double penalty_auto_objective_scale;    /* 10 */
  double penalty_auto_min;                /* 1e-8 */
  double penalty_auto_max;                /* 1e8 */
  int32_t warmup_max_inner_iterations;    /* 10 */
  double warmup_inner_gradient_tolerance; /* 1e-2 */
  double multiplier_max;                  /* 1e20 */
  double kkt_gradient_tolerance;          /* 1e-4 (carried, unused by the reference's loop) */
} cno_al_config_t;

/* The fields of the OUTER solver's stopping_progress the constrained branch of
 * Progress::Update reads (progress.h:212-252). */
typedef struct cno_al_stop {
  uint64_t num_iterations;           /* 0 = unlimited */
  double constraint_threshold;       /* 1e-5 in both presets (progress.h:378,416) */
  double kkt_stationarity_threshold; /* 1e-4 (progress.h:126); <= 0 disables */
} cno_al_stop_t;

/* Per-instance results.  The oracle accepts NULL for any of them; cno_al_minimize
 * needs all of them (they double as the solver's state between outer iterations). */
typedef struct cno_al_out {
  void* x;                       /* [B, d]     AugmentedLagrangeState::x (best iterate) */
  void* equality_multipliers;    /* [B, n_eq] */
  void* inequality_multipliers;  /* [B, n_ineq] */
  void* penalty;                 /* [B] */
  void* max_violation;           /* [B] */
  void* max_lagrangian_gradient; /* [B] */
  uint32_t* num_iterations;      /* [B] outer iterations */
  int8_t* status;                /* [B] cno_status_t of the outer loop */
  uint32_t* nfev;                /* [B] evaluations of the OBJECTIVE functor, all uses */
  void* x_delta;                 /* [B] outer Progress values (composite of prev / cur state) */
  void* f_delta;
  void* gradient_norm;
} cno_al_out_t;

void cno_al_default_config(cno_al_config_t* c);
void cno_al_default_stop(cno_al_stop_t* s);

/* CNO_OK if a device path is compiled for this objective (First mode) with these
 * constraint counts (n_eq, n_ineq <= 32 each). */
int cno_al_supported(const cno_problem_t* objective, const cno_constraints_t* constraints);

/* Bytes of device scratch cno_al_minimize needs for this batch. */
int cno_al_workspace_bytes(const cno_problem_t* objective, const cno_constraints_t* constraints,
                           int64_t batch, size_t* bytes);

/* AugmentedLagrangian<Problem, Lbfgs>::Minimize for every instance; all pointers
 * (x0, eq0, ineq0, penalty0, constraints->kinds/data, out->*) are DEVICE pointers.
 * eq0 / ineq0 / penalty0 may be NULL (zeros; penalty 0 = auto-scale,
 * augmented_lagrangian.h:312-318).  inner_stop: the inner Lbfgs template's
 * stopping_progress (NULL = default preset).  One outer iteration = [auto-scale
 * kernel on the first] + the fused L-BFGS kernel on the composite + one outer-step
 * kernel; the host reads one counter back per outer iteration. */
int cno_al_minimize(const cno_problem_t* objective, const cno_constraints_t* constraints,
                    int64_t batch, const void* x0, const void* eq0, const void* ineq0,
                    const void* penalty0, const cno_stop_t* inner_stop,
                    const cno_al_stop_t* outer_stop, const cno_al_config_t* config,
                    const cno_al_out_t* out, void* workspace, size_t workspace_bytes, void* stream,
                    cno_launch_info_t* info);

#ifdef __cplusplus
}
#endif
#endif /* CNO_AL_H_ */
