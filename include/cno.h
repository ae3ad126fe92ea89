/*
 * cno.h -- C ABI of the H100-native batched unconstrained-minimisation engine.
 *
 * This is the drop-in boundary for ONE path of PatWie/CppNumericalSolvers
 * (cppoptlib 2.0.0): solver::{Lbfgs,Bfgs,NewtonDescent}::Minimize with the
 * MoreThuente / Armijo line searches and the Progress stopping rules, with a
 * batch axis added (B independent instances, one warp per instance on sm_90a).
 *
 * Plain C: pointers and sizes only, no C++/torch types.  All citations are
 * relative to the reference tree (include/cppoptlib/...).
 *
 *   reference interface                         replaced / mirrored here
 *   ------------------------------------------  -----------------------------
 *   solver/progress.h:37-47   enum Status       cno_status_t
 *   solver/progress.h:82-140  Progress fields   cno_stop_t (stop thresholds)
 *                                               cno_batch_out_t (per-instance
 *                                               progress values)
 *   solver/progress.h:353-431 Default preset    cno_default_stop()
 *   solver/progress.h:456-464 Conservative      cno_conservative_stop()
 *   solver/solver.h:181-224   Solver::Minimize  cno_minimize() /
 *                                               cno_minimize_host()
 *   solver/solver.h:226-228   OptimizationStep  cno_minimize_steps() (K iterations
 *   solver/solver.h:163-176   SetCallback       per call; the host runs its callback
 *                                               between calls)
 *   solver/lbfgs.h:40-324     Lbfgs<F,m=10>     solver = CNO_LBFGS
 *   solver/bfgs.h:39-145      Bfgs<F>           solver = CNO_BFGS
 *   solver/newton_descent.h:38-85 NewtonDescent solver = CNO_NEWTON
 *   solver/gradient_descent.h:37-75 GradientDescent (MoreThuente)
 *                                               solver = CNO_GRADIENT_DESCENT
 *   solver/conjugated_gradient_descent.h:38-92 ConjugatedGradientDescent
 *                                               solver = CNO_CONJUGATED_GRADIENT_DESCENT
 *   solver/lbfgsb.h:44-538    Lbfgsb<F, m = 5>  cno_lbfgsb_minimize() + cno_bounds_t (SetBounds),
 *                                               cno_lbfgsb_default_stop() (the Lbfgsb() preset)
 *   function_base.h:96-126    FunctionCRTP      cno_problem_t names a functor
 *                                               that was compiled for the
 *                                               device (see INTEGRATION.md)
 *   function_base.h:298-332   FunctionState     x / value / gradient arrays
 *
 * Error behaviour (solver/progress.h: numerical outcomes are reported through
 * Progress::status, never thrown): every entry point returns 0 on success or a
 * negative cno_error_t; numerical outcomes are per-instance status codes.
 * There is NO CPU fallback: without a CUDA device every compute entry point
 * returns CNO_ERR_NO_DEVICE.
 */
#ifndef CNO_H_
#define CNO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CNO_VERSION_MAJOR 0
#define CNO_VERSION_MINOR 2

/* solver/progress.h:37-47 (same numeric values as the reference enum). */
typedef enum cno_status {
  CNO_STATUS_NOT_STARTED = -1,
  CNO_STATUS_CONTINUE = 0,
  CNO_STATUS_ITERATION_LIMIT = 1,
  CNO_STATUS_X_DELTA_VIOLATION = 2,
  CNO_STATUS_F_DELTA_VIOLATION = 3,
  CNO_STATUS_GRADIENT_NORM_VIOLATION = 4,
  CNO_STATUS_HESSIAN_CONDITION_VIOLATION = 5,
  CNO_STATUS_FINISHED = 6
} cno_status_t;

typedef enum cno_error {
  CNO_OK = 0,
  CNO_ERR_INVALID_ARGUMENT = -1,
  CNO_ERR_UNSUPPORTED = -2,   /* no kernel instantiated for <solver,functor,T,d> */
  CNO_ERR_NO_DEVICE = -3,     /* no CUDA device: there is no CPU fallback */
  CNO_ERR_CUDA = -4,          /* see cno_last_cuda_error() */
  CNO_ERR_WORKSPACE = -5      /* workspace too small / misaligned */
} cno_error_t;

typedef enum cno_solver {
  CNO_LBFGS = 0,  /* solver/lbfgs.h, m = 10, MoreThuente */
  CNO_BFGS = 1,   /* solver/bfgs.h, MoreThuente */
  CNO_NEWTON = 2, /* solver/newton_descent.h, Armijo<F,2> */
  CNO_GRADIENT_DESCENT = 3,            /* solver/gradient_descent.h, MoreThuente */
  CNO_CONJUGATED_GRADIENT_DESCENT = 4, /* solver/conjugated_gradient_descent.h, Armijo<F,1>;
                                          fp64 only (the reference computes beta in double) */
  /* the same solvers with LineSearch = linesearch::HagerZhang (linesearch/hager_zhang.h:54-552;
   * the template parameter at lbfgs.h:41, bfgs.h:40, gradient_descent.h:38) */
  CNO_LBFGS_HAGER_ZHANG = 5,
  CNO_BFGS_HAGER_ZHANG = 6,
  CNO_GRADIENT_DESCENT_HAGER_ZHANG = 7
} cno_solver_t;

typedef enum cno_dtype { CNO_F64 = 0, CNO_F32 = 1 } cno_dtype_t;

/* Objective families with a device functor compiled into libcno.so.  Users add
 * their own with CNO_INSTANTIATE_* (include/cppoptlib_b200/device.cuh). */
typedef enum cno_family {
  /* chained Rosenbrock; reduces to src/test/verify.cc:58-69 at d = 2 */
  CNO_FN_ROSENBROCK = 0,
  /* sum_i c_i x_i^2 + c0 with c = (5, 100), c0 = 5: Dockerfile.test:21-29 */
  CNO_FN_DIAG_QUADRATIC = 1,
  /* 0.5 * ||x||^2: src/test/augmented_lagrangian_test.cc:123-130 */
  CNO_FN_HALF_SQUARED_NORM = 2,
  /* sum_j log1p(exp(-y_j x_j.w)) + lambda/2 ||w||^2, per-instance data */
  CNO_FN_LOGISTIC = 3,
  /* 0.5 x'Ax - b'x (Second mode), per-instance A,b: src/examples/debug.cc:43-65 */
  CNO_FN_DENSE_QUADRATIC = 4
} cno_family_t;

/* Reduction-order policy = the arithmetic specification every dot/norm on the
 * path follows (DESIGN.md "Arithmetic specification").  Oracle and kernel are
 * bit-identical under the same policy. */
typedef enum cno_policy {
  CNO_POLICY_WARP_TREE = 0,  /* lane-blocked partials + xor butterfly (fp32 kernels) */
  CNO_POLICY_EIGEN_SSE2 = 1, /* model of Eigen 3.4 SSE2 redux (oracle only) */
  CNO_POLICY_DMMA_TREE = 2,  /* lane-blocked partials + two FP64 tensor-core MMAs (fp64 kernels) */
  /* CNO_POLICY_DMMA_TREE for every sum, and hessian.lu().solve (newton_descent.h:76) with every
   * multiply-subtract of the elimination and of both substitutions FUSED (a - l*u rounded once, the
   * contraction a -march=native build of the reference makes): the form the FP64 tensor core
   * evaluates, so the blocked elimination's trailing update runs as DMMA.8x8x4 (NewtonDescent,
   * d = 64 fp64; csrc/cno_newton_dmma.cuh).  Oracle twin: lu_solve(..., fused = 1). */
  CNO_POLICY_DMMA_LU = 3
} cno_policy_t;

/* Stopping thresholds: the fields of solver::Progress that
 * DefaultStoppingSolverProgress() sets (solver/progress.h:87-136). */
typedef struct cno_stop {
  uint64_t num_iterations;        /* :87  0 = unlimited */
  double x_delta;                 /* :88 */
  int32_t x_delta_violations;     /* :89 */
  double f_delta;                 /* :90 */
  int32_t f_delta_violations;     /* :91 */
  int32_t f_delta_relative;       /* :98 */
  double gradient_norm;           /* :99 */
  int32_t gradient_norm_relative; /* :109 */
  double condition_hessian;       /* :110 */
  int32_t past;                   /* :135 (<= CNO_MAX_PAST) */
  double past_delta;              /* :136 */
} cno_stop_t;

#define CNO_MAX_PAST 8
#define CNO_LBFGS_M 10

/* Which objective, which scalar type, which dimension. */
typedef struct cno_problem {
  int32_t family;      /* cno_family_t */
  int32_t dtype;       /* cno_dtype_t */
  int32_t d;           /* dimension of x */
  int32_t n;           /* CNO_FN_LOGISTIC: samples per instance */
  double param;        /* CNO_FN_LOGISTIC: lambda */
  const void* data;    /* per-instance data, [B, data_stride] scalars (device ptr
                          for cno_minimize, host ptr for cno_minimize_host/oracle) */
  int64_t data_stride; /* scalars per instance */
  int32_t policy;      /* cno_policy_t */
  int32_t mode;        /* 0/1 = use the functor as a First-mode function; 2 = Second mode:
                          Lbfgs then takes its diagonal-preconditioner branch
                          (solver/lbfgs.h:116-139,177-179).  NewtonDescent is always Second. */
  int32_t lbfgs_m;     /* the `m` of Lbfgs<F, m, LineSearch> (solver/lbfgs.h:40-41): pairs kept; 0 = the
                          reference's default 10.  Compiled: 5, 10, 20 (cno_supported tells). */
  int32_t reserved_;
} cno_problem_t;

/* Per-instance outputs.  Any pointer may be NULL (not written).  x, value,
 * gradient = the returned FunctionState (function_base.h:298-332); the rest =
 * the returned Progress (solver/progress.h:87-127). Scalars are of problem.dtype. */
typedef struct cno_batch_out {
  void* x;                 /* [B, d] */
  void* value;             /* [B] */
  void* gradient;          /* [B, d] */
  uint32_t* num_iterations;/* [B] */
  int8_t* status;          /* [B] cno_status_t */
  uint32_t* nfev;          /* [B] objective evaluations (not exposed by the reference) */
  void* x_delta;           /* [B] */
  void* f_delta;           /* [B] */
  void* gradient_norm;     /* [B] */
} cno_batch_out_t;

/* Launch record of the last cno_minimize* call on this thread. */
typedef struct cno_launch_info {
  int32_t kernel_launches; /* kernels of this library launched by the call */
  int32_t grid;            /* CTAs */
  int32_t block;           /* threads per CTA */
  int32_t warps_per_cta;   /* solver warps = resident instances per CTA (block / 32 is twice that for a functor with a helper warp per instance) */
  int64_t dynamic_smem;    /* bytes per CTA */
  float kernel_ms;         /* device time of the solve kernel(s), CUDA events */
  float total_ms;          /* cno_minimize_host: including H2D/D2H */
  int64_t h2d_bytes;
  int64_t d2h_bytes;
} cno_launch_info_t;

void cno_version(int* major, int* minor);
const char* cno_error_string(int err);
/* cudaError_t of the last CNO_ERR_CUDA on this thread and its string. */
int cno_last_cuda_error(const char** msg);

/* solver/progress.h:353-431 and :456-464. */
void cno_default_stop(cno_stop_t* stop);
void cno_conservative_stop(cno_stop_t* stop);

/* 0 if a kernel is instantiated for (solver, problem), else CNO_ERR_UNSUPPORTED. */
int cno_supported(int solver, const cno_problem_t* problem);

/* Scratch the caller must provide for cno_minimize (may be 0). */
int cno_workspace_bytes(int solver, const cno_problem_t* problem, int64_t batch,
                        size_t* bytes);

/* Batched Solver::Minimize (solver/solver.h:181-224).  All pointers are DEVICE
 * pointers on the current device; stream is a cudaStream_t (NULL = default).
 * Asynchronous with respect to the host unless info != NULL (timing needs a
 * synchronisation). */
int cno_minimize(int solver, const cno_problem_t* problem, int64_t batch,
                 const void* x0, const cno_stop_t* stop,
                 const cno_batch_out_t* out, void* workspace,
                 size_t workspace_bytes, void* stream, cno_launch_info_t* info);

/* Stepwise Minimize = batched OptimizationStep (solver/solver.h:226-228) + the
 * per-iteration callback hook (solver/solver.h:163-176,197): runs at most
 * max_iterations iterations of every unfinished instance and parks the solver's
 * members (lbfgs.h:305-323) and Progress counters in `state`
 * (cno_state_bytes() bytes, device memory, owned by the caller).  first_call != 0
 * starts from x0; later calls continue from `state` and the previous outputs
 * (out->x, value, gradient, status, num_iterations must be the same non-NULL
 * arrays in every call).  An instance is finished when its status != CONTINUE;
 * the sequence of calls produces bit for bit what one cno_minimize call does. */
int cno_state_bytes(int solver, const cno_problem_t* problem, int64_t batch, size_t* bytes);
int cno_minimize_steps(int solver, const cno_problem_t* problem, int64_t batch, const void* x0,
                       const cno_stop_t* stop, const cno_batch_out_t* out, void* state,
                       size_t state_bytes, int32_t max_iterations, int32_t first_call,
                       void* workspace, size_t workspace_bytes, void* stream,
                       cno_launch_info_t* info);

/* Same call with HOST pointers (x0, problem->data and every non-NULL member of
 * out): stages through pinned memory, copies H2D, solves, copies D2H.  This is
 * the call a host-side user of the reference makes; bench.py times it for e2e. */
int cno_minimize_host(int solver, const cno_problem_t* problem, int64_t batch,
                      const void* x0, const cno_stop_t* stop,
                      const cno_batch_out_t* out, cno_launch_info_t* info);

/* ---- Lbfgsb<F, m = 5, MoreThuente> (solver/lbfgsb.h:44-538): box constraints lower <= x <= upper -------------
 * SetBounds (:88-92) with a batch axis: lower / upper are DEVICE arrays of problem.dtype, [d] (stride = 0: one
 * box for the whole batch) or [B, d] (stride = d); a NULL side is unbounded (numeric_limits lowest / max, as
 * InitializeSolver does at :122-128). */
typedef struct cno_bounds {
  const void* lower;
  const void* upper;
  int64_t stride;
} cno_bounds_t;
/* The Lbfgsb() constructor's stopping preset (:78-81): cno_default_stop + f_delta = 2.22e-9, relative. */
void cno_lbfgsb_default_stop(cno_stop_t* stop);
/* 0 if a kernel is instantiated for Lbfgsb on this problem, else CNO_ERR_UNSUPPORTED. */
int cno_lbfgsb_supported(const cno_problem_t* problem);
/* Batched Lbfgsb::Minimize (:238-286: the projected-gradient sup-norm drives stop->gradient_norm).  Device
 * pointers; bounds may be NULL (unbounded); stop NULL = cno_lbfgsb_default_stop; workspace as for cno_minimize.
 * Compiled: the built-in families up to d = 128 (one warp per instance), and Rosenbrock fp64 with m = 5 and the
 * default policy at d = 256, 512 and 1024 (one group of d / 128 warps per instance). */
int cno_lbfgsb_minimize(const cno_problem_t* problem, const cno_bounds_t* bounds, int64_t batch, const void* x0,
                        const cno_stop_t* stop, const cno_batch_out_t* out, void* workspace, size_t workspace_bytes,
                        void* stream, cno_launch_info_t* info);

/* Batched F::operator()(x, &gradient) (function_base.h:103-120; the evaluating FunctionState constructor,
 * :315-326): value [B] and/or gradient [B, d] of the built-in family at x [B, d].  DEVICE pointers; either
 * output may be NULL.  Families that stage per-instance data on chip (CNO_FN_LOGISTIC) are not evaluated
 * stand-alone: CNO_ERR_UNSUPPORTED. */
int cno_evaluate(const cno_problem_t* problem, int64_t batch, const void* x, void* value, void* gradient,
                 void* stream);

/* cno_minimize_host keeps its device staging arena between calls (grown on demand, one per process);
 * this frees it.  Returns 0 or CNO_ERR_CUDA. */
int cno_release_host_arena(void);

/* Counter-based start generator (SURVEY.md 8(d)): element with global counter
 * n = first + k gets lo + (hi - lo) * u, u = (mix64(seed + (n+1)*GOLDEN) >> 11)
 * * 2^-53 (f64) or (>> 40) * 2^-24 (f32).  dst is a device pointer. */
int cno_fill_uniform(int dtype, void* dst, int64_t first, int64_t count,
                     uint64_t seed, double lo, double hi, void* stream);

/* Packs status != CONTINUE into a bitmap, one bit per instance ([ceil(B/32)]
 * uint32 words, device pointers): the per-GPU convergence bitmap that ranks
 * all-gather for the global stop test. */
int cno_done_bitmap(const int8_t* status, int64_t batch, uint32_t* words,
                    void* stream);

/* The ONE collective of the path (SURVEY.md 8(e)): all-gathers the per-GPU convergence bitmaps for the global
 * stop test.  comm = an ncclComm_t of the caller (one rank per GPU), local_words / all_words device pointers
 * ([words] and [nranks * words] uint32), stream a cudaStream_t.  NCCL is resolved at first use (dlopen of
 * libnccl.so.2 -- the copy already loaded by the process, e.g. PyTorch's, or the system one); without it the
 * call returns CNO_ERR_UNSUPPORTED.  cno_count_done then counts the set bits of the first `bits` bits of each
 * of the `ranks` bitmaps on the device and returns the total through a host pointer (synchronises the stream). */
int cno_allgather_done(void* comm, const uint32_t* local_words, uint32_t* all_words, size_t words, void* stream);
int cno_count_done(const uint32_t* all_words, int32_t ranks, size_t words_per_rank, const int64_t* bits_per_rank,
                   int64_t* total_done, void* stream);

/* Progress::condition_hessian on request (solver/progress.h:203-210): condition[b] = H(x_b).norm() *
 * H(x_b).inverse().norm(), the value the reference's Progress::Update computes for a Second-mode function at
 * every iteration (one Hessian evaluation and a full inverse) and no preset tests.  The fused solve kernels do
 * not carry it (a non-zero cno_stop_t::condition_hessian is rejected); call this on the states whose condition
 * number is wanted -- the returned x of a solve gives the reference's final progress.condition_hessian.
 * x [B, d] and condition [B]: DEVICE pointers; workspace: >= 8 bytes of device scratch, 8-byte aligned.
 * Second-mode built-ins under the dtype's default policy (CNO_FN_DENSE_QUADRATIC f64 d = 64 / 12, f32 d = 64;
 * CNO_FN_ROSENBROCK f64 d = 2 / 8); otherwise CNO_ERR_UNSUPPORTED. */
int cno_condition_hessian(const cno_problem_t* problem, int64_t batch, const void* x, void* condition,
                          void* workspace, size_t workspace_bytes, void* stream);

/* Device-side known-answer hook for MoreThuente::cstep
 * (linesearch/more_thuente.h:261-407): runs the device cstep on one thread.
 * io = {stx, fx, dx, sty, fy, dy, stp, fp, dp, stpmin, stpmax} (host, f64),
 * brackt/info in-out, ret = cstep's return value. */
int cno_device_cstep(double io[11], int* brackt, int* info, int* ret);

/* Device-side check hook for the division helper of csrc/cno_newton_dmma.cuh (the reciprocal refinement of a
 * divisor computed once, the quotient finished in three operations): for i < n it writes
 * helper[i] = div_with(a[i], b[i], div_rcp(b[i])) where the helper's range test accepts the operands (else the plain
 * quotient, as the kernels do), plain[i] = a[i] / b[i], accepted[i] = the range test.  Host pointers, f64. */
int cno_device_div_check(const double* a, const double* b, int64_t n, double* helper, double* plain,
                         int32_t* accepted);

#ifdef __cplusplus
} /* extern "C" */
#endif

#endif /* CNO_H_ */
