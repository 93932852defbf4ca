/*
 * mtg_b200.h -- C-ABI of the H100-native batched linear min-derivative solver.
 *
 * Drop-in boundary for ONE path of ethz-asl/mav_trajectory_generation:
 * PolynomialOptimization<N>::solveLinear() and the per-segment assembly feeding it.
 * The reference has no FFI layer; what these entry points replace is the body of the
 * following members (paths under mav_trajectory_generation/include/mav_trajectory_generation/):
 *
 *   mtg_solve_linear_batch_*      impl/polynomial_optimization_linear_impl.h:338-379 solveLinear()
 *                                 + :285-305 updateSegmentTimes() (A^-1, Q per segment)
 *                                 + :307-336 constructR()
 *                                 + :262-283 updateSegmentsFromCompactConstraints()
 *   mtg_coeffs_from_constraints_* impl/...linear_impl.h:499-508 setFreeConstraints()
 *                                 -> :262-283 updateSegmentsFromCompactConstraints()
 *   mtg_compute_cost_batch_*      impl/...linear_impl.h:123-140 computeCost()
 *   mtg_problem_layout            impl/...linear_impl.h:181-260 setupConstraintReorderingMatrix()
 *                                 (the 0/1 matrix C as one column index per row; host only)
 *
 * Conventions
 *   - plain C, no torch / Eigen / STL types cross this boundary; every buffer is caller-owned.
 *   - all arithmetic fp64; polynomial coefficients in INCREASING powers
 *     (polynomial_optimization_linear.h:43-44).
 *   - a "problem" is a constraint TOPOLOGY shared by the whole batch: N coefficients,
 *     derivative_to_optimize r, K segments, D dimensions, and which derivatives each of the
 *     K+1 vertices fixes.  Per trajectory only the segment times and the fixed constraint
 *     VALUES differ (the reference re-uses one factorisation for all D for the same reason,
 *     linear_impl.h:369-375).
 *   - d_fixed / d_free use the reference's compact ordering: constraints sorted by
 *     (vertex, derivative) (polynomial_optimization_linear.h:287-295), i.e. exactly
 *     getFixedConstraints()/getFreeConstraints() (polynomial_optimization_linear.h:194-206).
 *   - nothing here aborts or throws: argument errors return a negative code
 *     (the reference CHECK-aborts, e.g. linear_impl.h:60,76,289,297); per-trajectory numeric
 *     trouble is reported in status[] and never stops the batch.
 *   - a handle is bound to one CUDA device and is single-caller (the reference object is not
 *     thread-safe either); use one handle per host thread / per GPU.
 *   - there is NO CPU fallback: every compute entry point launches sm_90a kernels or fails.
 */
#ifndef MTG_B200_H_
#define MTG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MTG_MAX_N 12 /* Polynomial::kMaxN, polynomial.h:44 */

/* return codes */
#define MTG_OK 0
#define MTG_ERR_BAD_ARG (-1)      /* null pointer, odd N, r out of [0, N/2-1], K < 1, D < 1 ... */
#define MTG_ERR_CUDA (-2)         /* CUDA runtime error; see mtg_last_error() */
#define MTG_ERR_NO_DEVICE (-3)    /* no sm_90 device / extension cannot run */
#define MTG_ERR_ALLOC (-4)

/* per-trajectory status bits (status[b] == 0 means solved) */
#define MTG_STATUS_BAD_TIME 1     /* some segment time <= 0, NaN or +inf (reference: CHECK_GT, linear_impl.h:297) */
#define MTG_STATUS_NOT_SPD 2      /* non-positive / NaN / infinite pivot in the R_pp factorisation */
#define MTG_STATUS_FEAS_CAPACITY 4 /* input feasibility: a candidate list (48 entries) or the roll/pitch walk (64 levels)
                                      ran out of room, or (sampling) a segment needs more than 2^24 samples; the
                                      segment is reported Indeterminable */

/* which kernel family a problem is routed to (introspection for tests / profiles) */
#define MTG_KERNEL_WAYPOINT 1     /* specialised block-tridiagonal Cholesky kernels, waypoint topology */
#define MTG_KERNEL_GENERIC 2      /* arbitrary per-vertex masks: masked block-tridiagonal Cholesky */
#define MTG_KERNEL_NOFREE 3       /* n_free == 0: back-substitution only (linear_impl.h:343-349) */

typedef struct mtg_handle mtg_handle;

typedef struct mtg_problem {
  int32_t N; /* coefficients per polynomial, even, 2..12   (template parameter _N, linear.h:45-51) */
  int32_t r; /* derivative_to_optimize in [0, N/2-1]        (setupFromVertices arg, linear.h:67-69) */
  int32_t K; /* number of segments (= vertices - 1) >= 1 */
  int32_t D; /* dimensions >= 1 */
  /* fixed_mask[(K+1)*(N/2)], row-major [vertex][derivative]: 1 = the vertex has a constraint on
   * that derivative (Vertex::hasConstraint, vertex.h:84), 0 = free.  NULL selects the
   * createRandomVertices / "waypoint" topology (vertex.cpp:27-82): first and last vertex fix
   * derivatives 0..N/2-1, interior vertices fix position only. */
  const uint8_t* fixed_mask;
} mtg_problem;

typedef struct mtg_layout {
  int32_t n_all;    /* K*N          getNumberAllConstraints()   */
  int32_t n_fixed;  /*              getNumberFixedConstraints() */
  int32_t n_free;   /*              getNumberFreeConstraints()  */
  int32_t kernel;   /* MTG_KERNEL_* this problem is routed to   */
} mtg_layout;

/* ---- lifecycle ------------------------------------------------------------------------- */
int mtg_create(int device, mtg_handle** out);
void mtg_destroy(mtg_handle* h);
/* last error text of this handle (or of the last failed mtg_create when h == NULL) */
const char* mtg_last_error(const mtg_handle* h);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t mtg_launch_count(const mtg_handle* h);
/* 1 when the visible device of the handle is compute capability 10.x */
int mtg_device_is_sm90(const mtg_handle* h);

/* tuning knobs (results are identical to rounding; used by tests and profiles)
 *   MTG_OPT_WAYPOINT_VARIANT: 0 = default (6 where it applies, else 4 for K <= 8, 3 while the factor fits on chip at
 *                                 two CTAs per SM, 5 beyond),
 *                             1 = one thread per trajectory, 2 = twisted (state in shared memory),
 *                             3 = twisted with the sweep state in shared memory + TMA tensor stores,
 *                             4 = persistent version of 3 with deep input prefetch,
 *                             5 = chunked kernel (outer sweep blocks parked in global memory), any K (default for
 *                                 K too large for 3),
 *                             6 = 4 with the inputs moved by TMA bulk copies (B % 16 == 0, 16-byte aligned inputs, K
 *                                 small enough for an input tile beside the state: K <= 16 at N = 10, D = 3). */
#define MTG_OPT_WAYPOINT_VARIANT 1
#define MTG_OPT_RING_DEPTH 2      /* reserved (the persistent kernel is built with a 3-deep input ring) */
#define MTG_OPT_CTAS_PER_SM 3     /* variant 4: cap on resident CTAs per SM, 0 = as many as fit, 9 = one CTA per tile;
                                     chunked kernel: cap on resident warps per SM, 0 = as many as fit */
#define MTG_OPT_STAGGER_US 4      /* reserved (accepted, no effect: the start-time stagger experiment was removed, DESIGN.md 4) */
#define MTG_OPT_CHUNK_BLOCKS 6    /* chunked (large-K) kernel: vertex blocks per lane kept in shared memory (the
                                     outer ones are parked in global memory), 0 = auto */
#define MTG_OPT_GENERIC_VARIANT 7 /* arbitrary masks: 0 = masked block kernel (default), 1 = banded kernel in global scratch */
#define MTG_OPT_MELLINGER_UNFUSED 8 /* 1 = batched Mellinger gradient through expand + solve + cost kernels */
#define MTG_OPT_TMA_INPUTS 9      /* 0 = never, 1 = the TMA-input kernel (v5) where two input tiles fit (double buffered),
                                    2 (default) = also where only one fits (single buffered) */
#define MTG_OPT_EARLY_REFILL 10   /* TMA-input kernel with one tile buffer: 0 = the buffer is refilled with the next tile two
                                   * outward-sweep steps before the tile ends (default), -1 = while the last segment is emitted */
#define MTG_OPT_CHUNK_WARPS 11    /* chunked kernel: warps per CTA, 1 or 4, 0 = auto (1: shared memory is allocated per warp,
                                     so more warps fit per SM) */
#define MTG_OPT_L2_HINTS 12       /* chunked kernel: 0 = no cache hints (default), 1 = inputs and coefficient stores marked
                                     evict-first in L2 (meant to keep the parked blocks there; measured slower on H100) */
#define MTG_OPT_DYNAMIC_TILES 5   /* persistent kernel: warps draw tiles from a global counter: 0 = auto, 1 = always, 2 = never */
int mtg_set_option(mtg_handle* h, int key, int value);

/* ---- host-only layout: the constraint reordering (linear_impl.h:181-260) ---------------- */
/* slot_col (nullable) receives K*N entries: row i*N+s of C (segment i, slot s; s < N/2 is
 * derivative s at the segment start, s >= N/2 derivative s-N/2 at its end) has its single 1 in
 * column slot_col[i*N+s]; columns [0,n_fixed) are d_fixed, [n_fixed, n_fixed+n_free) are d_free. */
int mtg_problem_layout(const mtg_problem* p, mtg_layout* out, int32_t* slot_col);

/* ---- the hot path, DEVICE pointers, asynchronous on `stream` (a cudaStream_t, may be 0) --- */
/* seg_times [B][K], d_fixed [B][D][n_fixed]  ->  coeffs [B][K][D][N]
 * optional: d_free [B][D][n_free], status [B] (int32). */
int mtg_solve_linear_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                               const double* d_fixed, double* coeffs, double* d_free, int32_t* status,
                               void* stream);

/* SURVEY.md 8f-1 ("next" row): time allocation + constraint packing fused into the solve, for the
 * createRandomVertices topology.  positions [B][K+1][D]; segment times are computed on the device as
 * estimateSegmentTimesNfabian(v_max, a_max, magic) (reference src/vertex.cpp:255-272; pass magic = 6.5
 * for the reference default), start/end derivatives 1..N/2-1 are zero (Vertex::makeStartOrEnd,
 * src/vertex.cpp:147-153).  coeffs [B][K][D][N]; seg_times_out [B][K] and status are optional.
 * Reads 8*(K+1)*D bytes per trajectory instead of 8*(K + D*n_fixed). */
int mtg_solve_waypoints_nfabian_batch_f64(mtg_handle* h, int32_t N, int32_t r, int32_t K, int32_t D, int64_t B,
                                          const double* positions, double v_max, double a_max, double magic,
                                          double* coeffs, double* seg_times_out, int32_t* status, void* stream);

/* updateSegmentsFromCompactConstraints for given d_free (setFreeConstraints path). */
int mtg_coeffs_from_constraints_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B,
                                          const double* seg_times, const double* d_fixed,
                                          const double* d_free, double* coeffs, void* stream);

/* computeCost(): cost[b] = 0.5 * sum_{segments, dims} c^T Q(T) c. */
int mtg_compute_cost_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                               const double* coeffs, double* cost, void* stream);

/* SURVEY.md 8f-2 ("next" row): the nonlinear time optimiser's numerical gradient, batched.
 * PolynomialOptimizationNonLinear::getCostAndGradientMellinger (reference
 * impl/polynomial_optimization_nonlinear_impl.h:286-364): cost[b] = computeCost() at seg_times[b], grad[b][n] =
 * (cost with +0.1 s on segment n and -0.1/(K-1) s on the others, clamped at 0.1 s, re-solved) - cost) / 0.1.
 * The K+1 solves of every trajectory run as ONE cost-only launch over the expanded batch: the perturbed times are
 * generated inside the kernel and the cost 0.5 d^T H d is accumulated from the solved end-point derivatives, so no
 * perturbed input and no coefficient is ever written (shapes without a fused kernel take expand + solve + cost
 * kernels).  cost may be NULL. */
int mtg_cost_gradient_mellinger_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                          const double* d_fixed, double* cost, double* grad, void* stream);

/* SURVEY.md 8f-3 ("next" row): batched Trajectory::evaluate on a uniform grid t_s = t_start + s*dt,
 * s < n_samples (reference src/trajectory.cpp:48-79 conventions per sample: a time on a vertex belongs to the
 * segment on its right, t == total time is the end of the last segment, beyond the end yields zeros;
 * Horner form of Polynomial::evaluate, polynomial.h:134-149).  coeffs [B][K][D][N] -> out [B][n_samples][D].
 * t_s is rounded twice, fl(t_start + fl(s*dt)) (never a fused multiply-add), so a sample lands on a vertex exactly
 * when the same expression computed by the caller does. */
int mtg_evaluate_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                           const double* coeffs, int32_t derivative, double t_start, double dt, int32_t n_samples,
                           double* out, void* stream);

/* SURVEY.md 8f-3: batched Trajectory::evaluateRange (reference src/trajectory.cpp:81-141) -- and with
 * derivs = {0,1,2,3,4} the sample set of sampleTrajectoryInRange (src/trajectory_sampling.cpp:45-110) -- for B
 * trajectories at once.  The reference's sequential walk is replayed exactly (running time_in_segment += dt; the
 * sample clock starts at the start of the segment that contains t_start; a sample on a segment end belongs to the
 * left segment; the walk ends after the last segment), and every sample is Polynomial::evaluate's arithmetic
 * (separate multiply and add), so samples are bit-identical to an x86 build of the reference.
 *   out            [B][max_samples][n_derivs][D]   (rows >= n_samples[b] are zero)
 *   n_samples      [B]  number of samples the reference would produce (may exceed max_samples: only the first
 *                       max_samples are stored); -1 when t_start lies beyond the trajectory (reference: LOG(ERROR),
 *                       empty result)
 *   sampling_times [B][max_samples] or NULL: the reference's `sampling_times` output
 * derivs is a HOST array of n_derivs (<= 8) derivative orders. */
int mtg_evaluate_range_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                 const double* coeffs, double t_start, double t_end, double dt, int32_t n_derivs,
                                 const int32_t* derivs, int32_t max_samples, double* out, int32_t* n_samples,
                                 double* sampling_times, void* stream);

/* computeMaximumOfMagnitude (impl/polynomial_optimization_linear_impl.h:465-497), B trajectories x n_derivs orders.
 * Candidates per segment are 0, T and every real root in [0, T] of sum_d p_d^(k) p_d^(k+1) (p^(k+1) for D = 1;
 * src/segment.cpp:83-184); the largest |p^(k)(t)| wins, the first one on a tie; all zero gives Extremum() = (0, 0, 0).
 * N even in [2, 12].  derivs: HOST array, n_derivs <= 8, each in [0, N-2].  value/time/segment: [B][n_derivs]; time is
 * relative to the segment start (Extremum::time); time, segment, status nullable.  A segment time <= 0 or non-finite:
 * status MTG_STATUS_BAD_TIME, value and time NaN, segment -1. */
int mtg_max_magnitude_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                const double* coeffs, int32_t n_derivs, const int32_t* derivs, double* value,
                                double* time, int32_t* segment, int32_t* status, void* stream);

/* The soft constraints and time cost of PolynomialOptimizationNonLinear (impl/polynomial_optimization_nonlinear_impl.h). */
typedef struct mtg_soft_constraint {
  int32_t derivative; /* in [0, N-2] */
  double max_value;   /* > 0 and finite (the reference would divide by 0 at max_value == 0) */
} mtg_soft_constraint;
typedef struct mtg_time_objective {
  int32_t time_cost;             /* 0: penalty * T_total^2 (kSquaredTime*), 1: penalty * T_total (kRichterTime*) */
  double time_penalty;           /* reference default 500 */
  double soft_constraint_weight; /* reference default 100 */
  double maximum_cost;           /* clamp of each soft term: 1e12 in the objectives, 1e9 in getTotalCostWithSoftConstraints */
  int32_t n_constraints;         /* 0..8; 0 = use_soft_constraints == false */
  const mtg_soft_constraint* constraints; /* HOST array, summed in array order like inequality_constraints_ */
} mtg_time_objective;

/* objectiveFunctionTime (nonlinear_impl.h:556-615) when d_free == NULL: the solve of mtg_solve_linear_batch_f64 at
 * seg_times; else objectiveFunctionTimeAndConstraints (:660-742): setFreeConstraints with d_free [B][D][n_free], as
 * mtg_coeffs_from_constraints_batch_f64.  coeffs [B][K][D][N] is a required output (the extrema read it).
 * objective[b] = computeCost() + time cost + sum_c min(maximum_cost, exp((max_c - max_value_c) / max_value_c * weight))
 * (evaluateMaximumMagnitudeAsSoftConstraint, :766-795), summed in that order; the time sum runs left to right.
 * terms [B][3] nullable = (trajectory cost, time cost, soft cost).  status [B] nullable; a trajectory with status != 0
 * (MTG_STATUS_BAD_TIME, MTG_STATUS_NOT_SPD) has objective NaN. */
int mtg_time_objective_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                 const double* d_fixed, const double* d_free, const mtg_time_objective* obj,
                                 double* coeffs, double* objective, double* terms, int32_t* status, void* stream);

/* Trajectory::scaleSegmentTimesToMeetConstraints (src/trajectory.cpp:382-429, Liu et al., RA-L 2017) for B
 * trajectories: up to 20 times, find max |v| and max |a| (as mtg_max_magnitude_batch_f64 with derivs {1, 2}), stop
 * when v / v_max <= 1.001 and a / a_max <= 1.001, else stretch every segment time by
 * s = std::max(1, std::max(v / v_max, sqrt(a / a_max))) and scale coefficient n by (1 / s)^n
 * (Polynomial::scalePolynomialInTime, src/polynomial.cpp:199-205), with the reference's arithmetic.  The whole loop
 * runs in one kernel launch.
 *   seg_times [B][K], coeffs [B][K][D][N] -> seg_times_out, coeffs_out; the outputs may be the input buffers (in-place
 *   use, as the reference mutates its Trajectory), but must not overlap them otherwise.
 *   within_range [B] int32: the reference's return value (1 = the last check met both limits; 0 after 20 stretches).
 *   maxima [B][2] = (max |v|, max |a|) at the last check.  status [B]: MTG_STATUS_BAD_TIME.  All three nullable.
 * N even in [4, 12]; v_max, a_max > 0 (not NaN), +inf = no limit on that order.  A row with a segment time <= 0 or
 * non-finite gets status MTG_STATUS_BAD_TIME, within_range 0, maxima NaN, and its times and coefficients unchanged.
 * A NaN violation (an infinite maximum against an infinite limit) gives s = 1 every round, as std::max does in the
 * reference: 20 unchanged rounds, within_range 0. */
int mtg_scale_to_constraints_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                       const double* seg_times, const double* coeffs, double v_max, double a_max,
                                       double* seg_times_out, double* coeffs_out, int32_t* within_range,
                                       double* maxima, int32_t* status, void* stream);

/* PolynomialOptimizationNonLinear::scaleSegmentTimesWithViolation (impl/polynomial_optimization_nonlinear_impl.h:
 * 366-406): solve at seg_times (as mtg_solve_linear_batch_f64), stretch as mtg_scale_to_constraints_batch_f64, then
 * solve again at the stretched times seg_times_out (may be seg_times) into coeffs [B][K][D][N].  The limits follow
 * mtg_scale_to_constraints_batch_f64 (+inf where the reference passes 0 for a missing constraint, :373-381).  A row
 * whose first solve fails keeps its input times and gets within_range 0 and maxima NaN.  status [B] is the OR of the
 * three steps' status bits.  within_range, maxima, status nullable. */
int mtg_scale_times_with_violation_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                             const double* d_fixed, double v_max, double a_max, double* coeffs,
                                             double* seg_times_out, int32_t* within_range, double* maxima,
                                             int32_t* status, void* stream);

/* Result codes of mtg_optimize_time_mellinger_batch_f64 and mtg_optimize_time_batch_f64: the public nlopt_result values, so that callers of the
 * reference read stopping reasons as before. */
#define MTG_OPTIMIZE_RESULT_FAILURE (-1)
#define MTG_OPTIMIZE_RESULT_ROUNDOFF_LIMITED (-4)
#define MTG_OPTIMIZE_RESULT_SUCCESS 1
#define MTG_OPTIMIZE_RESULT_FTOL_REACHED 3
#define MTG_OPTIMIZE_RESULT_XTOL_REACHED 4
#define MTG_OPTIMIZE_RESULT_MAXEVAL_REACHED 5

/* The stopping rules of NonlinearOptimizationParameters that the Mellinger outer loop reads.  A negative tolerance
 * disables its test.  Reference defaults: f_abs -1, f_rel 0.05, x_rel -1, x_abs -1, initial_stepsize_rel 0.1,
 * max_iterations 3000. */
typedef struct mtg_mellinger_params {
  double f_abs, f_rel, x_rel, x_abs;
  double initial_stepsize_rel; /* <= 0: 0.1 ("heuristic if negative") */
  int32_t max_iterations;      /* gradient evaluations; < 0: no limit */
} mtg_mellinger_params;

/* PolynomialOptimizationNonLinear::optimize() with kMellingerOuterLoop (impl/polynomial_optimization_nonlinear_impl.h:
 * 171-259) for B trajectories: a descent on the segment times with the gradient of
 * mtg_cost_gradient_mellinger_batch_f64, times bounded below by 0.1 s, then mtg_scale_times_with_violation_batch_f64.
 * The reference drives the descent with NLopt; this entry defines its own projected-gradient descent, per row, with
 * x = the K segment times, l = 0.1, and k counting gradient evaluations from 0:
 *   1. (J_k, g_k) = getCostAndGradientMellinger(x_k), exactly as mtg_cost_gradient_mellinger_batch_f64.
 *   2. alpha_0 = fl(fl(initial_stepsize_rel * max_i x_0,i) / max_i |g_0,i|).
 *   3. Every g_k,i == 0 (always for K = 1): stop, SUCCESS.
 *   4. Candidates j = 0..7 at step a_j = fl(alpha_k * 2^(1-j)): x_j,i = max(l, fl(x_k,i - fl(a_j * g_k,i))) (two roundings,
 *      no FMA, `v > l ? v : l`).  J_j = computeCost() of the solve at x_j.
 *   5. Accept the smallest j with J_j <= fl(J_k + fl(1e-4 * s_j)), s_j = sum_i fl(g_k,i * fl(x_j,i - x_k,i)) summed left
 *      to right: x_k+1 = x_j, alpha_k+1 = a_j.  No candidate accepted: stop, ROUNDOFF_LIMITED, keep x_k (so the cost
 *      never rises above the start).
 *   6. After an accepted step, in this order: k+1 >= max_iterations (when >= 0): MAXEVAL_REACHED; |J_j - J_k| <=
 *      f_rel * |J_j| or <= f_abs: FTOL_REACHED; for every i, |x_k+1,i - x_k,i| <= x_rel * |x_k+1,i| or <= x_abs:
 *      XTOL_REACHED.  Otherwise iterate.  max_iterations == 0: every valid row stops at once with MAXEVAL_REACHED.
 * Then every row that iterated goes through mtg_scale_times_with_violation_batch_f64 at (v_max, a_max).
 * Outputs: seg_times_out [B][K] the scaled times (may be seg_times), coeffs [B][K][D][N] the re-solve at them;
 * relative_times [B][K] the times before scaling (the reference's "RELATIVE Solution"); cost [B] computeCost() at the
 * final times (getCost()); iterations [B] accepted steps; result [B] MTG_OPTIMIZE_RESULT_*; within_range, maxima as the
 * scaling entry; status [B] the scaling's status bits, with MTG_STATUS_NOT_SPD when the loop stopped on a failed solve.
 * Everything after seg_times_out is nullable.  Edge rows:
 *   a segment time <= 0 or non-finite: FAILURE, status MTG_STATUS_BAD_TIME, times unchanged, 0 iterations;
 *   a start time in (0, 0.1): FAILURE, neither iterated nor scaled (decision: the reference returns before the scaling
 *     when its optimiser aborts without a cost, which NLopt does for a start below the lower bound); coeffs are the
 *     solve at the start times;
 *   any solve of a row reporting MTG_STATUS_NOT_SPD (gradient or candidates): FAILURE, keeps x_k, then scaled.
 * A row's result does not depend on the other rows of the batch.  Unlike the other entries this one WAITS on `stream`
 * once per iteration: it reads the number of rows still iterating (pinned memory, one event wait), and every
 * launch after that covers only those rows.  Refused (MTG_ERR_BAD_ARG, no launch): what
 * mtg_scale_times_with_violation_batch_f64 refuses, a null params, and params with every tolerance negative and
 * max_iterations < 0. */
int mtg_optimize_time_mellinger_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                          const double* d_fixed, const mtg_mellinger_params* params, double v_max,
                                          double a_max, double* coeffs, double* seg_times_out, double* relative_times,
                                          double* cost, int32_t* iterations, int32_t* result, int32_t* within_range,
                                          double* maxima, int32_t* status, void* stream);

/* PolynomialOptimizationNonLinear::optimize() with kSquaredTime or kRichterTime (optimizeTime(), impl/
 * polynomial_optimization_nonlinear_impl.h:132-168) for B trajectories: the K segment times minimise the objective of
 * mtg_time_objective_batch_f64 (d_free == NULL) with the caller's `obj`, bounded below by 0.1 s.  obj->time_cost picks
 * the method (0 kSquaredTime, 1 kRichterTime).  The reference drives the search with NLopt's LN_BOBYQA; this entry
 * defines its own derivative-free compass search, per row, with x = the K segment times, l = 0.1, f(x) = that
 * objective, and e counting objective evaluations (OptimizationInfo::n_iterations):
 *   1. Start.  A segment time <= 0 or non-finite: FAILURE, status MTG_STATUS_BAD_TIME, times unchanged, e = 0.  A time
 *      in (0, 0.1): FAILURE, not iterated, e = 1 (the Mellinger entry's decision).  Otherwise f_0 = f(x_0), e = 1; a
 *      start solve reporting MTG_STATUS_NOT_SPD gives FAILURE.
 *   2. Steps.  delta_i = fl(rho * x_0,i), rho = initial_stepsize_rel (<= 0: 0.1), NLopt's initial_step as the
 *      reference sets it (:139-147).
 *   3. Poll, only if max_iterations < 0 or e + 2K <= max_iterations (else stop: MAXEVAL_REACHED).  Candidate j = 2i
 *      has y_i = fl(x_i + delta_i), j = 2i + 1 has y_i = max(l, fl(x_i - delta_i)) (`v > l ? v : l`, no FMA); every
 *      other coordinate equals x.  All 2K are evaluated: e += 2K.
 *   4. Accept.  j* = the candidate with the smallest objective, the lowest j on a tie.  f(y_j*) < f(x) (strict; a NaN
 *      never wins): x = y_j*, f = f(y_j*), delta unchanged.  Otherwise every delta_i = delta_i / 2.  Any candidate
 *      solve reporting MTG_STATUS_NOT_SPD ends the row: FAILURE, keeps x, status bit set.
 *   5. Stop, tested in this order after each poll.  After an accepted poll: |df| <= f_rel * |f_new| (f_rel >= 0) or
 *      <= f_abs (f_abs >= 0): FTOL_REACHED; else, when x_rel >= 0 or x_abs >= 0, every |dx_i| <= x_rel * |x_i| or
 *      <= x_abs: XTOL_REACHED.  After a failed poll: when x_rel >= 0 or x_abs >= 0, every halved delta_i <= x_rel *
 *      |x_i| or <= x_abs: XTOL_REACHED; else, every candidate of the next poll equal to x bit for bit:
 *      ROUNDOFF_LIMITED.  Otherwise the next poll (step 3).
 * The objective strictly decreases over finitely many fp64 points and delta reaches rounding after about 55 halvings,
 * so every row stops even without tolerances.  params: the fields of mtg_mellinger_params are read as NLopt reads
 * NonlinearOptimizationParameters; max_iterations counts OBJECTIVE EVALUATIONS (NLopt's maxeval), not gradient
 * evaluations as in mtg_optimize_time_mellinger_batch_f64.
 * Outputs: seg_times_out [B][K] the BEST point the search found (may be seg_times; the reference leaves its problem at
 * the last point NLopt evaluated, which need not be the best); coeffs [B][K][D][N] the solve at it; objective [B] and
 * terms [B][3] as mtg_time_objective_batch_f64 there; evaluations [B] e; result [B] MTG_OPTIMIZE_RESULT_*; status [B]
 * the objective's status bits at the returned times, with MTG_STATUS_NOT_SPD when a candidate's solve failed.  No
 * scaleSegmentTimesWithViolation follows (optimizeTime() does not call it).  Everything after seg_times_out is
 * nullable.  A row's result does not depend on the other rows of the batch.  Like the Mellinger entry this one WAITS
 * on `stream` once per poll to read the number of rows still iterating.  Refused (MTG_ERR_BAD_ARG, no launch): what
 * mtg_time_objective_batch_f64 refuses, a null params, and params with every tolerance negative and
 * max_iterations < 0. */
int mtg_optimize_time_batch_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                const double* d_fixed, const mtg_time_objective* obj,
                                const mtg_mellinger_params* params, double* coeffs, double* seg_times_out,
                                double* objective, double* terms, int32_t* evaluations, int32_t* result,
                                int32_t* status, void* stream);

/* FeasibilityAnalytic::checkInputFeasibility per segment and checkInputFeasibilityTrajectory per trajectory (reference
 * mav_trajectory_generation_ros/src/feasibility_analytic.cpp, feasibility_base.cpp).  result[b] is an MTG_FEAS_* code
 * (InputFeasibilityResult): the first segment that is not Feasible decides, in the reference's order of checks --
 * thrust in [f_min, f_max] (ThrustLow before ThrustHigh; run when f_min, f_max or omega_xy_max is present), speed over
 * dims 0..2, yaw rate and yaw acceleration (D = 4 only), then the recursive roll/pitch bound sqrt(j_max / f_min) over
 * halved sections down to min_section_time.  The roll/pitch step returns only Feasible or Indeterminable (a section
 * shorter than min_section_time, the whole segment included, is Indeterminable); MTG_FEAS_ROLL_PITCH_RATES is never
 * returned.  Candidates are 0, T and the exact real roots of each critical polynomial in [0, T] (the reference's
 * Jenkins-Traub |imag| > eps filter is not reproduced); their values use the reference's arithmetic.
 *   segment[b]: index of the deciding segment, -1 when the row is Feasible or has a bad time.  segment, status nullable.
 *   D not 3 or 4: every row Indeterminable at segment 0, as the reference.
 *   A segment time <= 0 or non-finite: status MTG_STATUS_BAD_TIME, result Indeterminable, segment -1.
 *   status MTG_STATUS_FEAS_CAPACITY: see above (not met by trajectories with distinct roots and T / min_section_time
 *   below 2^60).
 * N even in [4, 12].  The limits are final values: InputConstraints::addConstraint's abs() and f_min / f_max
 * corrections belong to the caller (the host mirror's InputConstraints applies them).  Refused (MTG_ERR_BAD_ARG, no
 * launch): a present limit that is NaN or negative, unknown `present` bits, a non-finite gravity, min_section_time <= 0
 * or non-finite.  An absent limit's value is ignored; +inf never fails. */
#define MTG_FEAS_FEASIBLE 0
#define MTG_FEAS_INDETERMINABLE 1
#define MTG_FEAS_THRUST_HIGH 2
#define MTG_FEAS_THRUST_LOW 3
#define MTG_FEAS_VELOCITY 4
#define MTG_FEAS_ROLL_PITCH_RATES 5
#define MTG_FEAS_YAW_RATES 6
#define MTG_FEAS_YAW_ACC 7
/* mtg_input_constraints::present bits (InputConstraintType order) */
#define MTG_INPUT_F_MIN (1u << 0)
#define MTG_INPUT_F_MAX (1u << 1)
#define MTG_INPUT_V_MAX (1u << 2)
#define MTG_INPUT_OMEGA_XY_MAX (1u << 3)
#define MTG_INPUT_OMEGA_Z_MAX (1u << 4)
#define MTG_INPUT_OMEGA_Z_DOT_MAX (1u << 5)
#define MTG_INPUT_ALL 0x3fu
typedef struct mtg_input_constraints {
  uint32_t present;        /* MTG_INPUT_* bits: which limits apply */
  double f_min;            /* normalized thrust [m/s^2] */
  double f_max;
  double v_max;            /* [m/s] */
  double omega_xy_max;     /* roll/pitch rate [rad/s] */
  double omega_z_max;      /* yaw rate [rad/s] */
  double omega_z_dot_max;  /* yaw acceleration [rad/s^2] */
  double gravity;          /* added to the z acceleration for the thrust (mav_msgs::kGravity in the reference) */
  double min_section_time; /* FeasibilityAnalytic / FeasibilityRecursive::Settings, reference default 0.05 s */
} mtg_input_constraints;
int mtg_input_feasibility_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                    const double* coeffs, const mtg_input_constraints* constraints, int32_t* result,
                                    int32_t* segment, int32_t* status, void* stream);

/* FeasibilityRecursive::checkInputFeasibility per segment and checkInputFeasibilityTrajectory per trajectory
 * (reference mav_trajectory_generation_ros/src/feasibility_recursive.cpp).  Same arguments, outputs, refusals, bad-time
 * rule and D rule as mtg_input_feasibility_batch_f64; min_section_time is FeasibilityRecursive::Settings'.  Per segment:
 * the recursion over [0, T], then (D = 4, only when it gives Feasible) yaw rate and yaw acceleration over the whole
 * segment.  Per section [t1, t2], depth first and left half first:
 *   t2 - t1 < min_section_time: Indeterminable (also with no limit present, so a segment shorter than
 *   min_section_time is always Indeterminable, unlike the analytic check);
 *   thrust |p'' + (0, 0, g)| at t1 and t2 against f_min (ThrustLow) and f_max (ThrustHigh); speed |p'| over dims 0..2
 *   at t1 and t2 (Velocity);
 *   per axis, from t1, t2 and the roots in [t1, t2]: a single-axis speed above v_max (Velocity), a single-axis thrust
 *   above f_max (ThrustHigh), and upper / lower bounds on speed, thrust and jerk summed over the axes;
 *   thrust upper bound < f_min: ThrustLow; lower bound > f_max: ThrustHigh;
 *   a bound beyond its limit (or the roll/pitch bound sqrt(j_max^2 / f_min^2), DBL_MAX when f_min^2 <= 1e-6, above
 *   omega_xy_max) halves the section; otherwise the section is Feasible.
 * Reachable results: Feasible, Indeterminable, ThrustLow, ThrustHigh, Velocity, YawRates, YawAcc; never
 * MTG_FEAS_ROLL_PITCH_RATES.  The roots are the exact real roots of p_i'', p_i''' and p_i'''' in [0, T] (the
 * reference's Jenkins-Traub roots with their |imag| > eps filter are not reproduced, and root finding never fails
 * here); every value uses the reference's arithmetic (Polynomial::evaluate, then g added to z; std::pow(x, 2) as
 * x * x, which is what an optimised x86 build of the reference computes).
 *   status MTG_STATUS_FEAS_CAPACITY (result Indeterminable): the roots of one axis and order k (k = 1, 2, 3) needed
 *   more than N - 2 - k + 2 entries (only clusters of roots unresolved at 2^-24 T add entries), or the bisection went
 *   64 levels deep (a section with f_min^2 <= 1e-6 at a min_section_time below T / 2^64). */
int mtg_input_feasibility_recursive_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                              const double* seg_times, const double* coeffs,
                                              const mtg_input_constraints* constraints, int32_t* result,
                                              int32_t* segment, int32_t* status, void* stream);

/* FeasibilitySampling::checkInputFeasibility per segment and checkInputFeasibilityTrajectory per trajectory
 * (reference mav_trajectory_generation_ros/src/feasibility_sampling.cpp).  Same outputs, refusals of the limits and
 * gravity, bad-time rule and D rule as mtg_input_feasibility_batch_f64; min_section_time is neither read nor
 * validated, and sampling_interval (FeasibilitySampling::Settings, reference default 0.01 s) takes its place.  Per
 * segment the samples are t = 0, fl(t + sampling_interval), ... while t <= T (the reference's running fp64 sum, not
 * k * sampling_interval, so T itself may be missed), and at each one the flat state goes through mav_msgs'
 * EigenMavStateFromEigenTrajectoryPoint with the given gravity:
 *   f = a + (0, 0, g), thrust = |f|, zb = f * (1 / thrust), xc = (cos yaw, sin yaw, 0), yb = normalized(zb x xc),
 *   xb = yb x zb, acceleration_B = R^T (zb thrust) with R = [xb yb zb], h = (1 / thrust) (j - (zb . j) zb),
 *   omega_B = (-h . yb, h . xb, yaw_rate zb_z), omega_dot_B,z = yaw_acc zb_z
 * (yaw, yaw rate, yaw acceleration from dim 3 when D = 4, through the quaternion round trip of setFromYaw / getYaw;
 * 0 when D = 3).  The checks, in order, the first failing sample and check deciding: only when f_min or f_max is
 * present |acceleration_B| < f_min (ThrustLow) and > f_max (ThrustHigh); |v| over dims 0..2 > v_max (Velocity);
 * |omega_B,xy| > omega_xy_max (RollPitchRates); |omega_B,z| > omega_z_max (YawRates); |omega_dot_B,z| >
 * omega_z_dot_max (YawAcc).  Values use Polynomial::evaluate's Horner and one rounding per operation; a NaN state (a
 * thrust of exactly 0) passes every comparison, as in the reference.  This is the only entry that returns
 * MTG_FEAS_ROLL_PITCH_RATES; it never returns MTG_FEAS_INDETERMINABLE for a good row with D 3 or 4 below the cap.
 *   status MTG_STATUS_FEAS_CAPACITY (result Indeterminable): fl(T / sampling_interval) > 2^24 for the deciding
 *   segment, which is then not sampled at all.
 * Refused (MTG_ERR_BAD_ARG, no launch): everything mtg_input_feasibility_batch_f64 refuses except min_section_time,
 * and a sampling_interval <= 0, NaN or infinite. */
int mtg_input_feasibility_sampling_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                             const double* seg_times, const double* coeffs,
                                             const mtg_input_constraints* constraints, double sampling_interval,
                                             int32_t* result, int32_t* segment, int32_t* status, void* stream);

/* FeasibilityBase::checkHalfPlaneFeasibility per segment and per trajectory (reference
 * mav_trajectory_generation_ros/src/feasibility_base.cpp:109-154): a segment passes plane (point q, normal n) when
 * (p(t) - q) . n > 0 at 0, T and every real root in [0, T] of the derivative of the projection n . p(t); the first
 * segment with a failing plane decides, and within it the first plane.  Values use the reference's arithmetic
 * (Horner per dimension, the subtraction, the dot product in dimension order), so a NaN value passes, as there.
 *   feasible[b]: 1 or 0.  segment[b], plane[b]: the first failing pair, -1 when none.  status[b]: 0 or
 *   MTG_STATUS_BAD_TIME.  segment, plane and status are nullable.
 *   planes: a HOST array of n_planes entries, read before the call returns (the caller may reuse it at once).  The
 *   planes are used as given: the reference's HalfPlane constructor normalises the normal, and so do the host mirror's
 *   HalfPlane and the Python helpers; a normal of another length scales every distance but changes no sign.
 *   n_planes = 0: every row with D in {3, 4} is feasible.
 *   D not 3 or 4: every row infeasible with segment 0 and plane -1, as the reference.
 *   A segment time <= 0 or non-finite: status MTG_STATUS_BAD_TIME, feasible 0, segment and plane -1 (the reference
 *   would pass it: its candidate list is empty when T < 0).
 *   Candidates are exact real roots, not Jenkins-Traub's: a row whose smallest distance lies within rounding of 0 can
 *   be decided differently from the reference.
 * N even in [2, 12].  Refused (MTG_ERR_BAD_ARG, no launch): n_planes < 0 or > MTG_MAX_HALF_PLANES, a null planes with
 * n_planes > 0, a non-finite point or normal component, an all-zero normal. */
#define MTG_MAX_HALF_PLANES 64
typedef struct mtg_half_plane {
  double point[3];   /* a point on the plane */
  double normal[3];  /* points into the allowed half-space */
} mtg_half_plane;
int mtg_half_plane_feasibility_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                         const double* seg_times, const double* coeffs, int32_t n_planes,
                                         const mtg_half_plane* planes, int32_t* feasible, int32_t* segment,
                                         int32_t* plane, int32_t* status, void* stream);

/* Flat states: mav_msgs::EigenTrajectoryPoint of sampleTrajectoryInRange, sampleWholeTrajectory and
 * sampleTrajectoryAtTime (reference src/trajectory_sampling.cpp:27-110), one fixed record of MTG_FLAT_STATE_DOUBLES
 * doubles per sample, fields at the offsets below:
 *   position_W, velocity_W, acceleration_W, jerk_W, snap_W   dims 0..2 of derivatives 0..4 (Polynomial::evaluate's
 *                                                            arithmetic: bit for bit mtg_evaluate_range_batch_f64's)
 *   orientation (w, x, y, z), angular_velocity_W, angular_acceleration_W:
 *     D = 4: setFromYaw / setFromYawRate / setFromYawAcc of dim 3: (cos y/2, 0, 0, sin y/2), (0, 0, y'), (0, 0, y'')
 *     D = 6: the rotation vector phi of dims 3..5: orientation exp(phi) with w >= 0, angular velocity J(phi) phi' and
 *            acceleration J phi'' + J' phi' (J the left Jacobian of SO(3)).  The reference converts through
 *            Eigen::Quaterniond(Matrix3d), whose sign can make w < 0 past a rotation angle of 2 pi / 3: the same
 *            rotation with the opposite sign.
 *     other D >= 3: identity, zero angular terms.
 * degrees_of_freedom is not stored: DOF6 when D = 6, DOF4 otherwise.  Trigonometry is the device's, a few ulps from
 * glibc's. */
#define MTG_FLAT_STATE_DOUBLES 25
#define MTG_FLAT_STATE_POSITION 0
#define MTG_FLAT_STATE_VELOCITY 3
#define MTG_FLAT_STATE_ACCELERATION 6
#define MTG_FLAT_STATE_JERK 9
#define MTG_FLAT_STATE_SNAP 12
#define MTG_FLAT_STATE_ORIENTATION 15
#define MTG_FLAT_STATE_ANGULAR_VELOCITY 19
#define MTG_FLAT_STATE_ANGULAR_ACCELERATION 22

/* sampleTrajectoryInRange (whole = 0) / sampleWholeTrajectory (whole = 1) for B trajectories at once.  The samples are
 * those of mtg_evaluate_range_batch_f64 over [min_time, max_time] (the reference's walk, replayed exactly); with
 * whole = 1 min_time and max_time are not read and each row uses [0, its total time], the left-to-right sum of its
 * segment times (Trajectory::getMaxTime).
 *   states     [B][max_samples][MTG_FLAT_STATE_DOUBLES]   (records >= n_samples[b] are zero)
 *   time_ns    [B][max_samples] int64 or NULL: (int64)((min_time + sampling_interval * s) * 1e9), each operation
 *              rounded on its own, truncated toward zero (min_time = 0 when whole = 1); 0 past n_samples[b]
 *   n_samples  [B]  the number of states the reference would produce (may exceed max_samples: only the first
 *              max_samples are stored); -1 where the reference returns false: min_time < 0, max_time above the row's
 *              total time, or D < 3 (every row).  A min_time beyond the trajectory gives 0 (the reference logs an error
 *              and returns true with no states).
 * N in [1, 12].  Refused (MTG_ERR_BAD_ARG, no launch): sampling_interval <= 0 or non-finite, max_samples < 0, K < 1,
 * D < 1, B < 0, a null seg_times, coeffs or n_samples with B > 0, a null states with B > 0 and max_samples > 0. */
int mtg_sample_flat_states_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                     const double* coeffs, double min_time, double max_time, double sampling_interval,
                                     int32_t whole, int32_t max_samples, double* states, int64_t* time_ns,
                                     int32_t* n_samples, void* stream);

/* sampleTrajectoryAtTime for B trajectories, each at its own time sample_times[b] (B vehicles at one control tick).
 * The segment follows Trajectory::evaluate (mtg_evaluate_batch_f64's conventions: a time on a vertex belongs to the
 * segment on its right, the total time is the end of the last segment).
 *   states   [B][MTG_FLAT_STATE_DOUBLES]
 *   time_ns  [B] int64 or NULL: (int64)(t * 1e9)
 *   ok       [B] 1, or 0 with a zero record and time stamp where the reference returns false: t outside [0, the row's
 *            total time] (a NaN t included), or D < 3.
 * N in [1, 12].  Refused (MTG_ERR_BAD_ARG, no launch): K < 1, D < 1, B < 0, a null seg_times, coeffs, sample_times, states
 * or ok with B > 0. */
int mtg_sample_flat_state_at_time_batch_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                            const double* seg_times, const double* coeffs, const double* sample_times,
                                            double* states, int64_t* time_ns, int32_t* ok, void* stream);

/* ---- the hot path, HOST pointers (what PolynomialOptimization<N>::solveLinear() calls) ---- */
/* Same contract with host buffers: each call refuses what its device entry refuses, before any copy, and
 * returns when the results are in the host buffers.  Pinned buffers (mtg_host_alloc) make the copies
 * asynchronous; pageable buffers work but serialise.  The three below are pipelined: up to 4096
 * trajectories run as one chunk, larger batches in chunks of ceil(B / 3) (at most 32768) whose H2D, kernels
 * and D2H overlap on three internal streams. */
int mtg_solve_linear_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                    const double* d_fixed, double* coeffs, double* d_free,
                                    int32_t* status);
int mtg_solve_waypoints_nfabian_batch_host_f64(mtg_handle* h, int32_t N, int32_t r, int32_t K, int32_t D, int64_t B,
                                               const double* positions, double v_max, double a_max, double magic,
                                               double* coeffs, double* seg_times_out, int32_t* status);
int mtg_coeffs_from_constraints_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B,
                                               const double* seg_times, const double* d_fixed,
                                               const double* d_free, double* coeffs);

/* The other host-pointer entry points run the whole batch as one copy in, launch and copy out on one
 * internal stream. */
int mtg_compute_cost_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                    const double* coeffs, double* cost);
int mtg_cost_gradient_mellinger_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                               const double* d_fixed, double* cost, double* grad);
int mtg_evaluate_range_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                      const double* coeffs, double t_start, double t_end, double dt, int32_t n_derivs,
                                      const int32_t* derivs, int32_t max_samples, double* out, int32_t* n_samples,
                                      double* sampling_times);
int mtg_max_magnitude_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B, const double* seg_times,
                                     const double* coeffs, int32_t n_derivs, const int32_t* derivs, double* value,
                                     double* time, int32_t* segment, int32_t* status);
int mtg_time_objective_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                      const double* d_fixed, const double* d_free, const mtg_time_objective* obj,
                                      double* coeffs, double* objective, double* terms, int32_t* status);
int mtg_scale_to_constraints_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                            const double* seg_times, const double* coeffs, double v_max, double a_max,
                                            double* seg_times_out, double* coeffs_out, int32_t* within_range,
                                            double* maxima, int32_t* status);
int mtg_scale_times_with_violation_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B,
                                                  const double* seg_times, const double* d_fixed, double v_max,
                                                  double a_max, double* coeffs, double* seg_times_out,
                                                  int32_t* within_range, double* maxima, int32_t* status);
int mtg_optimize_time_mellinger_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                               const double* d_fixed, const mtg_mellinger_params* params, double v_max,
                                               double a_max, double* coeffs, double* seg_times_out,
                                               double* relative_times, double* cost, int32_t* iterations,
                                               int32_t* result, int32_t* within_range, double* maxima,
                                               int32_t* status);
int mtg_optimize_time_batch_host_f64(mtg_handle* h, const mtg_problem* p, int64_t B, const double* seg_times,
                                     const double* d_fixed, const mtg_time_objective* obj,
                                     const mtg_mellinger_params* params, double* coeffs, double* seg_times_out,
                                     double* objective, double* terms, int32_t* evaluations, int32_t* result,
                                     int32_t* status);

int mtg_input_feasibility_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                         const double* seg_times, const double* coeffs,
                                         const mtg_input_constraints* constraints, int32_t* result, int32_t* segment,
                                         int32_t* status);
int mtg_input_feasibility_recursive_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                                   const double* seg_times, const double* coeffs,
                                                   const mtg_input_constraints* constraints, int32_t* result,
                                                   int32_t* segment, int32_t* status);
int mtg_input_feasibility_sampling_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                                  const double* seg_times, const double* coeffs,
                                                  const mtg_input_constraints* constraints, double sampling_interval,
                                                  int32_t* result, int32_t* segment, int32_t* status);
int mtg_half_plane_feasibility_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                              const double* seg_times, const double* coeffs, int32_t n_planes,
                                              const mtg_half_plane* planes, int32_t* feasible, int32_t* segment,
                                              int32_t* plane, int32_t* status);
int mtg_sample_flat_states_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                          const double* seg_times, const double* coeffs, double min_time,
                                          double max_time, double sampling_interval, int32_t whole, int32_t max_samples,
                                          double* states, int64_t* time_ns, int32_t* n_samples);
int mtg_sample_flat_state_at_time_batch_host_f64(mtg_handle* h, int32_t N, int32_t K, int32_t D, int64_t B,
                                                 const double* seg_times, const double* coeffs,
                                                 const double* sample_times, double* states, int64_t* time_ns,
                                                 int32_t* ok);

/* ---- memory helpers (so host code above the ABI needs no CUDA headers) -------------------- */
void* mtg_host_alloc(mtg_handle* h, uint64_t bytes);   /* pinned */
void mtg_host_free(mtg_handle* h, void* ptr);
void* mtg_device_alloc(mtg_handle* h, uint64_t bytes);
void mtg_device_free(mtg_handle* h, void* ptr);
int mtg_memcpy_h2d(mtg_handle* h, void* dst, const void* src, uint64_t bytes, void* stream);
int mtg_memcpy_d2h(mtg_handle* h, void* dst, const void* src, uint64_t bytes, void* stream);
int mtg_memcpy_d2d(mtg_handle* h, void* dst, const void* src, uint64_t bytes, void* stream);  /* incl. peer memory */
int mtg_stream_synchronize(mtg_handle* h, void* stream);

/* ---- NVLink peer memory between the one-process-per-GPU ranks of a job ----------------------------------------
 * The owner exports a device buffer (64-byte CUDA IPC handle + offset of `ptr` inside its allocation), another
 * rank imports it with ITS device current, which makes the buffer directly addressable by the kernels of that
 * rank: handing a slice of the root's coefficient buffer to mtg_solve_linear_batch_f64 as `coeffs` makes the solve
 * kernels store their results over NVLink straight into their final place -- the gather of BASELINE config C5
 * fused into the solve (mav_trajectory_generation_b200/sharding.py:peer_solve_into_root). */
int mtg_ipc_export(mtg_handle* h, const void* ptr, uint8_t handle_out[64], uint64_t* offset_out);
int mtg_ipc_import(mtg_handle* h, const uint8_t handle[64], uint64_t offset, void** ptr_out, void** base_out);
int mtg_ipc_close(mtg_handle* h, void* base);

/* library version (major*10000 + minor*100 + patch) */
int mtg_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MTG_B200_H_ */
