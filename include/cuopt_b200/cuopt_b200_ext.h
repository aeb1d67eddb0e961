/*
 * Extension entry points of the H100-native libcuopt LP build.
 *
 * The reference C ABI (cuopt_c.h) has no way to read the iteration count, the dual objective or the
 * residuals of an LP solve: they live in additional_termination_information_t
 * (cpp/include/cuopt/linear_programming/pdlp/solver_solution.hpp:47-87), reachable from C++ / Python only.
 * These clearly-prefixed additions expose them, plus a white-box "solver session" used by the parity
 * tests and by bench.py (device-resident timing, per-kernel roofline) and the multi-GPU bootstrap.
 * Nothing here changes the behaviour of the 41 reference symbols.
 */
#ifndef CUOPT_B200_EXT_H
#define CUOPT_B200_EXT_H

#include <cuopt/linear_programming/cuopt_c.h>

#ifdef __cplusplus
extern "C" {
#endif

/* additional_termination_information_t (solver_solution.hpp:47-87) + timing of this build */
typedef struct cuOptB200LPStats {
  cuopt_int_t number_of_steps_taken;           /* accepted PDLP iterations */
  cuopt_int_t total_number_of_attempted_steps; /* PDHG attempts incl. rejected step sizes */
  cuopt_float_t l2_primal_residual;
  cuopt_float_t l2_relative_primal_residual;
  cuopt_float_t l2_dual_residual;
  cuopt_float_t l2_relative_dual_residual;
  cuopt_float_t primal_objective;
  cuopt_float_t dual_objective;
  cuopt_float_t gap;
  cuopt_float_t relative_gap;
  cuopt_int_t solved_by_pdlp;
  cuopt_int_t n_major_iterations; /* termination / restart evaluations */
  cuopt_int_t n_restarts;
  cuopt_int_t method_stand_in; /* 0: the requested method ran; 1: CUOPT_METHOD_CONCURRENT was served by PDLP alone (no
                                * simplex race in this build); 2: CUOPT_METHOD_DUAL_SIMPLEX was served by PDLP with strict
                                * infeasibility detection and tolerances tightened to <= 1e-8 (INTEGRATION.md) */
  cuopt_float_t solve_time;          /* seconds, wall clock of the solver loop (reference semantics) */
  cuopt_float_t setup_seconds;       /* host->device upload, transpose, diagonal scaling */
  cuopt_float_t pdhg_loop_seconds;   /* device time (CUDA events) spent in PDHG batches */
  cuopt_float_t termination_seconds; /* device time spent in termination / restart passes */
  cuopt_float_t initial_step_size;
  cuopt_float_t initial_primal_weight;
  cuopt_float_t final_step_size;
  cuopt_float_t final_primal_weight;
  int64_t kernel_launches; /* kernels of this library launched by the solve */
} cuOptB200LPStats;

/* Statistics of an LP solution returned by cuOptSolve. */
cuopt_int_t cuOptB200GetLPStats(cuOptSolution solution, cuOptB200LPStats* stats);

/* ---- presolve --------------------------------------------------------------------------------------------------
 * Bool parameter (cuOptSetIntegerParameter / cuOptSetParameter / cuopt_cli --presolve true), default false.  When on, the
 * solver first removes, in rounds on the device, fixed columns, empty rows, singleton rows (turned into column bounds) and
 * empty columns, runs PDLP on what is left and maps the solution back to the original rows and columns (postsolve of
 * primal, dual and reduced costs).  Reported objectives include the removed columns; residuals are those of the reduced
 * problem.  Refused with CUOPT_VALIDATION_ERROR together with a warm start, warm-start capture or
 * cuOptB200SolveDistributed.  INTEGRATION.md "presolve". */
#define CUOPT_B200_PRESOLVE "presolve"

typedef struct cuOptB200PresolveStats {
  cuopt_int_t ran; /* 1 when the solve was presolved */
  cuopt_int_t original_m, original_n, original_nnz;
  cuopt_int_t reduced_m, reduced_n, reduced_nnz; /* stored zeros are dropped from the reduced matrix */
  cuopt_int_t fixed_columns, empty_rows, singleton_rows, empty_columns; /* removed by each rule */
  cuopt_int_t rounds;
  cuopt_float_t presolve_seconds, postsolve_seconds; /* device time */
} cuOptB200PresolveStats;

/* Presolve statistics of a solution (all zero when presolve was off). */
cuopt_int_t cuOptB200GetPresolveStats(cuOptSolution solution, cuOptB200PresolveStats* stats);

/* ---- solver session: the same solver cuOptSolve runs, driven step by step -------------------- */
typedef void* cuOptB200Solver;

typedef struct cuOptB200KernelProfile {
  cuopt_float_t ms_primal_step, ms_dual_step, ms_transpose_step; /* mean device time per launch */
  cuopt_float_t bytes_primal_step, bytes_dual_step, bytes_transpose_step; /* algorithmic bytes per launch */
  cuopt_float_t ms_iteration; /* mean per attempt, all three kernels back to back */
  cuopt_int_t reps;
  cuopt_int_t grid_primal, grid_dual, grid_transpose;
  /* the payload-free partial transpose product of the sharded solve (k_transpose_partial) on this problem's A^T:
   * blocks of <= 32 rows, and the wide schedule (<= 256 rows; 0 when A^T has >= 4 nonzeros per row on average) */
  cuopt_float_t ms_transpose_partial, ms_transpose_partial_wide;
  /* gather blocking: > 1 means the "dual" / "transpose" step is that many k_block_pass launches + one element-wise
   * epilogue instead of the single fused kernel (their times above are those of the whole group) */
  cuopt_int_t blocks_dual, blocks_transpose;
} cuOptB200KernelProfile;

/* Upload the problem to the current CUDA device (A, A^T, row-block schedules). */
cuopt_int_t cuOptB200SolverCreate(cuOptOptimizationProblem problem,
                                  cuOptSolverSettings settings,
                                  cuOptB200Solver* solver_ptr);
void cuOptB200SolverDestroy(cuOptB200Solver* solver_ptr);
/* Diagonal scaling + initial step size / primal weight (what cuOptSolve does before iterating). */
cuopt_int_t cuOptB200SolverInitialise(cuOptB200Solver solver);
/* Run the outer loop for `accepted_steps` more accepted PDLP iterations (<0: to termination).
 * *finished_ptr = 1 once a termination status was reached. */
cuopt_int_t cuOptB200SolverAdvance(cuOptB200Solver solver, cuopt_int_t accepted_steps, cuopt_int_t* finished_ptr);
/* Named state: scalars "step_size", "primal_weight", "tau", "sigma", "sum_w", "k_total", "k_pdhg",
 * "its_since_restart", "interaction", "norm_dx2", "norm_dy2", "l2_norm_b", "l2_norm_c", "n_restarts";
 * launch geometry (read-only): "sm_count", "occ_spmv" / "occ_spmv2" (resident CTAs per SM of the SpMV kernels with one /
 * two payload row groups), "grid_k1", "grid_k2", "grid_k3" (CTAs of the primal step and of the fused K2 / K3 as they
 * launch: on the last column block when gather blocking is on), "grid_n", "grid_m" (element-wise grids), "k2_npre"
 * (payload row groups of the fused K2), "n_std_a", "n_blk_a", "n_std_at", "n_blk_at" (interleaved blocks and all
 * blocks, long rows included, of the scaled A and A^T), "staged_fills" (pinned staging-ring slots filled while this
 * session uploaded its arrays; 0 when every array took the plain copy.  The ring is shared by the device: sessions built
 * at the same time on the same device count each other's fills too), "device_cache_hits" (device allocations served
 * from the block cache so far in this process, by any session);
 * vectors "x", "y", "aty", "x_next", "y_next", "aty_next", "x_bar", "sum_x", "sum_y", "x_avg", "y_avg",
 * "row_scaling", "col_scaling", "scaled_values", "scaled_values_t", "scaled_c", "scaled_l", "scaled_u",
 * "scaled_lc", "scaled_uc", "x_last_restart", "y_last_restart" (scaled space unless noted).
 * Presolved sessions: the vectors above are of the reduced problem; "presolve_row_map", "presolve_col_map" (original
 * index of each kept row / column), "presolve_c", "presolve_l", "presolve_u", "presolve_lc", "presolve_uc" (the reduced
 * problem, unscaled, in minimisation form: c negated when maximising) and the scalar "presolve_offset" (objective of the
 * removed columns, same form).  cuOptB200SolverGetSolution returns the postsolved solution. */
cuopt_int_t cuOptB200SolverGetScalar(cuOptB200Solver solver, const char* name, cuopt_float_t* value_ptr);
cuopt_int_t cuOptB200SolverGetVector(cuOptB200Solver solver,
                                     const char* name,
                                     cuopt_float_t* values,
                                     cuopt_int_t capacity,
                                     cuopt_int_t* size_ptr);
/* Read-only: lower / upper bound of the trust-region restart of Methodical1 (bound_optimal_objective) at a point of
 * the SCALED space (px: num_variables values, py: num_constraints values) for a radius >= 0, from the same kernels the
 * restart runs.  The session must be initialised with pdlp_solver_mode Methodical1; its iterates, restart state and
 * statistics are not changed. */
cuopt_int_t cuOptB200SolverTrustRegionBounds(cuOptB200Solver solver,
                                             const cuopt_float_t* px,
                                             const cuopt_float_t* py,
                                             cuopt_float_t radius,
                                             cuopt_float_t* lower_ptr,
                                             cuopt_float_t* upper_ptr);
/* Read-only: the infeasibility-detection statistics of the termination check at a caller-given current point (x_cur,
 * y_cur) and average point (x_avg, y_avg), from the products and kernels the evaluation runs.  The points are in the space
 * the evaluation works in: unscaled, minimisation form (c negated when maximising), and of the reduced problem in a
 * presolved session (x: num_variables values, y: num_constraints values).  stats receives 12 values per iterate, current
 * first: max |x|, max bound violation of the ray, max homogeneous row violation, c.x, max |y|, max |reduced cost|, dual
 * residual and dual-ray objective as summed, primal-ray objective c.x / max |x|, max primal residual / max |x|, and the
 * dual residual and dual-ray objective divided by max(max |y|, max |reduced cost|); status receives the verdict of each
 * iterate as the solve would draw it (2 PrimalInfeasible, 3 DualInfeasible, 6 none) under the session's
 * primal_infeasible_tolerance, dual_infeasible_tolerance and reduced-cost rule.  Works whether or not
 * infeasibility_detection is set; refused with CUOPT_INVALID_ARGUMENT before cuOptB200SolverInitialise and in multi-GPU
 * sessions.  The iterates, the statistics and the launch count of the session are not changed. */
cuopt_int_t cuOptB200SolverInfeasibilityStats(cuOptB200Solver solver,
                                              const cuopt_float_t* x_cur,
                                              const cuopt_float_t* y_cur,
                                              const cuopt_float_t* x_avg,
                                              const cuopt_float_t* y_avg,
                                              cuopt_float_t* stats,
                                              cuopt_int_t* status);
/* Solution object (same type cuOptSolve returns) of a finished session. */
cuopt_int_t cuOptB200SolverGetSolution(cuOptB200Solver solver, cuOptSolution* solution_ptr);
/* Time the three PDHG kernels in situ (CUDA events on the solver's stream) after `warmup_steps`. */
cuopt_int_t cuOptB200SolverProfileKernels(cuOptB200Solver solver,
                                          cuopt_int_t warmup_steps,
                                          cuopt_int_t reps,
                                          cuOptB200KernelProfile* profile);

/* ---- multi-GPU (one process per GPU, rows of A sharded over the ranks; SURVEY.md 8(e)) ---------------------
 * The reference cannot use several GPUs for one LP (docs/cuopt/source/faq.rst:53); this is new functionality.
 * Bootstrap: rank 0 calls cuOptB200DistGetUniqueId and broadcasts the 128 bytes by any means (torch.distributed,
 * MPI, a file); every rank then calls cuOptB200DistInit on its own CUDA device.
 * cuOptB200SolveDistributed is collective: each rank passes a problem holding ITS contiguous block of constraint
 * rows (all columns, global column indices; objective, variable bounds and types replicated).  Every rank gets the
 * full primal solution and reduced costs; the dual solution returned is the rank's own block of rows. */
typedef void* cuOptB200Dist;
cuopt_int_t cuOptB200DistGetUniqueId(char* unique_id_128_bytes);
cuopt_int_t cuOptB200DistInit(cuopt_int_t rank, cuopt_int_t world_size, const char* unique_id_128_bytes, cuOptB200Dist* dist_ptr);
void cuOptB200DistDestroy(cuOptB200Dist* dist_ptr);
cuopt_int_t cuOptB200SolveDistributed(cuOptOptimizationProblem local_rows_problem,
                                      cuOptSolverSettings settings,
                                      cuOptB200Dist dist,
                                      cuOptSolution* solution_ptr);

/* ---- Warm start across solves --------------------------------------------------------------------------------
 * The reference exposes pdlp_warm_start_data_t only through C++/Python
 * (cpp/include/cuopt/linear_programming/pdlp/pdlp_warm_start_data.hpp:28-72, solver_settings.cu set_pdlp_warm_start_data,
 * solver_solution.hpp get_pdlp_warm_start_data); these entry points carry it through the C ABI.
 *   cuOptB200SetWarmStartCapture(settings, 1);  cuOptSolve(...);            // the solution now carries the state
 *   cuOptB200GetWarmStart(solution, &ws);       cuOptB200SetWarmStart(settings2, ws);   cuOptSolve(...);
 * Vector names: current_primal_solution, current_dual_solution, initial_primal_average, initial_dual_average,
 * current_ATY, sum_primal_solutions, sum_dual_solutions, last_restart_duality_gap_primal_solution,
 * last_restart_duality_gap_dual_solution.  Scalar names: initial_primal_weight, initial_step_size,
 * total_pdlp_iterations, total_pdhg_iterations, last_candidate_kkt_score, last_restart_kkt_score,
 * sum_solution_weight, iterations_since_last_restart.  The same scaling (same problem, same pdlp_solver_mode) is
 * assumed, as in the reference. */
typedef void* cuOptB200WarmStart;
cuopt_int_t cuOptB200SetWarmStartCapture(cuOptSolverSettings settings, cuopt_int_t enable);
/* new handle sharing the solution's state; CUOPT_INVALID_ARGUMENT when the solve did not capture it */
cuopt_int_t cuOptB200GetWarmStart(cuOptSolution solution, cuOptB200WarmStart* warm_start_ptr);
/* the settings keep a reference (the handle may be destroyed afterwards); NULL clears */
cuopt_int_t cuOptB200SetWarmStart(cuOptSolverSettings settings, cuOptB200WarmStart warm_start);
/* from raw host arrays: 9 vectors in the order listed above (primal-sized ones hold num_variables values, dual-sized
 * ones num_constraints), 8 scalars in the order listed above */
cuopt_int_t cuOptB200CreateWarmStart(cuopt_int_t num_constraints,
                                     cuopt_int_t num_variables,
                                     const cuopt_float_t* const* vectors_9,
                                     const cuopt_float_t* scalars_8,
                                     cuOptB200WarmStart* warm_start_ptr);
void cuOptB200DestroyWarmStart(cuOptB200WarmStart* warm_start_ptr);
cuopt_int_t cuOptB200WarmStartGetScalar(cuOptB200WarmStart warm_start, const char* name, cuopt_float_t* value_ptr);
/* values == NULL: only *size_ptr is written */
cuopt_int_t cuOptB200WarmStartGetVector(cuOptB200WarmStart warm_start,
                                        const char* name,
                                        cuopt_float_t* values,
                                        cuopt_int_t* size_ptr);

/* cuOptReadProblem with an explicit format switch (the reference C ABI always parses free format;
 * its C++ parse_mps(file, fixed_mps_format) has the flag: cpp/libmps_parser/include/mps_parser/parser.hpp:33). */
cuopt_int_t cuOptB200ReadProblem(const char* filename, cuopt_int_t fixed_format, cuOptOptimizationProblem* problem_ptr);

/* Library identification: "cuopt-b200 <version> sm_90a". */
const char* cuOptB200Version(void);

#ifdef __cplusplus
}
#endif

#endif /* CUOPT_B200_EXT_H */
