/*
 * libcuopt LP C interface — H100-native (sm_90a) PDLP build.
 *
 * This header declares, with identical names, argument order, scalar types and
 * status codes, the 41 entry points of the reference C API
 * (NVIDIA/cuopt 25.08, cpp/include/cuopt/linear_programming/cuopt_c.h; the
 * `ref:` tag on each declaration gives the line it replaces, implementation
 * semantics follow cpp/src/linear_programming/cuopt_c.cpp).  A client built
 * against the reference header can be relinked against this library.
 *
 * Scope: LP only, solved by PDLP on one (or, through the cuopt_b200_ext.h
 * extension, several) H100 GPUs.  A problem that declares integer variables
 * is reported by cuOptIsMIP, and cuOptSolve answers it with an error solution
 * (CUOPT_VALIDATION_ERROR) instead of running a MIP search.
 *
 * Conventions (same as the reference):
 *   - every array argument is copied at call time; the caller keeps ownership
 *   - handles are opaque heap objects, released by the matching Destroy call,
 *     which also nulls the caller's handle
 *   - functions return CUOPT_SUCCESS or one of the CUOPT_* error codes; no
 *     C++ exception crosses this boundary
 *   - array pointers may be HOST or DEVICE / managed pointers on either side
 *     (inputs of the Create calls, destinations of the getters), like the
 *     reference's raft::copy-based C layer (cuopt_c.cpp:110-135, :261-266)
 */
#ifndef CUOPT_C_API_H
#define CUOPT_C_API_H

#include <cuopt/linear_programming/constants.h>

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* cuOptOptimizationProblem; /* ref: cuopt_c.h:31-35 */
typedef void* cuOptSolverSettings;      /* ref: cuopt_c.h:37-40 */
typedef void* cuOptSolution;            /* ref: cuopt_c.h:42-45 */

#if CUOPT_INSTANTIATE_FLOAT
typedef float cuopt_float_t;
#endif
#if CUOPT_INSTANTIATE_DOUBLE
typedef double cuopt_float_t; /* ref: cuopt_c.h:50-66 */
#endif
#if CUOPT_INSTANTIATE_INT32
typedef int32_t cuopt_int_t; /* ref: cuopt_c.h:68-82 */
#endif
#if CUOPT_INSTANTIATE_INT64
typedef int64_t cuopt_int_t;
#endif

/* sizeof(cuopt_float_t) == 8.  ref: cuopt_c.h:89 */
int8_t cuOptGetFloatSize();
/* sizeof(cuopt_int_t) == 4.  ref: cuopt_c.h:94 */
int8_t cuOptGetIntSize();

/* Parse an MPS file (free format; fixed-format files that are also valid free
 * format are accepted) into a new problem.  CUOPT_MPS_FILE_ERROR if the file
 * cannot be opened, CUOPT_MPS_PARSE_ERROR if it is malformed; *problem_ptr is
 * NULL on failure.  ref: cuopt_c.h:106, cuopt_c.cpp:62-86 */
cuopt_int_t cuOptReadProblem(const char* filename, cuOptOptimizationProblem* problem_ptr);

/* Build a problem  min/max c'x + offset  s.t.  A x {<=,>=,=} rhs,  lb <= x <= ub
 * from a CSR matrix and per-row sense characters ('L','G','E').
 * objective_sense: CUOPT_MINIMIZE or CUOPT_MAXIMIZE; variable_types: 'C'/'I'.
 * Any NULL pointer -> CUOPT_INVALID_ARGUMENT.  ref: cuopt_c.h:151-164 */
cuopt_int_t cuOptCreateProblem(cuopt_int_t num_constraints,
                               cuopt_int_t num_variables,
                               cuopt_int_t objective_sense,
                               cuopt_float_t objective_offset,
                               const cuopt_float_t* objective_coefficients,
                               const cuopt_int_t* constraint_matrix_row_offsets,
                               const cuopt_int_t* constraint_matrix_column_indices,
                               const cuopt_float_t* constraint_matrix_coefficent_values,
                               const char* constraint_sense,
                               const cuopt_float_t* rhs,
                               const cuopt_float_t* lower_bounds,
                               const cuopt_float_t* upper_bounds,
                               const char* variable_types,
                               cuOptOptimizationProblem* problem_ptr);

/* Same, with two-sided rows  constraint_lower_bounds <= A x <= constraint_upper_bounds
 * (use +-CUOPT_INFINITY for one-sided rows).  ref: cuopt_c.h:220-233 */
cuopt_int_t cuOptCreateRangedProblem(cuopt_int_t num_constraints,
                                     cuopt_int_t num_variables,
                                     cuopt_int_t objective_sense,
                                     cuopt_float_t objective_offset,
                                     const cuopt_float_t* objective_coefficients,
                                     const cuopt_int_t* constraint_matrix_row_offsets,
                                     const cuopt_int_t* constraint_matrix_column_indices,
                                     const cuopt_float_t* constraint_matrix_coefficients,
                                     const cuopt_float_t* constraint_lower_bounds,
                                     const cuopt_float_t* constraint_upper_bounds,
                                     const cuopt_float_t* variable_lower_bounds,
                                     const cuopt_float_t* variable_upper_bounds,
                                     const char* variable_types,
                                     cuOptOptimizationProblem* problem_ptr);

/* Free a problem and set *problem_ptr = NULL.  ref: cuopt_c.h:240 */
void cuOptDestroyProblem(cuOptOptimizationProblem* problem_ptr);

/* Problem getters: each copies into caller storage sized from the dimension
 * getters.  ref: cuopt_c.h:251-418 */
cuopt_int_t cuOptGetNumConstraints(cuOptOptimizationProblem problem,
                                   cuopt_int_t* num_constraints_ptr);                      /* ref: 251 */
cuopt_int_t cuOptGetNumVariables(cuOptOptimizationProblem problem,
                                 cuopt_int_t* num_variables_ptr);                          /* ref: 263 */
cuopt_int_t cuOptGetObjectiveSense(cuOptOptimizationProblem problem,
                                   cuopt_int_t* objective_sense_ptr);                      /* ref: 274 */
cuopt_int_t cuOptGetObjectiveOffset(cuOptOptimizationProblem problem,
                                    cuopt_float_t* objective_offset_ptr);                  /* ref: 286 */
cuopt_int_t cuOptGetObjectiveCoefficients(cuOptOptimizationProblem problem,
                                          cuopt_float_t* objective_coefficients_ptr);      /* ref: 299 */
cuopt_int_t cuOptGetNumNonZeros(cuOptOptimizationProblem problem,
                                cuopt_int_t* num_non_zeros_ptr);                           /* ref: 312 */
cuopt_int_t cuOptGetConstraintMatrix(cuOptOptimizationProblem problem,
                                     cuopt_int_t* constraint_matrix_row_offsets_ptr,
                                     cuopt_int_t* constraint_matrix_column_indices_ptr,
                                     cuopt_float_t* constraint_matrix_coefficients_ptr);   /* ref: 332 */
cuopt_int_t cuOptGetConstraintSense(cuOptOptimizationProblem problem,
                                    char* constraint_sense_ptr);                           /* ref: 346 */
cuopt_int_t cuOptGetConstraintRightHandSide(cuOptOptimizationProblem problem,
                                            cuopt_float_t* rhs_ptr);                       /* ref: 357 */
cuopt_int_t cuOptGetConstraintLowerBounds(cuOptOptimizationProblem problem,
                                          cuopt_float_t* lower_bounds_ptr);                /* ref: 369 */
cuopt_int_t cuOptGetConstraintUpperBounds(cuOptOptimizationProblem problem,
                                          cuopt_float_t* upper_bounds_ptr);                /* ref: 381 */
cuopt_int_t cuOptGetVariableLowerBounds(cuOptOptimizationProblem problem,
                                        cuopt_float_t* lower_bounds_ptr);                  /* ref: 393 */
cuopt_int_t cuOptGetVariableUpperBounds(cuOptOptimizationProblem problem,
                                        cuopt_float_t* upper_bounds_ptr);                  /* ref: 405 */
cuopt_int_t cuOptGetVariableTypes(cuOptOptimizationProblem problem,
                                  char* variable_types_ptr);                               /* ref: 418 */

/* Settings object with the reference's defaults (all six tolerances 1e-4,
 * pdlp_solver_mode Stable2, method Concurrent, no limits).
 * ref: cuopt_c.h:427-434, math_optimization/solver_settings.cu:63-125 */
cuopt_int_t cuOptCreateSolverSettings(cuOptSolverSettings* settings_ptr);
void cuOptDestroySolverSettings(cuOptSolverSettings* settings_ptr);

/* Parameter access by name (names in constants.h).  Unknown name, unparsable
 * or out-of-range value -> CUOPT_INVALID_ARGUMENT.  The integer setter/getter
 * also reaches boolean parameters.  ref: cuopt_c.h:444-522 */
cuopt_int_t cuOptSetParameter(cuOptSolverSettings settings,
                              const char* parameter_name,
                              const char* parameter_value);
cuopt_int_t cuOptGetParameter(cuOptSolverSettings settings,
                              const char* parameter_name,
                              cuopt_int_t parameter_value_size,
                              char* parameter_value);
cuopt_int_t cuOptSetIntegerParameter(cuOptSolverSettings settings,
                                     const char* parameter_name,
                                     cuopt_int_t parameter_value);
cuopt_int_t cuOptGetIntegerParameter(cuOptSolverSettings settings,
                                     const char* parameter_name,
                                     cuopt_int_t* parameter_value);
cuopt_int_t cuOptSetFloatParameter(cuOptSolverSettings settings,
                                   const char* parameter_name,
                                   cuopt_float_t parameter_value);
cuopt_int_t cuOptGetFloatParameter(cuOptSolverSettings settings,
                                   const char* parameter_name,
                                   cuopt_float_t* parameter_value);

/* *is_mip_ptr = 1 if any variable is integer.  ref: cuopt_c.h:533 */
cuopt_int_t cuOptIsMIP(cuOptOptimizationProblem problem, cuopt_int_t* is_mip_ptr);

/* Solve.  Always allocates *solution_ptr (also on failure, so the error string
 * can be read); the return value is the solution's ERROR status, not its
 * termination status.  Blocking.  ref: cuopt_c.h:546, cuopt_c.cpp:580-620 */
cuopt_int_t cuOptSolve(cuOptOptimizationProblem problem,
                       cuOptSolverSettings settings,
                       cuOptSolution* solution_ptr);

/* Free a solution and set *solution_ptr = NULL.  ref: cuopt_c.h:555 */
void cuOptDestroySolution(cuOptSolution* solution_ptr);

/* Solution getters.  ref: cuopt_c.h:566-668 */
cuopt_int_t cuOptGetTerminationStatus(cuOptSolution solution,
                                      cuopt_int_t* termination_status_ptr);   /* ref: 566 */
cuopt_int_t cuOptGetErrorStatus(cuOptSolution solution,
                                cuopt_int_t* error_status_ptr);               /* ref: 577 */
cuopt_int_t cuOptGetErrorString(cuOptSolution solution,
                                char* error_string_ptr,
                                cuopt_int_t error_string_size);               /* ref: 590 */
cuopt_int_t cuOptGetPrimalSolution(cuOptSolution solution,
                                   cuopt_float_t* solution_values);           /* ref: 603 */
cuopt_int_t cuOptGetObjectiveValue(cuOptSolution solution,
                                   cuopt_float_t* objective_value_ptr);       /* ref: 614 */
cuopt_int_t cuOptGetSolveTime(cuOptSolution solution,
                              cuopt_float_t* solve_time_ptr);                 /* ref: 624 */
/* MIP-only: return CUOPT_INVALID_ARGUMENT for LP solutions (as the reference does). */
cuopt_int_t cuOptGetMIPGap(cuOptSolution solution, cuopt_float_t* mip_gap_ptr);               /* ref: 635 */
cuopt_int_t cuOptGetSolutionBound(cuOptSolution solution, cuopt_float_t* solution_bound_ptr); /* ref: 646 */
/* LP-only. */
cuopt_int_t cuOptGetDualSolution(cuOptSolution solution,
                                 cuopt_float_t* dual_solution_ptr);           /* ref: 657 */
cuopt_int_t cuOptGetReducedCosts(cuOptSolution solution,
                                 cuopt_float_t* reduced_cost_ptr);            /* ref: 668 */

#ifdef __cplusplus
}
#endif

#endif /* CUOPT_C_API_H */
