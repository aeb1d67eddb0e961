/*
 * Drop-in ABI constants for the libcuopt LP C interface (H100-native PDLP build).
 *
 * The numeric values and parameter-name strings below are the wire contract of
 * the reference header cpp/include/cuopt/linear_programming/constants.h:26-113
 * (NVIDIA/cuopt 25.08): a caller compiled against the reference header links
 * and runs against this library unchanged.  Only the LP path is implemented;
 * MIP-only parameters are accepted and stored so that client code that sets
 * them keeps working, but have no effect (see INTEGRATION.md).
 */
#ifndef CUOPT_CONSTANTS_H
#define CUOPT_CONSTANTS_H

#ifdef __cplusplus
#include <limits>
#else
#include <math.h>
#endif

/* Instantiated scalar types: cuopt_float_t = double, cuopt_int_t = int32_t. */
#define CUOPT_INSTANTIATE_FLOAT  0
#define CUOPT_INSTANTIATE_DOUBLE 1
#define CUOPT_INSTANTIATE_INT32  1
#define CUOPT_INSTANTIATE_INT64  0

/* Parameter names understood by cuOptSet*Parameter / cuOptGet*Parameter. */
#define CUOPT_ABSOLUTE_DUAL_TOLERANCE     "absolute_dual_tolerance"
#define CUOPT_RELATIVE_DUAL_TOLERANCE     "relative_dual_tolerance"
#define CUOPT_ABSOLUTE_PRIMAL_TOLERANCE   "absolute_primal_tolerance"
#define CUOPT_RELATIVE_PRIMAL_TOLERANCE   "relative_primal_tolerance"
#define CUOPT_ABSOLUTE_GAP_TOLERANCE      "absolute_gap_tolerance"
#define CUOPT_RELATIVE_GAP_TOLERANCE      "relative_gap_tolerance"
#define CUOPT_INFEASIBILITY_DETECTION     "infeasibility_detection"
#define CUOPT_STRICT_INFEASIBILITY        "strict_infeasibility"
#define CUOPT_PRIMAL_INFEASIBLE_TOLERANCE "primal_infeasible_tolerance"
#define CUOPT_DUAL_INFEASIBLE_TOLERANCE   "dual_infeasible_tolerance"
#define CUOPT_ITERATION_LIMIT             "iteration_limit"
#define CUOPT_TIME_LIMIT                  "time_limit"
#define CUOPT_PDLP_SOLVER_MODE            "pdlp_solver_mode"
#define CUOPT_METHOD                      "method"
#define CUOPT_PER_CONSTRAINT_RESIDUAL     "per_constraint_residual"
#define CUOPT_SAVE_BEST_PRIMAL_SO_FAR     "save_best_primal_so_far"
#define CUOPT_FIRST_PRIMAL_FEASIBLE       "first_primal_feasible"
#define CUOPT_LOG_FILE                    "log_file"
#define CUOPT_LOG_TO_CONSOLE              "log_to_console"
#define CUOPT_CROSSOVER                   "crossover"
#define CUOPT_MIP_ABSOLUTE_TOLERANCE      "mip_absolute_tolerance"
#define CUOPT_MIP_RELATIVE_TOLERANCE      "mip_relative_tolerance"
#define CUOPT_MIP_INTEGRALITY_TOLERANCE   "mip_integrality_tolerance"
#define CUOPT_MIP_ABSOLUTE_GAP            "mip_absolute_gap"
#define CUOPT_MIP_RELATIVE_GAP            "mip_relative_gap"
#define CUOPT_MIP_HEURISTICS_ONLY         "mip_heuristics_only"
#define CUOPT_MIP_SCALING                 "mip_scaling"
#define CUOPT_SOLUTION_FILE               "solution_file"
#define CUOPT_NUM_CPU_THREADS             "num_cpu_threads"
#define CUOPT_USER_PROBLEM_FILE           "user_problem_file"

/* Termination status codes (spelling "TERIMINATION" is part of the reference ABI). */
#define CUOPT_TERIMINATION_STATUS_NO_TERMINATION   0
#define CUOPT_TERIMINATION_STATUS_OPTIMAL          1
#define CUOPT_TERIMINATION_STATUS_INFEASIBLE       2
#define CUOPT_TERIMINATION_STATUS_UNBOUNDED        3
#define CUOPT_TERIMINATION_STATUS_ITERATION_LIMIT  4
#define CUOPT_TERIMINATION_STATUS_TIME_LIMIT       5
#define CUOPT_TERIMINATION_STATUS_NUMERICAL_ERROR  6
#define CUOPT_TERIMINATION_STATUS_PRIMAL_FEASIBLE  7
#define CUOPT_TERIMINATION_STATUS_FEASIBLE_FOUND   8
#define CUOPT_TERIMINATION_STATUS_CONCURRENT_LIMIT 9

/* Objective sense. */
#define CUOPT_MINIMIZE 1
#define CUOPT_MAXIMIZE -1

/* Constraint sense characters. */
#define CUOPT_LESS_THAN    'L'
#define CUOPT_GREATER_THAN 'G'
#define CUOPT_EQUAL        'E'

/* Variable type characters. */
#define CUOPT_CONTINUOUS 'C'
#define CUOPT_INTEGER    'I'

/* +infinity for bounds. */
#ifdef __cplusplus
#define CUOPT_INFINITY std::numeric_limits<double>::infinity()
#else
#define CUOPT_INFINITY INFINITY
#endif

/* pdlp_solver_mode values. */
#define CUOPT_PDLP_SOLVER_MODE_STABLE1     0
#define CUOPT_PDLP_SOLVER_MODE_STABLE2     1
#define CUOPT_PDLP_SOLVER_MODE_METHODICAL1 2
#define CUOPT_PDLP_SOLVER_MODE_FAST1       3

/* method values. */
#define CUOPT_METHOD_CONCURRENT   0
#define CUOPT_METHOD_PDLP         1
#define CUOPT_METHOD_DUAL_SIMPLEX 2

/* Return / error status codes. */
#define CUOPT_SUCCESS          0
#define CUOPT_INVALID_ARGUMENT 1
#define CUOPT_MPS_FILE_ERROR   2
#define CUOPT_MPS_PARSE_ERROR  3
#define CUOPT_VALIDATION_ERROR 4
#define CUOPT_OUT_OF_MEMORY    5
#define CUOPT_RUNTIME_ERROR    6

#endif /* CUOPT_CONSTANTS_H */
