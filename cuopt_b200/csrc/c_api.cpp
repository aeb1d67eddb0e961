// extern "C" boundary: the 41 reference symbols of cuopt_c.h plus the cuOptB200* extension.
// Semantics follow cpp/src/linear_programming/cuopt_c.cpp of the reference (line tags below).
#include <cuopt_b200/cuopt_b200_ext.h>

#include "dist_comm.hpp"
#include "lp_problem.hpp"
#include "pdlp_solver.hpp"
#include "solver_settings.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>

using namespace cuopt_b200;

namespace cuopt_b200 {
bool write_problem_as_mps(const lp_problem_t& p, const std::string& path);  // file_writers.cpp
bool write_solution_file(const lp_problem_t& p, const lp_solution_t& s, const std::string& path);
}  // namespace cuopt_b200

namespace {

struct solution_handle_t {
  lp_solution_t sol;
  bool is_mip = false;
};

struct solver_handle_t {
  std::unique_ptr<pdlp_solver_t> solver;
  bool finished = false;
};

// The reference's C layer moves every array with raft::copy, which takes host or device pointers on either side
// (cuopt_c.cpp:110-135 for the inputs, :261-266 for the getters).  Same here: a pointer the CUDA runtime knows as device or
// managed memory is copied with cudaMemcpy, anything else (also: no driver on this host) is plain host memory.
bool is_device_pointer(const void* p)
{
  if (p == nullptr) return false;
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
template <typename T, typename A>
void copy_out(T* dst, const std::vector<T, A>& src)
{
  if (src.empty()) return;
  if (is_device_pointer(dst)) {  // getters have no error channel beyond their status: a failed copy leaves dst untouched
    if (cudaMemcpy(dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) cudaGetLastError();
    return;
  }
  std::memcpy(dst, src.data(), src.size() * sizeof(T));
}
template <typename T>
void copy_in(hvec<T>& dst, const T* src, size_t n)
{
  if (n > 0 && is_device_pointer(src)) {
    dst.resize(n);
    if (cudaMemcpy(dst.data(), src, n * sizeof(T), cudaMemcpyDeviceToHost) != cudaSuccess)
      throw lp_error(error_type_t::RuntimeError, "copy from a device buffer failed");
    return;
  }
  parallel_assign(dst, src, n);
}
void copy_in(std::vector<char>& dst, const char* src, size_t n)
{
  dst.resize(n);
  if (n > 0 && is_device_pointer(src)) {
    if (cudaMemcpy(dst.data(), src, n, cudaMemcpyDeviceToHost) != cudaSuccess)
      throw lp_error(error_type_t::RuntimeError, "copy from a device buffer failed");
    return;
  }
  if (n > 0) std::memcpy(dst.data(), src, n);
}

cuopt_int_t fill_problem_common(lp_problem_t& p,
                                cuopt_int_t m,
                                cuopt_int_t n,
                                cuopt_int_t sense,
                                cuopt_float_t offset,
                                const cuopt_float_t* c,
                                const cuopt_int_t* off,
                                const cuopt_int_t* idx,
                                const cuopt_float_t* val,
                                const cuopt_float_t* lb,
                                const cuopt_float_t* ub,
                                const char* types)
{
  if (m < 0 || n < 0) return CUOPT_INVALID_ARGUMENT;
  p.n_constraints    = m;
  p.n_variables      = n;
  p.maximize         = (sense == CUOPT_MAXIMIZE);
  p.objective_offset = offset;
  copy_in(p.objective_coefficients, c, (size_t)n);
  copy_in(p.A_offsets, off, (size_t)m + 1);
  const cuopt_int_t nnz = p.A_offsets[m];
  if (nnz < 0) return CUOPT_INVALID_ARGUMENT;
  copy_in(p.A_indices, idx, (size_t)nnz);
  copy_in(p.A_values, val, (size_t)nnz);
  copy_in(p.variable_lower_bounds, lb, (size_t)n);
  copy_in(p.variable_upper_bounds, ub, (size_t)n);
  copy_in(p.variable_types, types, (size_t)n);
  for (int j = 0; j < n; ++j) p.variable_types[j] = p.variable_types[j] == CUOPT_CONTINUOUS ? 'C' : 'I';  // cuopt_c.cpp:127-131
  return CUOPT_SUCCESS;
}

// reference log line formats: pdlp.cu:1078-1080, termination_strategy.cu:380-390, solve.cu:376-380
void log_solution(const pdlp_settings_t& st, const lp_problem_t& p, const lp_solution_t& s)
{
  auto emit = [&](FILE* f) {
    std::fprintf(f, "Solving a problem with %d constraints %d variables (%d integers) and %d nonzeros\n", p.n_constraints,
                 p.n_variables, 0, p.nnz());
    if (s.stats.method_stand_in == 1)
      std::fprintf(f, "method Concurrent: this build has no CPU simplex to race, PDLP runs alone\n");
    if (s.stats.method_stand_in == 2)
      std::fprintf(f, "method DualSimplex: this build has no CPU simplex; PDLP stands in with strict infeasibility detection "
                      "and tolerances tightened to <= 1e-8\n");
    if (s.presolve.ran)
      std::fprintf(f, "Presolve: %d rows, %d columns, %d nonzeros remain of %d, %d, %d (%d fixed columns, %d empty rows, "
                      "%d singleton rows, %d empty columns; %d rounds, %.3f ms)\n", s.presolve.reduced_m, s.presolve.reduced_n,
                   s.presolve.reduced_nnz, s.presolve.original_m, s.presolve.original_n, s.presolve.original_nnz,
                   s.presolve.fixed_columns, s.presolve.empty_rows, s.presolve.singleton_rows, s.presolve.empty_columns,
                   s.presolve.rounds, 1e3 * s.presolve.presolve_seconds);
    std::fprintf(f, "   Iter    Primal Obj.      Dual Obj.    Gap        Primal Res.  Dual Res.   Time\n");
    std::fprintf(f, "%7d %+.8e %+.8e  %8.2e   %8.2e     %8.2e   %.3fs\n", s.stats.number_of_steps_taken,
                 s.stats.primal_objective, s.stats.dual_objective, s.stats.gap, s.stats.l2_primal_residual,
                 s.stats.l2_dual_residual, s.stats.solve_time);
    std::fprintf(f, "PDLP finished\n");
    std::fprintf(f, "Status: %s   Objective: %.8e  Iterations: %d  Time: %.3fs\n",
                 termination_status_string(s.termination_status), s.stats.primal_objective,
                 s.stats.number_of_steps_taken, s.stats.solve_time);
  };
  if (st.log_to_console) emit(stdout);
  if (!st.log_file.empty()) {
    if (FILE* f = std::fopen(st.log_file.c_str(), "w")) {
      emit(f);
      std::fclose(f);
    }
  }
}

// Maps anything thrown on the host side of a solve to an error solution: no C++ exception crosses the C boundary.
template <typename F>
void guarded(lp_solution_t& sol, F&& body)
{
  try {
    body();
  } catch (const std::bad_alloc&) {
    sol                = lp_solution_t{};
    sol.error_status   = CUOPT_OUT_OF_MEMORY;
    sol.error_message  = "Memory allocation failed";
  } catch (const std::exception& e) {
    sol                = lp_solution_t{};
    sol.error_status   = CUOPT_RUNTIME_ERROR;
    sol.error_message  = e.what();
  }
}

}  // namespace

extern "C" {

int8_t cuOptGetFloatSize() { return sizeof(cuopt_float_t); }
int8_t cuOptGetIntSize() { return sizeof(cuopt_int_t); }

cuopt_int_t cuOptReadProblem(const char* filename, cuOptOptimizationProblem* problem_ptr)  // cuopt_c.cpp:62-86
{
  if (filename == nullptr || problem_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  *problem_ptr = nullptr;
  try {
    auto* p      = new lp_problem_t(read_mps(filename, false));
    *problem_ptr = p;
    return CUOPT_SUCCESS;
  } catch (const lp_error& e) {
    return e.type == error_type_t::MpsFileError ? CUOPT_MPS_FILE_ERROR : CUOPT_MPS_PARSE_ERROR;
  } catch (const std::exception&) {
    return CUOPT_MPS_PARSE_ERROR;
  }
}

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
                               cuOptOptimizationProblem* problem_ptr)  // cuopt_c.cpp:88-141
{
  if (problem_ptr == nullptr || objective_coefficients == nullptr || constraint_matrix_row_offsets == nullptr ||
      constraint_matrix_column_indices == nullptr || constraint_matrix_coefficent_values == nullptr ||
      constraint_sense == nullptr || rhs == nullptr || lower_bounds == nullptr || upper_bounds == nullptr ||
      variable_types == nullptr)
    return CUOPT_INVALID_ARGUMENT;
  try {
    auto p = std::make_unique<lp_problem_t>();
    if (auto rc = fill_problem_common(*p, num_constraints, num_variables, objective_sense, objective_offset,
                                      objective_coefficients, constraint_matrix_row_offsets,
                                      constraint_matrix_column_indices, constraint_matrix_coefficent_values, lower_bounds,
                                      upper_bounds, variable_types))
      return rc;
    copy_in(p->row_types, constraint_sense, (size_t)num_constraints);
    copy_in(p->constraint_bounds, rhs, (size_t)num_constraints);
    *problem_ptr = p.release();
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}

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
                                     cuOptOptimizationProblem* problem_ptr)  // cuopt_c.cpp:143-198
{
  if (problem_ptr == nullptr || objective_coefficients == nullptr || constraint_matrix_row_offsets == nullptr ||
      constraint_matrix_column_indices == nullptr || constraint_matrix_coefficients == nullptr ||
      constraint_lower_bounds == nullptr || constraint_upper_bounds == nullptr || variable_lower_bounds == nullptr ||
      variable_upper_bounds == nullptr || variable_types == nullptr)
    return CUOPT_INVALID_ARGUMENT;
  try {
    auto p = std::make_unique<lp_problem_t>();
    if (auto rc = fill_problem_common(*p, num_constraints, num_variables, objective_sense, objective_offset,
                                      objective_coefficients, constraint_matrix_row_offsets,
                                      constraint_matrix_column_indices, constraint_matrix_coefficients,
                                      variable_lower_bounds, variable_upper_bounds, variable_types))
      return rc;
    copy_in(p->constraint_lower_bounds, constraint_lower_bounds, (size_t)num_constraints);
    copy_in(p->constraint_upper_bounds, constraint_upper_bounds, (size_t)num_constraints);
    *problem_ptr = p.release();
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}

void cuOptDestroyProblem(cuOptOptimizationProblem* problem_ptr)  // cuopt_c.cpp:200-206
{
  if (problem_ptr == nullptr || *problem_ptr == nullptr) return;
  delete static_cast<lp_problem_t*>(*problem_ptr);
  *problem_ptr = nullptr;
}

#define PROBLEM_OR_FAIL(out)                                             \
  if (problem == nullptr || (out) == nullptr) return CUOPT_INVALID_ARGUMENT; \
  const lp_problem_t& p = *static_cast<const lp_problem_t*>(problem)

cuopt_int_t cuOptGetNumConstraints(cuOptOptimizationProblem problem, cuopt_int_t* num_constraints_ptr)
{
  PROBLEM_OR_FAIL(num_constraints_ptr);
  *num_constraints_ptr = p.n_constraints;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetNumVariables(cuOptOptimizationProblem problem, cuopt_int_t* num_variables_ptr)
{
  PROBLEM_OR_FAIL(num_variables_ptr);
  *num_variables_ptr = p.n_variables;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetObjectiveSense(cuOptOptimizationProblem problem, cuopt_int_t* objective_sense_ptr)
{
  PROBLEM_OR_FAIL(objective_sense_ptr);
  *objective_sense_ptr = p.maximize ? CUOPT_MAXIMIZE : CUOPT_MINIMIZE;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetObjectiveOffset(cuOptOptimizationProblem problem, cuopt_float_t* objective_offset_ptr)
{
  PROBLEM_OR_FAIL(objective_offset_ptr);
  *objective_offset_ptr = p.objective_offset;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetObjectiveCoefficients(cuOptOptimizationProblem problem, cuopt_float_t* objective_coefficients_ptr)
{
  PROBLEM_OR_FAIL(objective_coefficients_ptr);
  copy_out(objective_coefficients_ptr, p.objective_coefficients);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetNumNonZeros(cuOptOptimizationProblem problem, cuopt_int_t* num_non_zeros_ptr)
{
  PROBLEM_OR_FAIL(num_non_zeros_ptr);
  *num_non_zeros_ptr = p.nnz();
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetConstraintMatrix(cuOptOptimizationProblem problem,
                                     cuopt_int_t* constraint_matrix_row_offsets_ptr,
                                     cuopt_int_t* constraint_matrix_column_indices_ptr,
                                     cuopt_float_t* constraint_matrix_coefficients_ptr)
{
  PROBLEM_OR_FAIL(constraint_matrix_row_offsets_ptr);
  if (constraint_matrix_column_indices_ptr == nullptr || constraint_matrix_coefficients_ptr == nullptr)
    return CUOPT_INVALID_ARGUMENT;
  copy_out(constraint_matrix_row_offsets_ptr, p.A_offsets);
  copy_out(constraint_matrix_column_indices_ptr, p.A_indices);
  copy_out(constraint_matrix_coefficients_ptr, p.A_values);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetConstraintSense(cuOptOptimizationProblem problem, char* constraint_sense_ptr)
{
  PROBLEM_OR_FAIL(constraint_sense_ptr);
  copy_out(constraint_sense_ptr, p.row_types);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetConstraintRightHandSide(cuOptOptimizationProblem problem, cuopt_float_t* rhs_ptr)
{
  PROBLEM_OR_FAIL(rhs_ptr);
  copy_out(rhs_ptr, p.constraint_bounds);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetConstraintLowerBounds(cuOptOptimizationProblem problem, cuopt_float_t* lower_bounds_ptr)
{
  PROBLEM_OR_FAIL(lower_bounds_ptr);
  copy_out(lower_bounds_ptr, p.constraint_lower_bounds);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetConstraintUpperBounds(cuOptOptimizationProblem problem, cuopt_float_t* upper_bounds_ptr)
{
  PROBLEM_OR_FAIL(upper_bounds_ptr);
  copy_out(upper_bounds_ptr, p.constraint_upper_bounds);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetVariableLowerBounds(cuOptOptimizationProblem problem, cuopt_float_t* lower_bounds_ptr)
{
  PROBLEM_OR_FAIL(lower_bounds_ptr);
  copy_out(lower_bounds_ptr, p.variable_lower_bounds);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetVariableUpperBounds(cuOptOptimizationProblem problem, cuopt_float_t* upper_bounds_ptr)
{
  PROBLEM_OR_FAIL(upper_bounds_ptr);
  copy_out(upper_bounds_ptr, p.variable_upper_bounds);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetVariableTypes(cuOptOptimizationProblem problem, char* variable_types_ptr)
{
  PROBLEM_OR_FAIL(variable_types_ptr);
  for (size_t j = 0; j < p.variable_types.size(); ++j)
    variable_types_ptr[j] = p.variable_types[j] == 'I' ? CUOPT_INTEGER : CUOPT_CONTINUOUS;
  return CUOPT_SUCCESS;
}

cuopt_int_t cuOptCreateSolverSettings(cuOptSolverSettings* settings_ptr)
{
  if (settings_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  *settings_ptr = new (std::nothrow) solver_settings_t();
  return *settings_ptr ? CUOPT_SUCCESS : CUOPT_OUT_OF_MEMORY;
}
void cuOptDestroySolverSettings(cuOptSolverSettings* settings_ptr)
{
  if (settings_ptr == nullptr) return;
  delete static_cast<solver_settings_t*>(*settings_ptr);
  *settings_ptr = nullptr;
}

cuopt_int_t cuOptSetParameter(cuOptSolverSettings settings, const char* parameter_name, const char* parameter_value)
{
  if (settings == nullptr || parameter_name == nullptr || parameter_value == nullptr) return CUOPT_INVALID_ARGUMENT;
  try {
    static_cast<solver_settings_t*>(settings)->set_from_string(parameter_name, parameter_value);
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetParameter(cuOptSolverSettings settings,
                              const char* parameter_name,
                              cuopt_int_t parameter_value_size,
                              char* parameter_value)
{
  if (settings == nullptr || parameter_name == nullptr || parameter_value == nullptr || parameter_value_size <= 0)
    return CUOPT_INVALID_ARGUMENT;
  try {
    const std::string s = static_cast<solver_settings_t*>(settings)->get_as_string(parameter_name);
    std::snprintf(parameter_value, parameter_value_size, "%s", s.c_str());
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptSetIntegerParameter(cuOptSolverSettings settings, const char* parameter_name, cuopt_int_t parameter_value)
{
  if (settings == nullptr || parameter_name == nullptr) return CUOPT_INVALID_ARGUMENT;
  try {
    static_cast<solver_settings_t*>(settings)->set_int(parameter_name, parameter_value);
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetIntegerParameter(cuOptSolverSettings settings, const char* parameter_name, cuopt_int_t* parameter_value)
{
  if (settings == nullptr || parameter_name == nullptr || parameter_value == nullptr) return CUOPT_INVALID_ARGUMENT;
  try {
    *parameter_value = static_cast<solver_settings_t*>(settings)->get_int(parameter_name);
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptSetFloatParameter(cuOptSolverSettings settings, const char* parameter_name, cuopt_float_t parameter_value)
{
  if (settings == nullptr || parameter_name == nullptr) return CUOPT_INVALID_ARGUMENT;
  try {
    static_cast<solver_settings_t*>(settings)->set_float(parameter_name, parameter_value);
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetFloatParameter(cuOptSolverSettings settings, const char* parameter_name, cuopt_float_t* parameter_value)
{
  if (settings == nullptr || parameter_name == nullptr || parameter_value == nullptr) return CUOPT_INVALID_ARGUMENT;
  try {
    *parameter_value = static_cast<solver_settings_t*>(settings)->get_float(parameter_name);
  } catch (const std::exception&) {
    return CUOPT_INVALID_ARGUMENT;
  }
  return CUOPT_SUCCESS;
}

cuopt_int_t cuOptIsMIP(cuOptOptimizationProblem problem, cuopt_int_t* is_mip_ptr)
{
  PROBLEM_OR_FAIL(is_mip_ptr);
  *is_mip_ptr = p.is_mip() ? 1 : 0;
  return CUOPT_SUCCESS;
}

cuopt_int_t cuOptSolve(cuOptOptimizationProblem problem, cuOptSolverSettings settings, cuOptSolution* solution_ptr)
{
  if (problem == nullptr || settings == nullptr || solution_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  *solution_ptr               = nullptr;
  const lp_problem_t& p       = *static_cast<const lp_problem_t*>(problem);
  const solver_settings_t& ss = *static_cast<const solver_settings_t*>(settings);
  std::unique_ptr<solution_handle_t> h(new (std::nothrow) solution_handle_t());
  if (!h) return CUOPT_OUT_OF_MEMORY;
  guarded(h->sol, [&]() {
    if (!ss.pdlp().user_problem_file.empty()) {  // solve.cu:586-589, before anything touches the GPU
      if (!write_problem_as_mps(p, ss.pdlp().user_problem_file))
        std::fprintf(stderr, "Could not open file %s for writing\n", ss.pdlp().user_problem_file.c_str());
    }
    if (p.is_mip()) {
      // LP-only build: answer with an error solution instead of a MIP search (INTEGRATION.md)
      h->is_mip            = false;
      h->sol.error_status  = CUOPT_VALIDATION_ERROR;
      h->sol.error_message = "cuopt-b200 implements the LP (PDLP) path only; the problem declares integer variables";
      return;
    }
    // This build has no CPU simplex and no crossover (SURVEY.md 8f rank 2).  What each `method` gets, and how the caller
    // is told (log line below + cuOptB200LPStats.method_stand_in, INTEGRATION.md "method"):
    //   PDLP        the requested method.
    //   Concurrent  (the reference races PDLP against the dual simplex, solve.cu:467-536): PDLP alone, caller's settings.
    //   DualSimplex PDLP stands in with what the simplex would tell apart or deliver: strict infeasibility detection (the
    //               reference's test_infeasible_problem asks exactly that of CUOPT_METHOD_DUAL_SIMPLEX) and tolerances
    //               tightened to 1e-8 where the caller's are looser (a simplex answer is a vertex, accurate to ~1e-9: the
    //               reference's test_ranged_problem expects 32.0 +- 1e-3, PDLP at 1e-4 stops at 31.9983).  Tolerances the
    //               caller already set below 1e-8, iteration_limit and time_limit are respected as given.
    pdlp_settings_t run = ss.pdlp();
    int stand_in        = 0;
    if (run.method == 0 /* CUOPT_METHOD_CONCURRENT */) stand_in = 1;
    if (run.method == 2 /* CUOPT_METHOD_DUAL_SIMPLEX */) {
      stand_in                 = 2;
      run.detect_infeasibility = true;
      run.strict_infeasibility = true;
      for (double* t : {&run.absolute_dual_tolerance, &run.relative_dual_tolerance, &run.absolute_primal_tolerance,
                        &run.relative_primal_tolerance, &run.absolute_gap_tolerance, &run.relative_gap_tolerance})
        *t = std::min(*t, 1e-8);
    }
    h->sol                       = solve_lp(p, run);
    h->sol.stats.method_stand_in = stand_in;
    if (h->sol.error_status == 0) log_solution(ss.pdlp(), p, h->sol);
    if (h->sol.error_status == 0 && !ss.pdlp().sol_file.empty()) {  // solve.cu:598-601
      if (!write_solution_file(p, h->sol, ss.pdlp().sol_file))
        std::fprintf(stderr, "Could not open file: %s for solution output\n", ss.pdlp().sol_file.c_str());
    }
  });
  const cuopt_int_t status = h->sol.error_status;
  *solution_ptr            = h.release();  // allocated even on failure: the error string stays retrievable (cuopt_c.cpp:611-618)
  return status;
}

void cuOptDestroySolution(cuOptSolution* solution_ptr)
{
  if (solution_ptr == nullptr || *solution_ptr == nullptr) return;
  delete static_cast<solution_handle_t*>(*solution_ptr);
  *solution_ptr = nullptr;
}

#define SOLUTION_OR_FAIL(out)                                               \
  if (solution == nullptr || (out) == nullptr) return CUOPT_INVALID_ARGUMENT; \
  const solution_handle_t& s = *static_cast<const solution_handle_t*>(solution)

cuopt_int_t cuOptGetTerminationStatus(cuOptSolution solution, cuopt_int_t* termination_status_ptr)
{
  SOLUTION_OR_FAIL(termination_status_ptr);
  *termination_status_ptr = (cuopt_int_t)s.sol.termination_status;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetErrorStatus(cuOptSolution solution, cuopt_int_t* error_status_ptr)
{
  SOLUTION_OR_FAIL(error_status_ptr);
  *error_status_ptr = s.sol.error_status;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetErrorString(cuOptSolution solution, char* error_string_ptr, cuopt_int_t error_string_size)
{
  SOLUTION_OR_FAIL(error_string_ptr);
  if (error_string_size > 0) std::snprintf(error_string_ptr, error_string_size, "%s", s.sol.error_message.c_str());
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetPrimalSolution(cuOptSolution solution, cuopt_float_t* solution_values)
{
  SOLUTION_OR_FAIL(solution_values);
  copy_out(solution_values, s.sol.primal);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetObjectiveValue(cuOptSolution solution, cuopt_float_t* objective_value_ptr)
{
  SOLUTION_OR_FAIL(objective_value_ptr);
  *objective_value_ptr = s.sol.stats.primal_objective;  // solver_solution.cu:307-310
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetSolveTime(cuOptSolution solution, cuopt_float_t* solve_time_ptr)
{
  SOLUTION_OR_FAIL(solve_time_ptr);
  *solve_time_ptr = s.sol.stats.solve_time;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetMIPGap(cuOptSolution solution, cuopt_float_t* mip_gap_ptr)
{
  SOLUTION_OR_FAIL(mip_gap_ptr);
  (void)s;
  return CUOPT_INVALID_ARGUMENT;  // LP solution (cuopt_c.cpp:776-779)
}
cuopt_int_t cuOptGetSolutionBound(cuOptSolution solution, cuopt_float_t* solution_bound_ptr)
{
  SOLUTION_OR_FAIL(solution_bound_ptr);
  (void)s;
  return CUOPT_INVALID_ARGUMENT;
}
cuopt_int_t cuOptGetDualSolution(cuOptSolution solution, cuopt_float_t* dual_solution_ptr)
{
  SOLUTION_OR_FAIL(dual_solution_ptr);
  copy_out(dual_solution_ptr, s.sol.dual);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptGetReducedCosts(cuOptSolution solution, cuopt_float_t* reduced_cost_ptr)
{
  SOLUTION_OR_FAIL(reduced_cost_ptr);
  copy_out(reduced_cost_ptr, s.sol.reduced_cost);
  return CUOPT_SUCCESS;
}

// ------------------------------------------------------------------------------ extension
static void export_stats(const lp_stats_t& t, cuOptB200LPStats* o)
{
  std::memset(o, 0, sizeof(*o));
  o->number_of_steps_taken           = t.number_of_steps_taken;
  o->total_number_of_attempted_steps = t.total_number_of_attempted_steps;
  o->l2_primal_residual              = t.l2_primal_residual;
  o->l2_relative_primal_residual     = t.l2_relative_primal_residual;
  o->l2_dual_residual                = t.l2_dual_residual;
  o->l2_relative_dual_residual       = t.l2_relative_dual_residual;
  o->primal_objective                = t.primal_objective;
  o->dual_objective                  = t.dual_objective;
  o->gap                             = t.gap;
  o->relative_gap                    = t.relative_gap;
  o->solved_by_pdlp                  = t.solved_by_pdlp;
  o->n_major_iterations              = t.n_major_iterations;
  o->n_restarts                      = t.n_restarts;
  o->method_stand_in                 = t.method_stand_in;
  o->solve_time                      = t.solve_time;
  o->setup_seconds                   = t.setup_seconds;
  o->pdhg_loop_seconds               = t.pdhg_loop_seconds;
  o->termination_seconds             = t.termination_seconds;
  o->initial_step_size               = t.initial_step_size;
  o->initial_primal_weight           = t.initial_primal_weight;
  o->final_step_size                 = t.final_step_size;
  o->final_primal_weight             = t.final_primal_weight;
  o->kernel_launches                 = t.kernel_launches;
}

cuopt_int_t cuOptB200GetLPStats(cuOptSolution solution, cuOptB200LPStats* stats)
{
  SOLUTION_OR_FAIL(stats);
  export_stats(s.sol.stats, stats);
  return CUOPT_SUCCESS;
}

cuopt_int_t cuOptB200GetPresolveStats(cuOptSolution solution, cuOptB200PresolveStats* stats)
{
  SOLUTION_OR_FAIL(stats);
  const presolve_stats_t& t = s.sol.presolve;
  std::memset(stats, 0, sizeof(*stats));
  stats->ran               = t.ran;
  stats->original_m        = t.original_m;
  stats->original_n        = t.original_n;
  stats->original_nnz      = t.original_nnz;
  stats->reduced_m         = t.reduced_m;
  stats->reduced_n         = t.reduced_n;
  stats->reduced_nnz       = t.reduced_nnz;
  stats->fixed_columns     = t.fixed_columns;
  stats->empty_rows        = t.empty_rows;
  stats->singleton_rows    = t.singleton_rows;
  stats->empty_columns     = t.empty_columns;
  stats->rounds            = t.rounds;
  stats->presolve_seconds  = t.presolve_seconds;
  stats->postsolve_seconds = t.postsolve_seconds;
  return CUOPT_SUCCESS;
}

// ---- warm start (cuopt_b200_ext.h) ----
namespace {
struct warm_start_handle_t {
  std::shared_ptr<const pdlp_warm_start_t> data;
};
const char* const WS_VECTORS[9] = {"current_primal_solution", "current_dual_solution", "initial_primal_average",
                                   "initial_dual_average", "current_ATY", "sum_primal_solutions", "sum_dual_solutions",
                                   "last_restart_duality_gap_primal_solution", "last_restart_duality_gap_dual_solution"};
const bool WS_IS_PRIMAL[9]      = {true, false, true, false, true, true, false, true, false};
std::vector<double> pdlp_warm_start_t::*const WS_MEMBERS[9] = {
  &pdlp_warm_start_t::current_primal_solution, &pdlp_warm_start_t::current_dual_solution,
  &pdlp_warm_start_t::initial_primal_average, &pdlp_warm_start_t::initial_dual_average, &pdlp_warm_start_t::current_ATY,
  &pdlp_warm_start_t::sum_primal_solutions, &pdlp_warm_start_t::sum_dual_solutions,
  &pdlp_warm_start_t::last_restart_duality_gap_primal_solution, &pdlp_warm_start_t::last_restart_duality_gap_dual_solution};
}  // namespace

cuopt_int_t cuOptB200SetWarmStartCapture(cuOptSolverSettings settings, cuopt_int_t enable)
{
  if (settings == nullptr) return CUOPT_INVALID_ARGUMENT;
  static_cast<solver_settings_t*>(settings)->set_capture_warm_start(enable != 0);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200GetWarmStart(cuOptSolution solution, cuOptB200WarmStart* warm_start_ptr)
{
  SOLUTION_OR_FAIL(warm_start_ptr);
  *warm_start_ptr = nullptr;
  if (!s.sol.warm_start) return CUOPT_INVALID_ARGUMENT;
  *warm_start_ptr = new warm_start_handle_t{s.sol.warm_start};
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SetWarmStart(cuOptSolverSettings settings, cuOptB200WarmStart warm_start)
{
  if (settings == nullptr) return CUOPT_INVALID_ARGUMENT;
  static_cast<solver_settings_t*>(settings)->set_warm_start(
    warm_start ? static_cast<warm_start_handle_t*>(warm_start)->data : nullptr);
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200CreateWarmStart(cuopt_int_t num_constraints, cuopt_int_t num_variables,
                                     const cuopt_float_t* const* vectors_9, const cuopt_float_t* scalars_8,
                                     cuOptB200WarmStart* warm_start_ptr)
{
  if (warm_start_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  *warm_start_ptr = nullptr;
  if (vectors_9 == nullptr || scalars_8 == nullptr || num_constraints < 0 || num_variables < 0) return CUOPT_INVALID_ARGUMENT;
  for (int q = 0; q < 9; ++q)
    if (vectors_9[q] == nullptr && (WS_IS_PRIMAL[q] ? num_variables : num_constraints) > 0) return CUOPT_INVALID_ARGUMENT;
  try {
    auto w = std::make_shared<pdlp_warm_start_t>();
    for (int q = 0; q < 9; ++q) {
      const int size = WS_IS_PRIMAL[q] ? num_variables : num_constraints;
      ((*w).*WS_MEMBERS[q]).assign(vectors_9[q], vectors_9[q] + size);
    }
    w->initial_primal_weight         = scalars_8[0];
    w->initial_step_size             = scalars_8[1];
    w->total_pdlp_iterations         = (int)scalars_8[2];
    w->total_pdhg_iterations         = (int)scalars_8[3];
    w->last_candidate_kkt_score      = scalars_8[4];
    w->last_restart_kkt_score        = scalars_8[5];
    w->sum_solution_weight           = scalars_8[6];
    w->iterations_since_last_restart = (int)scalars_8[7];
    *warm_start_ptr                  = new warm_start_handle_t{w};
  } catch (const std::bad_alloc&) {
    return CUOPT_OUT_OF_MEMORY;
  }
  return CUOPT_SUCCESS;
}
void cuOptB200DestroyWarmStart(cuOptB200WarmStart* warm_start_ptr)
{
  if (warm_start_ptr == nullptr || *warm_start_ptr == nullptr) return;
  delete static_cast<warm_start_handle_t*>(*warm_start_ptr);
  *warm_start_ptr = nullptr;
}
cuopt_int_t cuOptB200WarmStartGetScalar(cuOptB200WarmStart warm_start, const char* name, cuopt_float_t* value_ptr)
{
  if (warm_start == nullptr || name == nullptr || value_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  const pdlp_warm_start_t& w = *static_cast<warm_start_handle_t*>(warm_start)->data;
  const std::string s(name);
  if (s == "initial_primal_weight") *value_ptr = w.initial_primal_weight;
  else if (s == "initial_step_size") *value_ptr = w.initial_step_size;
  else if (s == "total_pdlp_iterations") *value_ptr = w.total_pdlp_iterations;
  else if (s == "total_pdhg_iterations") *value_ptr = w.total_pdhg_iterations;
  else if (s == "last_candidate_kkt_score") *value_ptr = w.last_candidate_kkt_score;
  else if (s == "last_restart_kkt_score") *value_ptr = w.last_restart_kkt_score;
  else if (s == "sum_solution_weight") *value_ptr = w.sum_solution_weight;
  else if (s == "iterations_since_last_restart") *value_ptr = w.iterations_since_last_restart;
  else return CUOPT_INVALID_ARGUMENT;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200WarmStartGetVector(cuOptB200WarmStart warm_start, const char* name, cuopt_float_t* values,
                                        cuopt_int_t* size_ptr)
{
  if (warm_start == nullptr || name == nullptr || size_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  const pdlp_warm_start_t& w = *static_cast<warm_start_handle_t*>(warm_start)->data;
  for (int q = 0; q < 9; ++q) {
    if (std::strcmp(name, WS_VECTORS[q]) != 0) continue;
    const std::vector<double>& v = w.*WS_MEMBERS[q];
    *size_ptr                    = (cuopt_int_t)v.size();
    if (values != nullptr && !v.empty()) std::memcpy(values, v.data(), v.size() * sizeof(double));
    return CUOPT_SUCCESS;
  }
  return CUOPT_INVALID_ARGUMENT;
}

cuopt_int_t cuOptB200SolverCreate(cuOptOptimizationProblem problem, cuOptSolverSettings settings, cuOptB200Solver* solver_ptr)
{
  if (problem == nullptr || settings == nullptr || solver_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  *solver_ptr = nullptr;
  try {
    auto h    = std::make_unique<solver_handle_t>();
    h->solver = std::make_unique<pdlp_solver_t>(*static_cast<const lp_problem_t*>(problem),
                                                static_cast<const solver_settings_t*>(settings)->pdlp());
    *solver_ptr = h.release();
  } catch (const lp_error& e) {
    std::fprintf(stderr, "cuOptB200SolverCreate: %s\n", e.what());
    return e.type == error_type_t::Success ? CUOPT_VALIDATION_ERROR : (cuopt_int_t)e.type;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "cuOptB200SolverCreate: %s\n", e.what());
    return CUOPT_RUNTIME_ERROR;
  }
  return CUOPT_SUCCESS;
}
void cuOptB200SolverDestroy(cuOptB200Solver* solver_ptr)
{
  if (solver_ptr == nullptr || *solver_ptr == nullptr) return;
  delete static_cast<solver_handle_t*>(*solver_ptr);
  *solver_ptr = nullptr;
}

#define SOLVER_GUARD(expr)                                     \
  try {                                                        \
    expr;                                                      \
  } catch (const lp_error& e) {                                \
    std::fprintf(stderr, "cuopt-b200: %s\n", e.what());        \
    return (cuopt_int_t)e.type;                                \
  } catch (const std::exception& e) {                          \
    std::fprintf(stderr, "cuopt-b200: %s\n", e.what());        \
    return CUOPT_RUNTIME_ERROR;                                \
  }

cuopt_int_t cuOptB200SolverInitialise(cuOptB200Solver solver)
{
  if (solver == nullptr) return CUOPT_INVALID_ARGUMENT;
  SOLVER_GUARD(static_cast<solver_handle_t*>(solver)->solver->initialise());
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SolverAdvance(cuOptB200Solver solver, cuopt_int_t accepted_steps, cuopt_int_t* finished_ptr)
{
  if (solver == nullptr) return CUOPT_INVALID_ARGUMENT;
  auto* h = static_cast<solver_handle_t*>(solver);
  SOLVER_GUARD(h->finished = h->solver->advance(accepted_steps));
  if (finished_ptr) *finished_ptr = h->finished ? 1 : 0;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SolverGetScalar(cuOptB200Solver solver, const char* name, cuopt_float_t* value_ptr)
{
  if (solver == nullptr || name == nullptr || value_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  SOLVER_GUARD(*value_ptr = static_cast<solver_handle_t*>(solver)->solver->scalar(name));
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SolverGetVector(cuOptB200Solver solver,
                                     const char* name,
                                     cuopt_float_t* values,
                                     cuopt_int_t capacity,
                                     cuopt_int_t* size_ptr)
{
  if (solver == nullptr || name == nullptr) return CUOPT_INVALID_ARGUMENT;
  SOLVER_GUARD({
    auto v = static_cast<solver_handle_t*>(solver)->solver->vector(name);
    if (size_ptr) *size_ptr = (cuopt_int_t)v.size();
    if (values) {
      if ((size_t)capacity < v.size()) return CUOPT_INVALID_ARGUMENT;
      copy_out(values, v);
    }
  });
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SolverTrustRegionBounds(cuOptB200Solver solver,
                                             const cuopt_float_t* px,
                                             const cuopt_float_t* py,
                                             cuopt_float_t radius,
                                             cuopt_float_t* lower_ptr,
                                             cuopt_float_t* upper_ptr)
{
  if (solver == nullptr || px == nullptr || py == nullptr || lower_ptr == nullptr || upper_ptr == nullptr)
    return CUOPT_INVALID_ARGUMENT;
  SOLVER_GUARD(static_cast<solver_handle_t*>(solver)->solver->trust_region_bounds(px, py, radius, *lower_ptr, *upper_ptr));
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SolverInfeasibilityStats(cuOptB200Solver solver,
                                              const cuopt_float_t* x_cur,
                                              const cuopt_float_t* y_cur,
                                              const cuopt_float_t* x_avg,
                                              const cuopt_float_t* y_avg,
                                              cuopt_float_t* stats,
                                              cuopt_int_t* status)
{
  if (solver == nullptr || x_cur == nullptr || y_cur == nullptr || x_avg == nullptr || y_avg == nullptr ||
      stats == nullptr || status == nullptr)
    return CUOPT_INVALID_ARGUMENT;
  SOLVER_GUARD({
    int st[2];
    static_cast<solver_handle_t*>(solver)->solver->infeasibility_stats(x_cur, y_cur, x_avg, y_avg, stats, st);
    status[0] = st[0];
    status[1] = st[1];
  });
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SolverGetSolution(cuOptB200Solver solver, cuOptSolution* solution_ptr)
{
  if (solver == nullptr || solution_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  auto* h   = static_cast<solver_handle_t*>(solver);
  auto* out = new (std::nothrow) solution_handle_t();
  if (!out) return CUOPT_OUT_OF_MEMORY;
  out->sol      = h->solver->solution();
  *solution_ptr = out;
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200SolverProfileKernels(cuOptB200Solver solver,
                                          cuopt_int_t warmup_steps,
                                          cuopt_int_t reps,
                                          cuOptB200KernelProfile* profile)
{
  if (solver == nullptr || profile == nullptr || reps <= 0) return CUOPT_INVALID_ARGUMENT;
  SOLVER_GUARD({
    const kernel_profile_t k      = static_cast<solver_handle_t*>(solver)->solver->profile_kernels(warmup_steps, reps);
    profile->ms_primal_step       = k.ms_primal_step;
    profile->ms_dual_step         = k.ms_dual_step;
    profile->ms_transpose_step    = k.ms_transpose_step;
    profile->bytes_primal_step    = k.bytes_primal_step;
    profile->bytes_dual_step      = k.bytes_dual_step;
    profile->bytes_transpose_step = k.bytes_transpose_step;
    profile->ms_iteration         = k.ms_iteration;
    profile->reps                 = k.reps;
    profile->grid_primal          = k.grid_primal;
    profile->grid_dual            = k.grid_dual;
    profile->grid_transpose       = k.grid_transpose;
    profile->ms_transpose_partial      = k.ms_transpose_partial;
    profile->ms_transpose_partial_wide = k.ms_transpose_partial_wide;
    profile->blocks_dual               = k.blocks_dual;
    profile->blocks_transpose          = k.blocks_transpose;
  });
  return CUOPT_SUCCESS;
}

cuopt_int_t cuOptB200DistGetUniqueId(char* unique_id_128_bytes)
{
  if (unique_id_128_bytes == nullptr) return CUOPT_INVALID_ARGUMENT;
  SOLVER_GUARD(dist_get_unique_id(unique_id_128_bytes));
  return CUOPT_SUCCESS;
}
cuopt_int_t cuOptB200DistInit(cuopt_int_t rank, cuopt_int_t world_size, const char* unique_id_128_bytes, cuOptB200Dist* dist_ptr)
{
  if (unique_id_128_bytes == nullptr || dist_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  *dist_ptr = nullptr;
  SOLVER_GUARD(*dist_ptr = dist_create(rank, world_size, unique_id_128_bytes));
  return CUOPT_SUCCESS;
}
void cuOptB200DistDestroy(cuOptB200Dist* dist_ptr)
{
  if (dist_ptr == nullptr || *dist_ptr == nullptr) return;
  dist_destroy(static_cast<dist_context_t*>(*dist_ptr));
  *dist_ptr = nullptr;
}
cuopt_int_t cuOptB200SolveDistributed(cuOptOptimizationProblem local_rows_problem,
                                      cuOptSolverSettings settings,
                                      cuOptB200Dist dist,
                                      cuOptSolution* solution_ptr)
{
  if (local_rows_problem == nullptr || settings == nullptr || dist == nullptr || solution_ptr == nullptr)
    return CUOPT_INVALID_ARGUMENT;
  const lp_problem_t& p       = *static_cast<const lp_problem_t*>(local_rows_problem);
  const solver_settings_t& ss = *static_cast<const solver_settings_t*>(settings);
  *solution_ptr = nullptr;
  std::unique_ptr<solution_handle_t> h(new (std::nothrow) solution_handle_t());
  if (!h) return CUOPT_OUT_OF_MEMORY;
  guarded(h->sol, [&]() {
    if (ss.pdlp().presolve) {  // each rank holds a block of rows; presolve needs the whole matrix (checked before `dist` is used)
      h->sol.error_status  = CUOPT_VALIDATION_ERROR;
      h->sol.error_message = "presolve is not available in multi-GPU solves: it needs the whole matrix";
      return;
    }
    if (p.is_mip()) {
      h->sol.error_status  = CUOPT_VALIDATION_ERROR;
      h->sol.error_message = "cuopt-b200 implements the LP (PDLP) path only; the problem declares integer variables";
      return;
    }
    auto* d = static_cast<dist_context_t*>(dist);
    h->sol  = solve_lp(p, ss.pdlp(), d);
    if (h->sol.error_status == 0 && d->rank == 0) log_solution(ss.pdlp(), p, h->sol);
  });
  const cuopt_int_t status = h->sol.error_status;
  *solution_ptr            = h.release();
  return status;
}

cuopt_int_t cuOptB200ReadProblem(const char* filename, cuopt_int_t fixed_format, cuOptOptimizationProblem* problem_ptr)
{
  if (filename == nullptr || problem_ptr == nullptr) return CUOPT_INVALID_ARGUMENT;
  *problem_ptr = nullptr;
  try {
    *problem_ptr = new lp_problem_t(read_mps(filename, fixed_format != 0));
    return CUOPT_SUCCESS;
  } catch (const lp_error& e) {
    return e.type == error_type_t::MpsFileError ? CUOPT_MPS_FILE_ERROR : CUOPT_MPS_PARSE_ERROR;
  } catch (const std::exception&) {
    return CUOPT_MPS_PARSE_ERROR;
  }
}

const char* cuOptB200Version(void) { return "cuopt-b200 0.1.0 sm_90a"; }

}  // extern "C"
