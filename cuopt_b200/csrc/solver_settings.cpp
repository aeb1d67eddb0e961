#include "solver_settings.hpp"

#include <cuopt/linear_programming/constants.h>
#include <cuopt_b200/cuopt_b200_ext.h>

#include <limits>

namespace cuopt_b200 {

namespace {
bool parse_bool(const std::string& v, bool& out)  // solver_settings.cu:48-62
{
  if (v == "true" || v == "True" || v == "TRUE" || v == "1" || v == "t" || v == "T") { out = true; return true; }
  if (v == "false" || v == "False" || v == "FALSE" || v == "0" || v == "f" || v == "F") { out = false; return true; }
  return false;
}
}  // namespace

solver_settings_t::solver_settings_t()
  : mip_time_limit_(std::numeric_limits<double>::infinity()),
    mip_abs_tol_(1e-4), mip_rel_tol_(1e-4), mip_int_tol_(1e-5), mip_abs_gap_(1e-10), mip_rel_gap_(1e-4),
    mip_num_cpu_threads_(-1), mip_scaling_(true), mip_heuristics_only_(false), mip_log_to_console_(true)
{
  const double inf = std::numeric_limits<double>::infinity();
  const int imax   = std::numeric_limits<int>::max();
  // name, storage, min, max  (defaults live in pdlp_settings_t / the initialisers above)
  floats_ = {
    {CUOPT_TIME_LIMIT, &mip_time_limit_, 0.0, inf},
    {CUOPT_TIME_LIMIT, &pdlp_.time_limit, 0.0, inf},
    {CUOPT_ABSOLUTE_DUAL_TOLERANCE, &pdlp_.absolute_dual_tolerance, 0.0, 1e-1},
    {CUOPT_RELATIVE_DUAL_TOLERANCE, &pdlp_.relative_dual_tolerance, 0.0, 1e-1},
    {CUOPT_ABSOLUTE_PRIMAL_TOLERANCE, &pdlp_.absolute_primal_tolerance, 0.0, 1e-1},
    {CUOPT_RELATIVE_PRIMAL_TOLERANCE, &pdlp_.relative_primal_tolerance, 0.0, 1e-1},
    {CUOPT_ABSOLUTE_GAP_TOLERANCE, &pdlp_.absolute_gap_tolerance, 0.0, 1e-1},
    {CUOPT_RELATIVE_GAP_TOLERANCE, &pdlp_.relative_gap_tolerance, 0.0, 1e-1},
    {CUOPT_MIP_ABSOLUTE_TOLERANCE, &mip_abs_tol_, 0.0, 1e-1},
    {CUOPT_MIP_RELATIVE_TOLERANCE, &mip_rel_tol_, 0.0, 1e-1},
    {CUOPT_MIP_INTEGRALITY_TOLERANCE, &mip_int_tol_, 0.0, 1e-1},
    {CUOPT_MIP_ABSOLUTE_GAP, &mip_abs_gap_, 0.0, 1e-1},
    {CUOPT_MIP_RELATIVE_GAP, &mip_rel_gap_, 0.0, 1e-1},
    {CUOPT_PRIMAL_INFEASIBLE_TOLERANCE, &pdlp_.primal_infeasible_tolerance, 0.0, 1e-1},
    {CUOPT_DUAL_INFEASIBLE_TOLERANCE, &pdlp_.dual_infeasible_tolerance, 0.0, 1e-1},
  };
  ints_ = {
    {CUOPT_ITERATION_LIMIT, &pdlp_.iteration_limit, 0, imax},
    {CUOPT_PDLP_SOLVER_MODE, &pdlp_.pdlp_solver_mode, CUOPT_PDLP_SOLVER_MODE_STABLE1, CUOPT_PDLP_SOLVER_MODE_FAST1},
    {CUOPT_METHOD, &pdlp_.method, CUOPT_METHOD_CONCURRENT, CUOPT_METHOD_DUAL_SIMPLEX},
    {CUOPT_NUM_CPU_THREADS, &mip_num_cpu_threads_, -1, imax},
  };
  bools_ = {
    {CUOPT_INFEASIBILITY_DETECTION, &pdlp_.detect_infeasibility, false, true},
    {CUOPT_STRICT_INFEASIBILITY, &pdlp_.strict_infeasibility, false, true},
    {CUOPT_PER_CONSTRAINT_RESIDUAL, &pdlp_.per_constraint_residual, false, true},
    {CUOPT_SAVE_BEST_PRIMAL_SO_FAR, &pdlp_.save_best_primal_so_far, false, true},
    {CUOPT_FIRST_PRIMAL_FEASIBLE, &pdlp_.first_primal_feasible, false, true},
    {CUOPT_MIP_SCALING, &mip_scaling_, false, true},
    {CUOPT_MIP_HEURISTICS_ONLY, &mip_heuristics_only_, false, true},
    {CUOPT_LOG_TO_CONSOLE, &pdlp_.log_to_console, false, true},
    {CUOPT_LOG_TO_CONSOLE, &mip_log_to_console_, false, true},
    {CUOPT_CROSSOVER, &pdlp_.crossover, false, true},
    {CUOPT_B200_PRESOLVE, &pdlp_.presolve, false, true},
  };
  strings_ = {
    {CUOPT_LOG_FILE, &mip_log_file_, "", ""},
    {CUOPT_LOG_FILE, &pdlp_.log_file, "", ""},
    {CUOPT_SOLUTION_FILE, &mip_sol_file_, "", ""},
    {CUOPT_SOLUTION_FILE, &pdlp_.sol_file, "", ""},
    {CUOPT_USER_PROBLEM_FILE, &mip_user_problem_file_, "", ""},
    {CUOPT_USER_PROBLEM_FILE, &pdlp_.user_problem_file, "", ""},
  };
}

void solver_settings_t::set_from_string(const std::string& name, const std::string& value)
{
  bool found = false;
  for (auto& p : ints_)
    if (p.name == name) {
      int v;
      try {
        v = std::stoi(value);
      } catch (const std::exception&) {
        throw std::invalid_argument("Parameter " + name + " value " + value + " is not an integer");
      }
      if (v < p.lo || v > p.hi) throw std::invalid_argument("Parameter " + name + " value " + value + " out of range");
      *p.ptr = v;
      found  = true;
    }
  for (auto& p : floats_)
    if (p.name == name) {
      double v;
      try {
        v = std::stod(value);
      } catch (const std::exception&) {
        throw std::invalid_argument("Parameter " + name + " value " + value + " is not a float");
      }
      if (v < p.lo || v > p.hi) throw std::invalid_argument("Parameter " + name + " value " + value + " out of range");
      *p.ptr = v;
      found  = true;
    }
  for (auto& p : bools_)
    if (p.name == name) {
      bool v;
      if (!parse_bool(value, v)) throw std::invalid_argument("Parameter " + name + " value " + value + " must be true or false");
      *p.ptr = v;
      found  = true;
    }
  for (auto& p : strings_)
    if (p.name == name) {
      *p.ptr = value;
      found  = true;
    }
  if (!found) throw std::invalid_argument("Parameter " + name + " not found");
}

std::string solver_settings_t::get_as_string(const std::string& name) const
{
  for (auto& p : ints_)
    if (p.name == name) return std::to_string(*p.ptr);
  for (auto& p : floats_)
    if (p.name == name) return std::to_string(*p.ptr);
  for (auto& p : bools_)
    if (p.name == name) return *p.ptr ? "true" : "false";
  for (auto& p : strings_)
    if (p.name == name) return *p.ptr;
  throw std::invalid_argument("Parameter " + name + " not found");
}

void solver_settings_t::set_int(const std::string& name, int value)
{
  bool found = false;
  for (auto& p : ints_)
    if (p.name == name) {
      if (value < p.lo || value > p.hi) throw std::out_of_range("Parameter " + name + " out of range");
      *p.ptr = value;
      found  = true;
    }
  if (found) return;
  for (auto& p : bools_)
    if (p.name == name) {
      *p.ptr = value != 0;
      found  = true;
    }
  if (!found) throw std::invalid_argument("Parameter " + name + " not found");
}

int solver_settings_t::get_int(const std::string& name) const
{
  for (auto& p : ints_)
    if (p.name == name) return *p.ptr;
  for (auto& p : bools_)
    if (p.name == name) return *p.ptr ? 1 : 0;
  throw std::invalid_argument("Parameter " + name + " not found");
}

void solver_settings_t::set_float(const std::string& name, double value)
{
  bool found = false;
  for (auto& p : floats_)
    if (p.name == name) {
      if (value < p.lo || value > p.hi) throw std::out_of_range("Parameter " + name + " out of range");
      *p.ptr = value;
      found  = true;
    }
  if (!found) throw std::invalid_argument("Parameter " + name + " not found");
}

double solver_settings_t::get_float(const std::string& name) const
{
  for (auto& p : floats_)
    if (p.name == name) return *p.ptr;
  throw std::invalid_argument("Parameter " + name + " not found");
}

}  // namespace cuopt_b200
