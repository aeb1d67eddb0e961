// Plain value types shared by the host driver, the CUDA solver and the C ABI.
#pragma once

#include <limits>
#include <memory>
#include <string>
#include <vector>

namespace cuopt_b200 {

// Same numeric values as the reference's pdlp_termination_status_t
// (cpp/include/cuopt/linear_programming/pdlp/solver_solution.hpp, constants.h:62-72).
enum class termination_status_t : int {
  NoTermination    = 0,
  Optimal          = 1,
  PrimalInfeasible = 2,
  DualInfeasible   = 3,
  IterationLimit   = 4,
  TimeLimit        = 5,
  NumericalError   = 6,
  PrimalFeasible   = 7,
  FeasibleFound    = 8,
  ConcurrentLimit  = 9
};

inline const char* termination_status_string(termination_status_t s)
{
  switch (s) {
    case termination_status_t::NoTermination: return "NoTermination";
    case termination_status_t::Optimal: return "Optimal";
    case termination_status_t::PrimalInfeasible: return "PrimalInfeasible";
    case termination_status_t::DualInfeasible: return "DualInfeasible";
    case termination_status_t::IterationLimit: return "IterationLimit";
    case termination_status_t::TimeLimit: return "TimeLimit";
    case termination_status_t::NumericalError: return "NumericalError";
    case termination_status_t::PrimalFeasible: return "PrimalFeasible";
    case termination_status_t::FeasibleFound: return "FeasibleFound";
    case termination_status_t::ConcurrentLimit: return "ConcurrentLimit";
  }
  return "Unknown";
}

// The reference keeps these 30 values in process-global variables
// (cpp/src/linear_programming/pdlp_hyper_params.cu:22-80) that the presets in
// solve.cu:64-199 overwrite.  Here they travel by value with each solve, so two
// solves with different modes can run in one process.
struct pdlp_hyper_params_t {
  double initial_step_size_scaling                                  = 1.0;
  int default_l_inf_ruiz_iterations                                 = 10;
  bool do_pock_chambolle_scaling                                    = true;
  bool do_ruiz_scaling                                              = true;
  double default_alpha_pock_chambolle_rescaling                     = 1.0;
  double default_artificial_restart_threshold                       = 0.36;
  bool compute_initial_step_size_before_scaling                     = false;
  bool compute_initial_primal_weight_before_scaling                 = false;
  double initial_primal_weight_c_scaling                            = 1.0;
  double initial_primal_weight_b_scaling                            = 1.0;
  int major_iteration                                               = 40;
  int min_iteration_restart                                         = 10;
  int restart_strategy                                              = 1;  // 0 none, 1 KKT, 2 trust region
  bool never_restart_to_average                                     = false;
  double reduction_exponent                                         = 0.3;
  double growth_exponent                                            = 0.6;
  double primal_weight_update_smoothing                             = 0.5;
  double sufficient_reduction_for_restart                           = 0.2;
  double necessary_reduction_for_restart                            = 0.8;
  double primal_importance                                          = 1.0;
  double primal_distance_smoothing                                  = 0.5;
  double dual_distance_smoothing                                    = 0.5;
  bool compute_last_restart_before_new_primal_weight                = true;
  bool artificial_restart_in_main_loop                              = false;
  bool rescale_for_restart                                          = true;
  bool update_primal_weight_on_initial_solution                     = false;
  bool update_step_size_on_initial_solution                         = false;
  bool handle_some_primal_gradients_on_finite_bounds_as_residuals   = false;
  bool project_initial_primal                                       = true;

  // solve.cu:64-199.  mode: 0 Stable1, 1 Stable2 (default), 2 Methodical1, 3 Fast1.
  static pdlp_hyper_params_t preset(int mode)
  {
    pdlp_hyper_params_t p;  // default member values == Stable2 (solve.cu:99-131)
    if (mode == 0) {        // Stable1, solve.cu:64-95
      p.initial_step_size_scaling                    = 1.6;
      p.default_l_inf_ruiz_iterations                = 1;
      p.default_alpha_pock_chambolle_rescaling       = 1.3;
      p.default_artificial_restart_threshold         = 0.5;
      p.compute_initial_primal_weight_before_scaling = true;
      p.initial_primal_weight_c_scaling              = 2.2;
      p.initial_primal_weight_b_scaling              = 4.6;
      p.major_iteration                              = 52;
      p.min_iteration_restart                        = 0;
      p.reduction_exponent                           = 0.5;
      p.growth_exponent                              = 0.9;
      p.primal_weight_update_smoothing               = 0.3;
      p.sufficient_reduction_for_restart             = 0.2;
      p.necessary_reduction_for_restart              = 0.5;
      p.primal_importance                            = 1.8;
      p.primal_distance_smoothing                    = 0.6;
      p.dual_distance_smoothing                      = 0.2;
      p.compute_last_restart_before_new_primal_weight = false;
      p.rescale_for_restart                          = false;
      p.handle_some_primal_gradients_on_finite_bounds_as_residuals = true;
      p.project_initial_primal                       = false;
    } else if (mode == 2) {  // Methodical1, solve.cu:133-165
      p.default_l_inf_ruiz_iterations        = 5;
      p.default_artificial_restart_threshold = 0.5;
      p.major_iteration                      = 64;
      p.min_iteration_restart                = 0;
      p.restart_strategy                     = 2;
      p.sufficient_reduction_for_restart     = 0.1;
      p.necessary_reduction_for_restart      = 0.9;
      p.rescale_for_restart                  = false;
      p.handle_some_primal_gradients_on_finite_bounds_as_residuals = true;
      p.project_initial_primal               = false;
    } else if (mode == 3) {  // Fast1, solve.cu:167-199
      p.initial_step_size_scaling                    = 0.8;
      p.default_l_inf_ruiz_iterations                = 6;
      p.do_ruiz_scaling                              = false;
      p.default_alpha_pock_chambolle_rescaling       = 2.0;
      p.default_artificial_restart_threshold         = 0.3;
      p.compute_initial_primal_weight_before_scaling = true;
      p.initial_primal_weight_c_scaling              = 1.2;
      p.initial_primal_weight_b_scaling              = 1.2;
      p.major_iteration                              = 76;
      p.min_iteration_restart                        = 6;
      p.never_restart_to_average                     = true;
      p.reduction_exponent                           = 0.4;
      p.growth_exponent                              = 0.6;
      p.sufficient_reduction_for_restart             = 0.3;
      p.necessary_reduction_for_restart              = 0.9;
      p.primal_importance                            = 0.8;
      p.primal_distance_smoothing                    = 0.8;
      p.dual_distance_smoothing                      = 0.3;
      p.artificial_restart_in_main_loop              = true;
      p.handle_some_primal_gradients_on_finite_bounds_as_residuals = true;
      p.project_initial_primal                       = false;
    }
    return p;
  }
};

// Everything a later solve needs to continue this one where it stopped (reference:
// include/cuopt/linear_programming/pdlp/pdlp_warm_start_data.hpp:28-72, filled by pdlp.cu:469-489 at termination,
// consumed by pdlp.cu:131-181 / :1074-1136).  Spaces as in the reference: the current iterate and the averages are
// UNSCALED (termination happens after the in-place unscaling), A^T y, the running sums and the last-restart point
// live in the scaled space.  Host vectors; in a sharded solve the dual-side vectors cover this rank's rows.
struct pdlp_warm_start_t {
  std::vector<double> current_primal_solution, current_dual_solution;
  std::vector<double> initial_primal_average, initial_dual_average;
  std::vector<double> current_ATY;
  std::vector<double> sum_primal_solutions, sum_dual_solutions;
  std::vector<double> last_restart_duality_gap_primal_solution, last_restart_duality_gap_dual_solution;
  double initial_primal_weight       = -1;
  double initial_step_size           = -1;
  int total_pdlp_iterations          = -1;
  int total_pdhg_iterations          = -1;
  double last_candidate_kkt_score    = -1;
  double last_restart_kkt_score      = -1;
  double sum_solution_weight         = -1;
  int iterations_since_last_restart  = -1;
  bool empty() const { return last_restart_duality_gap_dual_solution.empty(); }  // the reference's test, pdlp.cu:131
};

// pdlp_solver_settings_t as seen by the C ABI (solver_settings.cu:63-125 for defaults / ranges).
struct pdlp_settings_t {
  double absolute_dual_tolerance     = 1e-4;
  double relative_dual_tolerance     = 1e-4;
  double absolute_primal_tolerance   = 1e-4;
  double relative_primal_tolerance   = 1e-4;
  double absolute_gap_tolerance      = 1e-4;
  double relative_gap_tolerance      = 1e-4;
  double primal_infeasible_tolerance = 1e-8;
  double dual_infeasible_tolerance   = 1e-8;
  int iteration_limit                = std::numeric_limits<int>::max();
  double time_limit                  = std::numeric_limits<double>::infinity();
  int pdlp_solver_mode               = 1;  // Stable2
  int method                         = 0;  // Concurrent
  bool detect_infeasibility          = false;
  bool strict_infeasibility          = false;
  bool per_constraint_residual       = false;
  bool save_best_primal_so_far       = false;
  bool first_primal_feasible         = false;
  bool log_to_console                = true;
  bool crossover                     = false;
  std::string log_file, sol_file, user_problem_file;
  // extension (cuopt_b200_ext.h): continue from a previous solve / make the solution carry the state to do so
  std::shared_ptr<const pdlp_warm_start_t> warm_start;
  bool capture_warm_start = false;
  bool presolve           = false;  // extension: presolve.cu before PDLP, postsolve after
};

// additional_termination_information_t (pdlp/solver_solution.hpp:47-87) plus timing of this build.
struct lp_stats_t {
  int number_of_steps_taken           = 0;
  int total_number_of_attempted_steps = 0;
  double l2_primal_residual           = 0;
  double l2_relative_primal_residual  = 0;
  double l2_dual_residual             = 0;
  double l2_relative_dual_residual    = 0;
  double primal_objective             = 0;
  double dual_objective               = 0;
  double gap                          = 0;
  double relative_gap                 = 0;
  int solved_by_pdlp                  = 1;
  int method_stand_in                 = 0;  // 0: the requested method ran; 1: Concurrent -> PDLP alone; 2: DualSimplex -> PDLP stand-in (c_api.cpp)
  double solve_time                   = 0;  // seconds, wall clock of run_solver (reference semantics)
  // --- this build ---
  double setup_seconds       = 0;  // H2D upload + transpose + scaling
  double pdhg_loop_seconds   = 0;  // device time (CUDA events) inside the PDHG iterations
  double termination_seconds = 0;  // device time inside the termination / restart passes
  int n_major_iterations     = 0;
  int n_restarts             = 0;
  long long kernel_launches  = 0;
  double initial_step_size   = 0;
  double initial_primal_weight = 0;
  double final_step_size     = 0;
  double final_primal_weight = 0;
};

// What presolve removed and what it and postsolve cost (cuOptB200PresolveStats).
struct presolve_stats_t {
  int ran = 0;  // 1 when the solve was presolved
  int original_m = 0, original_n = 0, original_nnz = 0;
  int reduced_m = 0, reduced_n = 0, reduced_nnz = 0;
  int fixed_columns = 0, empty_rows = 0, singleton_rows = 0, empty_columns = 0;
  int rounds = 0;
  double presolve_seconds = 0, postsolve_seconds = 0;  // device time (CUDA events)
};

struct lp_solution_t {
  termination_status_t termination_status = termination_status_t::NoTermination;
  int error_status                        = 0;  // error_type_t
  std::string error_message;
  std::vector<double> primal, dual, reduced_cost;
  lp_stats_t stats;
  std::shared_ptr<pdlp_warm_start_t> warm_start;  // filled when settings.capture_warm_start
  presolve_stats_t presolve;
};

}  // namespace cuopt_b200
