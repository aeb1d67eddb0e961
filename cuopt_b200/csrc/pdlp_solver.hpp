// Host-visible interface of the PDLP solver (no CUDA types: c_api.cpp includes this).
//
// Counterpart of the reference's pdlp_solver_t / solve_lp
// (cpp/src/linear_programming/pdlp.cuh, solve.cu:554-613) for the PDLP method.
#pragma once

#include "lp_problem.hpp"
#include "pdlp_types.hpp"

#include <memory>

namespace cuopt_b200 {

// Average device time per launch of the three PDHG kernels (profiling entry point, bench.py roofline).
struct kernel_profile_t {
  double ms_primal_step = 0, ms_dual_step = 0, ms_transpose_step = 0;
  double bytes_primal_step = 0, bytes_dual_step = 0, bytes_transpose_step = 0;  // algorithmic bytes / launch
  double ms_iteration = 0;  // average per attempt inside a batched run (all three kernels, back to back)
  int reps = 0;
  int grid_dual = 0, grid_transpose = 0, grid_primal = 0;
  double ms_transpose_partial = 0, ms_transpose_partial_wide = 0;  // k_transpose_partial<1> / <WARP_WIDE_RPL>
  int blocks_dual = 1, blocks_transpose = 1;                       // gather blocking (1 = fused kernel)
};

// Optional multi-GPU context: rows of A are sharded over `world` ranks (see pdlp_dist.cu).
struct dist_context_t;

class pdlp_solver_t {
 public:
  // Uploads the problem to the current CUDA device, builds A^T, the row-block schedules and the
  // diagonal scaling.  Throws lp_error.
  pdlp_solver_t(const lp_problem_t& problem, const pdlp_settings_t& settings, dist_context_t* dist = nullptr);
  ~pdlp_solver_t();

  // pdlp_solver_t::run_solver (pdlp.cu:984-1185)
  lp_solution_t run();

  // White-box access for the parity tests / profiling (cuopt_b200_ext.h).
  void initialise();                                 // scaling + initial step size / primal weight
  bool advance(int accepted_steps);                  // run the outer loop for N more accepted steps
  double scalar(const std::string& name);
  std::vector<double> vector(const std::string& name);
  kernel_profile_t profile_kernels(int warmup_steps, int reps);
  // Lower / upper bound of the trust-region restart (Methodical1) at a point (px: n, py: m values) of the scaled space,
  // radius >= 0; reads the solver state, changes none of it.
  void trust_region_bounds(const double* px, const double* py, double radius, double& lower, double& upper);
  // Infeasibility-detection statistics (12 per iterate) and the status the tests give, at current / average points of the
  // unscaled minimisation form (x: n, y: m values); reads the solver state, changes none of it.
  void infeasibility_stats(const double* x_cur, const double* y_cur, const double* x_avg, const double* y_avg,
                           double* stats, int* status);
  const lp_solution_t& solution() const;

  struct impl_t;

 private:
  std::unique_ptr<impl_t> impl_;
};

// solve_lp for method == PDLP (and what Concurrent / DualSimplex fall back to in this build).
// `dist` != nullptr: `problem` holds THIS RANK'S block of rows (all columns); collective over the communicator.
lp_solution_t solve_lp(const lp_problem_t& problem, const pdlp_settings_t& settings, dist_context_t* dist = nullptr);

}  // namespace cuopt_b200
