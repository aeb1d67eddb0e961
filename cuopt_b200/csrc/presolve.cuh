// Opt-in presolve of an LP on the device (settings.presolve, presolve.cu): empty rows and columns, fixed columns and
// singleton rows, removed in rounds; postsolve of primal, dual and reduced costs back to the original sizes.
//
// Both act on the problem in the minimisation form the solver uses (c already negated for maximisation, defaults applied).
#pragma once

#include "device_utils.cuh"
#include "pdlp_types.hpp"

namespace cuopt_b200 {

// What presolve keeps on the device for postsolve.  Per original column: alive or removed (then x_fix holds its value),
// and for each side of its bounds the singleton row that supplied it (-1: the column's own bound) with its coefficient.
struct presolve_state_t {
  int m0 = 0, n0 = 0, nnz0 = 0;  // original sizes
  int m1 = 0, n1 = 0, nnz1 = 0;  // reduced sizes
  termination_status_t verdict = termination_status_t::NoTermination;  // decided without PDLP (Optimal / infeasible / unbounded)
  double offset = 0.0;           // sum of c_j * x_fix_j over the removed columns (minimisation form)
  presolve_stats_t stats;
  dvec<int> toff, tidx;  // original A^T (postsolve products)
  dvec<double> tval;
  dvec<double> c0;       // original c (minimisation form)
  dvec<unsigned char> row_alive, col_alive;
  dvec<int> row_new, col_new;  // exclusive sums of the alive flags: new index of a kept row / column
  dvec<int> row_map, col_map;  // original index of each kept row / column
  dvec<double> x_fix;
  dvec<int> src_lo, src_hi;
  dvec<double> a_lo, a_hi;
  bool removed_nothing() const { return m1 == m0 && n1 == n0 && nnz1 == nnz0; }
};

// Presolves the m x n problem held in off / idx / val, c, l, u, lc, uc (device, unscaled, minimisation form); on return those
// arrays and m, n hold the reduced problem (the original A is freed) and ps the postsolve data.  `tol`: absolute primal
// tolerance of the infeasibility tests.  One small block of counters comes back to the host per round.
void presolve_device(int& m, int& n, dvec<int>& off, dvec<int>& idx, dvec<double>& val, dvec<double>& c, dvec<double>& l,
                     dvec<double>& u, dvec<double>& lc, dvec<double>& uc, double tol, presolve_state_t& ps,
                     cudaStream_t stream, bool trace);

// Postsolve of a reduced-space solution (host vectors of the reduced sizes, empty when there is none) into original-size
// host vectors.  certificate: the vectors are an infeasibility certificate — scattered, zeros on the removed entries; with
// dual_ray (a PrimalInfeasible ending) the singleton rows then get the duals that carry the bounds they supplied into the
// ray's objective on the original problem (r0 = -A^T y in the rule below).  Otherwise removed columns take their fixed
// value, removed rows dual 0, the singleton rows that supply an active bound get the dual that zeroes the column's reduced
// cost, and r = c - A^T y with the original A^T.
void postsolve_device(const presolve_state_t& ps, const std::vector<double>& x_red, const std::vector<double>& y_red,
                      const std::vector<double>& rc_red, bool certificate, bool dual_ray, std::vector<double>& x,
                      std::vector<double>& y, std::vector<double>& rc, cudaStream_t stream);

}  // namespace cuopt_b200
