"""Methodical1 (trust-region restart, pdlp_restart_strategy.cu:278-364, :983-1678) on the CUDA path
(cuopt_b200/csrc/trust_region.cuh), against the oracle restatement that is pinned to the reference's tests:
  * the reference's test_very_low_tolerance (test_lp_solver.py:101-121),
  * the iterates across the first trust-region restarts against the oracle,
  * the objectives of the golden instances (the oracle's are pinned to the reference's dual simplex)."""
import numpy as np
import pytest

from cases import lp_relaxation, make_pair
from conftest import mps_path, problem_arrays
from cuopt_b200 import capi
from exact import rel_err
from oracle import pdlp_oracle as po

pytestmark = pytest.mark.gpu

# 6 x 64 steps crossing trust-region restarts (sort + prefix sums + bisection feed the restart decision), iterates compared
# with the sequential oracle at every checkpoint.  PDHG with adaptive steps is a discontinuous map (accept / reject, restart
# candidate): two summation orders of the same algorithm agree to rounding for a while and then part ways while converging to
# the same solution: the block-interleaved core (rows that span lanes: carry + part) adds in another order than the oracle,
# and the grids follow the device's SM count.  Asserted: rounding-level agreement over the first 128 steps (two restarts), equal restart counts throughout, and no blow-up afterwards; the end result of
# the preset is pinned by the other tests of this file.
CHECKPOINT_BOUNDS = [1e-6, 1e-6, 1e-1, 1e-1, 1e-1, 1e-1]


def test_very_low_tolerance_afiro():
    p = capi.Problem.read(mps_path("linear_programming/afiro_original.mps"))
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=2)
    s.set("optimality_tolerance", 1e-12)
    sol = capi.solve(p, s)
    assert sol.return_code == 0, sol.error_string
    assert sol.termination_status == 1
    assert sol.stats().primal_objective == pytest.approx(-464.7531)
    assert sol.stats().n_restarts >= 1


def test_iterates_across_trust_region_restarts_match_the_oracle():
    g, o, _ = make_pair(capi.Problem.read(mps_path("linear_programming/afiro_original.mps")), mode=2, tol=1e-12)
    g.initialise(); o.initialise()
    worst, restarts = [], []
    for _ in range(6):  # major iterations every 64 steps
        g.advance(64); o.run(64)
        worst.append(max(rel_err(g.vector(name), o.vector(name))
                         for name in ("x", "y", "aty", "sum_x", "sum_y", "x_last_restart", "y_last_restart")))
        restarts.append((g.scalar("n_restarts"), o.scalar("n_restarts")))
        for name in ("step_size", "primal_weight"):
            worst[-1] = max(worst[-1], abs(g.scalar(name) - o.scalar(name)) / abs(o.scalar(name)))
    report = f"worst relative differences per checkpoint {worst}, restarts (gpu, oracle) {restarts}"
    assert all(a == b for a, b in restarts), report
    assert restarts[-1][1] >= 1, report
    assert all(w <= bound for w, bound in zip(worst, CHECKPOINT_BOUNDS)), report


@pytest.mark.parametrize("rel", ["mip/sudoku.mps", "mip/sample.mps", "mip/bb_optimality.mps"])
def test_objective_against_the_oracle(rel):
    p = lp_relaxation(rel)
    a = problem_arrays(p)
    o = po.Oracle(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"],
                  maximize=a["maximize"], objective_offset=a["objective_offset"], mode=po.METHODICAL1, tol=1e-8,
                  iteration_limit=400000)
    assert o.run(-1) and o.stats().termination_status == 1
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=2)
    s.set("optimality_tolerance", 1e-8)
    sol = capi.solve(p, s)
    assert sol.termination_status == 1
    assert sol.stats().primal_objective == pytest.approx(o.stats().primal_objective, rel=1e-6, abs=1e-6)
