"""`save_best_primal_so_far` (pdlp.cu:333-463, :265-331): when a limit stops the solve, the best of the current / average
iterates seen at the major iterations — primal feasible first, then objective; otherwise least l2 primal residual — is
returned instead of the last iterate.  Property of the reference's tests best_primal_so_far_iteration / _time
(pdlp_test.cu:717-772): the returned l2 primal residual is smaller with the flag than without."""
import pytest

from conftest import mps_path, problem_arrays
from cuopt_b200 import capi
from oracle import pdlp_oracle as po

CASES = [("mip/50v-10-free-bound.mps", 300), ("mip/neos5-free-bound.mps", 200), ("linear_programming/afiro_original.mps", 100)]


def oracle_run(a, limit, flag):
    o = po.Oracle(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"],
                  maximize=a["maximize"], objective_offset=a["objective_offset"], tol=1e-8, iteration_limit=limit,
                  save_best_primal_so_far=flag)
    assert o.run(-1)
    return o.stats()


def relaxed(rel):
    from cases import lp_relaxation
    return lp_relaxation(rel)


@pytest.mark.parametrize("rel,limit", CASES)
def test_oracle_returns_a_better_primal_point_at_the_iteration_limit(rel, limit):
    a = problem_arrays(capi.Problem.read(mps_path(rel)))
    plain, best = oracle_run(a, limit, False), oracle_run(a, limit, True)
    assert plain.termination_status == best.termination_status == 4
    assert best.l2_primal_residual < plain.l2_primal_residual
    assert best.number_of_steps_taken <= plain.number_of_steps_taken   # stats are those of the recorded iterate


@pytest.mark.gpu
@pytest.mark.parametrize("rel,limit", CASES)
def test_gpu_matches_the_oracle(rel, limit):
    p = relaxed(rel)
    a = problem_arrays(p)
    want = oracle_run(a, limit, True)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, iteration_limit=limit,
                      save_best_primal_so_far=True)
    s.set("optimality_tolerance", 1e-8)
    sol = capi.solve(p, s)
    assert sol.return_code == 0 and sol.termination_status == 4
    st = sol.stats()
    assert st.number_of_steps_taken == want.number_of_steps_taken
    # same recorded iterate (equal step counts); values to the drift of a 100-300 step trajectory on these degenerate
    # relaxations
    assert st.l2_primal_residual == pytest.approx(want.l2_primal_residual, rel=1e-4, abs=1e-9)
    assert st.primal_objective == pytest.approx(want.primal_objective, rel=1e-4, abs=1e-9)
