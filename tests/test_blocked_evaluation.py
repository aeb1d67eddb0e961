"""Termination evaluation and the restart's A^T y on gather-blocked matrices.

With gather blocking on, the evaluation forms A [x, x_avg] and A^T [y, y_avg] over the column blocks of the UNSCALED matrix,
both iterates in one stream of each block, and a restart to the average rebuilds A^T y with the same column-block passes
that K3 runs.  Blocking is forced on small LPs with CUOPT_B200_GATHER_BLOCK_BYTES, as in test_gpu_parity.py.  Blocked and
fused runs differ only in the summation order of row sums, so their evaluations agree to 1e-12 relative."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import problem_arrays
from cuopt_b200 import capi, lpgen
from exact import ELEMENTWISE, rel_err

pytestmark = pytest.mark.gpu

STATS = ("primal_objective", "dual_objective", "gap", "l2_primal_residual", "l2_dual_residual")


def problem(lp, **changes):
    a = dict(offsets=lp.offsets, indices=lp.indices, values=lp.values, con_lb=lp.con_lb, con_ub=lp.con_ub, c=lp.c,
             var_lb=lp.var_lb, var_ub=lp.var_ub)
    a.update(changes)
    return capi.Problem.create_ranged(a["offsets"], a["indices"], a["values"], a["con_lb"], a["con_ub"], a["c"],
                                      a["var_lb"], a["var_ub"])


def solve_fused_and_blocked(p, n, monkeypatch, **settings):
    out = []
    for nbytes in (None, 8 * n / 2.5):  # unblocked, then 3 column blocks of A and 3 of A^T
        if nbytes is None:
            monkeypatch.delenv("CUOPT_B200_GATHER_BLOCK_BYTES", raising=False)
        else:
            monkeypatch.setenv("CUOPT_B200_GATHER_BLOCK_BYTES", str(int(nbytes)))
        s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, **settings)
        sol = capi.solve(p, s)
        assert sol.return_code == 0, sol.error_string
        out.append(sol)
    monkeypatch.delenv("CUOPT_B200_GATHER_BLOCK_BYTES", raising=False)
    return out


def assert_same_evaluation(fused, blocked):
    assert blocked.termination_status == fused.termination_status
    fs, bs = fused.stats(), blocked.stats()
    assert bs.number_of_steps_taken == fs.number_of_steps_taken
    for name in STATS:
        f, b = getattr(fs, name), getattr(bs, name)
        assert b == pytest.approx(f, rel=ELEMENTWISE, abs=ELEMENTWISE), name
    assert rel_err(blocked.reduced_costs(), fused.reduced_costs()) <= ELEMENTWISE
    assert rel_err(blocked.primal(), fused.primal()) <= ELEMENTWISE
    assert rel_err(blocked.dual(), fused.dual()) <= ELEMENTWISE


@pytest.mark.parametrize("iterations", [1, 8, 12])
def test_blocked_evaluation_matches_unblocked(iterations, monkeypatch):
    """Iterations 1..10 are all major iterations: every step is evaluated, and restarts follow from the evaluations."""
    lp = lpgen.sparse_lp(3000, 2500, 6, seed=11)
    fused, blocked = solve_fused_and_blocked(problem(lp), lp.n, monkeypatch, iteration_limit=iterations)
    assert fused.termination_reason == "IterationLimit"
    assert_same_evaluation(fused, blocked)


@pytest.mark.parametrize("infeasible", [False, True])
def test_blocked_evaluation_with_detection_and_per_constraint_residual(infeasible, monkeypatch):
    lp = lpgen.sparse_lp(3000, 2500, 6, seed=5)
    changes = {}
    if infeasible:  # every variable fixed at 0, yet row 0 asks for A_0 x >= 1
        lb = np.array(lp.con_lb, float).copy()
        ub = np.array(lp.con_ub, float).copy()
        lb[0], ub[0] = 1.0, np.inf
        changes = dict(var_lb=np.zeros(lp.n), var_ub=np.zeros(lp.n), con_lb=lb, con_ub=ub)
    fused, blocked = solve_fused_and_blocked(problem(lp, **changes), lp.n, monkeypatch, iteration_limit=40,
                                             infeasibility_detection=True, strict_infeasibility=True,
                                             per_constraint_residual=True)
    assert_same_evaluation(fused, blocked)


def blocked_session(lp, monkeypatch, nbytes):
    monkeypatch.setenv("CUOPT_B200_GATHER_BLOCK_BYTES", str(int(nbytes)))
    p = problem(lp)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False)
    s.set("optimality_tolerance", 1e-9)
    g = capi.Solver(p, s)
    g.initialise()
    monkeypatch.delenv("CUOPT_B200_GATHER_BLOCK_BYTES", raising=False)
    return p, g


def test_blocked_solve_evaluates_over_the_unscaled_column_blocks(monkeypatch):
    """The blocked runs compared above really evaluate over column blocks (3 of A, 3 of A^T here); an unblocked one in a
    single pass."""
    lp = lpgen.sparse_lp(3000, 2500, 6, seed=11)
    _, g = blocked_session(lp, monkeypatch, 8 * lp.n / 2.5)
    assert g.scalar("eval_blocks") == 3
    assert g.scalar("eval_blocks_t") == 3
    g = capi.Solver(problem(lp), capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False))
    g.initialise()
    assert g.scalar("eval_blocks") == g.scalar("eval_blocks_t") == 1


def test_restart_to_average_rebuilds_aty_over_the_column_blocks(monkeypatch):
    """After a restart to the average the next primal step uses A^T y of the new y, summed over the column blocks.  Checked
    through that step: x' = clamp(x - tau (c - A^T y), l, u) on the scaled problem, for every step taken right after a
    restart to the average."""
    lp = lpgen.sparse_lp(3000, 2500, 6, seed=11)
    p, g = blocked_session(lp, monkeypatch, 8 * lp.n / 3.2)
    assert g.scalar("eval_blocks_t") > 1
    a = problem_arrays(p)
    m, n = len(a["con_lb"]), len(a["c"])
    AT = sp.csr_matrix((g.vector("scaled_values"), a["indices"], a["offsets"]), shape=(m, n)).T.tocsr()
    c, l, u = g.vector("scaled_c"), g.vector("scaled_l"), g.vector("scaled_u")
    checked = 0
    for _ in range(60):
        restarts = g.scalar("n_restarts")
        g.advance(1)
        if g.scalar("n_restarts") == restarts or g.scalar("last_restart_was_average") != 1.0:
            continue
        aty = AT @ g.vector("y")
        x, tau, attempts, restarts = g.vector("x"), g.scalar("tau"), g.scalar("k_pdhg"), g.scalar("n_restarts")
        g.advance(1)
        if g.scalar("k_pdhg") != attempts + 1 or g.scalar("n_restarts") != restarts:
            continue  # the first attempt was rejected, or this step ended in another restart
        want = np.maximum(np.minimum(x - tau * (c - aty), u), l)
        assert rel_err(g.vector("x"), want) <= ELEMENTWISE
        checked += 1
    assert checked > 0
