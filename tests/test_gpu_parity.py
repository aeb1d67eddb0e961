"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle on the same inputs, against the
committed golden fixtures, and - at full BASELINE sizes - through size-independent properties.

fp64 tolerances (stated once, used below):
  ELEMENTWISE  1e-12 relative : vectors after a fixed number of PDHG steps from the same state (the only difference
                                is summation order inside SpMV rows / reductions and libm ulps in pow/log/exp)
  TRAJECTORY   1e-7  relative : state after tens of iterations including restarts
  OBJECTIVE    1e-6  relative : final objectives vs the reference's CPU dual simplex at PDLP tolerance <= 1e-8
  ITERATIONS   within one major iteration (40) of the oracle; +-30 % on the two degenerate MIP relaxations
                                (iteration counts are not pinned by any reference test)
"""
import numpy as np
import pytest

from cases import RANGED_LP, lp_relaxation, make_pair, problem_of as lp_problem
from conftest import has_gpu, load_golden, mps_path, problem_arrays
from cuopt_b200 import capi, lpgen
from device_model import gather_block_bytes  # noqa: F401
from exact import ELEMENTWISE, OBJECTIVE, TRAJECTORY, rel_err
from oracle import pdlp_oracle as po

pytestmark = pytest.mark.gpu


SMALL = ["linear_programming/afiro_original.mps", "mip/50v-10-free-bound.mps", "mip/sudoku.mps",
         "mip/neos5-free-bound.mps"]


@pytest.mark.parametrize("rel", SMALL + ["mip/cod105_max.mps"])
@pytest.mark.parametrize("mode", [0, 1, 3])
def test_scaling_and_initial_step_match_oracle(rel, mode):
    g, o, _ = make_pair(capi.Problem.read(mps_path(rel)), mode=mode)
    g.initialise(); o.initialise()
    for name in ("row_scaling", "col_scaling", "scaled_values", "scaled_values_t", "scaled_c", "scaled_lc", "scaled_uc"):
        gv, ov = g.vector(name), o.vector(name)
        fin = np.isfinite(ov)
        assert np.array_equal(np.isfinite(gv), fin), name
        assert rel_err(gv[fin], ov[fin]) <= ELEMENTWISE, name
    for name in ("step_size", "primal_weight", "l2_norm_b", "l2_norm_c"):
        assert g.scalar(name) == pytest.approx(o.scalar(name), rel=1e-13), name


def test_afiro_methodical1_initial_values_pin(pins):
    # reference test pdlp_test.cu:237-283, evaluated on the GPU path (initialisation does not need the restart scheme)
    p = capi.Problem.read(mps_path("linear_programming/afiro_original.mps"))
    g = capi.Solver(p, capi.Settings(pdlp_solver_mode=capi.CUOPT_PDLP_SOLVER_MODE_METHODICAL1, log_to_console=False))
    g.initialise()
    assert abs(g.scalar("step_size") - pins["afiro_methodical1_initial_step_size"]["value"]) <= 1e-4
    assert abs(g.scalar("primal_weight") - pins["afiro_methodical1_initial_primal_weight"]["value"]) <= 1e-4


@pytest.mark.parametrize("rel", SMALL)
def test_first_steps_match_oracle_elementwise(rel):
    g, o, _ = make_pair(capi.Problem.read(mps_path(rel)))
    for steps in (1, 1, 3):
        g.advance(steps); o.run(steps)
        for name in ("x", "y", "aty", "sum_x", "sum_y"):
            assert rel_err(g.vector(name), o.vector(name)) <= 1e-11, (name, steps)
        for name in ("step_size", "primal_weight", "sum_w"):
            assert g.scalar(name) == pytest.approx(o.scalar(name), rel=1e-11), name
        assert g.scalar("k_pdhg") == o.scalar("k_pdhg")


@pytest.mark.parametrize("seed", [1, 2])
def test_single_attempt_kernels_on_synthetic(seed):
    # kernel-level parity at a size with thousands of row blocks: K1+K2+K3 of ONE attempt vs the oracle's
    # primal_projection / dual_projection / interaction_and_movement from the same state
    lp = lpgen.sparse_lp(60_000, 50_000, 8, seed=seed)
    g, o, _ = make_pair(lp_problem(lp))
    g.advance(7); o.run(7)  # a non-trivial state
    x, y, aty = g.vector("x"), g.vector("y"), g.vector("aty")
    want = o.single_attempt(x, y, aty, g.scalar("tau"), g.scalar("sigma"))
    g.advance(1)
    # after one more accepted step the GPU "current" buffers hold x', y', A^T y'
    if g.scalar("k_pdhg") == 8:
        assert rel_err(g.vector("x"), want["x_next"]) <= ELEMENTWISE
        assert rel_err(g.vector("y"), want["y_next"]) <= ELEMENTWISE
        assert rel_err(g.vector("aty"), want["aty_next"]) <= 1e-11
        assert g.scalar("norm_dx2") == pytest.approx(want["norm_dx2"], rel=1e-11)
        assert g.scalar("norm_dy2") == pytest.approx(want["norm_dy2"], rel=1e-11)
        assert g.scalar("interaction") == pytest.approx(want["interaction"], rel=1e-9, abs=1e-9 * want["norm_dx2"])


@pytest.mark.parametrize("rel", SMALL)
def test_trajectory_with_restarts_matches_oracle(rel):
    g, o, _ = make_pair(capi.Problem.read(mps_path(rel)), tol=1e-12)
    g.advance(120); o.run(120)  # crosses major iterations 40, 80, 120 and several KKT restarts
    assert g.scalar("n_restarts") == o.scalar("n_restarts")
    assert g.scalar("k_pdhg") == o.scalar("k_pdhg")
    for name in ("x", "y"):
        assert rel_err(g.vector(name), o.vector(name)) <= TRAJECTORY, name
    assert g.scalar("primal_weight") == pytest.approx(o.scalar("primal_weight"), rel=TRAJECTORY)
    assert g.scalar("step_size") == pytest.approx(o.scalar("step_size"), rel=TRAJECTORY)


def solve_capi(p, expect_ok=True, **kw):
    tol = kw.pop("tol", 1e-4)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, **kw)
    s.set("optimality_tolerance", tol)
    sol = capi.solve(p, s)
    if expect_ok:
        assert sol.return_code == 0, f"cuOptSolve error {sol.return_code}: {sol.error_string}"
    return sol


def test_afiro_default_settings_golden_vector(pins):
    # test_lp_solver.py:430-476 through cuOptReadProblem + cuOptSolve + cuOptGetPrimalSolution
    p = capi.Problem.read(mps_path("linear_programming/afiro_original.mps"))
    sol = capi.solve(p, capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False))
    assert sol.return_code == 0 and sol.termination_reason == "Optimal"
    want = list(pins["afiro_default_primal"]["values"].values())
    got = sol.primal()
    # json preserves the reference test's dict order == variable order of the file
    for g_, w_ in zip(got, want):
        assert g_ == pytest.approx(w_, rel=1e-4)
    assert sol.objective_value == pytest.approx(-464.0, rel=1e-2)  # pdlp_test.cu:58-84


def test_afiro_tight_tolerance_objective(pins):
    # pdlp_test.cu:86-110 (tolerance floor still converges) / test_lp_solver.py:101-121
    p = capi.Problem.read(mps_path("linear_programming/afiro_original.mps"))
    sol = solve_capi(p, tol=1e-10)
    assert sol.termination_reason == "Optimal"
    assert sol.objective_value == pytest.approx(pins["afiro_objective"]["value"], rel=1e-6)


@pytest.mark.parametrize("rel,key", [("linear_programming/good-max.mps", "good_max_objective"),
                                     ("linear_programming/max_offset.mps", "max_offset_objective")])
def test_maximisation_pins(pins, rel, key):
    sol = solve_capi(capi.Problem.read(mps_path(rel)))
    assert sol.termination_reason == "Optimal"
    assert abs(sol.objective_value - pins[key]["value"]) <= pins[key]["abs"]


def test_c_api_ranged_problem(pins):
    d = RANGED_LP
    p = capi.Problem.create_ranged(d["offsets"], d["indices"], d["values"], d["con_lb"], d["con_ub"], d["c"],
                                   d["var_lb"], d["var_ub"], maximize=True)
    sol = solve_capi(p, tol=1e-6)
    assert sol.termination_reason == "Optimal"
    assert abs(sol.objective_value - pins["c_api_ranged_objective"]["value"]) <= pins["c_api_ranged_objective"]["abs"]


CASES = [("linear_programming/afiro_original.mps", 1e-8, 1e-6), ("mip/50v-10-free-bound.mps", 1e-8, 1e-6),
         ("mip/neos5-free-bound.mps", 1e-8, 1e-6), ("mip/sudoku.mps", 1e-8, 1e-6), ("mip/cod105_max.mps", 1e-8, 1e-6),
         ("mip/sample.mps", 1e-8, 1e-6), ("mip/bb_optimality.mps", 1e-8, 1e-6)]


@pytest.mark.parametrize("rel,tol,otol", CASES)
def test_full_solve_vs_reference_simplex_and_oracle(simplex_golden, rel, tol, otol):
    # configs[0] and configs[4]: LP (relaxations) from the reference's datasets, PDLP to tolerance
    p = lp_relaxation(rel)
    sol = solve_capi(p, tol=tol, iteration_limit=400000)
    assert sol.termination_reason == "Optimal"
    want = simplex_golden[rel]["objective"]
    st = sol.stats()
    assert st.primal_objective == pytest.approx(want, rel=otol, abs=otol)
    assert st.dual_objective == pytest.approx(want, rel=otol, abs=otol)
    a = problem_arrays(p)
    o = po.Oracle(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"],
                  maximize=a["maximize"], objective_offset=a["objective_offset"], tol=tol, iteration_limit=400000)
    r = o.solve()
    assert r["status"] == "Optimal"
    # iteration counts: identical on most instances; the two degenerate MIP
    # relaxations (50v-10, neos5) drift chaotically at deep tolerances: summation order flips a restart decision
    band = 0.30 if rel in ("mip/50v-10-free-bound.mps", "mip/neos5-free-bound.mps") else 0.0
    assert abs(st.number_of_steps_taken - r["iterations"]) <= max(40, band * r["iterations"])
    # post-solve invariants the reference checks on the CPU (pdlp_test_utilities.cuh:42-139)
    x = sol.primal()
    sign = -1.0 if a["maximize"] else 1.0
    assert float(a["c"] @ x) + a["objective_offset"] == pytest.approx(st.primal_objective, rel=1e-6, abs=1e-6)
    import scipy.sparse as sp
    A = sp.csr_matrix((a["values"], a["indices"], a["offsets"]), shape=(len(a["con_lb"]), len(a["c"])))
    ax = A @ x
    viol = np.maximum(a["con_lb"] - ax, 0) + np.maximum(ax - a["con_ub"], 0)
    assert np.linalg.norm(viol) == pytest.approx(st.l2_primal_residual, abs=1e-6)
    assert np.all(x >= a["var_lb"] - 1e-6) and np.all(x <= a["var_ub"] + 1e-6)
    del sign


@pytest.mark.parametrize("mode", [0, 3])
def test_other_kkt_presets(mode):
    p = capi.Problem.read(mps_path("linear_programming/afiro_original.mps"))
    sol = solve_capi(p, tol=1e-8, pdlp_solver_mode=mode)
    assert sol.termination_reason == "Optimal"
    assert sol.objective_value == pytest.approx(-464.75314285714285, rel=1e-6)


def test_limits_and_error_paths():
    p = lp_relaxation("mip/50v-10-free-bound.mps")
    sol = solve_capi(p, iteration_limit=1)  # c_api_tests: iteration limit 1
    assert sol.termination_status == 4 and sol.return_code == 0
    sol = solve_capi(p, tol=1e-12, time_limit=0.05)
    assert sol.termination_status in (5, 1)
    assert sol.solve_time < 5.0
    # empty matrix -> NumericalError (pdlp_test.cu:875-889)
    pe = capi.Problem.read(mps_path("linear_programming/empty_matrix.mps"))
    se = solve_capi(pe)
    assert se.termination_status == 6
    # Methodical1 (trust-region restart) is a regular preset since round 2: tests/test_methodical1.py
    sm = solve_capi(capi.Problem.read(mps_path("linear_programming/afiro_original.mps")), pdlp_solver_mode=2)
    assert sm.return_code == 0 and sm.termination_status == 1


def test_run_to_run_determinism_and_graph_equivalence(monkeypatch):
    lp = lpgen.sparse_lp(30_000, 30_000, 8, seed=5)
    p = lp_problem(lp)
    a = solve_capi(p, tol=1e-6, iteration_limit=800)
    b = solve_capi(p, tol=1e-6, iteration_limit=800)
    assert a.stats().number_of_steps_taken == b.stats().number_of_steps_taken
    assert np.array_equal(a.primal(), b.primal()) and np.array_equal(a.dual(), b.dual())
    monkeypatch.setenv("CUOPT_B200_NO_GRAPH", "1")
    c = solve_capi(p, tol=1e-6, iteration_limit=800)
    assert np.array_equal(a.primal(), c.primal())


def test_synthetic_planted_optimum_medium():
    # configs[1] generator at 1/10 size, compared with the closed-form optimum and the oracle
    lp = lpgen.sparse_lp(100_000, 100_000, 8, seed=1234)
    p = lp_problem(lp)
    sol = solve_capi(p, tol=1e-8, iteration_limit=200000)
    assert sol.termination_reason == "Optimal"
    assert sol.objective_value == pytest.approx(lp.optimal_objective, rel=OBJECTIVE)
    assert sol.stats().dual_objective == pytest.approx(lp.optimal_objective, rel=OBJECTIVE)


@pytest.mark.slow
def test_full_size_config1_properties():
    # configs[1] at full size (1M x 1M, 8 nnz/row): size-independent properties
    lp = lpgen.sparse_lp(1_000_000, 1_000_000, 8, seed=1234)
    p = lp_problem(lp)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False)
    s.set("optimality_tolerance", 1e-4)
    g = capi.Solver(p, s)
    g.initialise()
    # (1) linearity of the fused SpMV: A^T y computed by K3 equals scipy's product with the scaled matrix
    g.advance(41)
    import scipy.sparse as sp
    dr, dc = g.vector("row_scaling"), g.vector("col_scaling")
    A = sp.csr_matrix((lp.values, lp.indices, lp.offsets), shape=(lp.m, lp.n))
    As = sp.diags(dr) @ A @ sp.diags(dc)
    y, aty = g.vector("y"), g.vector("aty")
    assert rel_err(aty, As.T @ y) <= 1e-11
    # (2) running sums: sum_x / sum_w is a convex combination of iterates => inside the variable bounds
    sx = g.vector("sum_x") / g.scalar("sum_w")
    assert np.all(sx >= g.vector("scaled_l") - 1e-9)
    # (3) convergence to the planted optimum through the plain C ABI
    sol = solve_capi(p, tol=1e-6, iteration_limit=100000)
    assert sol.termination_reason == "Optimal"
    assert sol.objective_value == pytest.approx(lp.optimal_objective, rel=1e-5)


# ---------------------------------------------------------------------------------- gather blocking (large-LP path)
@pytest.mark.parametrize("mode", [1, 3])
def test_blocked_kernels_follow_the_oracle_step_by_step(gather_block_bytes, mode):
    lp = lpgen.sparse_lp(3000, 2500, 6, seed=11)
    gather_block_bytes(8 * 2500 / 3.2)  # 4 column blocks for A (n = 2500), 4-5 for A^T (m = 3000)
    g, o, _ = make_pair(lp_problem(lp), mode=mode, tol=1e-9)
    g.initialise(); o.initialise()
    for steps in (1, 7, 33):
        g.advance(steps); o.run(steps)
        for name in ("x", "y", "aty", "sum_x", "sum_y"):
            assert rel_err(g.vector(name), o.vector(name)) <= TRAJECTORY, (steps, name)
        for name in ("step_size", "primal_weight", "k_total", "its_since_restart"):
            assert g.scalar(name) == pytest.approx(o.scalar(name), rel=1e-9), (steps, name)


def test_blocked_and_fused_paths_solve_identically(gather_block_bytes):
    """Fused kernels vs gather-blocked passes (+ fused last pass) on the same LP, solved to 1e-8: the same optimum to 1e-6 in
    the objective (at tolerance 1e-6 two such runs can differ by far more than 1e-6, which says nothing; at 1e-8 the bound
    holds).  Iteration counts still react to last-bit differences through the restart decisions."""
    for lp in (lpgen.sparse_lp(3000, 2500, 6, seed=11), lpgen.multicommodity(60, 200, 4, seed=2)):
        p = lp_problem(lp)
        s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False)
        s.set("optimality_tolerance", 1e-8)
        gather_block_bytes(None)
        fused = capi.solve(p, s)
        gather_block_bytes(8 * lp.n / 2.5)
        blocked = capi.solve(p, s)
        assert fused.termination_status == blocked.termination_status == 1
        fs, bs = fused.stats(), blocked.stats()
        assert abs(bs.number_of_steps_taken - fs.number_of_steps_taken) <= max(40, 0.4 * fs.number_of_steps_taken)
        assert bs.primal_objective == pytest.approx(fs.primal_objective, rel=OBJECTIVE, abs=1e-9)
        assert bs.dual_objective == pytest.approx(fs.dual_objective, rel=OBJECTIVE, abs=1e-9)
        assert np.linalg.norm(blocked.primal() - fused.primal()) <= 1e-3 * max(1.0, np.linalg.norm(fused.primal()))


def test_pds_shaped_config2_against_reference_dual_simplex():
    """configs[2]: the three pds-shaped multicommodity LPs (up to 126K x 297K, 0.89M nnz) solved to 1e-6 through the C
    ABI, against the optimal objectives of the reference's own CPU dual simplex (tests/golden/c3_reference_simplex.json;
    the largest took the simplex 41.7 s on one host core)."""
    import json
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "c3_reference_simplex.json")) as f:
        cases = json.load(f)["cases"]
    for case in cases:
        lp = lpgen.multicommodity(nodes=case["nodes"], arcs=case["arcs"], commodities=11, seed=1234)
        s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False)
        s.set("optimality_tolerance", 1e-6)
        sol = capi.solve(lp_problem(lp), s)
        assert sol.termination_status == 1
        st = sol.stats()
        assert st.primal_objective == pytest.approx(case["objective"], rel=1e-4)
        assert st.dual_objective == pytest.approx(case["objective"], rel=1e-4)
