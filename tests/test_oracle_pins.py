"""Pins the CPU oracle (oracle/pdlp_oracle.cpp) to the reference's OWN known answers before anything trusts it.

Sources of truth (all committed under tests/golden/, produced by scripts/gen_golden.py):
  reference_pins.json  values copied from the reference's tests (file:line inside the json)
  simplex_golden.json  optimal objectives computed by the reference's CPU dual simplex in this container
"""
import numpy as np
import pytest

from cases import RANGED_LP, c_api_infeasible_lp, unbounded_lp
from conftest import load_golden, mps_path, problem_arrays
from cuopt_b200 import capi
from oracle import pdlp_oracle as po


def oracle_for(rel, **kw):
    p = capi.Problem.read(mps_path(rel))
    a = problem_arrays(p)
    return po.Oracle(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"],
                     a["con_ub"], maximize=a["maximize"], objective_offset=a["objective_offset"], **kw), p


def test_afiro_methodical1_initial_step_size_and_primal_weight(pins):
    # cpp/tests/linear_programming/pdlp_test.cu:237-283 (iteration_limit 0, Methodical1)
    o, _ = oracle_for("linear_programming/afiro_original.mps", mode=po.METHODICAL1, iteration_limit=0)
    o.initialise()
    s, w = pins["afiro_methodical1_initial_step_size"], pins["afiro_methodical1_initial_primal_weight"]
    assert abs(o.scalar("step_size") - s["value"]) <= s["abs"]
    assert abs(o.scalar("primal_weight") - w["value"]) <= w["abs"]


def test_afiro_default_settings_primal_vector(pins):
    # python/cuopt/cuopt/tests/linear_programming/test_lp_solver.py:430-476: 32 named values, rel 1e-4
    o, p = oracle_for("linear_programming/afiro_original.mps")
    r = o.solve()
    assert r["status"] == "Optimal"
    want = pins["afiro_default_primal"]
    names = ["X01", "X02", "X03", "X04", "X06", "X07", "X08", "X09", "X10", "X11", "X12", "X13", "X14", "X15", "X16",
             "X22", "X23", "X24", "X25", "X26", "X28", "X29", "X30", "X31", "X32", "X33", "X34", "X35", "X36", "X37",
             "X38", "X39"]  # variable order of afiro_original.mps (test_lp_solver.py:395-428)
    assert len(names) == p.num_variables == len(want["values"])
    for name, got in zip(names, r["x"]):
        assert got == pytest.approx(want["values"][name], rel=want["rel"]), name


def test_afiro_objective_tight(pins):
    o, _ = oracle_for("linear_programming/afiro_original.mps", tol=1e-10, iteration_limit=100000)
    r = o.solve()
    assert r["status"] == "Optimal"
    assert r["primal_objective"] == pytest.approx(pins["afiro_objective"]["value"], rel=pins["afiro_objective"]["rel"])
    assert r["primal_objective"] == pytest.approx(-464.75314285714285, rel=1e-8)  # reference dual simplex


@pytest.mark.parametrize("rel,key", [("linear_programming/good-max.mps", "good_max_objective"),
                                     ("linear_programming/max_offset.mps", "max_offset_objective")])
def test_maximisation_pins(pins, rel, key):
    # pdlp_test.cu:909-943
    o, _ = oracle_for(rel)
    r = o.solve()
    assert r["status"] == "Optimal"
    assert abs(r["primal_objective"] - pins[key]["value"]) <= pins[key]["abs"]


def test_c_api_ranged_problem(pins):
    # c_api_test.c:761-874 / c_api_tests.cpp:89-96: maximize 5x + 8y ; 2x+3y <= 12 ; 3x+y <= 6 ; 2 <= x+2y <= 8 ;
    # 0 <= x,y <= 10  -> objective 32.0 +- 1e-3
    d = RANGED_LP
    o = po.Oracle(d["offsets"], d["indices"], d["values"], d["c"], d["var_lb"], d["var_ub"], d["con_lb"], d["con_ub"],
                  maximize=True, tol=1e-6)
    r = o.solve()
    assert r["status"] == "Optimal"
    want = pins["c_api_ranged_objective"]
    assert abs(r["primal_objective"] - want["value"]) <= want["abs"]


# (instance, PDLP tolerance, objective tolerance).  minrep_inf is a 6x4 big-M LP on which PDLP stalls below 1e-6.
SIMPLEX_CASES = [("linear_programming/afiro_original.mps", 1e-8, 1e-6), ("mip/50v-10-free-bound.mps", 1e-8, 1e-6),
                 ("mip/neos5-free-bound.mps", 1e-8, 1e-6), ("mip/sudoku.mps", 1e-8, 1e-6),
                 ("mip/cod105_max.mps", 1e-8, 1e-6), ("mip/sample.mps", 1e-8, 1e-6),
                 ("mip/minrep_inf.mps", 1e-6, 2e-5), ("mip/bb_optimality.mps", 1e-8, 1e-6),
                 ("linear_programming/good-mps-some-var-bounds.mps", 1e-8, 1e-6),
                 ("linear_programming/lp_model_with_var_bounds.mps", 1e-8, 1e-6)]


@pytest.mark.parametrize("rel,tol,otol", SIMPLEX_CASES)
def test_objective_matches_reference_dual_simplex(simplex_golden, rel, tol, otol):
    want = simplex_golden[rel]
    assert want["status"] == "OPTIMAL"
    o, _ = oracle_for(rel, tol=tol, iteration_limit=400000)
    r = o.solve()
    assert r["status"] == "Optimal", r
    assert r["primal_objective"] == pytest.approx(want["objective"], rel=otol, abs=otol)
    assert r["dual_objective"] == pytest.approx(want["objective"], rel=otol, abs=otol)


def test_methodical1_very_low_tolerance_afiro():
    """python/cuopt/cuopt/tests/linear_programming/test_lp_solver.py:101-121 (test_very_low_tolerance): Methodical1
    (trust-region restart), optimality tolerance 1e-12, no infeasibility detection -> Optimal, objective -464.7531."""
    o, _ = oracle_for("linear_programming/afiro_original.mps", mode=po.METHODICAL1, tol=1e-12, iteration_limit=2000000)
    r = o.solve()
    assert r["status"] == "Optimal"
    assert r["primal_objective"] == pytest.approx(-464.7531)          # the reference's assertion (rel 1e-6)
    assert r["primal_objective"] == pytest.approx(-464.75314285714285, rel=1e-10)
    assert o.stats().n_restarts >= 1                                  # the trust-region rule did fire


@pytest.mark.parametrize("rel,tol,otol", [c for c in SIMPLEX_CASES if "minrep" not in c[0]])
def test_methodical1_objective_matches_reference_dual_simplex(simplex_golden, rel, tol, otol):
    want = simplex_golden[rel]
    o, _ = oracle_for(rel, mode=po.METHODICAL1, tol=tol, iteration_limit=400000)
    r = o.solve()
    assert r["status"] == "Optimal", r
    assert r["primal_objective"] == pytest.approx(want["objective"], rel=otol, abs=otol)
    assert r["dual_objective"] == pytest.approx(want["objective"], rel=otol, abs=otol)


@pytest.mark.parametrize("mode", [po.STABLE1, po.STABLE2, po.FAST1, po.METHODICAL1])
def test_presets_converge_on_afiro(mode):
    o, _ = oracle_for("linear_programming/afiro_original.mps", mode=mode, tol=1e-8, iteration_limit=200000)
    r = o.solve()
    assert r["status"] == "Optimal"
    assert r["primal_objective"] == pytest.approx(-464.75314285714285, rel=1e-6)


def test_iteration_limit_and_determinism():
    o, _ = oracle_for("mip/50v-10-free-bound.mps", iteration_limit=1)  # c_api_tests: iteration limit 1 -> IterationLimit
    r = o.solve()
    assert r["status"] == "IterationLimit"
    a, _ = oracle_for("mip/50v-10-free-bound.mps", tol=1e-6)
    b, _ = oracle_for("mip/50v-10-free-bound.mps", tol=1e-6)
    ra, rb = a.solve(), b.solve()
    assert ra["iterations"] == rb["iterations"] and np.array_equal(ra["x"], rb["x"])


def test_warm_start_style_additivity_of_stepping():
    # the oracle can be advanced in pieces (used by the GPU trajectory tests): 25+15 steps == 40 steps
    a, _ = oracle_for("mip/sudoku.mps")
    b, _ = oracle_for("mip/sudoku.mps")
    a.run(25); a.run(15)
    b.run(40)
    assert np.array_equal(a.vector("x"), b.vector("x")) and a.scalar("step_size") == b.scalar("step_size")


def test_pds_shaped_lp_against_reference_dual_simplex():
    """configs[2] shape (multicommodity flow, synthesised): the oracle's PDLP against the optimal objective the
    reference's own CPU dual simplex found (tests/golden/c3_reference_simplex.json, scripts/gen_golden_c3.py)."""
    import json
    import os
    from cuopt_b200 import lpgen
    with open(os.path.join(os.path.dirname(__file__), "golden", "c3_reference_simplex.json")) as f:
        case = json.load(f)["cases"][0]
    lp = lpgen.multicommodity(nodes=case["nodes"], arcs=case["arcs"], commodities=11, seed=1234)
    assert (lp.m, lp.n, lp.nnz) == (case["rows"], case["cols"], case["nnz"])
    o = po.Oracle(lp.offsets, lp.indices, lp.values, lp.c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub, tol=1e-6)
    assert o.run(-1)
    assert o.stats().termination_status == 1
    assert o.stats().primal_objective == pytest.approx(case["objective"], rel=1e-5)
    assert o.stats().dual_objective == pytest.approx(case["objective"], rel=1e-5)


# ------------------------------------------------------------------ infeasibility detection (oracle only so far)
@pytest.mark.parametrize("strict", [False, True])
def test_infeasibility_detection_on_the_reference_c_api_infeasible_lp(strict):
    off, idx, val, c, l, u, lc, uc = c_api_infeasible_lp()
    # the reference's own verdict on it (its test expects CUOPT_TERIMINATION_STATUS_INFEASIBLE from the dual simplex)
    assert reference_verdict("c_api_infeasible_lp", off, idx, val, c, l, u, lc, uc) == "INFEASIBLE"
    o = po.Oracle(off, idx, val, c, l, u, lc, uc, tol=1e-4, detect_infeasibility=True, strict_infeasibility=strict,
                  iteration_limit=100000)
    assert o.run(-1)
    assert o.stats().termination_status == 2   # PrimalInfeasible == CUOPT_TERIMINATION_STATUS_INFEASIBLE
    # without detection PDLP cannot say so: it runs into its limit
    o = po.Oracle(off, idx, val, c, l, u, lc, uc, tol=1e-4, iteration_limit=2000)
    assert o.run(-1)
    assert o.stats().termination_status == 4


def reference_verdict(name, off, idx, val, c, l, u, lc, uc):
    """The reference CPU dual simplex's status: run live where oracle/_ref is built, else as stored by
    scripts/gen_golden_writer.py."""
    from oracle import ref_cpu
    if ref_cpu.available():
        return ref_cpu.dual_simplex(off, idx, val, lc, uc, c, l, u)["status"]
    return load_golden("writer_golden.json")["verdicts"][name]


def test_infeasibility_detection_flags_an_unbounded_lp():
    args = unbounded_lp()
    assert reference_verdict("unbounded_lp", *args) == "UNBOUNDED"
    o = po.Oracle(*args, tol=1e-4, detect_infeasibility=True, strict_infeasibility=True, iteration_limit=100000)
    assert o.run(-1)
    assert o.stats().termination_status == 3   # DualInfeasible == CUOPT_TERIMINATION_STATUS_UNBOUNDED
