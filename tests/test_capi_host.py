"""Host-side behaviour of the C ABI (no GPU needed): symbol export, handle lifecycle, problem getters,
parameter registry.  Mirrors cpp/tests/linear_programming/c_api_tests/c_api_test.c (test_int_size,
test_float_size, check_problem round-trips, invalid-parameter handling) of the reference."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from cases import RANGED_LP
from conftest import ROOT
from cuopt_b200 import capi

INF = float("inf")


def test_library_loads_and_exports_every_declared_symbol():
    L = capi.lib()
    for s in capi.REFERENCE_SYMBOLS + capi.EXTENSION_SYMBOLS:
        assert hasattr(L, s), s
    # every function the two public headers declare is in the lists above (and hence exported)
    declared = set()
    for hdr in ("include/cuopt/linear_programming/cuopt_c.h", "include/cuopt_b200/cuopt_b200_ext.h"):
        text = open(os.path.join(ROOT, hdr)).read()
        declared |= set(re.findall(r"\b(cuOpt[A-Za-z0-9]+)\s*\(", text))
    assert declared == set(capi.REFERENCE_SYMBOLS + capi.EXTENSION_SYMBOLS)
    assert len(capi.REFERENCE_SYMBOLS) == 41
    assert b"sm_90a" in L.cuOptB200Version()


def test_scalar_sizes():
    L = capi.lib()
    assert L.cuOptGetIntSize() == 4 and L.cuOptGetFloatSize() == 8  # c_api_tests.cpp: int32 / double


def test_create_problem_round_trip():
    # c_api_test.c check_problem: everything handed to cuOptCreateProblem comes back through the getters
    off = np.array([0, 2, 4], np.int32); idx = np.array([0, 1, 0, 1], np.int32); val = np.array([3.0, 4.0, 2.7, 10.1])
    rhs = np.array([5.4, 4.9]); c = np.array([0.2, 0.1]); lb = np.array([0.0, 0.0]); ub = np.array([2.0, INF])
    p = capi.Problem.create(off, idx, val, b"LL", rhs, c, lb, ub, objective_offset=1.5)
    assert (p.num_constraints, p.num_variables, p.num_nonzeros) == (2, 2, 4)
    assert p.objective_sense == capi.CUOPT_MINIMIZE and p.objective_offset == 1.5
    o2, i2, v2 = p.constraint_matrix()
    assert np.array_equal(o2, off) and np.array_equal(i2, idx) and np.array_equal(v2, val)
    assert p.constraint_sense() == b"LL"
    assert np.array_equal(p.rhs(), rhs) and np.array_equal(p.objective_coefficients(), c)
    assert np.array_equal(p.variable_lower_bounds(), lb) and np.array_equal(p.variable_upper_bounds(), ub)
    assert p.variable_types() == b"CC" and not p.is_mip
    pm = capi.Problem.create(off, idx, val, b"LL", rhs, c, lb, ub, maximize=True, variable_types=b"CI")
    assert pm.objective_sense == capi.CUOPT_MAXIMIZE and pm.is_mip and pm.variable_types() == b"CI"


def test_create_ranged_problem_round_trip():
    d = RANGED_LP
    p = capi.Problem.create_ranged(d["offsets"], d["indices"], d["values"], d["con_lb"], d["con_ub"], d["c"],
                                   d["var_lb"], d["var_ub"], maximize=True)
    assert np.array_equal(p.constraint_lower_bounds(), d["con_lb"])  # c_api_test.c:807-829
    assert np.array_equal(p.constraint_upper_bounds(), d["con_ub"])


def test_null_arguments_are_rejected():
    L = capi.lib()
    h = C.c_void_p()
    assert L.cuOptCreateProblem(1, 1, 1, 0.0, None, None, None, None, None, None, None, None, None, C.byref(h)) == 1
    assert L.cuOptGetNumConstraints(None, None) == capi.CUOPT_INVALID_ARGUMENT
    assert L.cuOptSolve(None, None, None) == capi.CUOPT_INVALID_ARGUMENT
    assert L.cuOptCreateSolverSettings(None) == capi.CUOPT_INVALID_ARGUMENT
    L.cuOptDestroyProblem(None)  # no crash
    L.cuOptDestroySolution(None)


def test_destroy_nulls_the_handle():
    p = capi.Problem.create(np.array([0, 1], np.int32), np.array([0], np.int32), np.array([1.0]), b"E",
                            np.array([1.0]), np.array([1.0]), np.array([0.0]), np.array([INF]))
    capi.lib().cuOptDestroyProblem(C.byref(p.h))
    assert not p.h  # cuopt_c.cpp:200-206
    s = capi.Settings()
    capi.lib().cuOptDestroySolverSettings(C.byref(s.h))
    assert not s.h


def test_settings_defaults_match_reference_registry():
    # math_optimization/solver_settings.cu:67-124
    s = capi.Settings()
    for name in capi.TOLERANCE_PARAMS:
        assert s.get_float(name) == 1e-4
    assert s.get_float("primal_infeasible_tolerance") == 1e-8 and s.get_float("dual_infeasible_tolerance") == 1e-8
    assert s.get_float("time_limit") == INF
    assert s.get_int("iteration_limit") == 2**31 - 1
    assert s.get_int("pdlp_solver_mode") == capi.CUOPT_PDLP_SOLVER_MODE_STABLE2
    assert s.get_int("method") == capi.CUOPT_METHOD_CONCURRENT
    for flag in ("infeasibility_detection", "strict_infeasibility", "per_constraint_residual",
                 "save_best_primal_so_far", "first_primal_feasible", "crossover"):
        assert s.get_int(flag) == 0
    assert s.get_int("log_to_console") == 1
    assert s.get_str("log_file") == "" and s.get_str("crossover") == "false"


def test_settings_set_get_and_errors():
    s = capi.Settings()
    s.set("absolute_gap_tolerance", 1e-6)
    assert s.get_float("absolute_gap_tolerance") == 1e-6
    s.set("iteration_limit", 7)
    assert s.get_int("iteration_limit") == 7 and s.get_str("iteration_limit") == "7"
    s.set("crossover", True)  # integer setter reaches bool parameters (cuopt_c.cpp:493-503)
    assert s.get_int("crossover") == 1
    s.set("log_file", "x.log")
    assert s.get_str("log_file") == "x.log"
    s.set("pdlp_solver_mode", "3")
    assert s.get_int("pdlp_solver_mode") == 3
    L = capi.lib()
    bad = capi.CUOPT_INVALID_ARGUMENT
    assert L.cuOptSetFloatParameter(s.h, b"bad_parameter_name", 1.0) == bad  # c_api_test.c test_bad_parameter_name
    assert L.cuOptSetIntegerParameter(s.h, b"bad_parameter_name", 1) == bad
    assert L.cuOptSetParameter(s.h, b"bad_parameter_name", b"1") == bad
    assert L.cuOptSetFloatParameter(s.h, b"absolute_gap_tolerance", 0.5) == bad  # range [0, 0.1]
    assert L.cuOptSetIntegerParameter(s.h, b"pdlp_solver_mode", 9) == bad
    assert L.cuOptSetParameter(s.h, b"iteration_limit", b"abc") == bad
    assert L.cuOptSetParameter(s.h, b"crossover", b"maybe") == bad
    v = C.c_double()
    assert L.cuOptGetFloatParameter(s.h, b"iteration_limit", C.byref(v)) == bad  # wrong type
    buf = C.create_string_buffer(8)
    assert L.cuOptGetParameter(s.h, b"time_limit", 0, buf) == bad


def test_mip_problem_is_answered_with_an_error_solution():
    # LP-only build: no GPU is touched for a MIP, the error is reported through the solution object
    p = capi.Problem.create(np.array([0, 1], np.int32), np.array([0], np.int32), np.array([1.0]), b"L",
                            np.array([1.5]), np.array([-1.0]), np.array([0.0]), np.array([5.0]), variable_types=b"I")
    sol = capi.solve(p, capi.Settings())
    assert sol.return_code == capi.CUOPT_VALIDATION_ERROR == sol.error_status
    assert "LP" in sol.error_string
    v = C.c_double()
    assert capi.lib().cuOptGetMIPGap(sol.h, C.byref(v)) == capi.CUOPT_INVALID_ARGUMENT


def test_solve_without_gpu_fails_loudly():
    from conftest import has_gpu
    if has_gpu():
        pytest.skip("GPU present")
    d = RANGED_LP
    p = capi.Problem.create_ranged(d["offsets"], d["indices"], d["values"], d["con_lb"], d["con_ub"], d["c"],
                                   d["var_lb"], d["var_ub"], maximize=True)
    sol = capi.solve(p, capi.Settings(log_to_console=False))
    assert sol.return_code == capi.CUOPT_RUNTIME_ERROR and "CUDA" in sol.error_string  # no CPU fallback exists
