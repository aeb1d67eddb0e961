"""ctypes binding of cuopt_b200/lib/libcuopt.so — the C ABI declared in include/cuopt/linear_programming/cuopt_c.h
(the reference's cuopt_c.h surface) plus the cuOptB200* extension of include/cuopt_b200/cuopt_b200_ext.h.

This is the stub a ctypes-based client of the reference library would write; tests and bench.py go through it so
that everything they exercise crosses the same extern "C" boundary a C caller uses.  There is no CPU fallback: if
the shared library is missing, import of `lib()` raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import build as _build

# constants.h
CUOPT_SUCCESS, CUOPT_INVALID_ARGUMENT, CUOPT_MPS_FILE_ERROR, CUOPT_MPS_PARSE_ERROR = 0, 1, 2, 3
CUOPT_VALIDATION_ERROR, CUOPT_OUT_OF_MEMORY, CUOPT_RUNTIME_ERROR = 4, 5, 6
CUOPT_MINIMIZE, CUOPT_MAXIMIZE = 1, -1
CUOPT_METHOD_CONCURRENT, CUOPT_METHOD_PDLP, CUOPT_METHOD_DUAL_SIMPLEX = 0, 1, 2
CUOPT_PDLP_SOLVER_MODE_STABLE1, CUOPT_PDLP_SOLVER_MODE_STABLE2 = 0, 1
CUOPT_PDLP_SOLVER_MODE_METHODICAL1, CUOPT_PDLP_SOLVER_MODE_FAST1 = 2, 3
TERMINATION = {0: "NoTermination", 1: "Optimal", 2: "Infeasible", 3: "Unbounded", 4: "IterationLimit",
               5: "TimeLimit", 6: "NumericalError", 7: "PrimalFeasible", 8: "FeasibleFound", 9: "ConcurrentLimit"}
TOLERANCE_PARAMS = ("absolute_dual_tolerance", "relative_dual_tolerance", "absolute_primal_tolerance",
                    "relative_primal_tolerance", "absolute_gap_tolerance", "relative_gap_tolerance")

c_int_p = C.POINTER(C.c_int32)
c_dbl_p = C.POINTER(C.c_double)


class LPStats(C.Structure):
    _fields_ = [("number_of_steps_taken", C.c_int32), ("total_number_of_attempted_steps", C.c_int32),
                ("l2_primal_residual", C.c_double), ("l2_relative_primal_residual", C.c_double),
                ("l2_dual_residual", C.c_double), ("l2_relative_dual_residual", C.c_double),
                ("primal_objective", C.c_double), ("dual_objective", C.c_double), ("gap", C.c_double),
                ("relative_gap", C.c_double), ("solved_by_pdlp", C.c_int32), ("n_major_iterations", C.c_int32),
                ("n_restarts", C.c_int32), ("method_stand_in", C.c_int32), ("solve_time", C.c_double),
                ("setup_seconds", C.c_double), ("pdhg_loop_seconds", C.c_double), ("termination_seconds", C.c_double),
                ("initial_step_size", C.c_double), ("initial_primal_weight", C.c_double),
                ("final_step_size", C.c_double), ("final_primal_weight", C.c_double), ("kernel_launches", C.c_int64)]


class PresolveStats(C.Structure):
    _fields_ = [("ran", C.c_int32), ("original_m", C.c_int32), ("original_n", C.c_int32), ("original_nnz", C.c_int32),
                ("reduced_m", C.c_int32), ("reduced_n", C.c_int32), ("reduced_nnz", C.c_int32),
                ("fixed_columns", C.c_int32), ("empty_rows", C.c_int32), ("singleton_rows", C.c_int32),
                ("empty_columns", C.c_int32), ("rounds", C.c_int32), ("presolve_seconds", C.c_double),
                ("postsolve_seconds", C.c_double)]


class KernelProfile(C.Structure):
    _fields_ = [("ms_primal_step", C.c_double), ("ms_dual_step", C.c_double), ("ms_transpose_step", C.c_double),
                ("bytes_primal_step", C.c_double), ("bytes_dual_step", C.c_double),
                ("bytes_transpose_step", C.c_double), ("ms_iteration", C.c_double), ("reps", C.c_int32),
                ("grid_primal", C.c_int32), ("grid_dual", C.c_int32), ("grid_transpose", C.c_int32),
                ("ms_transpose_partial", C.c_double), ("ms_transpose_partial_wide", C.c_double),
                ("blocks_dual", C.c_int32), ("blocks_transpose", C.c_int32)]


# every symbol include/*.h declares (tests check that the library exports all of them)
REFERENCE_SYMBOLS = [
    "cuOptGetFloatSize", "cuOptGetIntSize", "cuOptReadProblem", "cuOptCreateProblem", "cuOptCreateRangedProblem",
    "cuOptDestroyProblem", "cuOptGetNumConstraints", "cuOptGetNumVariables", "cuOptGetObjectiveSense",
    "cuOptGetObjectiveOffset", "cuOptGetObjectiveCoefficients", "cuOptGetNumNonZeros", "cuOptGetConstraintMatrix",
    "cuOptGetConstraintSense", "cuOptGetConstraintRightHandSide", "cuOptGetConstraintLowerBounds",
    "cuOptGetConstraintUpperBounds", "cuOptGetVariableLowerBounds", "cuOptGetVariableUpperBounds",
    "cuOptGetVariableTypes", "cuOptCreateSolverSettings", "cuOptDestroySolverSettings", "cuOptSetParameter",
    "cuOptGetParameter", "cuOptSetIntegerParameter", "cuOptGetIntegerParameter", "cuOptSetFloatParameter",
    "cuOptGetFloatParameter", "cuOptIsMIP", "cuOptSolve", "cuOptDestroySolution", "cuOptGetTerminationStatus",
    "cuOptGetErrorStatus", "cuOptGetErrorString", "cuOptGetPrimalSolution", "cuOptGetObjectiveValue",
    "cuOptGetSolveTime", "cuOptGetMIPGap", "cuOptGetSolutionBound", "cuOptGetDualSolution", "cuOptGetReducedCosts",
]
EXTENSION_SYMBOLS = [
    "cuOptB200GetLPStats", "cuOptB200SolverCreate", "cuOptB200SolverDestroy", "cuOptB200SolverInitialise",
    "cuOptB200SolverAdvance", "cuOptB200SolverGetScalar", "cuOptB200SolverGetVector", "cuOptB200SolverGetSolution",
    "cuOptB200SolverTrustRegionBounds", "cuOptB200SolverInfeasibilityStats",
    "cuOptB200SolverProfileKernels", "cuOptB200ReadProblem", "cuOptB200Version", "cuOptB200DistGetUniqueId",
    "cuOptB200DistInit", "cuOptB200DistDestroy", "cuOptB200SolveDistributed",
    "cuOptB200SetWarmStartCapture", "cuOptB200GetWarmStart", "cuOptB200SetWarmStart", "cuOptB200CreateWarmStart",
    "cuOptB200DestroyWarmStart", "cuOptB200WarmStartGetScalar", "cuOptB200WarmStartGetVector",
    "cuOptB200GetPresolveStats",
]
WARM_VECTORS = ("current_primal_solution", "current_dual_solution", "initial_primal_average", "initial_dual_average",
                "current_ATY", "sum_primal_solutions", "sum_dual_solutions", "last_restart_duality_gap_primal_solution",
                "last_restart_duality_gap_dual_solution")
WARM_IS_PRIMAL = (True, False, True, False, True, True, False, True, False)
WARM_SCALARS = ("initial_primal_weight", "initial_step_size", "total_pdlp_iterations", "total_pdhg_iterations",
                "last_candidate_kkt_score", "last_restart_kkt_score", "sum_solution_weight",
                "iterations_since_last_restart")
WARM_INT_SCALARS = ("total_pdlp_iterations", "total_pdhg_iterations", "iterations_since_last_restart")

_lib = None


def lib_path() -> str:
    return _build.LIB


def lib():
    """Load libcuopt.so (building it first when sources are newer).  Raises if it cannot be had."""
    global _lib
    if _lib is None:
        path = _build.LIB
        if _build.needs_build():
            try:
                _build.build()
            except Exception:
                if not os.path.exists(path):
                    raise
        L = C.CDLL(path)
        vp = C.c_void_p
        L.cuOptGetFloatSize.restype = C.c_int8
        L.cuOptGetIntSize.restype = C.c_int8
        L.cuOptReadProblem.argtypes = [C.c_char_p, C.POINTER(vp)]
        L.cuOptCreateProblem.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_double, c_dbl_p, c_int_p, c_int_p,
                                         c_dbl_p, C.c_char_p, c_dbl_p, c_dbl_p, c_dbl_p, C.c_char_p, C.POINTER(vp)]
        L.cuOptCreateRangedProblem.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_double, c_dbl_p, c_int_p, c_int_p,
                                               c_dbl_p, c_dbl_p, c_dbl_p, c_dbl_p, c_dbl_p, C.c_char_p,
                                               C.POINTER(vp)]
        L.cuOptDestroyProblem.argtypes = [C.POINTER(vp)]
        L.cuOptDestroyProblem.restype = None
        for name in ("cuOptGetNumConstraints", "cuOptGetNumVariables", "cuOptGetObjectiveSense",
                     "cuOptGetNumNonZeros", "cuOptIsMIP"):
            getattr(L, name).argtypes = [vp, c_int_p]
        L.cuOptGetObjectiveOffset.argtypes = [vp, c_dbl_p]
        for name in ("cuOptGetObjectiveCoefficients", "cuOptGetConstraintRightHandSide",
                     "cuOptGetConstraintLowerBounds", "cuOptGetConstraintUpperBounds", "cuOptGetVariableLowerBounds",
                     "cuOptGetVariableUpperBounds"):
            getattr(L, name).argtypes = [vp, c_dbl_p]
        L.cuOptGetConstraintMatrix.argtypes = [vp, c_int_p, c_int_p, c_dbl_p]
        L.cuOptGetConstraintSense.argtypes = [vp, C.c_char_p]
        L.cuOptGetVariableTypes.argtypes = [vp, C.c_char_p]
        L.cuOptCreateSolverSettings.argtypes = [C.POINTER(vp)]
        L.cuOptDestroySolverSettings.argtypes = [C.POINTER(vp)]
        L.cuOptDestroySolverSettings.restype = None
        L.cuOptSetParameter.argtypes = [vp, C.c_char_p, C.c_char_p]
        L.cuOptGetParameter.argtypes = [vp, C.c_char_p, C.c_int32, C.c_char_p]
        L.cuOptSetIntegerParameter.argtypes = [vp, C.c_char_p, C.c_int32]
        L.cuOptGetIntegerParameter.argtypes = [vp, C.c_char_p, c_int_p]
        L.cuOptSetFloatParameter.argtypes = [vp, C.c_char_p, C.c_double]
        L.cuOptGetFloatParameter.argtypes = [vp, C.c_char_p, c_dbl_p]
        L.cuOptSolve.argtypes = [vp, vp, C.POINTER(vp)]
        L.cuOptDestroySolution.argtypes = [C.POINTER(vp)]
        L.cuOptDestroySolution.restype = None
        L.cuOptGetTerminationStatus.argtypes = [vp, c_int_p]
        L.cuOptGetErrorStatus.argtypes = [vp, c_int_p]
        L.cuOptGetErrorString.argtypes = [vp, C.c_char_p, C.c_int32]
        for name in ("cuOptGetPrimalSolution", "cuOptGetObjectiveValue", "cuOptGetSolveTime", "cuOptGetMIPGap",
                     "cuOptGetSolutionBound", "cuOptGetDualSolution", "cuOptGetReducedCosts"):
            getattr(L, name).argtypes = [vp, c_dbl_p]
        L.cuOptB200GetLPStats.argtypes = [vp, C.POINTER(LPStats)]
        L.cuOptB200GetPresolveStats.argtypes = [vp, C.POINTER(PresolveStats)]
        L.cuOptB200SolverCreate.argtypes = [vp, vp, C.POINTER(vp)]
        L.cuOptB200SolverDestroy.argtypes = [C.POINTER(vp)]
        L.cuOptB200SolverDestroy.restype = None
        L.cuOptB200SolverInitialise.argtypes = [vp]
        L.cuOptB200SolverAdvance.argtypes = [vp, C.c_int32, c_int_p]
        L.cuOptB200SolverGetScalar.argtypes = [vp, C.c_char_p, c_dbl_p]
        L.cuOptB200SolverGetVector.argtypes = [vp, C.c_char_p, c_dbl_p, C.c_int32, c_int_p]
        L.cuOptB200SolverGetSolution.argtypes = [vp, C.POINTER(vp)]
        L.cuOptB200SolverTrustRegionBounds.argtypes = [vp, c_dbl_p, c_dbl_p, C.c_double, c_dbl_p, c_dbl_p]
        L.cuOptB200SolverInfeasibilityStats.argtypes = [vp, c_dbl_p, c_dbl_p, c_dbl_p, c_dbl_p, c_dbl_p, c_int_p]
        L.cuOptB200SolverProfileKernels.argtypes = [vp, C.c_int32, C.c_int32, C.POINTER(KernelProfile)]
        L.cuOptB200ReadProblem.argtypes = [C.c_char_p, C.c_int32, C.POINTER(vp)]
        L.cuOptB200Version.restype = C.c_char_p
        L.cuOptB200DistGetUniqueId.argtypes = [C.c_char_p]
        L.cuOptB200DistInit.argtypes = [C.c_int32, C.c_int32, C.c_char_p, C.POINTER(vp)]
        L.cuOptB200DistDestroy.argtypes = [C.POINTER(vp)]
        L.cuOptB200DistDestroy.restype = None
        L.cuOptB200SolveDistributed.argtypes = [vp, vp, vp, C.POINTER(vp)]
        L.cuOptB200SetWarmStartCapture.argtypes = [vp, C.c_int32]
        L.cuOptB200GetWarmStart.argtypes = [vp, C.POINTER(vp)]
        L.cuOptB200SetWarmStart.argtypes = [vp, vp]
        L.cuOptB200CreateWarmStart.argtypes = [C.c_int32, C.c_int32, C.POINTER(c_dbl_p), c_dbl_p, C.POINTER(vp)]
        L.cuOptB200DestroyWarmStart.argtypes = [C.POINTER(vp)]
        L.cuOptB200DestroyWarmStart.restype = None
        L.cuOptB200WarmStartGetScalar.argtypes = [vp, C.c_char_p, c_dbl_p]
        L.cuOptB200WarmStartGetVector.argtypes = [vp, C.c_char_p, c_dbl_p, c_int_p]
        _lib = L
    return _lib


class CuOptError(RuntimeError):
    def __init__(self, code, what=""):
        super().__init__(f"cuOpt status {code} {what}")
        self.code = code


def _check(code, what=""):
    if code != CUOPT_SUCCESS:
        raise CuOptError(code, what)


def _dp(a):
    return a.ctypes.data_as(c_dbl_p)


def _ip(a):
    return a.ctypes.data_as(c_int_p)


class Problem:
    """cuOptOptimizationProblem handle."""

    def __init__(self, handle):
        self.h = handle

    @classmethod
    def read(cls, path: str, fixed_format: bool | None = None) -> "Problem":
        h = C.c_void_p()
        if fixed_format is None:
            _check(lib().cuOptReadProblem(os.fsencode(path), C.byref(h)), f"cuOptReadProblem({path})")
        else:
            _check(lib().cuOptB200ReadProblem(os.fsencode(path), int(fixed_format), C.byref(h)),
                   f"cuOptB200ReadProblem({path})")
        return cls(h)

    @classmethod
    def create(cls, offsets, indices, values, sense, rhs, c, lb, ub, *, maximize=False, objective_offset=0.0,
               variable_types=None) -> "Problem":
        m, n = len(rhs), len(c)
        offsets = np.ascontiguousarray(offsets, np.int32); indices = np.ascontiguousarray(indices, np.int32)
        values, rhs, c, lb, ub = (np.ascontiguousarray(a, np.float64) for a in (values, rhs, c, lb, ub))
        sense = bytes(sense) if not isinstance(sense, (bytes, bytearray)) else bytes(sense)
        vt = variable_types if variable_types is not None else b"C" * n
        h = C.c_void_p()
        _check(lib().cuOptCreateProblem(m, n, CUOPT_MAXIMIZE if maximize else CUOPT_MINIMIZE, objective_offset,
                                        _dp(c), _ip(offsets), _ip(indices), _dp(values), sense, _dp(rhs), _dp(lb),
                                        _dp(ub), vt, C.byref(h)), "cuOptCreateProblem")
        return cls(h)

    @classmethod
    def create_ranged(cls, offsets, indices, values, con_lb, con_ub, c, lb, ub, *, maximize=False,
                      objective_offset=0.0, variable_types=None) -> "Problem":
        m, n = len(con_lb), len(c)
        offsets = np.ascontiguousarray(offsets, np.int32); indices = np.ascontiguousarray(indices, np.int32)
        values, con_lb, con_ub, c, lb, ub = (np.ascontiguousarray(a, np.float64)
                                             for a in (values, con_lb, con_ub, c, lb, ub))
        vt = variable_types if variable_types is not None else b"C" * n
        h = C.c_void_p()
        _check(lib().cuOptCreateRangedProblem(m, n, CUOPT_MAXIMIZE if maximize else CUOPT_MINIMIZE, objective_offset,
                                              _dp(c), _ip(offsets), _ip(indices), _dp(values), _dp(con_lb),
                                              _dp(con_ub), _dp(lb), _dp(ub), vt, C.byref(h)),
               "cuOptCreateRangedProblem")
        return cls(h)

    def close(self):
        if self.h and _lib is not None:
            _lib.cuOptDestroyProblem(C.byref(self.h))

    __del__ = close

    def _int(self, fn):
        v = C.c_int32()
        _check(getattr(lib(), fn)(self.h, C.byref(v)), fn)
        return v.value

    @property
    def num_constraints(self): return self._int("cuOptGetNumConstraints")
    @property
    def num_variables(self): return self._int("cuOptGetNumVariables")
    @property
    def num_nonzeros(self): return self._int("cuOptGetNumNonZeros")
    @property
    def objective_sense(self): return self._int("cuOptGetObjectiveSense")
    @property
    def is_mip(self): return bool(self._int("cuOptIsMIP"))

    @property
    def objective_offset(self):
        v = C.c_double()
        _check(lib().cuOptGetObjectiveOffset(self.h, C.byref(v)))
        return v.value

    def _vec(self, fn, size):
        out = np.full(size, np.nan)
        _check(getattr(lib(), fn)(self.h, _dp(out)), fn)
        return out

    def objective_coefficients(self): return self._vec("cuOptGetObjectiveCoefficients", self.num_variables)
    def rhs(self): return self._vec("cuOptGetConstraintRightHandSide", self.num_constraints)
    def constraint_lower_bounds(self): return self._vec("cuOptGetConstraintLowerBounds", self.num_constraints)
    def constraint_upper_bounds(self): return self._vec("cuOptGetConstraintUpperBounds", self.num_constraints)
    def variable_lower_bounds(self): return self._vec("cuOptGetVariableLowerBounds", self.num_variables)
    def variable_upper_bounds(self): return self._vec("cuOptGetVariableUpperBounds", self.num_variables)

    def constraint_matrix(self):
        m, nnz = self.num_constraints, self.num_nonzeros
        off = np.zeros(m + 1, np.int32); idx = np.zeros(nnz, np.int32); val = np.zeros(nnz)
        _check(lib().cuOptGetConstraintMatrix(self.h, _ip(off), _ip(idx), _dp(val)))
        return off, idx, val

    def constraint_sense(self):
        buf = C.create_string_buffer(max(self.num_constraints, 1) + 1)
        _check(lib().cuOptGetConstraintSense(self.h, buf))
        return buf.raw[: self.num_constraints]

    def variable_types(self):
        buf = C.create_string_buffer(max(self.num_variables, 1) + 1)
        _check(lib().cuOptGetVariableTypes(self.h, buf))
        return buf.raw[: self.num_variables]


class Settings:
    """cuOptSolverSettings handle."""

    def __init__(self, **params):
        self.h = C.c_void_p()
        _check(lib().cuOptCreateSolverSettings(C.byref(self.h)))
        for k, v in params.items():
            self.set(k, v)

    def close(self):
        if self.h and _lib is not None:
            _lib.cuOptDestroySolverSettings(C.byref(self.h))

    __del__ = close

    def set(self, name: str, value):
        if name == "optimality_tolerance":  # convenience: the reference's set_optimality_tolerance
            for p in TOLERANCE_PARAMS:
                self.set(p, value)
            return
        nb = name.encode()
        if isinstance(value, bool):
            _check(lib().cuOptSetIntegerParameter(self.h, nb, int(value)), name)
        elif isinstance(value, int):
            _check(lib().cuOptSetIntegerParameter(self.h, nb, value), name)
        elif isinstance(value, float):
            _check(lib().cuOptSetFloatParameter(self.h, nb, value), name)
        else:
            _check(lib().cuOptSetParameter(self.h, nb, str(value).encode()), name)

    def capture_warm_start(self, enable: bool = True):
        """Make solutions carry the state a later solve can continue from (cuOptB200SetWarmStartCapture)."""
        _check(lib().cuOptB200SetWarmStartCapture(self.h, int(enable)))

    def set_warm_start(self, warm_start: "WarmStart | None"):
        _check(lib().cuOptB200SetWarmStart(self.h, warm_start.h if warm_start is not None else None))

    def get_float(self, name):
        v = C.c_double()
        _check(lib().cuOptGetFloatParameter(self.h, name.encode(), C.byref(v)), name)
        return v.value

    def get_int(self, name):
        v = C.c_int32()
        _check(lib().cuOptGetIntegerParameter(self.h, name.encode(), C.byref(v)), name)
        return v.value

    def get_str(self, name, size=256):
        buf = C.create_string_buffer(size)
        _check(lib().cuOptGetParameter(self.h, name.encode(), size, buf), name)
        return buf.value.decode()


class Solution:
    """cuOptSolution handle."""

    def __init__(self, handle, m, n, rc=0):
        self.h, self.m, self.n, self.return_code = handle, m, n, rc

    def close(self):
        if self.h and _lib is not None:
            _lib.cuOptDestroySolution(C.byref(self.h))

    __del__ = close

    @property
    def termination_status(self):
        v = C.c_int32()
        _check(lib().cuOptGetTerminationStatus(self.h, C.byref(v)))
        return v.value

    @property
    def termination_reason(self): return TERMINATION.get(self.termination_status, "?")

    @property
    def error_status(self):
        v = C.c_int32()
        _check(lib().cuOptGetErrorStatus(self.h, C.byref(v)))
        return v.value

    @property
    def error_string(self):
        buf = C.create_string_buffer(1024)
        _check(lib().cuOptGetErrorString(self.h, buf, 1024))
        return buf.value.decode()

    def _scalar(self, fn):
        v = C.c_double()
        _check(getattr(lib(), fn)(self.h, C.byref(v)), fn)
        return v.value

    @property
    def objective_value(self): return self._scalar("cuOptGetObjectiveValue")
    @property
    def solve_time(self): return self._scalar("cuOptGetSolveTime")

    def primal(self):
        out = np.zeros(self.n); _check(lib().cuOptGetPrimalSolution(self.h, _dp(out))); return out

    def dual(self):
        out = np.zeros(self.m); _check(lib().cuOptGetDualSolution(self.h, _dp(out))); return out

    def reduced_costs(self):
        out = np.zeros(self.n); _check(lib().cuOptGetReducedCosts(self.h, _dp(out))); return out

    def stats(self) -> LPStats:
        s = LPStats()
        _check(lib().cuOptB200GetLPStats(self.h, C.byref(s)))
        return s

    def presolve_stats(self) -> PresolveStats:
        s = PresolveStats()
        _check(lib().cuOptB200GetPresolveStats(self.h, C.byref(s)))
        return s

    def warm_start(self) -> "WarmStart":
        h = C.c_void_p()
        _check(lib().cuOptB200GetWarmStart(self.h, C.byref(h)), "cuOptB200GetWarmStart (was capture_warm_start set?)")
        return WarmStart(h)


class WarmStart:
    """cuOptB200WarmStart handle: the reference's pdlp_warm_start_data_t through the C ABI."""

    def __init__(self, handle):
        self.h = handle

    @classmethod
    def create(cls, m: int, n: int, data: dict) -> "WarmStart":
        """From host arrays / scalars keyed by the reference's field names (see WARM_VECTORS, WARM_SCALARS)."""
        vecs = [np.ascontiguousarray(data[k], np.float64) for k in WARM_VECTORS]
        for v, primal, k in zip(vecs, WARM_IS_PRIMAL, WARM_VECTORS):
            if len(v) != (n if primal else m):
                raise ValueError(f"{k}: expected {n if primal else m} values, got {len(v)}")
        ptrs = (c_dbl_p * 9)(*[_dp(v) for v in vecs])
        sc = np.array([float(data[k]) for k in WARM_SCALARS])
        h = C.c_void_p()
        _check(lib().cuOptB200CreateWarmStart(m, n, ptrs, _dp(sc), C.byref(h)), "cuOptB200CreateWarmStart")
        return cls(h)

    def close(self):
        if self.h and _lib is not None:
            _lib.cuOptB200DestroyWarmStart(C.byref(self.h))

    __del__ = close

    def scalar(self, name: str):
        v = C.c_double()
        _check(lib().cuOptB200WarmStartGetScalar(self.h, name.encode(), C.byref(v)), name)
        return int(v.value) if name in WARM_INT_SCALARS else v.value

    def vector(self, name: str) -> np.ndarray:
        size = C.c_int32()
        _check(lib().cuOptB200WarmStartGetVector(self.h, name.encode(), None, C.byref(size)), name)
        out = np.zeros(size.value)
        _check(lib().cuOptB200WarmStartGetVector(self.h, name.encode(), _dp(out), C.byref(size)), name)
        return out

    def to_dict(self) -> dict:
        d = {k: self.vector(k) for k in WARM_VECTORS}
        d.update({k: self.scalar(k) for k in WARM_SCALARS})
        return d


def solve(problem: Problem, settings: Settings) -> Solution:
    h = C.c_void_p()
    rc = lib().cuOptSolve(problem.h, settings.h, C.byref(h))
    return Solution(h, problem.num_constraints, problem.num_variables, rc)


class Solver:
    """cuOptB200Solver session (white-box stepping, profiling)."""

    def __init__(self, problem: Problem, settings: Settings):
        self.h = C.c_void_p()
        self.m, self.n = problem.num_constraints, problem.num_variables
        _check(lib().cuOptB200SolverCreate(problem.h, settings.h, C.byref(self.h)), "cuOptB200SolverCreate")

    def close(self):
        if self.h and _lib is not None:
            _lib.cuOptB200SolverDestroy(C.byref(self.h))

    __del__ = close

    def initialise(self): _check(lib().cuOptB200SolverInitialise(self.h))

    def advance(self, steps: int) -> bool:
        f = C.c_int32()
        _check(lib().cuOptB200SolverAdvance(self.h, steps, C.byref(f)), "advance")
        return bool(f.value)

    def scalar(self, name):
        v = C.c_double()
        _check(lib().cuOptB200SolverGetScalar(self.h, name.encode(), C.byref(v)), name)
        return v.value

    def vector(self, name):
        sz = C.c_int32()
        _check(lib().cuOptB200SolverGetVector(self.h, name.encode(), None, 0, C.byref(sz)), name)
        out = np.zeros(sz.value)
        _check(lib().cuOptB200SolverGetVector(self.h, name.encode(), _dp(out), sz.value, C.byref(sz)), name)
        return out

    def trust_region_bounds(self, px, py, radius: float):
        """(lower, upper) of the Methodical1 trust-region restart at a point of the scaled space; changes no state."""
        px = np.ascontiguousarray(px, np.float64); py = np.ascontiguousarray(py, np.float64)
        if len(px) != self.n or len(py) != self.m:
            raise ValueError(f"expected {self.n} primal and {self.m} dual values, got {len(px)} and {len(py)}")
        lo, up = C.c_double(), C.c_double()
        _check(lib().cuOptB200SolverTrustRegionBounds(self.h, _dp(px), _dp(py), float(radius), C.byref(lo), C.byref(up)),
               "trust_region_bounds")
        return lo.value, up.value

    INFEASIBILITY_STATS = ("xinf", "max_viol", "hres", "cx", "yinf", "rcinf", "hdres_raw", "dobj_raw", "pobj",
                           "max_primal", "hdres", "dobj")

    def infeasibility_stats(self, x_cur, y_cur, x_avg, y_avg):
        """(stats, status): the 12 detection statistics of the current and the average point (a 2 x 12 array in the order
        of INFEASIBILITY_STATS) and the verdict each would draw (2, 3 or 6), at points of the unscaled minimisation form
        of the original problem; changes no state."""
        pts = [np.ascontiguousarray(v, np.float64) for v in (x_cur, y_cur, x_avg, y_avg)]
        if any(len(v) != (self.n if k % 2 == 0 else self.m) for k, v in enumerate(pts)):
            raise ValueError(f"expected {self.n} primal and {self.m} dual values per point")
        stats, status = np.zeros((2, 12)), (C.c_int32 * 2)()
        _check(lib().cuOptB200SolverInfeasibilityStats(self.h, *(_dp(v) for v in pts), _dp(stats), status),
               "infeasibility_stats")
        return stats, [status[0], status[1]]

    def solution(self) -> Solution:
        h = C.c_void_p()
        _check(lib().cuOptB200SolverGetSolution(self.h, C.byref(h)))
        return Solution(h, self.m, self.n)

    def profile_kernels(self, warmup_steps=50, reps=200) -> KernelProfile:
        p = KernelProfile()
        _check(lib().cuOptB200SolverProfileKernels(self.h, warmup_steps, reps, C.byref(p)))
        return p


class Dist:
    """cuOptB200Dist communicator (one per process / GPU)."""

    def __init__(self, rank: int, world: int, unique_id: bytes):
        self.rank, self.world = rank, world
        self.h = C.c_void_p()
        _check(lib().cuOptB200DistInit(rank, world, unique_id, C.byref(self.h)), "cuOptB200DistInit")

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _check(lib().cuOptB200DistGetUniqueId(buf), "cuOptB200DistGetUniqueId")
        return buf.raw

    def close(self):
        if self.h and _lib is not None:
            _lib.cuOptB200DistDestroy(C.byref(self.h))

    __del__ = close


def solve_distributed(local_problem: Problem, settings: Settings, dist: Dist) -> Solution:
    h = C.c_void_p()
    rc = lib().cuOptB200SolveDistributed(local_problem.h, settings.h, dist.h, C.byref(h))
    return Solution(h, local_problem.num_constraints, local_problem.num_variables, rc)
