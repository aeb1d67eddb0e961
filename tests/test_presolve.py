"""Opt-in presolve (settings `presolve`, cuopt_b200/csrc/presolve.cu): empty rows and columns, fixed columns and singleton
rows removed on the device in rounds, postsolve of primal, dual and reduced costs.

`presolve_reference` below restates the four rules in numpy, in the order the device applies them; it is the test
reference.  HiGHS confirms it on every fixture (the reduced problem plus its offset has the original's optimum, or the
original's verdict), the device's reduced problem is checked against it, and the postsolved solution is checked against the
KKT conditions of the ORIGINAL problem."""
import functools
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import mps_path, problem_arrays
from cuopt_b200 import build as b
from cuopt_b200 import capi, lpgen
from cases import planted_bounds
from exact import LP, STEPWISE, certifies, highs, rel_err, row_sum_tolerance
from oracle import pdlp_oracle as po

inf = np.inf
TOL = 1e-4              # absolute_primal_tolerance default: the infeasibility tests of presolve
MAX_ROUNDS = 32         # PRESOLVE_MAX_ROUNDS in presolve.cu
VERDICT = {"Optimal": 1, "PrimalInfeasible": 2, "DualInfeasible": 3}
HIGHS_STATUS = {"Optimal": 0, "PrimalInfeasible": 2, "DualInfeasible": 3}


# ------------------------------------------------------------------------------------------------ numpy restatement
def presolve_reference(offsets, indices, values, c, l, u, lc, uc, tol=TOL):
    """The four rules of presolve.cu in its order (minimisation form).  Returns a dict: reduced problem, maps, offset,
    counts per rule, rounds, verdict (None when PDLP has to run) and the per-row magnitude of the bound shifts."""
    offsets, indices, values = (np.asarray(a) for a in (offsets, indices, values))
    c, l, u, lc, uc = (np.array(v, float) for v in (c, l, u, lc, uc))
    m, n = len(lc), len(c)
    row_of = np.repeat(np.arange(m), np.diff(offsets))
    A = sp.csr_matrix((values, indices, offsets), shape=(m, n))
    T = A.T.tocsr()
    T.sort_indices()
    row_alive, col_alive = np.ones(m, bool), np.ones(n, bool)
    x_fix = np.zeros(n)
    shift_mag, shift_len = np.abs(lc.copy()), np.zeros(m)
    shift_mag[~np.isfinite(shift_mag)] = 0.0
    counts = dict(fixed_columns=0, empty_rows=0, singleton_rows=0, empty_columns=0)
    rounds, infeasible = 0, False
    for _ in range(MAX_ROUNDS):
        rounds += 1
        # 1. fixed columns
        fixed = col_alive & (l == u) & np.isfinite(l)
        col_alive[fixed] = False
        x_fix[fixed] = l[fixed]
        counts["fixed_columns"] += int(fixed.sum())
        # 2. row shifts, live counts, empty rows
        fe = fixed[indices] & row_alive[row_of]
        term = np.where(fe, values * x_fix[indices], 0.0)
        shift = np.bincount(row_of, weights=term, minlength=m)
        shift_mag += np.bincount(row_of, weights=np.abs(term), minlength=m)
        shift_len += np.bincount(row_of, weights=fe.astype(float), minlength=m)
        for v in (lc, uc):
            ok = row_alive & np.isfinite(v)
            v[ok] -= shift[ok]
        live = col_alive[indices] & (values != 0) & row_alive[row_of]
        cnt = np.bincount(row_of[live], minlength=m)
        single_col = np.full(m, -1)
        single_val = np.zeros(m)
        single_col[row_of[live]] = indices[live]
        single_val[row_of[live]] = values[live]
        empty = row_alive & (cnt == 0)
        infeasible |= bool(np.any((lc[empty] > tol) | (uc[empty] < -tol)))
        row_alive[empty] = False
        counts["empty_rows"] += int(empty.sum())
        # 3. singleton rows, ascending row order per column
        touched, singles = set(), 0
        for i in np.flatnonzero(row_alive & (cnt == 1)):
            j, a = single_col[i], single_val[i]
            lo, hi = (lc[i] / a, uc[i] / a) if a > 0 else (uc[i] / a, lc[i] / a)
            if lo > l[j]:
                l[j] = lo
            if hi < u[j]:
                u[j] = hi
            row_alive[i] = False
            singles += 1
            touched.add(j)
        for j in touched:
            if l[j] > u[j] + tol:
                infeasible = True
            elif l[j] > u[j]:
                u[j] = l[j]
        # 4. empty columns
        live = col_alive[indices] & (values != 0) & row_alive[row_of]
        ccount = np.bincount(indices[live], minlength=n)
        empty_c = col_alive & (ccount == 0)
        v = np.where(c > 0, l, np.where(c < 0, u, np.minimum(np.maximum(0.0, l), u)))
        gone = empty_c & np.isfinite(v)
        x_fix[gone] = v[gone]
        col_alive[gone] = False
        counts["empty_columns"] += int(gone.sum())
        counts["singleton_rows"] += singles
        removed = int(fixed.sum()) + int(empty.sum()) + singles + int(gone.sum())
        if infeasible or removed == 0:
            break
    verdict = "PrimalInfeasible" if infeasible else None
    if verdict is None and not row_alive.any():
        verdict = "Optimal" if not col_alive.any() else "DualInfeasible"
    row_map, col_map = np.flatnonzero(row_alive), np.flatnonzero(col_alive)
    R = A[row_map][:, col_map].tocsr()
    R.eliminate_zeros()
    R.sort_indices()
    return dict(offsets=R.indptr, indices=R.indices, values=R.data, c=c[col_map], l=l[col_map], u=u[col_map],
                lc=lc[row_map], uc=uc[row_map], row_map=row_map, col_map=col_map, rounds=rounds, verdict=verdict,
                offset=float(np.sum(c[~col_alive] * x_fix[~col_alive])), x_fix=x_fix, col_alive=col_alive,
                row_alive=row_alive, shift_mag=shift_mag[row_map], shift_len=shift_len[row_map], **counts)


# --------------------------------------------------------------------------------------------------------- fixtures
def arrays(offsets, indices, values, c, l, u, lc, uc, maximize=False, offset=0.0):
    return dict(offsets=np.asarray(offsets, np.int32), indices=np.asarray(indices, np.int32),
                values=np.asarray(values, float), c=np.asarray(c, float), l=np.asarray(l, float),
                u=np.asarray(u, float), lc=np.asarray(lc, float), uc=np.asarray(uc, float), maximize=maximize,
                offset=offset)


def from_rows(rows, n, c, l, u, lc, uc, **kw):
    """rows: list of {column: value}."""
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    idx = [j for r in rows for j in sorted(r)]
    val = [r[j] for r in rows for j in sorted(r)]
    return arrays(off, idx, val, c, l, u, lc, uc, **kw)


def singleton_zoo(seed):
    """Box-bounded random rows around a feasible point plus singleton rows of every kind: active at lc, at uc, inactive,
    negative coefficients, two on one column, one that fixes its column, and a chain (a fixed column turns a two-entry row
    into a singleton, whose removal empties its other column)."""
    rng = np.random.default_rng(seed)
    n, m = 40, 24
    x0 = rng.uniform(-2, 2, n)
    rows = []
    for _ in range(m):
        cols = rng.choice(n - 4, 5, replace=False)
        rows.append({int(j): float(rng.normal()) for j in cols})
    ax = np.array([sum(a * x0[j] for j, a in r.items()) for r in rows])
    lc = list(ax - rng.uniform(0.5, 2.0, m))
    uc = list(ax + rng.uniform(0.5, 2.0, m))
    c = rng.normal(0, 1, n)
    l, u = np.full(n, -5.0), np.full(n, 5.0)

    def single(j, a, lo, hi):
        rows.append({j: a})
        lc.append(lo)
        uc.append(hi)

    single(0, 2.0, 2.0 * (x0[0] - 0.5) if c[0] > 0 else -inf, inf)          # pushes x0 up: active at lc when c0 > 0
    single(1, 1.5, -inf, 1.5 * (x0[1] + 0.5))                                # upper bound on x1
    single(2, -3.0, -3.0 * (x0[2] + 0.7), inf)                               # negative coefficient: an upper bound
    single(3, -0.5, -inf, -0.5 * (x0[3] - 0.7))                              # negative coefficient: a lower bound
    single(4, 1.0, -100.0, 100.0)                                            # inactive
    single(5, 1.0, x0[5] - 1.0, inf)                                         # two on one column
    single(5, 2.0, 2.0 * (x0[5] - 0.5), 2.0 * (x0[5] + 3.0))
    single(6, 4.0, 4.0 * x0[6], 4.0 * x0[6])                                 # fixes its column
    # chain: column n-2 fixed, row {n-2, n-1} is then a singleton on n-1, which has no other entry
    l[n - 2] = u[n - 2] = 1.0
    x0[n - 2] = 1.0
    rows.append({n - 2: 1.0, n - 1: 2.0})
    lc.append(1.0 + 2.0 * (x0[n - 1] - 1.0))
    uc.append(1.0 + 2.0 * (x0[n - 1] + 1.0))
    # an empty column with a finite favoured bound and a column fixed from the start
    c[n - 3] = abs(c[n - 3]) + 0.1
    l[n - 4] = u[n - 4] = 0.25
    return from_rows(rows, n, c, l, u, lc, uc)


def planted_reductions(m, n, seed):
    """lpgen.sparse_lp past one launch wave of the presolve kernels and one 64K-row schedule segment, with planted fixed
    columns, singleton rows (bounds around x*) and empty rows; x* stays feasible."""
    lp = lpgen.sparse_lp(m, n, 4, seed=seed)
    rng = np.random.default_rng(seed + 1)
    l, u = lp.var_lb.copy(), lp.var_ub.copy()
    x = lp.x_star
    fix = rng.choice(n, 500, replace=False)
    l[fix] = u[fix] = x[fix]
    cols = rng.choice(n, 300, replace=False)
    k = len(cols)
    off = np.concatenate([lp.offsets, lp.offsets[-1] + np.arange(1, k + 1), np.full(40, lp.offsets[-1] + k)])
    idx = np.concatenate([lp.indices, cols])
    val = np.concatenate([lp.values, rng.choice([-2.0, 0.5, 3.0], k)])
    act = val[-k:] * x[cols]
    lc = np.concatenate([lp.con_lb, act - rng.uniform(0.0, 1.0, k), np.full(40, -1.0)])
    uc = np.concatenate([lp.con_ub, act + rng.uniform(0.5, 1.0, k), np.full(40, 1.0)])
    return arrays(off, idx, val, lp.c, l, u, lc, uc)


def from_problem(p):
    a = problem_arrays(p)
    return arrays(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"],
                  maximize=a["maximize"], offset=a["objective_offset"])


@functools.lru_cache(maxsize=None)
def fixture(name):
    if name == "bound_zoo":
        lp = planted_bounds(40, 30, 21)
        return arrays(lp.offsets, lp.indices, lp.values, lp.user_c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub)
    if name == "bound_zoo_max_offset":
        lp = planted_bounds(3000, 2500, 22, maximize=True, offset=123.25)
        return arrays(lp.offsets, lp.indices, lp.values, lp.user_c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub,
                      maximize=True, offset=123.25)
    if name.startswith("singleton_zoo"):
        return singleton_zoo(int(name.split("_")[-1]))
    if name == "afiro":
        return from_problem(capi.Problem.read(mps_path("linear_programming/afiro_original.mps")))
    if name == "sudoku":
        return from_problem(capi.Problem.read(mps_path("mip/sudoku.mps")))
    if name == "planted_large":
        return planted_reductions(70_000, 280_000, 5)
    if name == "infeasible_empty_row":
        return from_rows([{}, {0: 1, 1: 1}], 2, [1, 1], [0, 0], [inf, inf], [1, 1], [2, 4])
    if name == "crossing_singletons":
        # x0 >= 2 and -2 x0 >= -2 (x0 <= 1)
        return from_rows([{0: 1}, {0: -2}, {0: 1, 1: 1}], 2, [1, 1], [0, 0], [10, 10], [2, -2, 0], [inf, inf, 5])
    if name == "unbounded_empty_column":
        return from_rows([{0: 1}, {}], 2, [1, -1], [0, 0], [inf, inf], [1, -1], [3, 1])
    if name == "no_constraints":
        return arrays([0], [], [], [1.0, -1.0, 0.0, 2.0], [0, -5, -inf, -3], [inf, 5, inf, 4], [], [])
    # certificates through presolve: PDLP decides these on the reduced problem
    if name == "ray_singleton_lower":
        # x0 >= 1 (a singleton G row) but x0 + x1 <= 0, x >= 0
        return from_rows([{0: 1}, {0: 1, 1: 1}], 2, [1, 1], [0, 0], [inf, inf], [1, -inf], [inf, 0])
    if name == "ray_singleton_negative_upper":
        # -x0 >= 1 (x0 <= -1) but x0 - x1 >= 0, x1 >= 0
        return from_rows([{0: -1}, {0: 1, 1: -1}], 2, [1, 1], [-inf, 0], [inf, inf], [1, 0], [inf, inf])
    if name == "ray_singleton_ranged":
        # 2 <= 2 x0 <= 6 (a ranged singleton row) but x0 + x1 <= 0, x >= 0
        return from_rows([{0: 2}, {0: 1, 1: 1}], 2, [1, 1], [0, 0], [inf, inf], [2, -inf], [6, 0])
    if name == "ray_fixed_column":
        # x2 = 2 (fixed) turns x0 + x1 + x2 <= 1 into x0 + x1 <= -1, x >= 0
        return from_rows([{0: 1, 1: 1, 2: 1}, {0: 1, 1: -1}], 3, [1, 1, 1], [0, 0, 2], [inf, inf, 2], [-inf, -4],
                         [1, 4])
    if name == "ray_fixed_makes_singleton":
        # x2 = 1 (fixed) turns x0 + x2 >= 3 into the singleton x0 >= 2, but x0 + x1 <= 1, x >= 0
        return from_rows([{0: 1, 2: 1}, {0: 1, 1: 1}], 3, [1, 1, 1], [0, 0, 1], [inf, inf, 1], [3, -inf], [inf, 1])
    if name == "ray_unbounded_with_removed_columns":
        # the unbounded_free_var certificate of cases.py with a fixed column (x4 = 2) in its E row and a
        # bounded empty column (x5, c5 > 0) next to it; both are removed, the reduced problem is that certificate
        return from_rows([{0: 1, 1: 1, 3: -1, 4: 1}, {2: 1, 3: 1}], 6, [1, 0, 1, 0, 3, 1], [-inf, 0, -1, 0, 2, 0],
                         [inf, inf, 1, inf, 2, 4], [3, -2], [3, 2])
    raise KeyError(name)


OPTIMAL = ["bound_zoo", "bound_zoo_max_offset", "singleton_zoo_1", "singleton_zoo_2", "singleton_zoo_3", "afiro",
           "sudoku", "planted_large"]
# (fixture, status, what presolve removes: fixed columns, singleton rows, empty columns)
RAYS = [("ray_singleton_lower", "PrimalInfeasible", (0, 1, 0)),
        ("ray_singleton_negative_upper", "PrimalInfeasible", (0, 1, 0)),
        ("ray_singleton_ranged", "PrimalInfeasible", (0, 1, 0)),
        ("ray_fixed_column", "PrimalInfeasible", (1, 0, 0)),
        ("ray_fixed_makes_singleton", "PrimalInfeasible", (1, 1, 0)),
        ("ray_unbounded_with_removed_columns", "DualInfeasible", (1, 0, 1))]
VERDICTS = [("infeasible_empty_row", "PrimalInfeasible"), ("crossing_singletons", "PrimalInfeasible"),
            ("unbounded_empty_column", "DualInfeasible"), ("no_constraints", "Optimal")]


def min_form(f):
    return -f["c"] if f["maximize"] else f["c"]


@functools.lru_cache(maxsize=None)
def reference(name):
    f = fixture(name)
    return presolve_reference(f["offsets"], f["indices"], f["values"], min_form(f), f["l"], f["u"], f["lc"], f["uc"])


def highs_of(f, c=None):
    return highs(f["offsets"], f["indices"], f["values"], min_form(f) if c is None else c, f["l"], f["u"], f["lc"], f["uc"])


# ------------------------------------------------------------------------------------------------- CPU: the rules
@pytest.mark.parametrize("name", OPTIMAL)
def test_highs_confirms_the_reduced_problem(name):
    f, r = fixture(name), reference(name)
    assert r["verdict"] is None
    orig = highs_of(f)
    red = highs(r["offsets"], r["indices"], r["values"], r["c"], r["l"], r["u"], r["lc"], r["uc"])
    assert orig.status == 0 and red.status == 0, (orig.message, red.message)
    assert red.fun + r["offset"] == pytest.approx(orig.fun, rel=1e-7, abs=1e-7)


def test_the_fixtures_exercise_every_rule():
    for name in ("bound_zoo", "singleton_zoo_1"):
        r = reference(name)
        assert r["fixed_columns"] > 0 and r["empty_rows"] + r["singleton_rows"] > 0, (name, r)
    z = reference("singleton_zoo_1")
    assert z["singleton_rows"] >= 9 and z["empty_columns"] >= 2 and z["rounds"] >= 2
    assert reference("afiro")["singleton_rows"] == 2
    s = reference("sudoku")
    assert (len(fixture("sudoku")["lc"]) - len(s["row_map"]), len(fixture("sudoku")["c"]) - len(s["col_map"])) == (29, 30)
    big = reference("planted_large")
    assert big["fixed_columns"] >= 500 and big["singleton_rows"] >= 300 and big["empty_rows"] >= 40
    assert big["empty_columns"] > 0


@pytest.mark.parametrize("name,verdict", VERDICTS)
def test_verdicts_agree_with_highs(name, verdict):
    f, r = fixture(name), reference(name)
    assert r["verdict"] == verdict
    res = highs_of(f)
    assert res.status == HIGHS_STATUS[verdict], res.message


@pytest.mark.parametrize("name,verdict,removed", RAYS)
def test_ray_fixtures_reduce_as_named_and_leave_the_verdict_to_pdlp(name, verdict, removed):
    f, r = fixture(name), reference(name)
    assert r["verdict"] is None and r["empty_rows"] == 0
    assert (r["fixed_columns"], r["singleton_rows"], r["empty_columns"]) == removed
    assert highs_of(f).status == HIGHS_STATUS[verdict]
    red = highs(r["offsets"], r["indices"], r["values"], r["c"], r["l"], r["u"], r["lc"], r["uc"])
    assert red.status == HIGHS_STATUS[verdict], red.message


def test_nothing_to_remove_on_the_identity_fixtures():
    for lp in identity_lps():
        r = presolve_reference(lp.offsets, lp.indices, lp.values, lp.c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub)
        assert len(r["row_map"]) == lp.m and len(r["col_map"]) == lp.n and r["rounds"] == 1


def identity_lps():
    return [lpgen.multicommodity(60, 200, 4, seed=2), lpgen.sparse_lp(2000, 1000, 8, seed=11)]


# --------------------------------------------------------------------------------------- CPU: parameter and refusals
def test_registry_parses_presolve():
    s = capi.Settings()
    assert s.get_int("presolve") == 0 and s.get_str("presolve") == "false"
    s.set("presolve", True)
    assert s.get_int("presolve") == 1
    s.set("presolve", "false")
    assert s.get_str("presolve") == "false"
    with pytest.raises(capi.CuOptError):
        s.set("presolve", "maybe")


def test_cli_parses_presolve():
    exe = b.build_cli()
    afiro = mps_path("linear_programming/afiro_original.mps")
    r = subprocess.run([exe, afiro, "--presolve", "maybe"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 1 and "unknown parameter or bad value: --presolve maybe" in r.stderr
    r = subprocess.run([exe, afiro, "--presolve", "true", "--iteration-limit", "0"], capture_output=True, text=True,
                       timeout=300)
    assert "unknown parameter" not in r.stderr


def small_problem():
    f = fixture("singleton_zoo_1")
    return capi.Problem.create_ranged(f["offsets"], f["indices"], f["values"], f["lc"], f["uc"], f["c"], f["l"], f["u"]), f


def test_presolve_with_a_warm_start_is_refused():
    p, f = small_problem()
    m, n = len(f["lc"]), len(f["c"])
    data = {k: np.zeros(n if prim else m) for k, prim in zip(capi.WARM_VECTORS, capi.WARM_IS_PRIMAL)}
    data.update({k: 1.0 for k in capi.WARM_SCALARS})
    s = capi.Settings(presolve=True, log_to_console=False)
    s.set_warm_start(capi.WarmStart.create(m, n, data))
    sol = capi.solve(p, s)
    assert sol.return_code == capi.CUOPT_VALIDATION_ERROR and "warm start" in sol.error_string


def test_presolve_with_warm_start_capture_is_refused():
    p, _ = small_problem()
    s = capi.Settings(presolve=True, log_to_console=False)
    s.capture_warm_start()
    sol = capi.solve(p, s)
    assert sol.return_code == capi.CUOPT_VALIDATION_ERROR and "capture" in sol.error_string


def test_presolve_in_a_distributed_solve_is_refused():
    import ctypes as C
    p, _ = small_problem()
    s = capi.Settings(presolve=True, log_to_console=False)
    h = C.c_void_p()
    # the refusal comes before the communicator is used: any non-null handle reaches it
    rc = capi.lib().cuOptB200SolveDistributed(p.h, s.h, C.c_void_p(1), C.byref(h))
    sol = capi.Solution(h, p.num_constraints, p.num_variables, rc)
    assert rc == capi.CUOPT_VALIDATION_ERROR and "multi-GPU" in sol.error_string


# ------------------------------------------------------------------------------------------------------ GPU
def problem_of(f):
    return capi.Problem.create_ranged(f["offsets"], f["indices"], f["values"], f["lc"], f["uc"], f["c"], f["l"], f["u"],
                                      maximize=f["maximize"], objective_offset=f["offset"])


def settings(tol=1e-8, **kw):
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, presolve=True)
    s.set("optimality_tolerance", tol)
    for k, v in kw.items():
        s.set(k, v)
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("name", OPTIMAL)
def test_device_reduced_problem_matches_the_restatement(name):
    f, r = fixture(name), reference(name)
    g = capi.Solver(problem_of(f), settings())
    np.testing.assert_array_equal(g.vector("presolve_row_map"), r["row_map"])
    np.testing.assert_array_equal(g.vector("presolve_col_map"), r["col_map"])
    np.testing.assert_array_equal(g.vector("presolve_c"), r["c"])
    tol_rows = row_sum_tolerance(r["shift_mag"], np.maximum(r["shift_len"], 1.0))
    for k in ("lc", "uc"):
        got, want = g.vector("presolve_" + k), r[k]
        fin = np.isfinite(want)
        np.testing.assert_array_equal(np.isfinite(got), fin)
        assert np.all(np.abs(got[fin] - want[fin]) <= tol_rows[fin]), k
    for k in ("l", "u"):
        got, want = g.vector("presolve_" + k), r[k]
        fin = np.isfinite(want)
        np.testing.assert_array_equal(np.isfinite(got), fin)
        assert np.all(np.abs(got[fin] - want[fin]) <= 1e-12 * (1 + np.abs(want[fin]))), k
    assert g.scalar("presolve_offset") == pytest.approx(r["offset"], rel=1e-12, abs=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("name", ["singleton_zoo_1", "bound_zoo"])
def test_reduced_solve_follows_the_oracle_stepwise(name, mode):
    f, r = fixture(name), reference(name)
    g = capi.Solver(problem_of(f), settings(pdlp_solver_mode=mode))
    o = po.Oracle(r["offsets"], r["indices"], r["values"], r["c"], r["l"], r["u"], r["lc"], r["uc"], mode=mode, tol=1e-8)
    g.initialise(); o.initialise()
    for steps in (1, 2, 5, 20):
        g.advance(steps); o.run(steps)
        for v in ("x", "y", "aty"):
            assert rel_err(g.vector(v), o.vector(v)) <= STEPWISE, (steps, v)


def original_kkt(f, x, y, rc):
    A = sp.csr_matrix((f["values"], f["indices"], f["offsets"]), shape=(len(f["lc"]), len(f["c"])))
    ax = A @ x
    viol = np.maximum(f["lc"] - ax, 0) + np.maximum(ax - f["uc"], 0)
    c = min_form(f)
    # dual residual: the part of r = c - A^T y no finite bound can absorb
    dres = np.where((rc > 0) & ~np.isfinite(f["l"]), rc, 0.0) + np.where((rc < 0) & ~np.isfinite(f["u"]), rc, 0.0)
    return ax, viol, c, dres, A


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in OPTIMAL if n != "planted_large"])
def test_postsolved_solution_satisfies_the_original_kkt_conditions(name):
    f, r = fixture(name), reference(name)
    sol = capi.solve(problem_of(f), settings())
    assert sol.return_code == 0 and sol.termination_reason == "Optimal", sol.error_string
    st, ps = sol.stats(), sol.presolve_stats()
    assert ps.ran == 1 and ps.reduced_m == len(r["row_map"]) and ps.reduced_n == len(r["col_map"])
    assert (ps.fixed_columns, ps.empty_rows, ps.singleton_rows, ps.empty_columns, ps.rounds) == (
        r["fixed_columns"], r["empty_rows"], r["singleton_rows"], r["empty_columns"], r["rounds"])
    x, y, rc = sol.primal(), sol.dual(), sol.reduced_costs()
    ax, viol, c, dres, A = original_kkt(f, x, y, rc)
    removed_rows = ~r["row_alive"]
    scale = 1.0 + np.abs(np.where(np.isfinite(f["lc"]), f["lc"], 0)) + np.abs(np.where(np.isfinite(f["uc"]), f["uc"], 0))
    rounding = 1e-9 * scale
    assert np.all(viol[removed_rows] <= rounding[removed_rows])
    assert np.linalg.norm(viol) <= st.l2_primal_residual + 1e-9 * np.linalg.norm(scale)
    assert np.allclose(rc, c - A.T @ y, rtol=0, atol=1e-9 * (1 + np.abs(c)).max())
    assert np.linalg.norm(dres) <= st.l2_dual_residual + 1e-7 * (1 + np.linalg.norm(c))
    # complementarity on removed rows and columns: |multiplier| x distance to the bound its sign names
    for i in np.flatnonzero(removed_rows):
        bound = f["lc"][i] if y[i] > 0 else f["uc"][i]
        gap = abs(ax[i] - bound) if np.isfinite(bound) else (inf if y[i] != 0 else 0.0)
        assert abs(y[i]) * gap <= 1e-6 * (1 + abs(ax[i])), (i, y[i], ax[i], bound)
    for j in np.flatnonzero(~r["col_alive"]):
        if f["l"][j] == f["u"][j] or rc[j] == 0:
            continue
        bound = f["l"][j] if rc[j] > 0 else f["u"][j]
        assert np.isfinite(bound) and abs(rc[j]) * abs(x[j] - bound) <= 1e-6 * (1 + abs(x[j])), (j, rc[j], x[j], bound)
    want = highs_of(f, c=f["c"]).fun if not f["maximize"] else -highs_of(f).fun
    assert st.primal_objective == pytest.approx(want + f["offset"], rel=1e-6, abs=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("name,verdict", VERDICTS)
def test_verdicts_with_full_size_vectors(name, verdict):
    f = fixture(name)
    sol = capi.solve(problem_of(f), settings())
    assert sol.return_code == 0 and sol.termination_status == VERDICT[verdict], (sol.termination_reason, sol.error_string)
    x, y, rc = sol.primal(), sol.dual(), sol.reduced_costs()
    assert len(x) == len(f["c"]) and len(y) == len(f["lc"]) and len(rc) == len(f["c"])
    if verdict == "Optimal":
        assert sol.stats().primal_objective == pytest.approx(highs_of(f).fun, rel=1e-9, abs=1e-12)
        assert np.all((x >= f["l"]) & (x <= f["u"]))


@pytest.mark.gpu
@pytest.mark.parametrize("name,verdict,removed", RAYS)
def test_returned_ray_certifies_the_original_problem(name, verdict, removed):
    """With presolve on, the certificate PDLP finds on the reduced problem comes back through postsolve and certifies the
    ORIGINAL problem under the exact restatement of exact.py (Stable2: reduced-cost rule 0).  A dual ray needs the duals
    of the singleton rows whose bounds it rests on."""
    f = fixture(name)
    sol = capi.solve(problem_of(f), settings(tol=1e-4, infeasibility_detection=True, strict_infeasibility=True,
                                             iteration_limit=100000, pdlp_solver_mode=po.STABLE2))
    assert sol.return_code == 0 and sol.termination_status == VERDICT[verdict], (sol.termination_reason, sol.error_string)
    assert sol.presolve_stats().ran == 1
    lp = LP(name, f["offsets"], f["indices"], f["values"], min_form(f), f["l"], f["u"], f["lc"], f["uc"])
    ok, ratio = certifies(lp, sol.primal(), sol.dual(), VERDICT[verdict], 0)
    assert ok, (ratio, sol.primal().tolist(), sol.dual().tolist())


@pytest.mark.gpu
def test_identity_when_nothing_is_removed():
    for lp in identity_lps():
        p = capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb,
                                       lp.var_ub)
        out = []
        for on in (False, True):
            s = settings(tol=1e-6)
            s.set("presolve", on)
            sol = capi.solve(p, s)
            assert sol.return_code == 0
            out.append((sol.primal(), sol.dual(), sol.reduced_costs(), sol.stats().number_of_steps_taken,
                        sol.stats().primal_objective))
        for a, b_ in zip(*out):
            np.testing.assert_array_equal(a, b_)


@pytest.mark.gpu
@pytest.mark.parametrize("ending", ["iteration_limit", "save_best_primal_so_far", "infeasibility_detection",
                                    "per_constraint_residual", "solution_file"])
def test_every_ending_is_postsolved(ending, tmp_path):
    f = fixture("afiro")  # 2 singleton rows removed; several hundred iterations to 1e-6
    kw = {"iteration_limit": 20} if ending in ("iteration_limit", "save_best_primal_so_far") else {}
    if ending not in ("iteration_limit", "solution_file"):
        kw[ending] = True
    path = tmp_path / "afiro.sol"
    problem = problem_of(f)
    if ending == "solution_file":
        kw["solution_file"] = str(path)
        problem = capi.Problem.read(mps_path("linear_programming/afiro_original.mps"))  # with its names
    sol = capi.solve(problem, settings(tol=1e-6, **kw))
    assert sol.return_code == 0, sol.error_string
    assert sol.termination_reason == ("IterationLimit" if "iteration_limit" in kw else "Optimal")
    x, y, rc = sol.primal(), sol.dual(), sol.reduced_costs()
    assert len(x) == len(f["c"]) and len(y) == len(f["lc"]) and len(rc) == len(f["c"])
    assert sol.presolve_stats().ran == 1 and sol.presolve_stats().reduced_m == len(f["lc"]) - 2
    if ending == "solution_file":
        lines = path.read_text().splitlines()[2:]   # one line per named variable of the original problem
        assert len(lines) == len(f["c"])
        np.testing.assert_allclose([float(ln.split()[1]) for ln in lines], x, rtol=1e-15, atol=0)


@pytest.mark.gpu
def test_cli_presolve_on_the_sudoku_relaxation():
    exe = b.build_cli()
    r = subprocess.run([exe, mps_path("mip/sudoku.mps"), "--relaxation", "--method", "1", "--presolve", "true",
                        "--optimality-tolerance", "1e-8"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "Status: Optimal" in r.stdout and "Presolve:" in r.stdout
    want = highs_of(fixture("sudoku")).fun
    line = next(ln for ln in r.stdout.splitlines() if ln.startswith("Status:"))
    got = float(line.split("Objective:")[1].split()[0])
    assert got == pytest.approx(want, rel=1e-6, abs=1e-6)
