"""Infeasibility detection (k_infeasibility_rows / k_infeasibility_cols) against an exact restatement, at chosen points.

`detection_np` of exact.py restates termination_strategy/infeasibility_information.cu and termination_strategy.cu:229-249
in numpy with the kernels' order of operations: homogeneous row bounds (a finite bound becomes 0), max_violation of the
ray, g = -A^T y with both reduced-cost rules, bound_value_product, compute_remaining_stats (pobj = c.x * (1 / xinf), the
divisions by max(yinf, rcinf)) and the two tests.  Products are correctly rounded row sums (row_sums_hp), sums are fsum.

cuOptB200SolverInfeasibilityStats runs the evaluation's products and both detection kernels at caller-given current and
average points; the two slots always get different points, so a mix-up of the iterates shows.  Two families:
  exact  the synthetic certificate zoo of cases.py (small integer matrices) at integer or dyadic points: every product
         and partial sum is exact in any order, so all 24 statistics and both verdicts must be bit-equal;
  real   planted_bounds medium (also maximised: detection sees the negated c), and the wide cases tall / short_rows
         (past one launch wave and 256 partials per quantity) at random full-support points: maxima of exact inputs are
         bit-equal, the rest within the componentwise rounding bounds, after asserting on the CPU that no branch decision
         lies within rounding of its threshold.
Each runs unblocked and with forced cuts of 3 and 16 column blocks, under Stable2 (reduced-cost rule 0) and Stable1
(rule 1).  Planted rays are checked as exact Farkas certificates in fractions, and HiGHS confirms every LP's status.
"""
import functools
import math
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.optimize import linprog

from cases import BLOCKING, CERT_STATUS, CERTIFICATES, HIGHS_STATUS, certificate_args, planted_bounds, wide
from cuopt_b200 import capi
from device_model import gather_block_bytes  # noqa: F401
from device_model import session as dm_session
from exact import LP, U53, certifies, detection_np, dot_tolerance, highs, rule_of
from oracle import pdlp_oracle as po

inf = np.inf
STATS = capi.Solver.INFEASIBILITY_STATS
MAXIMA = ("xinf", "max_viol", "yinf")           # maxima of exact inputs: bit-equal in both families
RULE_MODES = [po.STABLE2, po.STABLE1]            # reduced-cost rule 0, rule 1
EDGE_DELTA = 1e-6                                # relative offset of a tolerance from the ratio it is set against


# ------------------------------------------------------------------------------------------------- the restatement
def branch_margins_clear(lp, x, aux, rule):
    """No branch decision lies within rounding of its threshold: each row against its homogeneous bounds, the sign of g,
    and rule 1's |x - bound| <= |x|."""
    ax, tol = aux["ax"], aux["ax_tol"]
    for h in (aux["hl"], aux["hu"]):
        fin = np.isfinite(h)
        assert np.all((np.abs(ax[fin] - h[fin]) > tol[fin]) | ((ax[fin] == h[fin]) & (tol[fin] <= 1e-300))), \
            "a row sum lies within rounding of a homogeneous bound"
    g, gtol = aux["g"], aux["g_tol"]
    assert np.all((np.abs(g) > gtol) | ((g == 0.0) & (gtol <= 1e-300))), "the sign of g is not decided"
    if rule:
        b = aux["bound"]
        with np.errstate(invalid="ignore"):
            fin = np.isfinite(b)
            d = np.abs(np.abs(x[fin] - b[fin]) - np.abs(x[fin]))
            assert np.all((d == 0.0) & (b[fin] == 0.0) | (d > 4 * U53 * (np.abs(x[fin]) + np.abs(b[fin])))), \
                "rule 1 is undecided on a column"


def real_tolerances(lp, aux, st):
    """Absolute bounds for the statistics of the real family that are not maxima of exact inputs."""
    cx_tol = dot_tolerance(aux["cx_terms"])
    d_tol = dot_tolerance(aux["dobj_terms"]) + 4 * U53 * abs(st["dobj_raw"])
    hd_tol = float(np.max(aux["g_tol"], initial=0.0))
    xinf, sc = st["xinf"], aux["scaling"]
    hr_tol = float(np.max(aux["ax_tol"], initial=0.0))
    t = dict(cx=cx_tol, hres=hr_tol, rcinf=hd_tol, hdres_raw=hd_tol, dobj_raw=d_tol,
             pobj=(cx_tol / xinf if xinf else 0.0) + 4 * U53 * abs(st["pobj"]),
             max_primal=(hr_tol / xinf if xinf else 0.0) + 4 * U53 * abs(st["max_primal"]))
    t["hdres"] = (hd_tol / sc if sc else 0.0) + 4 * U53 * abs(st["hdres"]) + (hd_tol * st["hdres"] / sc if sc else 0.0)
    t["dobj"] = (d_tol / sc if sc else 0.0) + 4 * U53 * abs(st["dobj"]) + (hd_tol * abs(st["dobj"]) / sc if sc else 0.0)
    return t


# ------------------------------------------------------------------------------------------------------- the LPs
def zoo_lp(name):
    return LP(name, *certificate_args(name))


def exact_ray(lp, status):
    """An integer ray found by HiGHS on the ray LP and made integral (the ray LPs are scale-invariant).
    status 2: y with y_i > 0 only on finite lc_i, < 0 only on finite uc_i, and g = -A^T y pressing only on finite
    variable bounds, maximising the dual-ray objective; status 3: x in the homogeneous bounds with c.x < 0."""
    A = sp.csr_matrix((lp.values, lp.indices, lp.offsets), shape=(lp.m, lp.n))
    if status == 2:
        # variables [yp, ym (m each), gp, gm (n each)], all >= 0: yp only on finite lc, ym on finite uc, gp on finite l,
        # gm on finite u
        fl, fu = np.isfinite(lp.l), np.isfinite(lp.u)
        ylo = np.where(np.isfinite(lp.uc), -1.0, 0.0)
        yhi = np.where(np.isfinite(lp.lc), 1.0, 0.0)
        # max lc.yp - uc.ym + l.gp - u.gm over y = yp - ym, -A^T y = gp - gm (an underestimate of the ray objective)
        Aeq = sp.hstack([A.T, -A.T, sp.identity(lp.n), -sp.identity(lp.n)]).tocsr()
        c = np.concatenate([-np.where(np.isfinite(lp.lc), lp.lc, 0.0), np.where(np.isfinite(lp.uc), lp.uc, 0.0),
                            -np.where(fl, lp.l, 0.0), np.where(fu, lp.u, 0.0)])
        bounds = np.column_stack([np.zeros(2 * lp.m + 2 * lp.n),
                                  np.concatenate([yhi, -ylo, np.where(fl, 10.0, 0.0), np.where(fu, 10.0, 0.0)])])
        res = linprog(c, A_eq=Aeq, b_eq=np.zeros(lp.n), bounds=bounds, method="highs")
        assert res.status == 0 and res.fun < 0, (lp.name, res.message)
        v = res.x[:lp.m] - res.x[lp.m:2 * lp.m]
    else:
        fl, fu = np.isfinite(lp.lc), np.isfinite(lp.uc)
        A_ub = sp.vstack([-A[fl], A[fu]]).tocsr()
        bounds = np.column_stack([np.where(np.isfinite(lp.l), 0.0, -1.0), np.where(np.isfinite(lp.u), 0.0, 1.0)])
        res = linprog(lp.c, A_ub=A_ub if A_ub.shape[0] else None, b_ub=np.zeros(A_ub.shape[0]) if A_ub.shape[0] else None,
                      bounds=bounds, method="highs")
        assert res.status == 0 and res.fun < 0, (lp.name, res.message)
        v = res.x
    fr = [Fraction(float(t)).limit_denominator(64) for t in v]
    den = math.lcm(*[f.denominator for f in fr])
    ray = np.array([float(f * den) for f in fr])
    assert is_certificate(lp, ray, status), lp.name
    return ray


def is_certificate(lp, ray, status):
    """The exact Farkas conditions in fractions (ray entries, matrix values and bounds are floats, held exactly)."""
    F = Fraction
    col_of = np.repeat(np.arange(lp.m), np.diff(lp.offsets))
    fin = lambda b: b is not None and math.isfinite(b)  # noqa: E731
    if status == 2:
        g = [F(0)] * lp.n
        for i, j, a in zip(col_of, lp.indices, lp.values):
            g[j] -= F(float(a)) * F(float(ray[i]))
        total = F(0)
        for i, yi in enumerate(ray):
            if yi > 0:
                if not fin(lp.lc[i]):
                    return False
                total += F(float(yi)) * F(float(lp.lc[i]))
            elif yi < 0:
                if not fin(lp.uc[i]):
                    return False
                total += F(float(yi)) * F(float(lp.uc[i]))
        for j, gj in enumerate(g):
            if gj > 0:
                if not fin(lp.l[j]):
                    return False
                total += gj * F(float(lp.l[j]))
            elif gj < 0:
                if not fin(lp.u[j]):
                    return False
                total += gj * F(float(lp.u[j]))
        return total > 0
    ax = [F(0)] * lp.m
    for i, j, a in zip(col_of, lp.indices, lp.values):
        ax[i] += F(float(a)) * F(float(ray[j]))
    ok_rows = all((not fin(lp.lc[i]) or ax[i] >= 0) and (not fin(lp.uc[i]) or ax[i] <= 0) for i in range(lp.m))
    ok_cols = all((not fin(lp.l[j]) or ray[j] >= 0) and (not fin(lp.u[j]) or ray[j] <= 0) for j in range(lp.n))
    return ok_rows and ok_cols and sum(F(float(c)) * F(float(r)) for c, r in zip(lp.c, ray)) < 0


# the synthetic zoo: the MPS fixtures carry decimal values (2.7, 10.1), whose products are not exact in fp64; they are
# checked through the certificates the solver returns (test_bound_structures.py::test_certificate_verdict)
ZOO_INFEASIBLE = [n for n in CERTIFICATES if CERT_STATUS[n] in (2, 3) and not n.startswith("good-mps")]


@functools.lru_cache(maxsize=None)
def zoo_ray(name):
    return exact_ray(zoo_lp(name), CERT_STATUS[name])


def exact_points(lp, status, ray):
    """Integer / dyadic (x, y) pairs of the exact family, each reaching a branch."""
    rng = np.random.default_rng(abs(hash(lp.name)) % 2**32)
    dy = lambda k: rng.integers(-16, 17, k) / 8.0  # noqa: E731
    x_ray = ray if status == 3 else np.zeros(lp.n)
    y_ray = ray if status == 2 else np.zeros(lp.m)
    x_ray_zero = x_ray
    # every variable bound kind's branch: components on each finite bound, beyond it and inside, duals of both signs
    xb = dy(lp.n)
    xb = np.where(np.isfinite(lp.l) & (rng.random(lp.n) < 0.3), lp.l, xb)
    xb = np.where(np.isfinite(lp.u) & (rng.random(lp.n) < 0.3), lp.u, xb)
    yb = dy(lp.m)
    if status == 2:  # x on the bound g = -A^T y presses on (exact: small integers), so rule 1 keeps that bound too
        g = -(sp.csr_matrix((lp.values, lp.indices, lp.offsets), shape=(lp.m, lp.n)).T @ ray)
        x_ray = np.where((g > 0) & np.isfinite(lp.l), lp.l, np.where((g < 0) & np.isfinite(lp.u), lp.u, dy(lp.n)))
    pts = [("ray", x_ray, y_ray if status == 2 else dy(lp.m)),
           ("ray_noise", x_ray_zero + dy(lp.n) / 8, y_ray + dy(lp.m) / 8),
           ("bound_branches", xb, yb),
           ("x_zero", np.zeros(lp.n), yb[::-1].copy()),
           ("y_zero", xb[::-1].copy(), np.zeros(lp.m)),
           ("dobj_nonpositive", -x_ray_zero, -y_ray)]
    return pts


EDGES = ["infeasible_ranged_row", "unbounded_free_var", "unbounded_upper_only_var_negative_cost"]


def real_points(lp, seed, x_star=None, y_star=None):
    rng = np.random.default_rng(seed)
    x = np.clip(rng.normal(0.0, 3.0, lp.n), np.where(np.isfinite(lp.l), lp.l - 1.0, -inf),
                np.where(np.isfinite(lp.u), lp.u + 1.0, inf))
    y = rng.normal(0.0, 1.0, lp.m)
    pts = [("random", x, y), ("random_2", rng.normal(0.0, 1.0, lp.n), rng.normal(0.0, 2.0, lp.m)),
           ("x_zero", np.zeros(lp.n), y * 0.5), ("y_zero", x * 0.5, np.zeros(lp.m))]
    if x_star is not None:
        pts.append(("optimum", x_star, y_star))
    return pts


@functools.lru_cache(maxsize=None)
def real_lp(name):
    """(LP as detection sees it, the problem as posed, planted optimum or None)."""
    if name.startswith("medium"):
        p = planted_bounds(3000, 2500, 22, maximize=name == "medium_max")
        lp = LP(name, p.offsets, p.indices, p.values, p.c, p.var_lb, p.var_ub, p.con_lb, p.con_ub)
        prob = capi.Problem.create_ranged(p.offsets, p.indices, p.values, p.con_lb, p.con_ub, p.user_c, p.var_lb,
                                          p.var_ub, maximize=p.maximize)
        return lp, prob, (p.x_star, p.y_star)
    case, p = wide(name)
    lp = LP(name, p.offsets, p.indices, p.values, p.c, p.var_lb, p.var_ub, p.con_lb, p.con_ub)
    prob = capi.Problem.create_ranged(p.offsets, p.indices, p.values, p.con_lb, p.con_ub, p.c, p.var_lb, p.var_ub)
    return lp, prob, (p.x_star, p.y_star)


REAL = ["medium", "medium_max", "tall", "short_rows"]


@functools.lru_cache(maxsize=None)
def real_reference(name, rule, k):
    """(statistics, status, tolerances) of point k of real_points, its branch margins asserted clear."""
    lp, _, (xs, ys) = real_lp(name)
    _, x, y = real_points(lp, 7, xs, ys)[k]
    want, status, aux = detection_np(lp, x, y, rule)
    branch_margins_clear(lp, x, aux, rule)
    return want, status, real_tolerances(lp, aux, want)


# ---------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("name", ZOO_INFEASIBLE)
def test_every_planted_ray_is_an_exact_farkas_certificate(name):
    lp, status = zoo_lp(name), CERT_STATUS[name]
    ray = zoo_ray(name)
    assert is_certificate(lp, ray, status)
    assert np.all(ray == np.round(ray)) and np.max(np.abs(ray)) < 2.0 ** 20
    st, verdict, _ = detection_np(lp, ray if status == 3 else np.zeros(lp.n), ray if status == 2 else np.zeros(lp.m),
                                  0)
    assert verdict == status and (st["hdres"] == 0.0 if status == 2 else st["max_primal"] == 0.0)


@pytest.mark.parametrize("name", ZOO_INFEASIBLE)
def test_highs_confirms_each_status(name):
    assert highs(*certificate_args(name)).status == HIGHS_STATUS[CERT_STATUS[name]]


def test_exact_family_is_exact():
    """Every product and partial sum of the exact family is an integer multiple of 2^-12 below 2^40: exact in fp64."""
    for name in ZOO_INFEASIBLE:
        lp = zoo_lp(name)
        assert np.all(lp.values == np.round(lp.values * 8) / 8) and np.max(np.abs(lp.values)) <= 64
        for b in (lp.c, lp.l, lp.u, lp.lc, lp.uc):
            f = b[np.isfinite(b)]
            assert np.all(f == np.round(f * 8) / 8) and np.all(np.abs(f) <= 2.0 ** 20)
        for _, x, y in exact_points(lp, CERT_STATUS[name], zoo_ray(name)):
            for v in (x, y):
                assert np.all(v * 64 == np.round(v * 64)) and np.all(np.abs(v) < 2.0 ** 20)


@pytest.mark.parametrize("name", ["medium", "medium_max", "tall"])
def test_restatement_reports_no_verdict_at_planted_optima(name):
    lp, _, (xs, ys) = real_lp(name)
    for rule in (0, 1):
        _, status, _ = detection_np(lp, xs, ys, rule)
        assert status == 6


@pytest.mark.parametrize("name", EDGES)
def test_edge_points_exist(name):
    edge_points(name)


def test_restatement_threshold_rules():
    """dobj > 0 and pobj < 0 are strict; the ratio tests are <=."""
    lp = zoo_lp("infeasible_equality_row")
    ray = zoo_ray("infeasible_equality_row")
    st, status, _ = detection_np(lp, np.zeros(lp.n), ray, 0, ptol=0.0)
    assert status == 2 and st["hdres"] == 0.0           # 0 <= 0
    st, status, _ = detection_np(lp, np.zeros(lp.n), -ray, 0)
    assert status == 6 and st["dobj"] < 0.0


# ------------------------------------------------------------------------------------------------------- GPU tests
def session(lp, prob, mode, force, blocks, **kw):
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=mode, **kw)
    return dm_session(lp, prob, s, blocks, force)


def zoo_problem(name):
    off, idx, val, c, l, u, lc, uc = certificate_args(name)
    return capi.Problem.create_ranged(off, idx, val, lc, uc, c, l, u)


def stats_of(g, pa, pb):
    stats, status = g.infeasibility_stats(pa[1], pa[2], pb[1], pb[2])
    return [dict(zip(STATS, stats[v])) for v in range(2)], status


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
@pytest.mark.parametrize("mode", RULE_MODES)
@pytest.mark.parametrize("name", ZOO_INFEASIBLE)
def test_statistics_bit_equal_on_the_exact_family(name, mode, blocks, gather_block_bytes):
    lp, status = zoo_lp(name), CERT_STATUS[name]
    g = session(lp, zoo_problem(name), mode, gather_block_bytes, blocks)
    pts = exact_points(lp, status, zoo_ray(name))
    rule = rule_of(mode)
    seen = set()
    for k in range(len(pts)):
        pair = (pts[k], pts[(k + 1) % len(pts)])
        got, got_status = stats_of(g, *pair)
        for v in range(2):
            want, want_status, _ = detection_np(lp, pair[v][1], pair[v][2], rule)
            for q in STATS:
                assert got[v][q] == want[q] or (math.isnan(got[v][q]) and math.isnan(want[q])), \
                    (pair[v][0], v, q, got[v][q], want[q])
            assert got_status[v] == want_status, (pair[v][0], v)
            seen.add(want_status)
    assert status in seen


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
@pytest.mark.parametrize("mode", RULE_MODES)
@pytest.mark.parametrize("name", REAL)
def test_statistics_within_rounding_on_the_real_family(name, mode, blocks, gather_block_bytes):
    lp, prob, (xs, ys) = real_lp(name)
    g = session(lp, prob, mode, gather_block_bytes, blocks)
    if blocks is not None:
        assert g.scalar("eval_blocks") >= 3 and g.scalar("eval_blocks_t") >= 3
    if name in ("tall", "short_rows"):
        assert g.scalar("grid_m") > 256 or g.scalar("grid_n") > 256
    pts = real_points(lp, 7, xs, ys)
    for k in range(len(pts)):
        pair = (pts[k], pts[(k + 1) % len(pts)])
        got, got_status = stats_of(g, *pair)
        for v in range(2):
            want, want_status, tol = real_reference(name, rule_of(mode), (k + v) % len(pts))
            for q in STATS:
                if q in MAXIMA:
                    assert got[v][q] == want[q], (pair[v][0], v, q, got[v][q], want[q])
                else:
                    assert abs(got[v][q] - want[q]) <= tol[q], (pair[v][0], v, q, got[v][q], want[q], tol[q])
            assert got_status[v] == want_status == 6, (pair[v][0], v)


def edge_points(name):
    """The planted ray plus dyadic noise whose ratio lies in (0, 0.09) (the first of a seeded search), the other side of
    the tests held at 0 so that it draws no verdict.  Returns (LP, status, x, y, ratio)."""
    lp, status = zoo_lp(name), CERT_STATUS[name]
    ray = zoo_ray(name)
    for seed in range(200):
        rng = np.random.default_rng(seed)
        scale = (1 / 64, 1 / 16, 1 / 4)[seed % 3]
        if status == 2:
            x, y = np.zeros(lp.n), ray + rng.integers(-4, 5, lp.m) * scale
        else:
            x, y = ray + rng.integers(-4, 5, lp.n) * scale, np.zeros(lp.m)
        st, _, _ = detection_np(lp, x, y, 0)
        if status == 2 and st["dobj"] > 0.0:
            ratio = st["hdres"] / st["dobj"]
        elif status == 3 and st["pobj"] < 0.0:
            ratio = st["max_primal"] / -st["pobj"]
        else:
            continue
        if 0.0 < ratio < 0.09:
            return lp, status, x, y, ratio
    raise AssertionError(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", EDGES)
def test_verdict_appears_exactly_on_the_le_side_of_the_threshold(name, gather_block_bytes):
    """The tolerance set to the reference ratio x (1 - delta), x 1 and x (1 + delta).  The exact family's ratio is the
    kernel's to the last bit, so delta (1e-6) is far above its rounding (one division, 2^-53)."""
    lp, status, x, y, ratio = edge_points(name)
    key = "primal_infeasible_tolerance" if status == 2 else "dual_infeasible_tolerance"
    other = np.zeros(lp.n), np.zeros(lp.m)
    for factor, want in ((1.0 - EDGE_DELTA, 6), (1.0, status), (1.0 + EDGE_DELTA, status)):
        g = session(lp, zoo_problem(name), po.STABLE2, gather_block_bytes, None, **{key: ratio * factor})
        _, got = stats_of(g, ("edge", x, y), ("zero",) + other)
        assert got[0] == want, (factor, ratio, got)


@pytest.mark.gpu
def test_the_call_leaves_the_session_unchanged(gather_block_bytes):
    lp, prob, (xs, ys) = real_lp("medium")
    runs = []
    for call in (False, True):
        g = session(lp, prob, po.STABLE2, gather_block_bytes, None, infeasibility_detection=True)
        g.advance(40)
        before = g.scalar("k_total")
        if call:
            stats, status = g.infeasibility_stats(xs, ys, xs * 0.5, ys * 0.5)
            assert status == [6, 6]
            assert g.scalar("k_total") == before
        g.advance(200)
        runs.append([g.vector(v) for v in ("x", "y", "aty", "x_avg", "y_avg", "sum_x", "sum_y")] +
                    [np.array([g.scalar(s) for s in ("step_size", "primal_weight", "k_total", "k_pdhg",
                                                     "its_since_restart", "n_restarts")])])
    for a, b in zip(*runs):
        np.testing.assert_array_equal(a, b)


@pytest.mark.gpu
def test_refusals_and_detection_off(gather_block_bytes):
    name = "infeasible_equality_row"
    lp = zoo_lp(name)
    gather_block_bytes(None)
    g = capi.Solver(zoo_problem(name), capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False))
    z = np.zeros(lp.n), np.zeros(lp.m)
    with pytest.raises(capi.CuOptError) as e:
        g.infeasibility_stats(z[0], z[1], z[0], z[1])
    assert e.value.code == capi.CUOPT_INVALID_ARGUMENT
    g.initialise()   # infeasibility_detection is off in this session
    _, status = g.infeasibility_stats(np.zeros(lp.n), zoo_ray(name), z[0], z[1])
    assert status == [2, 6]


def embedded(name):
    """The wide case `tall` with the zoo certificate `name` appended block-diagonally; the planted ray padded with
    zeros certifies the whole LP (its rows and columns meet none of tall's)."""
    _, t = wide("tall")
    off, idx, val, c, l, u, lc, uc = certificate_args(name)
    big = LP(f"tall+{name}", np.concatenate([t.offsets, t.offsets[-1] + off[1:]]),
             np.concatenate([t.indices, idx + t.n]), np.concatenate([t.values, val]), np.concatenate([t.c, c]),
             np.concatenate([t.var_lb, l]), np.concatenate([t.var_ub, u]), np.concatenate([t.con_lb, lc]),
             np.concatenate([t.con_ub, uc]))
    ray = zoo_ray(name)
    pad = np.concatenate([np.zeros(t.m), ray]) if CERT_STATUS[name] == 2 else np.concatenate([np.zeros(t.n), ray])
    return big, pad


def test_embedded_ray_certifies_the_wide_lp():
    big, ray = embedded("infeasible_equality_row")
    st, status, _ = detection_np(big, np.zeros(big.n), ray, 0)
    assert status == 2 and st["hdres"] == 0.0 and st["dobj"] > 0.0
    small = zoo_lp("infeasible_equality_row")
    assert is_certificate(small, zoo_ray("infeasible_equality_row"), 2)   # the padding adds only exact zeros


@pytest.mark.gpu
def test_primal_infeasibility_verdict_at_width():
    """PrimalInfeasible on tall (600 000 x 400 000, past one launch wave and 256 partials per quantity) with a certificate
    block: strict rule, Stable2, and the returned ray certifies the whole LP."""
    big, _ = embedded("infeasible_equality_row")
    p = capi.Problem.create_ranged(big.offsets, big.indices, big.values, big.lc, big.uc, big.c, big.l, big.u)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, infeasibility_detection=True,
                      strict_infeasibility=True, iteration_limit=100000, pdlp_solver_mode=po.STABLE2)
    sol = capi.solve(p, s)
    assert sol.return_code == 0, sol.error_string
    print(f"tall + infeasible_equality_row: {sol.termination_reason} after {sol.stats().number_of_steps_taken} steps")
    assert sol.termination_status == 2, sol.termination_reason
    ok, ratio = certifies(big, sol.primal(), sol.dual(), 2, 0)
    assert ok, ratio
