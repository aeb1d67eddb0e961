"""Every kind of variable and constraint bound against exact references, under all four presets.

The synthetic LPs of the other test files all have 0 <= x < +inf and rows of kind E, L or G, so the branches of the
kernels that depend on the BOUND KIND ran only on afiro and a few MIP relaxations, and were checked there only through
parity with the oracle or final objectives.  This file builds a seeded zoo of LPs that hold every kind in every role of
a planted optimum (numpy, complementary slackness as planted() of cases.py):

  variables  free; [l, +inf) with l < 0, l = 0, l > 0, at the bound or inside; (-inf, u] at the bound or inside;
             boxes at either bound or inside, straddling 0, entirely above 0, entirely below 0; one box 1e-6 |l| wide;
             fixed l == u with reduced costs of both signs, and l = u = 0
  rows       E; L and G active or inactive; ranged active at lc, at uc or inactive; free rows with entries; an empty
             ranged row containing 0

and a second family of small LPs that are infeasible or unbounded BECAUSE of one bound kind.  CPU tests prove the
census, confirm each planted optimum and each certificate with HiGHS, and check the oracle against every criterion
below before it serves as a witness.  GPU tests (every preset; unblocked and with 3 forced column blocks where a
product is involved) compare the setup, the primal and dual steps, the evaluation, the trust-region bounds and whole
solves with plain numpy / fsum references.

Sign conventions: y_i > 0 presses on lc_i, y_i < 0 on uc_i; r_j = (c - A^T y)_j > 0 presses on l_j, r_j < 0 on u_j.
A maximisation is solved as the minimisation of -c (problem_helpers.cuh:127 of the reference: c <- -c and the objective
scaling factor becomes -1), so the solver's y and reduced costs are those of min -c'x, and both reported objectives are
-(that objective) + offset.

The cases are planted_bounds() and certificates() of cases.py.  Tolerances: those of exact.py (componentwise
row-sum bound 4 len 2^-53 sum|a_ij v_j| for every product).
"""
import math

import numpy as np
import pytest
import scipy.sparse as sp

from cases import (BOUND_ZOO as ZOO, CERT_STATUS, CERTIFICATES, HIGHS_STATUS, VAR_ROLES, bound_zoo as zoo,
                   bounds_oracle as oracle_of, bounds_problem as problem_of, certificate_args, certificates, mps_arrays,
                   settings_of)
from cuopt_b200 import capi, lpgen
from device_model import block_bytes, gather_block_bytes  # noqa: F401
from device_model import session as dm_session
from exact import (ACROSS_TRUST_REGION, OBJECTIVE, STEPWISE, TRAJECTORY, U53, LP, bound_value_product, certifies,
                   close_counts, device_formulation, dual_step_reference, highs, reduced_costs_np, rel_err, row_sum_tolerance,
                   row_sums_hp, rule_of, scaled_problem, scaled_transpose, transpose_product)
from oracle import pdlp_oracle as po

inf = np.inf
FAST1_TRAJECTORY = 1e-5
BOUND_SLACK = 1e-12  # relative to max(1, |bound|)
MODES = [po.STABLE1, po.STABLE2, po.METHODICAL1, po.FAST1]

MPS_OPTIMA = [("lp_model_with_var_bounds", -2.0), ("good-mps-some-var-bounds", -0.2), ("good-mps-rhs-cost", -5.0)]
# PDLP tests for a ray only while the iterate is primal INFEASIBLE (termination_strategy.cu:141-227 of the reference:
# Optimal / PrimalFeasible are decided first).  On these two fixtures the diverging iterate stays primal feasible (one
# L row, a free variable), so PDLP (the reference, the oracle and this build alike) ends with NumericalError (6) when
# the iterate overflows, not with HiGHS's Unbounded; the synthetic certificates put an equality row in the way of the ray.
PDLP_STATUS = {**CERT_STATUS, "good-mps-free-var": 6, "good-mps-lower-bound-inf-var": 6}


# ------------------------------------------------------------------------------------------------- numpy references
def evaluation_np(lp, x, y, rc):
    """Primal / dual objectives of the posed problem, l2 residuals, gap, and the linf per-constraint criteria, from
    fsum over exact products, with `rc` the reduced costs the evaluation used; plus absolute tolerances."""
    ax, mag, lens = row_sums_hp(lp.offsets, lp.indices, lp.values, x)
    axtol = row_sum_tolerance(mag, lens)
    with np.errstate(invalid="ignore"):
        viol = np.where(ax < lp.con_lb, lp.con_lb - ax, np.where(ax > lp.con_ub, ax - lp.con_ub, 0.0))
    aty, magt, lenst = transpose_product(lp.offsets, lp.indices, lp.values, lp.n, y)
    g = lp.c - aty
    sgn = -1.0 if lp.maximize else 1.0
    prods = lp.c * x
    pobj = sgn * math.fsum(prods.tolist()) + lp.offset
    dterms = np.concatenate([bound_value_product(y, lp.con_lb, lp.con_ub), bound_value_product(rc, lp.var_lb, lp.var_ub)])
    dobj = sgn * math.fsum(dterms.tolist()) + lp.offset
    fin = lambda b: np.where(np.isfinite(b), np.abs(b), 0.0)  # noqa: E731
    b = np.maximum(fin(lp.con_lb), fin(lp.con_ub))
    return dict(primal_objective=pobj, dual_objective=dobj, gap=abs(pobj - dobj),
                l2_primal_residual=math.sqrt(math.fsum((viol * viol).tolist())),
                l2_dual_residual=math.sqrt(math.fsum(((g - rc) ** 2).tolist())),
                viol=viol, g=g, b=b,
                tol_primal=float(np.linalg.norm(axtol)) + 1e-300,
                tol_dual=float(np.linalg.norm(row_sum_tolerance(magt, lenst) + 4 * U53 * (np.abs(lp.c) + np.abs(aty)))),
                tol_objective=8 * U53 * (math.fsum(np.abs(prods).tolist()) + math.fsum(np.abs(dterms).tolist()) +
                                         abs(lp.offset)) + 1e-300)


def assert_evaluation(lp, x, y, rc, st):
    ref = evaluation_np(lp, x, y, rc)
    for v, tol in (("primal_objective", ref["tol_objective"]), ("dual_objective", ref["tol_objective"]),
                   ("gap", 2 * ref["tol_objective"]), ("l2_primal_residual", ref["tol_primal"]),
                   ("l2_dual_residual", ref["tol_dual"])):
        got = getattr(st, v)
        tol = tol + 1e-12 * abs(ref[v])  # the device sums in its own order: a relative rounding allowance
        assert abs(got - ref[v]) <= tol, (v, got, ref[v], tol)
    return ref


# ------------------------------------------------------------------------------------------------------- CPU tests
def test_every_case_has_every_bound_kind_in_the_role_it_is_named_for():
    for name in ZOO:
        lp = zoo(name)
        l, u, x, r, y = lp.var_lb, lp.var_ub, lp.x_star, lp.r_star, lp.y_star
        lc, uc = lp.con_lb, lp.con_ub
        lens = np.diff(lp.offsets)
        fl, fu = np.isfinite(l), np.isfinite(u)
        kinds = {
            "free": ~fl & ~fu & (r == 0),
            "lower_neg_at": fl & ~fu & (l < 0) & (x == l) & (r > 0), "lower_neg_in": fl & ~fu & (l < 0) & (x > l) & (r == 0),
            "lower_zero_at": (l == 0) & ~fu & (x == 0) & (r > 0), "lower_zero_in": (l == 0) & ~fu & (x > 0) & (r == 0),
            "lower_pos_at": fl & ~fu & (l > 0) & (x == l) & (r > 0), "lower_pos_in": fl & ~fu & (l > 0) & (x > l) & (r == 0),
            "upper_neg_at": ~fl & fu & (u < 0) & (x == u) & (r < 0), "upper_pos_at": ~fl & fu & (u > 0) & (x == u) & (r < 0),
            "upper_in": ~fl & fu & (x < u) & (r == 0),
            "box_at_l": fl & fu & (l < 0) & (u > 0) & (x == l) & (r > 0),
            "box_at_u": fl & fu & (l < 0) & (u > 0) & (x == u) & (r < 0),
            "box_in": fl & fu & (l < 0) & (u > 0) & (x > l) & (x < u) & (r == 0),
            "box_above_at_l": (l > 0) & fu & (l < u) & (x == l) & (r > 0), "box_above_at_u": (l > 0) & fu & (x == u) & (r < 0),
            "box_above_in": (l > 0) & fu & (x > l) & (x < u) & (r == 0),
            "box_below_at_l": fl & (u < 0) & (l < u) & (x == l) & (r > 0), "box_below_at_u": fl & (u < 0) & (x == u) & (r < 0),
            "box_below_in": fl & (u < 0) & (x > l) & (x < u) & (r == 0),
            "box_thin": fl & (u > l) & (u - l <= 2e-6 * np.abs(l)) & (x == l) & (r > 0),
            "fixed_r_pos": (l == u) & (r > 0), "fixed_r_neg": (l == u) & (r < 0), "fixed_zero": (l == 0) & (u == 0),
        }
        assert set(kinds) == set(VAR_ROLES)
        for k, mask in kinds.items():
            named = lp.var_role == k
            assert named.any() and mask[named].all(), (name, k)
        ax = row_sums_hp(lp.offsets, lp.indices, lp.values, x)[0]
        flc, fuc = np.isfinite(lc), np.isfinite(uc)
        close = lambda a, b: np.abs(a - b) <= 1e-9 * (1 + np.abs(b))  # noqa: E731
        rows = {
            "E": (lc == uc) & close(ax, lc),
            "L_active": ~flc & fuc & close(ax, uc) & (y < 0), "L_inactive": ~flc & fuc & (ax < uc - 0.1) & (y == 0),
            "G_active": flc & ~fuc & close(ax, lc) & (y > 0), "G_inactive": flc & ~fuc & (ax > lc + 0.1) & (y == 0),
            "ranged_at_lc": flc & fuc & (lc < uc) & close(ax, lc) & (y > 0),
            "ranged_at_uc": flc & fuc & (lc < uc) & close(ax, uc) & (y < 0),
            "ranged_inside": flc & fuc & (ax > lc + 0.1) & (ax < uc - 0.1) & (y == 0),
            "free": ~flc & ~fuc & (lens > 0) & (y == 0),
            "empty_ranged": (lens == 0) & (lc < 0) & (uc > 0) & (y == 0),
        }
        for k, mask in rows.items():
            named = lp.row_role == k
            assert named.any() and mask[named].all(), (name, k)
        assert (lp.y_star[lp.row_role == "E"] > 0).any() and (lp.y_star[lp.row_role == "E"] < 0).any()
        # the planted pair is optimal: primal feasible, dual feasible, equal objectives
        assert np.all(l <= x) and np.all(x <= u) and np.all(lc - 1e-9 * (1 + np.abs(lc)) <= ax)
        assert np.all(ax <= uc + 1e-9 * (1 + np.abs(uc)))
        dual = math.fsum(np.concatenate([bound_value_product(y, lc, uc), bound_value_product(r, l, u)]).tolist())
        assert dual == pytest.approx(float(lp.c @ x), rel=1e-12)
    assert zoo("medium").m == 3000 and zoo("medium").n == 2500 and np.all(np.diff(zoo("medium").offsets) <= 6)
    assert np.diff(zoo("heavy").offsets).max() > 100   # the heavy-tail rows are long enough to be long rows
    assert zoo("medium_max").maximize and zoo("medium_offset").offset != 0.0


@pytest.mark.parametrize("name", ZOO)
def test_highs_confirms_the_planted_optimum(name):
    lp = zoo(name)
    res = highs(lp.offsets, lp.indices, lp.values, lp.c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub)
    assert res.status == 0, res.message
    sgn = -1.0 if lp.maximize else 1.0
    assert sgn * res.fun + lp.offset == pytest.approx(lp.optimal_objective, rel=1e-9, abs=1e-9)


@pytest.mark.parametrize("name", CERTIFICATES)
def test_highs_confirms_each_certificate(name):
    assert highs(*certificate_args(name)).status == HIGHS_STATUS[CERT_STATUS[name]]
    if not name.startswith("good-mps"):  # ... and without the bound kind it is named for, the LP has an optimum
        k = next(k for k in certificates() if k.name == name)
        l, u, lc, uc = k.l.copy(), k.u.copy(), k.lc.copy(), k.uc.copy()
        if name in ("infeasible_fixed_var", "infeasible_upper_only_var"):
            l[0], u[0] = 0.0, inf
        elif "upper_only" in name or "minus_inf" in name:
            l[0] = -10.0
        elif "ranged" in name:
            lc[0], uc[0] = -inf, inf
        elif "equality" in name:
            lc[0] = -inf
            uc[0] = 10.0
        elif "free" in name:
            l[0] = -10.0
        elif "because_of_upper_bound" in name:
            u[0] = inf
        res = highs(k.offsets, k.indices, k.values, k.c, l, u, lc, uc)
        assert res.status == (3 if k.status == 1 else 0), (name, res.message)


@pytest.mark.parametrize("name,value", MPS_OPTIMA)
def test_highs_confirms_the_mps_optima(name, value):
    a = mps_arrays(name)
    res = highs(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"])
    assert res.status == 0 and res.fun + a["objective_offset"] == pytest.approx(value, rel=1e-9)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ZOO)
def test_oracle_meets_every_criterion(name, mode):
    """The oracle's setup, single attempt, evaluation and trust-region bounds against the numpy references."""
    lp = zoo(name)
    o = oracle_of(lp, mode)
    o.initialise()
    dr, dc = o.vector("row_scaling"), o.vector("col_scaling")
    with np.errstate(divide="ignore", invalid="ignore"):
        assert np.array_equal(o.vector("scaled_l"), np.where(dc == 0, 0.0, lp.var_lb / dc))
        assert np.array_equal(o.vector("scaled_u"), np.where(dc == 0, 0.0, lp.var_ub / dc))
    assert np.array_equal(o.vector("scaled_lc"), lp.con_lb * dr)
    assert np.array_equal(o.vector("scaled_uc"), lp.con_ub * dr)
    # one attempt from a point that sits on bounds, with duals of every sign
    rng = np.random.default_rng(5)
    ls, us = o.vector("scaled_l"), o.vector("scaled_u")
    x = np.clip(rng.normal(0.0, 3.0, lp.n), ls, us)
    y = rng.normal(0.0, 1.0, lp.m)
    case = lp
    scaled = o.vector("scaled_values")
    T = scaled_transpose(case, scaled, o.vector("scaled_values_t"))
    aty, mag, lens = row_sums_hp(*T, y)
    tau, sigma = 0.37, 0.61
    got = o.single_attempt(x, y, aty, tau, sigma)
    cs = o.vector("scaled_c")
    want = np.maximum(np.minimum(x - tau * (cs - aty), us), ls)
    tol = tau * row_sum_tolerance(mag, lens) + 8 * U53 * (np.abs(x) + tau * (np.abs(cs) + np.abs(aty)))
    assert np.all(np.abs(got["x_next"] - want) <= tol)
    assert np.all(got["x_next"] >= ls) and np.all(got["x_next"] <= us)
    want, tol = dual_step_reference(case, scaled, got["x_bar"], y, sigma, o.vector("scaled_lc"), o.vector("scaled_uc"))
    assert np.all(np.abs(got["y_next"] - want) <= tol)
    # the evaluation of an unscaled point with the preset's reduced-cost rule
    xu = np.clip(rng.normal(0.0, 3.0, lp.n), lp.var_lb, lp.var_ub)
    xu[::3] = np.where(np.isfinite(lp.var_lb[::3]), lp.var_lb[::3], xu[::3])   # on the lower bound
    yu = lp.y_star + rng.normal(0.0, 0.1, lp.m)
    cv = o.convergence(xu, yu)
    rc, g, tol, exempt = reduced_costs_np(lp, xu, yu, rule_of(mode))
    assert exempt.sum() <= 2
    assert np.all(np.abs(cv["reduced_cost"] - rc)[~exempt] <= tol[~exempt])
    ref = evaluation_np(lp, xu, yu, cv["reduced_cost"])
    assert cv["primal_objective"] == pytest.approx(ref["primal_objective"], abs=ref["tol_objective"], rel=1e-12)
    assert cv["dual_objective"] == pytest.approx(ref["dual_objective"], abs=ref["tol_objective"], rel=1e-12)
    assert cv["l2_primal_residual"] == pytest.approx(ref["l2_primal_residual"], abs=ref["tol_primal"], rel=1e-12)
    assert cv["l2_dual_residual"] == pytest.approx(ref["l2_dual_residual"], abs=ref["tol_dual"], rel=1e-12)
    if mode == po.METHODICAL1:
        o.run(7)
        prob = (sp.csr_matrix((scaled, lp.indices, lp.offsets), shape=(lp.m, lp.n)), cs, ls, us, o.vector("scaled_lc"),
                o.vector("scaled_uc"))
        for px, py in tr_points(lp, prob, o.vector("x"), o.vector("y")):
            for radius in (0.0, 1e-6, 0.5, 1e6):
                lo_want, up_want, _ = o.trust_region_bounds(px, py, radius)
                lo_got, up_got = device_formulation(*prob, o.scalar("tau"), o.scalar("sigma"), px, py, radius)
                scale = max(1.0, abs(lo_want), abs(up_want))
                assert abs(lo_got - lo_want) <= 1e-9 * scale and abs(up_got - up_want) <= 1e-9 * scale, (radius,)


def tr_points(lp, prob, x, y):
    """Points of the scaled space for the trust-region bounds: an iterate; the same with components put on each of
    their finite bounds (either gradient sign follows from the random duals) and duals of every sign, -0.0 among them;
    and the planted optimum (many components on bounds pressing outwards: a run of equal zero thresholds).  A zero
    threshold is always +0.0 (tr_direction returns early for a component on a bound pressing outwards, and a computed
    threshold is a ratio of two numbers of one sign), so -0.0 appears in the centres, not in the sorted keys."""
    _, _, ls, us, lcs, ucs = prob
    rng = np.random.default_rng(9)
    px = x.copy()
    on_l = np.isfinite(ls) & (rng.random(lp.n) < 0.4)
    on_u = np.isfinite(us) & ~on_l & (rng.random(lp.n) < 0.5)
    px[on_l], px[on_u] = ls[on_l], us[on_u]
    py = rng.normal(0.0, 1.0, lp.m)
    py[rng.random(lp.m) < 0.2] = 0.0
    # dual feasible, as every iterate is: y >= 0 where uc = +inf, y <= 0 where lc = -inf
    py = np.where(np.isfinite(ucs), py, np.maximum(py, 0.0))
    py = np.where(np.isfinite(lcs), py, np.minimum(py, 0.0))
    py[(py == 0.0) & (rng.random(lp.m) < 0.5)] = -0.0
    px[np.flatnonzero(px == 0.0)[::2]] = -0.0
    return [(x, y), (px, py)]


def test_oracle_reaches_each_certificate_verdict():
    for name in CERTIFICATES:
        for strict in (False, True):
            off, idx, val, c, l, u, lc, uc = certificate_args(name)
            o = po.Oracle(off, idx, val, c, l, u, lc, uc, tol=1e-4, detect_infeasibility=True,
                          strict_infeasibility=strict, iteration_limit=CERT_CAP)
            o.run(-1)
            assert o.stats().termination_status == PDLP_STATUS[name], (name, strict, o.stats().termination_status)


CERT_CAP = 100000


# ------------------------------------------------------------------------------------------------------- GPU tests
def session(lp, mode, blocks, force):
    g = dm_session(lp, problem_of(lp), settings_of(mode, 1e-9), blocks, force)
    if blocks is not None:
        assert g.scalar("eval_blocks") >= 3 and g.scalar("eval_blocks_t") >= 3
    return g


# the tiny case is below one column block: forcing blocks would not change what runs
PRODUCT_CASES = [(n, b) for n in ZOO for b in ((None,) if n == "tiny" else (None, 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,blocks", PRODUCT_CASES)
def test_setup_preserves_every_bound_kind(name, blocks, mode, gather_block_bytes):
    lp = zoo(name)
    g = session(lp, mode, blocks, gather_block_bytes)
    dr, dc = g.vector("row_scaling"), g.vector("col_scaling")
    ls, us, lcs, ucs = g.vector("scaled_l"), g.vector("scaled_u"), g.vector("scaled_lc"), g.vector("scaled_uc")
    with np.errstate(divide="ignore", invalid="ignore"):
        assert np.array_equal(ls, np.where(dc == 0, 0.0, lp.var_lb / dc))
        assert np.array_equal(us, np.where(dc == 0, 0.0, lp.var_ub / dc))
    assert np.array_equal(lcs, lp.con_lb * dr) and np.array_equal(ucs, lp.con_ub * dr)
    for got, want in ((ls, lp.var_lb), (us, lp.var_ub), (lcs, lp.con_lb), (ucs, lp.con_ub)):
        assert np.array_equal(np.isposinf(got), np.isposinf(want)) and np.array_equal(np.isneginf(got), np.isneginf(want))
    x0 = g.vector("x")
    hp = po.preset(mode)
    if hp.project_initial_primal:
        assert np.array_equal(x0, np.clip(0.0, ls, us))
        assert (x0 != 0.0).any()  # boxes above / below 0: the projection moves something
    else:
        assert not x0.any()
    # norms of the unscaled problem, initial step size and primal weight
    fin = lambda b: np.where(np.isfinite(b), np.abs(b), 0.0)  # noqa: E731
    comb = lambda lo, hi: np.maximum(fin(lo), fin(hi))  # noqa: E731  combine_finite_abs_bounds
    sumtol = lambda k: 2 * k * U53  # noqa: E731  a sum of k non-negative terms in any order
    assert g.scalar("l2_norm_c") == pytest.approx(math.sqrt(math.fsum((lp.c ** 2).tolist())), rel=sumtol(lp.n))
    assert g.scalar("l2_norm_b") == pytest.approx(math.sqrt(math.fsum((comb(lp.con_lb, lp.con_ub) ** 2).tolist())),
                                                  rel=sumtol(lp.m))
    assert g.scalar("step_size") == hp.initial_step_size_scaling / np.max(np.abs(g.vector("scaled_values")))
    if hp.compute_initial_primal_weight_before_scaling:
        cc, b = lp.c, comb(lp.con_lb, lp.con_ub)
    else:
        cc, b = g.vector("scaled_c"), comb(lcs, ucs)
    cn = math.sqrt(math.fsum((cc * cc * hp.initial_primal_weight_c_scaling).tolist()))
    bn = math.sqrt(math.fsum((b * b * hp.initial_primal_weight_b_scaling).tolist()))
    assert g.scalar("primal_weight") == pytest.approx(hp.primal_importance * cn / bn, rel=sumtol(lp.m + lp.n))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,blocks", PRODUCT_CASES)
def test_primal_and_dual_steps_respect_every_bound_kind(name, blocks, mode, gather_block_bytes):
    """K1 and K2 of every step accepted at its first attempt, element by element, and the exact invariants."""
    lp = zoo(name)
    g = session(lp, mode, blocks, gather_block_bytes)
    case = lp
    scaled = g.vector("scaled_values")
    T = scaled_transpose(case, scaled, g.vector("scaled_values_t"))
    c, l, u, lc, uc = (g.vector(v) for v in ("scaled_c", "scaled_l", "scaled_u", "scaled_lc", "scaled_uc"))
    fixed, free = lp.var_lb == lp.var_ub, ~np.isfinite(lp.con_lb) & ~np.isfinite(lp.con_ub)
    is_l, is_g = ~np.isfinite(lp.con_lb) & np.isfinite(lp.con_ub), np.isfinite(lp.con_lb) & ~np.isfinite(lp.con_ub)
    checked = 0
    for _ in range(30):
        if checked == 4:
            break
        x, y, tau, sigma = g.vector("x"), g.vector("y"), g.scalar("tau"), g.scalar("sigma")
        attempts, restarts = g.scalar("k_pdhg"), g.scalar("n_restarts")
        aty, mag, lens = row_sums_hp(*T, y)
        g.advance(1)
        if g.scalar("n_restarts") != restarts:
            continue  # a restart to the average rounds a weighted mean: the invariants below are those of a step
        xn, yn = g.vector("x"), g.vector("y")
        assert np.all(l <= xn) and np.all(xn <= u) and np.array_equal(xn[fixed], l[fixed])
        assert np.all(yn[free] == 0.0) and np.all(yn[is_l] <= 0.0) and np.all(yn[is_g] >= 0.0)
        if g.scalar("k_pdhg") != attempts + 1:
            continue
        want = np.maximum(np.minimum(x - tau * (c - aty), u), l)
        tol = tau * row_sum_tolerance(mag, lens) + 8 * U53 * (np.abs(x) + tau * (np.abs(c) + np.abs(aty)))
        bad = np.flatnonzero(~(np.abs(xn - want) <= tol))
        assert bad.size == 0, ("columns", bad[:8].tolist(), lp.var_role[bad[:8]].tolist(), xn[bad[:8]], want[bad[:8]])
        want, tol = dual_step_reference(case, scaled, g.vector("x_bar"), y, sigma, lc, uc)
        bad = np.flatnonzero(~(np.abs(yn - want) <= tol))
        assert bad.size == 0, ("rows", bad[:8].tolist(), lp.row_role[bad[:8]].tolist(), yn[bad[:8]], want[bad[:8]])
        checked += 1
    assert checked >= 3


def check_solution_evaluation(lp, sol, mode):
    x, y, st = sol.primal(), sol.dual(), sol.stats()
    rc_np, g, tol, exempt = reduced_costs_np(lp, x, y, rule_of(mode))
    rc = sol.reduced_costs()
    assert exempt.sum() <= 2, exempt.sum()
    bad = np.flatnonzero(~(np.abs(rc - rc_np) <= tol) & ~exempt)
    assert bad.size == 0, ("columns", bad[:8].tolist(), lp.var_role[bad[:8]].tolist(), rc[bad[:8]], rc_np[bad[:8]])
    return assert_evaluation(lp, x, y, rc, st)


@pytest.mark.gpu
@pytest.mark.parametrize("iterations", [1, 7, 40])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,blocks", PRODUCT_CASES)
def test_evaluation_of_every_bound_kind(name, blocks, mode, iterations, gather_block_bytes):
    """Reduced costs under the preset's rule, objectives (offset, maximisation), residuals and gap at the returned
    iterate.  The iteration limit is looked at where the preset evaluates (every major_iteration steps, and at the
    first step where it does), so a limit of 1, 7 or 40 returns the iterate of the first evaluation at or past it."""
    lp = zoo(name)
    gather_block_bytes(block_bytes(lp, blocks))
    sol = capi.solve(problem_of(lp), settings_of(mode, tol=1e-12, iteration_limit=iterations))
    assert sol.return_code == 0, sol.error_string
    assert sol.termination_reason == "IterationLimit"
    assert 1 <= sol.stats().number_of_steps_taken <= max(iterations, po.preset(mode).major_iteration)
    check_solution_evaluation(lp, sol, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ZOO)
def test_per_constraint_residual_verdict(name, mode):
    """per_constraint_residual: linf of (violation_i - rel max(|lc_i|, |uc_i|)) over rows (ranged and one-sided rows
    take the larger finite bound) and of ((g - rc)_j - rel c_j) over columns, against the absolute tolerances."""
    lp = zoo(name)
    probe = capi.solve(problem_of(lp), settings_of(mode, tol=1e-12, iteration_limit=PROBE_STEPS,
                                                   per_constraint_residual=True))
    assert probe.termination_reason == "IterationLimit"
    x, y, rc = probe.primal(), probe.dual(), probe.reduced_costs()
    ref = evaluation_np(lp, x, y, rc)
    rel = 1e-12
    lp_inf = float(np.max(ref["viol"] - rel * ref["b"], initial=0.0))
    ld_inf = float(np.max((ref["g"] - rc) - rel * lp.c, initial=0.0))
    # the settings accept at most 0.1; a criterion already met (0: the reduction is seeded with 0) is held to exactly 0
    assert lp_inf < 0.09 and ld_inf < 0.09 and max(lp_inf, ld_inf) > 0.0, (lp_inf, ld_inf)
    # absolute tolerances 1 % above both recomputed criteria (relative ones 1e-12, the gap loose): the same trajectory
    # must now stop as Optimal, at this iterate or an earlier one.  A device criterion that read a row kind's bound
    # wrongly, or dropped it, would exceed the recomputed one and keep going.
    s = settings_of(mode, tol=1e-12, iteration_limit=PROBE_STEPS, per_constraint_residual=True)
    s.set("absolute_primal_tolerance", lp_inf * 1.01)
    s.set("absolute_dual_tolerance", ld_inf * 1.01)
    s.set("absolute_gap_tolerance", 0.1)
    s.set("relative_gap_tolerance", 0.1)
    sol = capi.solve(problem_of(lp), s)
    assert sol.termination_reason == "Optimal", sol.termination_reason
    assert sol.stats().number_of_steps_taken <= probe.stats().number_of_steps_taken


PROBE_STEPS = 2000


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,blocks", PRODUCT_CASES)
def test_steps_match_oracle(name, blocks, mode, gather_block_bytes):
    """Step by step across the first major iteration of the preset and its restart."""
    lp = zoo(name)
    g = session(lp, mode, blocks, gather_block_bytes)
    o = oracle_of(lp, mode)
    o.initialise()
    last = po.preset(mode).major_iteration
    # Fast1 restarts inside the main loop and never to the average: its two trajectories separate faster across the
    # first major iteration (measured up to 1.1e-6 on the heavy case, H100)
    final = {po.METHODICAL1: ACROSS_TRUST_REGION, po.FAST1: FAST1_TRAJECTORY}.get(mode, TRAJECTORY)
    for steps, tol in ((1, STEPWISE), (1, STEPWISE), (3, STEPWISE), (last, final)):
        g.advance(steps); o.run(steps)
        for v in ("x", "y", "aty", "sum_x", "sum_y"):
            assert rel_err(g.vector(v), o.vector(v)) <= tol, (v, steps)
        for v in ("step_size", "primal_weight", "sum_w"):
            assert g.scalar(v) == pytest.approx(o.scalar(v), rel=tol), (v, steps)
        assert g.scalar("k_pdhg") == o.scalar("k_pdhg")


def tr_session_lp(name):
    """The zoo case, or on its tiny matrix: every threshold infinite (free variables, equality rows), or a gradient
    that vanishes at the origin (c = 0, ranged rows containing 0 and free rows)."""
    if name not in ("all_infinite", "zero_gradient"):
        return zoo(name)
    t = zoo("tiny")
    if name == "all_infinite":
        lp = lpgen.LP(t.offsets, t.indices, t.values, t.c, np.full(t.n, -inf), np.full(t.n, inf), np.ones(t.m),
                      np.ones(t.m))
    else:
        free = np.arange(t.m) % 3 == 0
        lp = lpgen.LP(t.offsets, t.indices, t.values, np.zeros(t.n), t.var_lb, t.var_ub, np.where(free, -inf, -1.0),
                      np.where(free, inf, 1.0))
    lp.user_c, lp.maximize, lp.offset = lp.c, False, 0.0
    return lp


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "medium", "heavy", "all_infinite", "zero_gradient"])
def test_trust_region_kernels_at_chosen_points(name):
    """k_tr_prepare / sort / k_tr_weights / k_tr_bisect / k_tr_bounds through the read-only session hook against the
    numpy transcription of the device formulation, at radii from 0 to 1e6."""
    lp = tr_session_lp(name)
    g = capi.Solver(problem_of(lp), settings_of(po.METHODICAL1, 1e-9))
    g.initialise()
    g.advance(5)
    prob = scaled_problem(lp, g)
    tau, sigma = g.scalar("tau"), g.scalar("sigma")
    x, y = g.vector("x"), g.vector("y")
    state = [g.vector(v) for v in ("x", "y", "aty", "sum_x", "sum_y", "x_last_restart")]
    if name == "zero_gradient":
        points = [(np.zeros(lp.n), np.zeros(lp.m))]
    elif name == "all_infinite":
        points = [(x, y), (x, y * 0.0 + 1.0)]
    else:
        points = tr_points(lp, prob, x, y) + [(lp.x_star / g.vector("col_scaling"), lp.y_star / g.vector("row_scaling"))]
    for px, py in points:
        for radius in (0.0, 1e-9, 1e-3, 0.5, 10.0, 1e6):
            want = device_formulation(*prob, tau, sigma, px, py, radius)
            got = g.trust_region_bounds(px, py, radius)
            scale = max(1.0, abs(want[0]), abs(want[1]))
            assert abs(got[0] - want[0]) <= 1e-9 * scale and abs(got[1] - want[1]) <= 1e-9 * scale, (radius, got, want)
            if name == "zero_gradient":
                assert got == (0.0, 0.0)
    for v, before in zip(("x", "y", "aty", "sum_x", "sum_y", "x_last_restart"), state):
        assert np.array_equal(g.vector(v), before), v   # the hook changes nothing
    with pytest.raises(capi.CuOptError):
        g.trust_region_bounds(x, y, -1.0)


# Fast1 does not reach 1e-8 on the medium cases within 400 000 iterations, on the CPU oracle either (IterationLimit at
# an objective within 3e-8 relative): a property of the preset, not of the kernels
FULL = [(n, m) for n in ZOO for m in MODES if not (m == po.FAST1 and n.startswith("medium"))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode", FULL)
def test_full_solve_reaches_planted_optimum(name, mode):
    lp = zoo(name)
    sol = capi.solve(problem_of(lp), settings_of(mode, tol=1e-8, iteration_limit=400000))
    assert sol.return_code == 0 and sol.termination_reason == "Optimal", sol.termination_reason
    st = sol.stats()
    scale = max(1.0, abs(lp.optimal_objective))
    assert abs(st.primal_objective - lp.optimal_objective) <= OBJECTIVE * scale
    assert abs(st.dual_objective - lp.optimal_objective) <= OBJECTIVE * scale
    # the returned x may be the average iterate, a rounded weighted mean unscaled by Dc: it meets the bounds to a few
    # tens of ulps (measured up to 6.6e-14 on |bound| ~ 10), not to 2 ulps as the current iterate would
    x = sol.primal()
    slack = lambda b: BOUND_SLACK * np.maximum(1.0, np.where(np.isfinite(b), np.abs(b), 0.0))  # noqa: E731
    assert np.all(x >= lp.var_lb - slack(lp.var_lb)) and np.all(x <= lp.var_ub + slack(lp.var_ub))
    fixed = lp.var_lb == lp.var_ub
    assert np.all(np.abs(x[fixed] - lp.var_lb[fixed]) <= slack(lp.var_lb)[fixed])


# Every preset under the strict rule; Stable2 under the non-strict rule too (Fast1's current and average iterates do not
# cross the threshold at the same major iteration on the unbounded cases within CERT_CAP, measured on an H100).
# Stable1 runs good-mps-free-var and good-mps-lower-bound-inf-var to the iteration limit (its iterate neither overflows
# nor passes the ray test within CERT_CAP, as the oracle shows), so those two are left out under Stable1.
VERDICT_CASES = [(n, m, strict) for n in CERTIFICATES for m in MODES for strict in (False, True)
                 if (strict or m == po.STABLE2)
                 and not (m == po.STABLE1 and n in ("good-mps-free-var", "good-mps-lower-bound-inf-var"))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode,strict", VERDICT_CASES)
def test_certificate_verdict(name, mode, strict):
    """The verdict under every preset, and the returned vectors re-evaluated on the LP by the exact restatement of
    exact.py with the preset's reduced-cost rule: they meet the criterion the solver reported."""
    off, idx, val, c, l, u, lc, uc = certificate_args(name)
    p = capi.Problem.create_ranged(off, idx, val, lc, uc, c, l, u)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, infeasibility_detection=True,
                      strict_infeasibility=strict, iteration_limit=CERT_CAP, pdlp_solver_mode=mode)
    sol = capi.solve(p, s)
    assert sol.return_code == 0, sol.error_string
    assert sol.termination_status == PDLP_STATUS[name], sol.termination_reason
    if sol.termination_status in (2, 3):
        ok, ratio = certifies(LP(name, off, idx, val, c, l, u, lc, uc), sol.primal(), sol.dual(),
                              sol.termination_status, rule_of(mode))
        assert ok, ratio
    if strict and mode == po.STABLE2:
        o = po.Oracle(off, idx, val, c, l, u, lc, uc, tol=1e-4, detect_infeasibility=True, strict_infeasibility=True,
                      iteration_limit=CERT_CAP)
        o.run(-1)
        assert close_counts(sol.stats().number_of_steps_taken, o.stats().number_of_steps_taken)
