"""Exact arithmetic and the references the tests build from it (support module: pytest does not collect it).

A row sum is compared COMPONENTWISE with the correctly rounded exact sum (`row_sums_hp`: error-free products,
math.fsum), never norm-wise: a dropped entry of a 6-entry row must not hide behind the magnitude of a dense row.

Tolerances:
  ROW_SUM      4 len 2^-53 sum_j |a_ij v_j| per row: the a-priori bound of ANY summation order of len products is
               len 2^-53 sum |.| to first order (with or without FMA); 4 is headroom for the second-order terms
  TINY         1e-300 absolute, so that an exact 0 compares with an exact 0
  ELEMENTWISE  1e-12 relative to the largest entry: setup vectors (a handful of roundings each, pow/sqrt in libm ulps)
  STEPWISE     1e-11 relative to the largest entry: iterates after the same steps from the same start, as
               test_gpu_parity.py::test_first_steps_match_oracle_elementwise
  TRAJECTORY   1e-7 relative: iterates after tens of steps across restarts (test_gpu_parity.py: a restart decision
               amplifies the last-bit differences of two summation orders)
  ACROSS_TRUST_REGION 1e-6 relative: the same across a trust-region restart of preset 2 (test_methodical1.py)
  OBJECTIVE    1e-6 relative: final objectives at PDLP tolerance 1e-8 against the planted optimum
"""
import functools
import math

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.optimize import linprog

from oracle import pdlp_oracle as po

U53 = 2.0 ** -53
ROW_SUM_FACTOR = 4.0
TINY = 1e-300
ELEMENTWISE, STEPWISE, TRAJECTORY, ACROSS_TRUST_REGION, OBJECTIVE = 1e-12, 1e-11, 1e-7, 1e-6, 1e-6


# ----------------------------------------------------------------------------------------- high-precision row sums
def two_product(a, b):
    """a b = p + e exactly (Veltkamp / Dekker; no overflow or underflow at the magnitudes used here)."""
    p = a * b
    ca, cb = 134217729.0 * a, 134217729.0 * b
    ah, bh = ca - (ca - a), cb - (cb - b)
    al, bl = a - ah, b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def row_sums_hp(offsets, indices, values, v):
    """(correctly rounded exact row sums of A v, sum_j |a_ij v_j|, row lengths)."""
    off = np.asarray(offsets, np.int64)
    a, g = np.asarray(values, float), np.asarray(v, float)[np.asarray(indices, np.int64)]
    p, e = two_product(a, g)
    pl, el = p.tolist(), e.tolist()
    sums = np.array([math.fsum(pl[lo:hi] + el[lo:hi]) for lo, hi in zip(off[:-1], off[1:])])
    lens = np.diff(off)
    mag = np.bincount(np.repeat(np.arange(len(lens)), lens), weights=np.abs(p), minlength=len(lens))
    return sums, mag, lens


def row_sum_tolerance(mag, lens):
    return ROW_SUM_FACTOR * lens * U53 * mag + TINY


def assert_row_sums(got, ref, what):
    sums, mag, lens = ref
    err = np.abs(np.asarray(got) - sums)
    bad = np.flatnonzero(~(err <= row_sum_tolerance(mag, lens)))
    assert bad.size == 0, (what, "rows", bad[:8].tolist(), "lengths", lens[bad[:8]].tolist(), "got", got[bad[:8]].tolist(),
                           "want", sums[bad[:8]].tolist())


def dot_tolerance(terms):
    return 2 * len(terms) * U53 * math.fsum(np.abs(terms).tolist()) + 1e-300


def rel_err(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b)))) if a.size else 0.0


def close_counts(gpu_steps, oracle_steps):
    """The certificate is reached on a DIVERGING iterate sequence, where rounding differences between the two
    implementations grow instead of being damped: same verdict, the
    iteration at which the 1e-8 threshold is crossed within a few major iterations / 50 %."""
    return abs(gpu_steps - oracle_steps) <= max(160, 0.5 * oracle_steps)


# -------------------------------------------------------------------------------------------------------- A^T
@functools.lru_cache(maxsize=None)
def _transpose(offsets, indices, n):
    m = len(offsets) // 8 - 1
    off, idx = np.frombuffer(offsets, np.int64), np.frombuffer(indices, np.int64)
    T = sp.csr_matrix((np.arange(1, len(idx) + 1, dtype=np.float64), idx, off), shape=(m, n)).T.tocsr()
    T.sort_indices()
    out = T.indptr, T.indices, T.data.astype(np.int64) - 1
    for a in out:
        a.flags.writeable = False
    return out


def transpose(offsets, indices, n):
    """(row offsets, column indices, source positions) of A^T for the CSR structure of A with n columns: entry k of A^T
    is entry positions[k] of A (stable order), so values[positions] are the values of A^T.  Cached; read-only."""
    return _transpose(np.asarray(offsets, np.int64).tobytes(), np.asarray(indices, np.int64).tobytes(), int(n))


def transpose_product(offsets, indices, values, n, y):
    """row_sums_hp of A^T y."""
    toff, tidx, pos = transpose(offsets, indices, n)
    return row_sums_hp(toff, tidx, np.asarray(values)[pos], y)


def scaled_transpose(case, scaled_values, scaled_values_t):
    """CSR of the scaled A^T: the structure of the input's transpose with the solver's own scaled values of A^T, after
    checking entry by entry that they are the scaled values of A at the transposed positions.  The two are scaled
    separately, (a Dr) Dc and (a Dc) Dr as the reference does, so they agree to two roundings, not bit for bit."""
    off, idx, pos = transpose(case.offsets, case.indices, case.n)
    moved = np.asarray(scaled_values)[pos]
    assert np.all(np.abs(scaled_values_t - moved) <= 4 * U53 * np.abs(moved))
    return off, idx, np.asarray(scaled_values_t)


# ----------------------------------------------------------------------------------------------- step references
def dual_step_reference(case, scaled_values, x_bar, y, sigma, lc, uc):
    """y' = max(ybar + sigma lc, min(ybar + sigma uc, 0)), ybar = y - sigma (A xbar), with its componentwise tolerance:
    the row-sum bound times sigma, plus a few roundings of the terms of the epilogue."""
    ax, mag, lens = row_sums_hp(case.offsets, case.indices, scaled_values, x_bar)
    nxt = y - sigma * ax
    with np.errstate(invalid="ignore"):
        want = np.maximum(nxt + sigma * lc, np.minimum(nxt + sigma * uc, 0.0))
    fin = lambda b: np.where(np.isfinite(b), np.abs(b), 0.0)  # noqa: E731
    tol = sigma * row_sum_tolerance(mag, lens) + 8 * U53 * (np.abs(y) + sigma * (np.abs(ax) + fin(lc) + fin(uc)))
    return want, tol


# ------------------------------------------------------------------------------------ reduced costs and the dual bound
def bound_value_product(v, lo, hi):
    """bound_value_product element-wise (the product rounded, as the kernel forms it)."""
    bound = np.where(v > 0.0, lo, np.where(v < 0.0, hi, 0.0))
    with np.errstate(invalid="ignore"):
        return np.where(np.isfinite(bound), v * bound, 0.0)


def rule_of(mode):
    """The reduced-cost rule of a preset: 0 keeps g_j where the bound it presses on is finite, 1 where
    |x_j - bound| <= |x_j|."""
    return po.preset(mode).handle_some_primal_gradients_on_finite_bounds_as_residuals


def reduced_cost(g, l, u, rule, x=None):
    """(reduced costs of the gradient g under rule 0 / rule 1, the bound each component presses on); rule 1 reads x."""
    bound = np.where(g > 0.0, l, u)
    with np.errstate(invalid="ignore"):
        keep = np.abs(x - bound) <= np.abs(x) if rule else np.isfinite(bound)
    return np.where((g != 0.0) & keep, g, 0.0), bound


def gradient_reference(lp, y):
    """(g = c - A^T y from exact row sums, A^T y, the componentwise tolerance of g)."""
    aty, mag, lens = transpose_product(lp.offsets, lp.indices, lp.values, lp.n, y)
    return lp.c - aty, aty, row_sum_tolerance(mag, lens) + 4 * U53 * (np.abs(lp.c) + np.abs(aty))


def reduced_cost_reference(lp, y):
    """Reduced costs of the default preset (rule 0) from exact row sums, and the componentwise tolerance; twice the
    row-sum bound, since a gradient within that bound of 0 may pick the other bound."""
    g, _, tol = gradient_reference(lp, y)
    return reduced_cost(g, lp.var_lb, lp.var_ub, 0)[0], g, 2.0 * tol


def reduced_costs_np(lp, x, y, rule):
    """(reduced costs under rule 0 / rule 1, g = c - A^T y, tolerance, exempt columns): exact products, fsum.
    Where |g| lies within its tolerance of 0 the bound it presses on may flip, but both answers (0 or g) then lie
    within twice that tolerance, which is what such a column is held to.  Exempt: under rule 1, |x - bound| and |x|
    within a few roundings of each other but not equal (the comparison itself may flip)."""
    g, _, tol = gradient_reference(lp, y)
    rc, bound = reduced_cost(g, lp.var_lb, lp.var_ub, rule, x)
    with np.errstate(invalid="ignore"):
        diff = np.abs(np.abs(x - bound) - np.abs(x))  # 0 for a zero bound: the comparison is then exact
        near = rule & np.isfinite(bound) & (diff > 0.0) & (diff < 4 * U53 * (np.abs(x) + np.abs(bound)))
    return rc, g, np.where(np.abs(g) <= tol, 2.0 * tol, tol), near


def check_evaluation(lp, sol, oracle):
    """stats() and reduced_costs() of a solution against a recomputation from its own primal() and dual(): the
    oracle's convergence of them, and the exact references."""
    assert sol.return_code == 0, sol.error_string
    x, y, st = sol.primal(), sol.dual(), sol.stats()
    cv = oracle.convergence(x, y)
    for v in ("l2_primal_residual", "l2_dual_residual", "primal_objective", "dual_objective", "gap"):
        assert getattr(st, v) == pytest.approx(cv[v], rel=STEPWISE, abs=STEPWISE), v
    rc, _, tol = reduced_cost_reference(lp, y)
    got = sol.reduced_costs()
    bad = np.flatnonzero(~(np.abs(got - rc) <= tol))
    assert bad.size == 0, ("columns", bad[:8].tolist(), got[bad[:8]].tolist(), rc[bad[:8]].tolist())
    ax = row_sums_hp(lp.offsets, lp.indices, lp.values, x)[0]
    viol = np.maximum(lp.con_lb - ax, 0.0) + np.maximum(ax - lp.con_ub, 0.0)
    assert st.l2_primal_residual == pytest.approx(np.linalg.norm(viol), rel=STEPWISE, abs=STEPWISE)


# ---------------------------------------------------------------------------------------- infeasibility detection
class LP:
    """A minimisation LP as detection sees it (c already negated for a maximisation)."""

    def __init__(self, name, offsets, indices, values, c, l, u, lc, uc):
        self.name = name
        self.offsets, self.indices = np.asarray(offsets, np.int32), np.asarray(indices, np.int32)
        self.values = np.asarray(values, float)
        self.c, self.l, self.u, self.lc, self.uc = (np.asarray(v, float) for v in (c, l, u, lc, uc))
        self.m, self.n = len(self.lc), len(self.c)


def detection_np(lp, x, y, rule, ptol=1e-8, dtol=1e-8):
    """termination_strategy/infeasibility_information.cu and termination_strategy.cu:229-249 of the reference in
    numpy, with the kernels' order of operations: homogeneous row bounds (a finite bound becomes 0), max_violation of
    the ray, g = -A^T y with either reduced-cost rule, bound_value_product, compute_remaining_stats (pobj = c.x *
    (1 / xinf), the divisions by max(yinf, rcinf)) and the two tests.  Products are correctly rounded row sums, sums
    are fsum.  -> (dict of the 12 statistics, status, dict of the data the branch margins and tolerances need)."""
    ax, amag, alen = row_sums_hp(lp.offsets, lp.indices, lp.values, x)
    aty, tmag, tlen = transpose_product(lp.offsets, lp.indices, lp.values, lp.n, y)
    hl, hu = np.where(np.isfinite(lp.lc), 0.0, lp.lc), np.where(np.isfinite(lp.uc), 0.0, lp.uc)
    viol = np.where(ax < hl, hl - ax, np.where(ax > hu, ax - hu, 0.0))
    hres = float(np.max(np.abs(viol), initial=0.0))
    yinf = float(np.max(np.abs(y), initial=0.0))
    dobj_rows = math.fsum(bound_value_product(y, lp.lc, lp.uc).tolist())
    xinf = float(np.max(np.abs(x), initial=0.0))
    max_viol = float(np.max(np.concatenate([np.where(np.isfinite(lp.l), -x, 0.0), np.where(np.isfinite(lp.u), x, 0.0),
                                            [0.0]])))
    g = -aty
    rc, bound = reduced_cost(g, lp.l, lp.u, rule, x)
    hdres_raw = float(np.max(np.abs(g - rc), initial=0.0))
    rcinf = float(np.max(np.abs(rc), initial=0.0))
    p, e = two_product(x, lp.c)
    cx = math.fsum(p.tolist() + e.tolist())
    dobj_cols = math.fsum(bound_value_product(rc, lp.l, lp.u).tolist())
    pobj = cx * (1.0 / xinf) if xinf != 0.0 else 0.0
    dobj_raw = dobj_rows + dobj_cols
    scaling = max(yinf, rcinf)
    hdres, dobj = (hdres_raw / scaling, dobj_raw / scaling) if scaling != 0.0 else (0.0, 0.0)
    if xinf > 0.0:
        max_primal = max(hres, max_viol) / xinf
    else:
        max_primal, pobj = 0.0, 0.0
    status = 6
    if dobj > 0.0 and hdres / dobj <= ptol:
        status = 2
    elif pobj < 0.0 and max_primal / -pobj <= dtol:
        status = 3
    st = dict(xinf=xinf, max_viol=max_viol, hres=hres, cx=cx, yinf=yinf, rcinf=rcinf, hdres_raw=hdres_raw,
              dobj_raw=dobj_raw, pobj=pobj, max_primal=max_primal, hdres=hdres, dobj=dobj)
    aux = dict(ax=ax, ax_tol=row_sum_tolerance(amag, alen), hl=hl, hu=hu, g=g, g_tol=row_sum_tolerance(tmag, tlen),
               bound=bound, rc=rc, cx_terms=lp.c * x,
               dobj_terms=np.concatenate([bound_value_product(y, lp.lc, lp.uc), bound_value_product(rc, lp.l, lp.u)]),
               scaling=scaling)
    return st, status, aux


def certifies(lp, x, y, status, rule, ptol=1e-8, dtol=1e-8):
    """Whether the returned (x, y) meet, on `lp` and within the rounding of the restatement, the criterion of the verdict
    `status` (2: y is a dual ray, 3: x a primal ray); returns (bool, the ratio)."""
    st, _, aux = detection_np(lp, x, y, rule)
    if status == 2:
        sc = aux["scaling"]
        if sc == 0.0:
            return False, np.inf
        hd = max(st["hdres_raw"] - float(np.max(aux["g_tol"], initial=0.0)), 0.0)
        d = st["dobj_raw"] + dot_tolerance(aux["dobj_terms"])
        return st["dobj"] > 0.0 and hd <= ptol * d, st["hdres"] / st["dobj"] if st["dobj"] > 0.0 else np.inf
    if st["xinf"] == 0.0:
        return False, np.inf
    mp = max(max(st["hres"] - float(np.max(aux["ax_tol"], initial=0.0)), 0.0), st["max_viol"])
    cx = st["cx"] - dot_tolerance(aux["cx_terms"])
    return st["pobj"] < 0.0 and mp <= dtol * -cx, st["max_primal"] / -st["pobj"] if st["pobj"] < 0.0 else np.inf


# ----------------------------------------------------------------------------------------------------------- HiGHS
def highs(offsets, indices, values, c, l, u, lc, uc):
    """linprog(method="highs") of min c'x, lc <= Ax <= uc, l <= x <= u (ranged rows as two inequalities)."""
    A = sp.csr_matrix((values, indices, offsets), shape=(len(lc), len(c)))
    eq = lc == uc
    up, lo = np.isfinite(uc) & ~eq, np.isfinite(lc) & ~eq
    A_ub = sp.vstack([A[up], -A[lo]]).tocsr()
    b_ub = np.concatenate([uc[up], -lc[lo]])
    return linprog(c, A_ub=A_ub if A_ub.shape[0] else None, b_ub=b_ub if A_ub.shape[0] else None,
                   A_eq=A[eq] if eq.any() else None, b_eq=lc[eq] if eq.any() else None,
                   bounds=np.column_stack([l, u]), method="highs")


# ------------------------------------------------------------------------------------ trust-region kernels (numpy)
def scaled_problem(lp, g):
    """scipy CSR of the scaled A and the scaled vectors of a session."""
    As = sp.csr_matrix((g.vector("scaled_values"), lp.indices, lp.offsets), shape=(lp.m, lp.n))
    return As, g.vector("scaled_c"), g.vector("scaled_l"), g.vector("scaled_u"), g.vector("scaled_lc"), g.vector("scaled_uc")


def device_formulation(As, cs, ls, us, lcs, ucs, tau, sigma, px, py, radius):
    """The trust-region solve as cuopt_b200/csrc/trust_region.cuh formulates it, transcribed: it does not re-reduce the
    active range at every trial threshold like the reference / the oracle, it sorts once, takes prefix sums of the two
    radius terms and evaluates every partial radius as a difference of prefix sums inside a single-thread bisection.
    -> (lower, upper) bound."""
    n, m = len(px), len(py)
    aty, ax = As.T @ py, As @ px
    # tr_component / tr_direction
    gp = cs - aty
    sub = np.where(py < 0, ucs, np.where(py > 0, lcs, 0.0))
    both_inf = ~np.isfinite(ucs) & ~np.isfinite(lcs)
    zero = py == 0
    sub = np.where(zero & both_inf, 0.0, sub)
    sub = np.where(zero & ~np.isfinite(ucs) & np.isfinite(lcs), lcs, sub)
    sub = np.where(zero & np.isfinite(ucs) & ~np.isfinite(lcs), ucs, sub)
    both_fin = zero & np.isfinite(ucs) & np.isfinite(lcs)
    sub = np.where(both_fin, np.clip(ax, np.where(both_fin, lcs, 0), np.where(both_fin, ucs, 0)), sub)
    gd = sub - ax
    center = np.concatenate([px, py])
    obj = np.concatenate([gp, -gd])
    lo = np.concatenate([ls, np.where(np.isfinite(ucs), -np.inf, 0.0)])
    up = np.concatenate([us, np.where(np.isfinite(lcs), np.inf, 0.0)])
    w = np.concatenate([np.full(n, 1.0 / tau), np.full(m, 1.0 / sigma)])
    lagrangian = px @ cs - px @ aty + py @ sub
    N = n + m
    # a component on a bound pressing outwards stays (direction 0, threshold 0); a zero gradient never stops (threshold inf)
    stay = ((center >= up) & (obj <= 0)) | ((center <= lo) & (obj >= 0))
    moves = ~stay & (obj != 0)
    dirv = np.where(moves, -obj / w, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        thr = np.where(moves, np.where(dirv > 0, (up - center) / dirv, (lo - center) / dirv),
                       np.where(stay, 0.0, np.inf))
    tr = center.copy()
    if not (radius == 0.0 or np.sqrt(obj @ obj) == 0.0):
        high_r2 = float(np.sum(np.where(np.isinf(thr), dirv * dirv * w, 0.0)))
        perm = np.argsort(thr, kind="stable")                       # cub::DeviceRadixSort (stable)
        ts, d, ww = thr[perm], dirv[perm], w[perm]
        with np.errstate(invalid="ignore"):
            A = np.where(np.isinf(ts), 0.0, (ts * d) ** 2 * ww)     # k_tr_weights
        B = d * d * ww
        PA, PB = np.cumsum(A), np.cumsum(B)                          # inclusive scans

        def rs(P, a, b):
            return (P[b - 1] - (P[a - 1] if a > 0 else 0.0)) if b > a else 0.0

        def first_ge(t, a, b):
            return a + int(np.searchsorted(ts[a:b], t, side="left"))

        def first_gt(t, a, b):
            return a + int(np.searchsorted(ts[a:b], t, side="right"))

        low, high, low_r2 = 0, first_ge(np.inf, 0, N), 0.0
        while low != high:                                            # k_tr_bisect
            size = high - low
            t = 0.5 * (ts[low + size // 2 - 1] + ts[low + size // 2]) if size % 2 == 0 else ts[low + size // 2]
            p = first_gt(t, low, high)
            test_r2 = rs(PA, low, p) + t * t * rs(PB, p, high)
            if low_r2 + test_r2 + t * t * high_r2 >= radius * radius:
                new_high = first_ge(t, low, high)
                high_r2 += rs(PB, new_high, high)
                high = new_high
            else:
                low_r2 += rs(PA, low, p)
                low = p
        T = ts[N - 1] if high_r2 <= 0.0 else np.sqrt((radius * radius - low_r2) / high_r2)
        moved = np.where(dirv == 0.0, center, center + T * dirv)     # k_tr_bounds
        tr = np.minimum(np.maximum(moved, lo), up)
    lower = lagrangian + (tr[:n] - px) @ gp
    upper = lagrangian + (tr[n:] - py) @ gd
    return lower, upper
