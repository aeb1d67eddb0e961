"""The device version of the trust-region solve (cuopt_b200/csrc/trust_region.cuh) does not re-reduce the active range
at every trial threshold like the reference / the oracle: it sorts once, takes prefix sums of the two radius terms and
evaluates every partial radius as a difference of prefix sums inside a single-thread bisection.  This file transcribes
exactly that formulation in numpy (same formulas, same search functions, same update rules) and checks it against the
oracle's direct restatement on real iterates — a CPU check of the reformulation, independent of CUDA."""
import numpy as np
import pytest
import scipy.sparse as sp

from conftest import mps_path, problem_arrays
from cuopt_b200 import capi, lpgen
from oracle import pdlp_oracle as po


def device_formulation(As, cs, ls, us, lcs, ucs, tau, sigma, px, py, radius):
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


def scaled_problem(o, a):
    dr, dc = o.vector("row_scaling"), o.vector("col_scaling")
    A = sp.csr_matrix((a["values"], a["indices"], a["offsets"]), shape=(len(a["con_lb"]), len(a["c"])))
    As = (sp.diags(dr) @ A @ sp.diags(dc)).tocsr()
    return As, o.vector("scaled_c"), o.vector("scaled_l"), o.vector("scaled_u"), o.vector("scaled_lc"), o.vector("scaled_uc")


CASES = ["afiro", "sparse", "multicommodity"]


@pytest.mark.parametrize("case", CASES)
def test_prefix_sum_bisection_equals_the_direct_restatement(case):
    if case == "afiro":
        a = problem_arrays(capi.Problem.read(mps_path("linear_programming/afiro_original.mps")))
    else:
        lp = lpgen.sparse_lp(400, 300, 5, seed=3) if case == "sparse" else lpgen.multicommodity(30, 90, 3, seed=2)
        a = dict(offsets=lp.offsets, indices=lp.indices, values=lp.values, c=lp.c, var_lb=lp.var_lb, var_ub=lp.var_ub,
                 con_lb=lp.con_lb, con_ub=lp.con_ub)
    o = po.Oracle(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"],
                  mode=po.METHODICAL1, tol=1e-10)
    o.initialise()
    prob = scaled_problem(o, a)
    for steps in (7, 20, 33):      # between restarts: the last-restart point is the origin / an earlier iterate
        o.run(steps)
        px, py = o.vector("x"), o.vector("y")
        tau, sigma = o.scalar("tau"), o.scalar("sigma")
        for radius in (-1.0, 1e-3, 0.5, 1e3):
            lo_want, up_want, used = o.trust_region_bounds(px, py, radius)
            lo_got, up_got = device_formulation(*prob, tau, sigma, px, py, used)
            scale = max(1.0, abs(lo_want), abs(up_want))
            assert abs(lo_got - lo_want) <= 1e-9 * scale, (case, steps, radius)
            assert abs(up_got - up_want) <= 1e-9 * scale, (case, steps, radius)
