"""Every kernel past one launch wave, one cut segment and one staging slot.

The grids of the solver follow the device's SM count, and several code paths start only once a problem outgrows one of
them (sizes for 132 SMs; the census below proves each case crosses them up to 144 SMs):

  SpMV wave         a warp takes blocks b, b + nwarps, ... and loads the indices of the next one ahead; long-row blocks are
                    dealt after the interleaved ones.  More than 8 x 4 x 132 = 4224 blocks (3168 for the fused K2 with two
                    payload row groups), or more long rows than warps
  grid-stride       element-wise kernels run ew_grid() = min(ceil(len / 256), 8 x SMs) CTAs: len > 270 336 strides
  partial folds     a grid of more than 256 CTAs publishes more partials than one CTA has threads
  scaling rounds    k_row_scaling_stat / k_scale_matrix run 16 x SMs CTAs of 256 / W row groups: every lane runs
                    ceil(rows / stride) rounds
  cut segments      the BICSR cut runs in 65 536-row segments on worker threads; no block crosses a segment boundary
  staging ring      host arrays of >= 8 MB go through 4 pinned slots of 32 MB: > 32 MB spans slots, a 5th fill waits
                    on the event of the copy that last read its slot

Cases (seeded, vectorised numpy, each with a planted optimum):
  tall           lpgen.sparse_lp(600 000, 400 000, 8): multi-wave A and A^T, 10 segments, values over two slots
  short_rows     1.1M x 1.1M, rows of 1 .. 3 entries: the fused K2 with two payload row groups over several waves,
                 element-wise kernels over 4+ rounds, seven arrays through the ring (it wraps)
  segment_edges  3 x 65 536 + 77 rows of 6 entries with >= 6000 long rows (more than the warps of a wave), and designed
                 rows at every segment boundary: long rows at 65 535 / 65 536, a run of 1-entry rows across 131 072,
                 empty rows across 196 608; A^T has ~70 entries per row (32 lanes per row group, 3 rounds)

The cases are wide() of cases.py; the cut, grids and staging model are those of device_model.py.  References and
tolerances are those of exact.py (componentwise row sums against the correctly rounded exact sum); setup values that
are one or two roundings of exact inputs are compared bit for bit.
"""
import functools
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import device_model as dm
from cases import (B1, B2, B3, EMPTY, RECYCLE, RUN, WIDE as CASES, cache_probe, host_threads, oracle_of, problem_of,
                   recycle_solve, settings_of, solve_arrays, wide, zoo)
from cuopt_b200 import capi
from device_model import gather_block_bytes  # noqa: F401
from device_model import (MAX_ROWS, RING, SEGMENT, SLOT, WARPS, cut, ew_grid, row_group_width, scaling_rounds,
                          staged_arrays, staged_fills)
from exact import (STEPWISE, TRAJECTORY, U53, assert_row_sums, check_evaluation, device_formulation, dot_tolerance,
                   dual_step_reference, reduced_cost_reference, rel_err, row_sum_tolerance, row_sums_hp, scaled_problem,
                   scaled_transpose, transpose)
from oracle import pdlp_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = (132, 144)                   # the H100 SXM and margin above it
UNSEGMENTED = 1 << 40


# ------------------------------------------------------------------------------------ the launch geometry of the cases
@functools.lru_cache(maxsize=None)
def structure_of(name):
    case, _ = wide(name)
    return dm.cut_counts(case.offsets, transpose(case.offsets, case.indices, case.n)[0])


def geometry(name, sms, occ=dm.OCC, occ2=dm.OCC2):
    """What the solver launches for the case on `sms` SMs (unblocked)."""
    return dm.geometry(structure_of(name), wide(name)[1], sms, occ, occ2)


def crossings(name, g, sms):
    """The thresholds the case is named for, on a device with `sms` SMs and launch geometry g -> {claim: holds}."""
    case, lp = wide(name)
    nnz = len(case.values)
    waves_a = g["n_std_a"] / (WARPS * g["grid_k2"])
    waves_at = g["n_std_at"] / (WARPS * g["grid_k3"])
    ew = lambda count: -(-count // (ew_grid(count, sms) * dm.EW_THREADS))  # noqa: E731  grid-stride rounds
    out = {"partials > 256": ew_grid(max(case.m, case.n), sms) > 256, "segments": case.m > SEGMENT}
    big = [b for b in staged_arrays(lp) if b >= SLOT // 4]
    if name == "tall":
        out.update({"A: 2 waves": waves_a >= 2, "A^T: 2 waves": waves_at >= 2, "EW m: 2 rounds": ew(case.m) >= 2,
                    "EW n: 2 rounds": ew(case.n) >= 2, "EW n + m: 3 rounds": ew(case.m + case.n) >= 3,
                    "scaling A: W 8, 2 rounds": row_group_width(case.m, nnz) == 8 and scaling_rounds(case.m, nnz, sms) >= 2,
                    "scaling A^T: W 16, 2 rounds":
                        row_group_width(case.n, nnz) == 16 and scaling_rounds(case.n, nnz, sms) >= 2,
                    "an array spans two slots": max(big) > SLOT, "10 segments": -(-case.m // SEGMENT) == 10})
    elif name == "short_rows":
        out.update({"K2 NPRE 2": g["k2_npre"] == 2, "A: 2 waves": waves_a >= 2, "EW: 4 rounds": ew(case.m) >= 4,
                    "scaling A: W 4, 2 rounds": row_group_width(case.m, nnz) == 4 and scaling_rounds(case.m, nnz, sms) >= 2,
                    "ring wraps": len(big) > RING, "empty columns": np.bincount(case.indices, minlength=case.n).min() == 0})
    else:
        out.update({"long rows > warps of a wave": g["n_long_a"] > WARPS * g["grid_k2"],
                    "scaling A^T: W 32, 2 rounds":
                        row_group_width(case.n, nnz) == 32 and scaling_rounds(case.n, nnz, sms) >= 2})
    return out


# ------------------------------------------------------------------------------------------------------- CPU tests
def test_segmented_cut_equals_the_plain_cut_below_one_segment():
    for c in zoo().values():
        assert cut(c.offsets) == cut(c.offsets, segment=UNSEGMENTED), c.name
    # and it is the unsegmented cut per segment
    off = wide("segment_edges")[0].offsets
    got = cut(off)
    want = ([], [])
    for s0 in range(0, len(off) - 1, SEGMENT):
        part = np.asarray(off[s0:min(len(off), s0 + SEGMENT + 1)], np.int64)
        std, lng = cut(part - part[0], segment=UNSEGMENTED)
        want[0].extend((a + s0, b + s0) for a, b in std)
        want[1].extend(r + s0 for r in lng)
    assert got == want


@pytest.mark.parametrize("name", CASES)
def test_census_every_case_crosses_what_it_is_named_for(name):
    case, lp = wide(name)
    assert case.offsets[-1] == len(case.indices) and len(case.offsets) == case.m + 1
    assert np.all(case.indices >= 0) and np.all(case.indices < case.n)
    assert lp.optimal_objective is not None and np.isfinite(lp.optimal_objective)
    for sms in range(SMS[0], SMS[1] + 1, 4):
        bad = [k for k, ok in crossings(name, geometry(name, sms), sms).items() if not ok]
        assert not bad, (name, sms, bad)
    if name == "tall":
        assert staged_fills(lp) >= 3
    if name == "short_rows":
        assert staged_fills(lp) == 7
    if name == "segment_edges":
        off = np.asarray(case.offsets, np.int64)
        lens = np.diff(off)
        std, lng = cut(off)
        plain_std, _ = cut(off, segment=UNSEGMENTED)
        starts = {a for a, _ in std} | set(lng)
        assert {B1 - 1, B1} <= set(lng)                       # long rows on both sides of the first boundary
        assert (B1 - 1, B1) not in std and B1 in starts       # ... so a block ends exactly on it
        assert np.all(lens[RUN[0]:RUN[1]] == 1) and np.all(lens[EMPTY[0]:EMPTY[1]] == 0)
        assert EMPTY[1] < case.m and np.all(lens[EMPTY[1]:] > 0)
        for b in (B2, B3):
            assert b in starts                                # the segment rule cuts here ...
            assert any(a < b < e for a, e in plain_std), b     # ... where an unsegmented cut would not
        assert len(lng) >= 6000
        assert any(e - a == MAX_ROWS for a, e in std if RUN[0] <= a < RUN[1])  # 256-row blocks of the run


@pytest.mark.parametrize("name", CASES)
def test_oracle_products_match_high_precision_reference(name):
    """The oracle serves as witness below: its A xbar (through y'), A^T y' and evaluation against exact row sums."""
    case, lp = wide(name)
    o = oracle_of(lp, num_threads=host_threads())
    o.initialise()
    rng = np.random.default_rng(3)
    x, y = rng.uniform(0.0, 2.0, case.n), rng.standard_normal(case.m)
    scaled = o.vector("scaled_values")
    T = scaled_transpose(case, scaled, o.vector("scaled_values_t"))
    aty = row_sums_hp(*T, y)[0]
    got = o.single_attempt(x, y, aty, 0.37, 0.61)
    assert_row_sums(got["aty_next"], row_sums_hp(*T, got["y_next"]), "A^T y'")
    want, tol = dual_step_reference(case, scaled, got["x_bar"], y, 0.61, o.vector("scaled_lc"), o.vector("scaled_uc"))
    assert np.all(np.abs(got["y_next"] - want) <= tol)
    cv = o.convergence(x, y)
    rc, g, tol = reduced_cost_reference(lp, y)
    assert np.all(np.abs(cv["reduced_cost"] - rc) <= tol)
    ax = row_sums_hp(case.offsets, case.indices, case.values, x)[0]
    viol = np.maximum(lp.con_lb - ax, 0.0) + np.maximum(ax - lp.con_ub, 0.0)
    assert cv["l2_primal_residual"] == pytest.approx(np.linalg.norm(viol), rel=1e-12)
    assert cv["primal_objective"] == pytest.approx(math.fsum(lp.c * x), rel=1e-12)


# ------------------------------------------------------------------------------------------ scaling reference (numpy)
def scaling_reference(case, mode):
    """compute_scaling_vectors transcribed: Ruiz passes (a max, a sqrt, a division: exact) then one Pock-Chambolle pass,
    whose sums come from fsum.  -> (Dr, Dc, componentwise relative tolerance of Dr, of Dc)."""
    hp = po.preset(mode)
    m, n = case.m, case.n
    off = np.asarray(case.offsets, np.int64)
    row = np.repeat(np.arange(m), np.diff(off))
    col = np.asarray(case.indices, np.int64)
    toff, tidx, pos = transpose(case.offsets, case.indices, case.n)
    a = np.asarray(case.values)
    lens, tlens = np.diff(off), np.diff(toff)

    def row_max(v, o, ln):
        out = np.zeros(len(ln))
        ne = ln > 0
        out[ne] = np.maximum.reduceat(v, o[:-1][ne]) if v.size else 0.0
        return out

    dr, dc = np.ones(m), np.ones(n)
    if hp.do_ruiz_scaling:
        for _ in range(hp.l_inf_ruiz_iterations):
            s = np.abs((a * dr[row]) * dc[col])
            sr, sc = row_max(s, off, lens), row_max(s[pos], toff, tlens)
            dr = np.where(sr > 0.0, dr / np.sqrt(np.where(sr > 0.0, sr, 1.0)), dr)
            dc = np.where(sc > 0.0, dc / np.sqrt(np.where(sc > 0.0, sc, 1.0)), dc)
    if hp.do_pock_chambolle_scaling:
        alpha = hp.alpha_pock_chambolle
        s = np.abs((a * dr[row]) * dc[col])
        sr = row_sums_hp(off, col, np.power(s, alpha), np.ones(n))[0]
        sc = row_sums_hp(toff, np.zeros(len(pos), np.int64), np.power(s[pos], 2.0 - alpha), np.ones(1))[0]
        dr = np.where(sr > 0.0, dr / np.sqrt(np.where(sr > 0.0, sr, 1.0)), dr)
        dc = np.where(sc > 0.0, dc / np.sqrt(np.where(sc > 0.0, sc, 1.0)), dc)
        # pow in libm ulps (2 per term), the sum in any order (len - 1), halved by the sqrt, plus the sqrt and division
        return dr, dc, (lens + 8) * U53, (tlens + 8) * U53
    return dr, dc, np.zeros(m), np.zeros(n)


# ------------------------------------------------------------------------------------------------------- GPU tests
def session(name, blocks, force, mode=1, tol=1e-9, **kw):
    """(case, LP, initialised GPU session) with the column blocking asked for."""
    case, lp = wide(name)
    g = dm.session(case, problem_of(lp), settings_of(mode, tol, **kw), blocks, force)
    if blocks is not None:
        assert g.scalar("eval_blocks") >= 3 and g.scalar("eval_blocks_t") >= 3
    return case, lp, g


GEOMETRY = ["n_std_a", "n_blk_a", "n_std_at", "n_blk_at", "k2_npre", "grid_k1", "grid_k2", "grid_k3", "grid_n", "grid_m",
            "staged_fills"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_census(name, gather_block_bytes):
    """The session's launch geometry equals the model, and every case crosses its thresholds on this card (no skip)."""
    _, _, g = session(name, None, gather_block_bytes)
    sms, occ, occ2 = (int(g.scalar(k)) for k in ("sm_count", "occ_spmv", "occ_spmv2"))
    want = geometry(name, sms, occ, occ2)
    got = {k: int(g.scalar(k)) for k in GEOMETRY}
    assert got == {k: want[k] for k in GEOMETRY}, (sms, occ, occ2)
    bad = [k for k, ok in crossings(name, dict(want), sms).items() if not ok]
    assert not bad, (sms, occ, occ2, bad)
    assert got["grid_m"] > 256 or got["grid_n"] > 256
    if name == "short_rows":
        assert got["k2_npre"] == 2 and got["staged_fills"] > RING


SETUP = [(n, 1) for n in CASES] + [("tall", m) for m in (0, 2, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode", SETUP)
def test_setup_bit_for_bit(name, mode, gather_block_bytes):
    """Scaling vectors, scaled matrix and vectors, norms, step size and primal weight: also the integrity check of every
    array that came through the staging ring and of every block of the segmented cut."""
    case, lp, g = session(name, None, gather_block_bytes, mode=mode)
    dr, dc = g.vector("row_scaling"), g.vector("col_scaling")
    rdr, rdc, tr, tc = scaling_reference(case, mode)
    for got, want, tol, what in ((dr, rdr, tr, "Dr"), (dc, rdc, tc, "Dc")):
        bad = np.flatnonzero(~(np.abs(got - want) <= tol * np.abs(want)))
        assert bad.size == 0, (what, bad[:8].tolist(), got[bad[:8]].tolist(), want[bad[:8]].tolist())
    row = np.repeat(np.arange(case.m), np.diff(case.offsets))
    col = np.asarray(case.indices, np.int64)
    assert np.array_equal(g.vector("scaled_values"), (case.values * dr[row]) * dc[col])
    toff, tidx, pos = transpose(case.offsets, case.indices, case.n)
    assert np.array_equal(g.vector("scaled_values_t"), (case.values[pos] * dc[col[pos]]) * dr[tidx])
    with np.errstate(divide="ignore", invalid="ignore"):
        assert np.array_equal(g.vector("scaled_l"), np.where(dc == 0, 0.0, lp.var_lb / dc))
        assert np.array_equal(g.vector("scaled_u"), np.where(dc == 0, 0.0, lp.var_ub / dc))
    assert np.array_equal(g.vector("scaled_c"), lp.c * dc)
    assert np.array_equal(g.vector("scaled_lc"), lp.con_lb * dr)
    assert np.array_equal(g.vector("scaled_uc"), lp.con_ub * dr)
    hp = po.preset(mode)
    fin = lambda b: np.where(np.isfinite(b), np.abs(b), 0.0)  # noqa: E731
    comb = lambda lo, hi: np.maximum(fin(lo), fin(hi))  # noqa: E731
    sumtol = lambda k: 2 * k * U53  # noqa: E731
    assert g.scalar("l2_norm_c") == pytest.approx(math.sqrt(math.fsum((lp.c ** 2).tolist())), rel=sumtol(lp.n))
    assert g.scalar("l2_norm_b") == pytest.approx(math.sqrt(math.fsum((comb(lp.con_lb, lp.con_ub) ** 2).tolist())),
                                                  rel=sumtol(lp.m))
    assert g.scalar("step_size") == hp.initial_step_size_scaling / np.max(np.abs(g.vector("scaled_values")))
    if hp.compute_initial_primal_weight_before_scaling:
        cc, b = lp.c, comb(lp.con_lb, lp.con_ub)
    else:
        cc, b = g.vector("scaled_c"), comb(g.vector("scaled_lc"), g.vector("scaled_uc"))
    cn = math.sqrt(math.fsum((cc * cc * hp.initial_primal_weight_c_scaling).tolist()))
    bn = math.sqrt(math.fsum((b * b * hp.initial_primal_weight_b_scaling).tolist()))
    assert g.scalar("primal_weight") == pytest.approx(hp.primal_importance * cn / bn, rel=sumtol(lp.m + lp.n))


STEP = [(n, None) for n in CASES] + [("tall", 3), ("tall", 16)]


def dot_tolerance(terms):
    return 2 * len(terms) * U53 * math.fsum(np.abs(terms).tolist()) + 1e-300


@pytest.mark.gpu
@pytest.mark.parametrize("name,blocks", STEP)
def test_one_pdhg_step_exactly(name, blocks, gather_block_bytes):
    """K1's x', K2's y', K3's A^T y' and the three dot products of every step accepted at its first attempt."""
    case, lp, g = session(name, blocks, gather_block_bytes)
    scaled = g.vector("scaled_values")
    T = scaled_transpose(case, scaled, g.vector("scaled_values_t"))
    c, l, u, lc, uc = (g.vector(v) for v in ("scaled_c", "scaled_l", "scaled_u", "scaled_lc", "scaled_uc"))
    checked, fresh = 0, True
    for _ in range(30):
        if checked == 3:
            break
        x, y, aty, tau, sigma = g.vector("x"), g.vector("y"), g.vector("aty"), g.scalar("tau"), g.scalar("sigma")
        attempts, restarts = g.scalar("k_pdhg"), g.scalar("n_restarts")
        g.advance(1)
        restarted = g.scalar("n_restarts") != restarts
        usable = fresh and not restarted and g.scalar("k_pdhg") == attempts + 1
        fresh = not restarted  # after a restart A^T y is rebuilt by the next step: its 'before' is not this aty
        if not usable:
            continue
        xn, yn, atyn = g.vector("x"), g.vector("y"), g.vector("aty")
        want = np.maximum(np.minimum(x - tau * (c - aty), u), l)
        tol = 4 * U53 * (np.abs(x) + tau * (np.abs(c) + np.abs(aty))) + 1e-300
        bad = np.flatnonzero(~(np.abs(xn - want) <= tol))
        assert bad.size == 0, ("K1 columns", bad[:8].tolist(), xn[bad[:8]].tolist(), want[bad[:8]].tolist())
        want, tol = dual_step_reference(case, scaled, g.vector("x_bar"), y, sigma, lc, uc)
        bad = np.flatnonzero(~(np.abs(yn - want) <= tol))
        assert bad.size == 0, ("K2 rows", bad[:8].tolist(), yn[bad[:8]].tolist(), want[bad[:8]].tolist())
        assert_row_sums(atyn, row_sums_hp(*T, yn), "K3 A^T y'")
        dx, dy = xn - x, yn - y
        for what, terms in (("interaction", dx * (atyn - aty)), ("norm_dx2", dx * dx), ("norm_dy2", dy * dy)):
            assert abs(g.scalar(what) - math.fsum(terms.tolist())) <= dot_tolerance(terms), what
        checked += 1
    assert checked >= 3


PARITY = [(n, None) for n in CASES] + [("tall", 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,blocks", PARITY)
def test_steps_match_oracle(name, blocks, gather_block_bytes):
    case, lp, g = session(name, blocks, gather_block_bytes)
    o = oracle_of(lp, tol=1e-9, num_threads=host_threads())
    o.initialise()
    for steps, tol in ((1, STEPWISE), (1, STEPWISE), (3, STEPWISE), (40, TRAJECTORY)):
        g.advance(steps); o.run(steps)
        for v in ("x", "y", "aty", "sum_x", "sum_y"):
            assert rel_err(g.vector(v), o.vector(v)) <= tol, (v, steps)
        for v in ("step_size", "primal_weight", "sum_w"):
            assert g.scalar(v) == pytest.approx(o.scalar(v), rel=tol), (v, steps)
        assert g.scalar("k_pdhg") == o.scalar("k_pdhg")
    assert g.scalar("n_restarts") >= 1 and g.scalar("n_restarts") == o.scalar("n_restarts")


@pytest.mark.gpu
@pytest.mark.parametrize("checks", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_evaluation_of_the_returned_iterate(name, checks):
    """The termination pass on the returned iterate; with per-constraint residuals and infeasibility detection on, the
    per-CTA maxima and the ray statistics fold more than 256 partials too."""
    _, lp = wide(name)
    kw = dict(per_constraint_residual=True, infeasibility_detection=True) if checks else {}
    sol = capi.solve(problem_of(lp), settings_of(tol=1e-12, iteration_limit=40, **kw))
    assert sol.termination_reason == "IterationLimit"
    check_evaluation(lp, sol, oracle_of(lp, **(dict(per_constraint_residual=True, detect_infeasibility=True) if checks else {})))


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", [None, 3])
def test_restart_to_average_rebuilds_aty(blocks, gather_block_bytes):
    """x' = clamp(x - tau (c - A^T y)) for the first step after a restart to the average, A^T y of the new y from exact
    row sums: on tall, A^T is several waves."""
    case, lp, g = session("tall", blocks, gather_block_bytes)
    T = scaled_transpose(case, g.vector("scaled_values"), g.vector("scaled_values_t"))
    c, l, u = g.vector("scaled_c"), g.vector("scaled_l"), g.vector("scaled_u")
    checked = 0
    for _ in range(400):
        restarts = g.scalar("n_restarts")
        g.advance(1)
        if g.scalar("n_restarts") == restarts or g.scalar("last_restart_was_average") != 1.0:
            continue
        aty, mag, lens = row_sums_hp(*T, g.vector("y"))
        x, tau, attempts, restarts = g.vector("x"), g.scalar("tau"), g.scalar("k_pdhg"), g.scalar("n_restarts")
        g.advance(1)
        if g.scalar("k_pdhg") != attempts + 1 or g.scalar("n_restarts") != restarts:
            continue
        want = np.maximum(np.minimum(x - tau * (c - aty), u), l)
        tol = tau * row_sum_tolerance(mag, lens) + 8 * U53 * (np.abs(x) + tau * (np.abs(c) + np.abs(aty)))
        assert np.all(np.abs(g.vector("x") - want) <= tol)
        checked += 1
        if checked == 2:
            break
    assert checked > 0


@pytest.mark.gpu
def test_trust_region_kernels_at_a_million_components():
    """Methodical1's trust-region kernels over N = n + m = 1M (several grid-stride rounds, > 256 partials)."""
    _, lp = wide("tall")
    g = capi.Solver(problem_of(lp), settings_of(po.METHODICAL1))
    g.initialise()
    g.advance(5)
    prob = scaled_problem(lp, g)
    tau, sigma = g.scalar("tau"), g.scalar("sigma")
    x, y = g.vector("x"), g.vector("y")
    for px, py in ((x, y), (lp.x_star / g.vector("col_scaling"), lp.y_star / g.vector("row_scaling"))):
        for radius in (0.0, 1e-9, 1e-3, 0.5, 10.0, 1e6):
            want = device_formulation(*prob, tau, sigma, px, py, radius)
            got = g.trust_region_bounds(px, py, radius)
            scale = max(1.0, abs(want[0]), abs(want[1]))
            assert abs(got[0] - want[0]) <= 1e-9 * scale and abs(got[1] - want[1]) <= 1e-9 * scale, (radius, got, want)


@pytest.mark.gpu
def test_two_solves_are_bit_identical_with_and_without_graphs(monkeypatch):
    """Repeated solves and the two launch paths give the same bits.  The cut's worker threads (as many as the host has
    cores, up to 32) finish their segments in a different order from run to run; the result must not depend on it.  That
    the joined cut is the sequential one is checked by the census (block counts) and by the exact row sums above."""
    _, lp = wide("segment_edges")
    runs = []
    for graphs in (True, False):
        if graphs:
            monkeypatch.delenv("CUOPT_B200_NO_GRAPH", raising=False)
        else:
            monkeypatch.setenv("CUOPT_B200_NO_GRAPH", "1")
        for _ in range(2):
            runs.append(solve_arrays(capi.solve(problem_of(lp), settings_of(tol=1e-12, iteration_limit=300))))
    x, y, rc, st = runs[0]
    assert st["number_of_steps_taken"] >= 300
    for other in runs[1:]:
        assert np.array_equal(x, other[0]) and np.array_equal(y, other[1]) and np.array_equal(rc, other[2])
        assert st == other[3]


@pytest.mark.gpu
def test_full_solve_reaches_planted_optimum():
    _, lp = wide("tall")
    s = settings_of(tol=1e-7, iteration_limit=200000, time_limit=600.0)
    sol = capi.solve(problem_of(lp), s)
    assert sol.return_code == 0 and sol.termination_reason == "Optimal", sol.termination_reason
    st = sol.stats()
    scale = max(1.0, abs(lp.optimal_objective))
    assert abs(st.primal_objective - lp.optimal_objective) <= 1e-5 * scale
    assert abs(st.dual_objective - lp.optimal_objective) <= 1e-5 * scale


# --------------------------------------------------------------------------------------------- recycled device memory
FRESH = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
from cases import cache_probe, recycle_solve, solve_arrays
x, y, rc, st = solve_arrays(recycle_solve({config!r}, {seed}))
assert cache_probe().scalar("device_cache_hits") == 0
np.savez({out!r}, x=x, y=y, rc=rc, **{{k: np.array(v) for k, v in st.items()}})
"""


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(RECYCLE))
def test_solve_on_recycled_memory_equals_fresh_memory(config, tmp_path):
    """From the second solve of a shape on, every device buffer comes from the block cache still holding the previous
    solve's data: LP B solved after LP A equals LP B solved alone with the cache off."""
    probe = cache_probe()
    recycle_solve(config, 41)
    hits = probe.scalar("device_cache_hits")
    x, y, rc, st = solve_arrays(recycle_solve(config, 42))
    assert probe.scalar("device_cache_hits") - hits >= 50  # solve B took its buffers from the cache
    out = str(tmp_path / "fresh.npz")
    env = dict(os.environ, CUOPT_B200_DEVICE_CACHE_MB="0")
    code = FRESH.format(root=ROOT, tests=os.path.join(ROOT, "tests"), config=config, seed=42, out=out)
    subprocess.run([sys.executable, "-c", code], env=env, check=True, timeout=900)
    f = np.load(out)
    assert np.array_equal(x, f["x"]) and np.array_equal(y, f["y"]) and np.array_equal(rc, f["rc"])
    assert st == {k: f[k].item() for k in st}
    assert st["number_of_steps_taken"] >= 64
