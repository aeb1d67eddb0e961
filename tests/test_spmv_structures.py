"""Every sparse product of the solver on adversarial row structures.

All SpMVs go through the block-interleaved core (cuopt_b200/csrc/spmv_bicsr.cuh), and several of its branches are
reached only by particular matrix STRUCTURES: rows longer than a block (one warp strides the plain CSR), matrices
without a single interleaved block, empty rows and whole blocks of them, blocks closed by the 256-row limit, rows that
span 2 .. 32 lanes of a block, column blocks without entries, long rows that a column split turns into a short and a
long part.  The generators of the other test files (k entries in every row, 2-3 per column) and the MPS fixtures
reach none of them, so cases.py builds a zoo of such structures (numpy, seeded); this file proves on the CPU, with the
cut and column blocks of device_model.py, that each case has the property it is named for, and runs the setup kernels,
K2, K3, the evaluation and full solves on them, unblocked and with gather blocking forced on.

References and tolerances are those of exact.py: a row sum is compared COMPONENTWISE with the correctly rounded exact
sum.  The CPU oracle is checked against the same reference on every structure (CPU tests below) before the GPU tests use
it as a witness.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

from cases import BLOCKING, ZOO, as_transpose, oracle_of, planted, problem_of, settings_of, zoo
from cuopt_b200 import capi
from device_model import CH, MAX_ROWS, SLOTS, block_bytes, column_blocks, cut, k2_npre, split_columns
from device_model import gather_block_bytes  # noqa: F401
from device_model import session as dm_session
from exact import (ACROSS_TRUST_REGION, ELEMENTWISE, OBJECTIVE, STEPWISE, TRAJECTORY, U53, assert_row_sums,
                   check_evaluation, dual_step_reference, reduced_cost_reference, rel_err, row_sum_tolerance, row_sums_hp,
                   scaled_transpose)


def structure(offsets):
    """The properties of a matrix that decide which branches of the SpMV core run."""
    off = np.asarray(offsets, np.int64)
    std, long_rows = cut(off)
    rows = len(off) - 1
    lanes_spanned = set()
    for r0, r1 in std:
        for r in range(r0, r1):
            if off[r + 1] > off[r]:
                lanes_spanned.add(int((off[r + 1] - 1 - off[r0]) // CH - (off[r] - off[r0]) // CH + 1))
    return dict(n_std=len(std), n_long=len(long_rows), long_rows=long_rows,
                block_with_256_rows=any(r1 - r0 == MAX_ROWS for r0, r1 in std),
                block_without_entries=any(off[r1] == off[r0] for r0, r1 in std),
                block_with_256_entries=any(off[r1] - off[r0] == SLOTS for r0, r1 in std),
                rows_past_two_groups=any(r1 - r0 > 64 for r0, r1 in std),
                two_payload_groups=k2_npre(rows, len(std)) == 2,
                lanes_spanned=lanes_spanned, empty_rows=int(np.sum(np.diff(off) == 0)))


# ------------------------------------------------------------------------------------------------------- CPU tests
def test_zoo_names_are_the_parametrisation():
    assert list(zoo()) == ZOO
    for c in zoo().values():
        assert c.offsets[0] == 0 and c.offsets[-1] == len(c.indices) == len(c.values) and len(c.offsets) == c.m + 1
        for r in range(c.m):
            cols = c.indices[c.offsets[r]:c.offsets[r + 1]]
            assert np.all(np.diff(cols) > 0) and (cols.size == 0 or (cols[0] >= 0 and cols[-1] < c.n)), (c.name, r)


def test_every_case_has_the_structure_it_is_named_for():
    z = zoo()
    S = {k: structure(c.offsets) for k, c in z.items()}
    ST = {k: structure(as_transpose(c).offsets) for k, c in z.items()}

    s = S["long_rows"]
    lens = np.diff(z["long_rows"].offsets)
    assert {255, 256, 257, 512, 513, 1000, z["long_rows"].n} <= set(lens.tolist())
    assert 0 in s["long_rows"] and z["long_rows"].m - 1 in s["long_rows"]
    assert any(b - a == 1 for a, b in zip(s["long_rows"], s["long_rows"][1:]))
    assert s["n_long"] >= 8 and s["n_std"] > 8
    assert ST["long_rows"]["n_long"] == 0  # the long rows are on one side only
    assert ST["dense_columns"]["n_long"] >= 8 and S["dense_columns"]["n_long"] == 0

    assert S["only_long"]["n_std"] == 0 and S["only_long"]["n_long"] == 40 and ST["only_long"]["n_long"] == 0

    for s in (S["empty_rows_and_columns"], ST["empty_rows_and_columns"]):
        assert s["block_without_entries"] and s["block_with_256_rows"] and s["empty_rows"] >= 300
    c = z["empty_rows_and_columns"]
    for cc in (c, as_transpose(c)):
        lens = np.diff(cc.offsets)
        assert lens[0] == 0 and lens[-1] == 0 and lens[50] == 0 and lens[49] > 0 and lens[51] > 0

    s = S["singleton_runs"]
    assert s["block_with_256_rows"] and s["rows_past_two_groups"] and s["two_payload_groups"]
    assert np.all(np.diff(z["singleton_runs"].offsets)[:1000] == 1)

    s = S["lane_spans"]
    # carry runs of many lengths, up to all 31 later lanes of a block
    assert {1, 2, 3, 4, 31, 32} <= s["lanes_spanned"] and len(s["lanes_spanned"]) >= 16, s["lanes_spanned"]
    assert s["block_with_256_entries"]
    off = z["lane_spans"].offsets
    std, _ = cut(off)
    shapes = [tuple(np.diff(off[r0:r1 + 1]).tolist()) for r0, r1 in std]
    for want in [(256,), (1, 255), (255, 1), (248, 8), (248,)]:
        assert want in shapes, (want, shapes[:12])
    assert shapes[shapes.index((248,)) + 1][0] == 9  # [248, 9] does not fit: the cut falls between them

    assert S["tiny_1x700"]["n_std"] == 0 and ST["tiny_1x700"]["block_with_256_rows"]
    assert ST["tiny_700x1"]["n_std"] == 0 and S["tiny_700x1"]["block_with_256_rows"]
    assert 1 < S["tiny_few_blocks"]["n_std"] < 8 and S["tiny_1x1"]["n_std"] == 1
    for k in ("heavy_tail_1", "heavy_tail_2"):
        assert S[k]["n_long"] > 0 and S[k]["empty_rows"] > 0 and len(S[k]["lanes_spanned"]) > 8

    # under the forced column blocks: blocking is on for both matrices, ...
    for k in ZOO:
        if k.startswith("tiny") or k == "only_long":
            continue
        for blocks in (3, 16):
            nbytes = block_bytes(z[k], blocks)
            assert column_blocks(z[k].n, 1, nbytes)[0] >= 3 and column_blocks(z[k].m, 1, nbytes)[0] >= 3, (k, blocks)
    # ... a column block holds no entry at all, ...
    for cc in (c, as_transpose(c)):
        for blocks in (3, 16):
            width = column_blocks(cc.n, 1, block_bytes(cc, blocks))[1]
            assert any(o[-1] == 0 for o, _ in split_columns(cc, width)), (cc.name, blocks)
    # ... and a long row keeps a long part in one block and a short, non-empty part in another
    for cc in (z["long_rows"], as_transpose(z["dense_columns"])):
        for blocks in (3, 16):
            width = column_blocks(cc.n, 1, block_bytes(cc, blocks))[1]
            parts = np.array([np.diff(o) for o, _ in split_columns(cc, width)])  # blocks x rows
            mixed = (parts > SLOTS).any(axis=0) & ((parts > 0) & (parts <= SLOTS)).any(axis=0)
            assert mixed.any(), (cc.name, blocks)
            long_blocks = (parts > SLOTS).any(axis=1)
            assert long_blocks.any()  # these blocks keep their plain unscaled values; those of the other side drop them


def test_row_sums_hp_is_exact_on_small_rows():
    rng = np.random.default_rng(0)
    for c in (zoo()["tiny_1x1"], zoo()["tiny_few_blocks"], zoo()["tiny_1x700"]):
        v = rng.standard_normal(c.n) * 10.0 ** rng.integers(-8, 8, c.n)
        sums, mag, lens = row_sums_hp(c.offsets, c.indices, c.values, v)
        for r in range(c.m):
            lo, hi = c.offsets[r], c.offsets[r + 1]
            exact = sum((Fraction(float(a)) * Fraction(float(v[j])) for a, j in zip(c.values[lo:hi], c.indices[lo:hi])),
                        Fraction(0))
            assert sums[r] == float(exact)
            assert mag[r] == pytest.approx(sum(abs(a * v[j]) for a, j in zip(c.values[lo:hi], c.indices[lo:hi])), rel=1e-13)
    assert row_sums_hp([0, 0, 0], [], [], np.zeros(3))[0].tolist() == [0.0, 0.0]


@pytest.mark.parametrize("name", ZOO)
def test_oracle_products_match_high_precision_reference(name):
    """The oracle's A xbar (through y'), A^T y', and the A x / A^T y of its evaluation, on every structure."""
    case = zoo()[name]
    lp = planted(case)
    o = oracle_of(lp)
    o.initialise()
    rng = np.random.default_rng(3)
    x, y = rng.uniform(0.0, 2.0, case.n), rng.standard_normal(case.m)
    scaled = o.vector("scaled_values")
    T = scaled_transpose(case, scaled, o.vector("scaled_values_t"))
    aty = row_sums_hp(*T, y)[0]
    tau, sigma = 0.37, 0.61
    got = o.single_attempt(x, y, aty, tau, sigma)
    assert_row_sums(got["aty_next"], row_sums_hp(*T, got["y_next"]), "A^T y'")
    want, tol = dual_step_reference(case, scaled, got["x_bar"], y, sigma, o.vector("scaled_lc"), o.vector("scaled_uc"))
    assert np.all(np.abs(got["y_next"] - want) <= tol)
    # evaluation on the unscaled problem
    cv = o.convergence(x, y)
    rc, g, tol = reduced_cost_reference(lp, y)
    assert np.all(np.abs(cv["reduced_cost"] - rc) <= tol)
    ax = row_sums_hp(case.offsets, case.indices, case.values, x)[0]
    viol = np.maximum(lp.con_lb - ax, 0.0) + np.maximum(ax - lp.con_ub, 0.0)
    assert cv["l2_primal_residual"] == pytest.approx(np.linalg.norm(viol), rel=1e-12)
    assert cv["l2_dual_residual"] == pytest.approx(np.linalg.norm(g - rc), rel=1e-12, abs=1e-12)
    assert cv["primal_objective"] == pytest.approx(math.fsum(lp.c * x), rel=1e-12)


# ------------------------------------------------------------------------------------------------------- GPU tests
def session(case, blocks, force, mode=1, tol=1e-9, seed=1):
    """(planted LP, initialised GPU session) with the column blocking asked for."""
    lp = planted(case, seed)
    return lp, dm_session(case, problem_of(lp), settings_of(mode, tol), blocks, force)


SETUP = [(n, mode) for n in ZOO for mode in ((0, 1, 3) if n in ("long_rows", "empty_rows_and_columns") else (1,))]


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
@pytest.mark.parametrize("name,mode", SETUP)
def test_setup_kernels_match_oracle(name, mode, blocks, gather_block_bytes):
    """Transpose, scaling statistics and matrix scaling with dense and empty rows / columns."""
    case = zoo()[name]
    lp, g = session(case, blocks, gather_block_bytes, mode=mode)
    o = oracle_of(lp, mode=mode, tol=1e-9)
    o.initialise()
    for v in ("row_scaling", "col_scaling", "scaled_values", "scaled_values_t", "scaled_c", "scaled_lc", "scaled_uc"):
        gv, ov = g.vector(v), o.vector(v)
        fin = np.isfinite(ov)
        assert np.array_equal(np.isfinite(gv), fin), v
        assert rel_err(gv[fin], ov[fin]) <= ELEMENTWISE, v
    for v in ("step_size", "primal_weight"):
        assert g.scalar(v) == pytest.approx(o.scalar(v), rel=ELEMENTWISE), v
    scaled_transpose(case, g.vector("scaled_values"), g.vector("scaled_values_t"))  # every value at its transposed position


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
@pytest.mark.parametrize("name", ZOO)
def test_transpose_step_row_sums(name, blocks, gather_block_bytes):
    """K3 (and the column-block passes before it): A^T y' of every accepted step, row by row."""
    case = zoo()[name]
    _, g = session(case, blocks, gather_block_bytes)
    T = scaled_transpose(case, g.vector("scaled_values"), g.vector("scaled_values_t"))
    checked = 0
    for _ in range(30):  # the first ten steps are all evaluated and often end in a restart
        if checked == 4:
            break
        attempts, restarts = g.scalar("k_pdhg"), g.scalar("n_restarts")
        g.advance(1)
        if g.scalar("k_pdhg") == attempts or g.scalar("n_restarts") != restarts:
            continue  # after a restart A^T y is rebuilt by the next step
        assert_row_sums(g.vector("aty"), row_sums_hp(*T, g.vector("y")), "A^T y'")
        checked += 1
    assert checked >= 3


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
@pytest.mark.parametrize("name", ZOO)
def test_dual_step_row_sums(name, blocks, gather_block_bytes):
    """K2 (and the column-block passes before it): y' from y, sigma and xbar of every step accepted at its first attempt."""
    case = zoo()[name]
    _, g = session(case, blocks, gather_block_bytes)
    scaled, lc, uc = g.vector("scaled_values"), g.vector("scaled_lc"), g.vector("scaled_uc")
    checked = 0
    for _ in range(30):
        if checked == 4:
            break
        y, sigma, attempts, restarts = g.vector("y"), g.scalar("sigma"), g.scalar("k_pdhg"), g.scalar("n_restarts")
        g.advance(1)
        if g.scalar("k_pdhg") != attempts + 1 or g.scalar("n_restarts") != restarts:
            continue
        want, tol = dual_step_reference(case, scaled, g.vector("x_bar"), y, sigma, lc, uc)
        got = g.vector("y")
        bad = np.flatnonzero(~(np.abs(got - want) <= tol))
        assert bad.size == 0, ("rows", bad[:8].tolist(), got[bad[:8]].tolist(), want[bad[:8]].tolist())
        checked += 1
    assert checked >= 3


STEPPED = [(n, 1) for n in ZOO] + [("long_rows", 2)]  # mode 2: its trust-region restart runs the plain single-vector SpMV


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
@pytest.mark.parametrize("name,mode", STEPPED)
def test_steps_match_oracle(name, mode, blocks, gather_block_bytes):
    case = zoo()[name]
    lp, g = session(case, blocks, gather_block_bytes, mode=mode)
    o = oracle_of(lp, mode=mode, tol=1e-9)
    o.initialise()
    # the last batch crosses a major iteration of the preset and its restarts
    for steps, tol in ((1, STEPWISE), (1, STEPWISE), (3, STEPWISE), (40, TRAJECTORY) if mode == 1 else (64, ACROSS_TRUST_REGION)):
        g.advance(steps); o.run(steps)
        for v in ("x", "y", "aty", "sum_x", "sum_y"):
            assert rel_err(g.vector(v), o.vector(v)) <= tol, (v, steps)
        for v in ("step_size", "primal_weight", "sum_w"):
            assert g.scalar(v) == pytest.approx(o.scalar(v), rel=tol), (v, steps)
        assert g.scalar("k_pdhg") == o.scalar("k_pdhg")


@pytest.mark.gpu
@pytest.mark.parametrize("iterations", [1, 7, 40])
@pytest.mark.parametrize("blocks", BLOCKING)
@pytest.mark.parametrize("name", ZOO)
def test_evaluation_of_both_operands(name, blocks, iterations, gather_block_bytes):
    """The termination pass (two vectors through one stream of A, and of A^T) on the returned iterate."""
    case = zoo()[name]
    lp = planted(case)
    gather_block_bytes(block_bytes(case, blocks))
    sol = capi.solve(problem_of(lp), settings_of(tol=1e-12, iteration_limit=iterations))
    assert 1 <= sol.stats().number_of_steps_taken <= iterations
    check_evaluation(lp, sol, oracle_of(lp))


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
def test_evaluation_with_per_constraint_residual(blocks, gather_block_bytes):
    case = zoo()["long_rows"]
    lp = planted(case)
    gather_block_bytes(block_bytes(case, blocks))
    sol = capi.solve(problem_of(lp), settings_of(tol=1e-12, iteration_limit=40, per_constraint_residual=True))
    assert sol.termination_reason == "IterationLimit"
    check_evaluation(lp, sol, oracle_of(lp, per_constraint_residual=True))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dense_columns", "empty_rows_and_columns"])
def test_restart_to_average_rebuilds_aty_unblocked(name, gather_block_bytes):
    """After a restart to the average the next primal step uses A^T y of the new y, here from the single-vector SpMV on the
    whole A^T: x' = clamp(x - tau (c - A^T y), l, u) for every step taken right after such a restart."""
    case = zoo()[name]
    _, g = session(case, None, gather_block_bytes)
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
            continue  # the first attempt was rejected, or this step ended in another restart
        want = np.maximum(np.minimum(x - tau * (c - aty), u), l)
        tol = tau * row_sum_tolerance(mag, lens) + 8 * U53 * (np.abs(x) + tau * (np.abs(c) + np.abs(aty)))
        assert np.all(np.abs(g.vector("x") - want) <= tol)
        checked += 1
        if checked == 3:
            break
    assert checked > 0


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", [None, 3])
@pytest.mark.parametrize("name", ["long_rows", "dense_columns", "singleton_runs", "heavy_tail_1"])
def test_full_solve_reaches_planted_optimum(name, blocks, gather_block_bytes):
    case = zoo()[name]
    lp = planted(case)
    gather_block_bytes(block_bytes(case, blocks))
    runs = [capi.solve(problem_of(lp), settings_of(tol=1e-8, iteration_limit=400000)) for _ in range(2)]
    sol = runs[0]
    assert sol.return_code == 0 and sol.termination_reason == "Optimal"
    st = sol.stats()
    scale = max(1.0, abs(lp.optimal_objective))
    assert abs(st.primal_objective - lp.optimal_objective) <= OBJECTIVE * scale
    assert abs(st.dual_objective - lp.optimal_objective) <= OBJECTIVE * scale
    x = sol.primal()
    assert np.all(x >= lp.var_lb - 1e-6) and np.all(x <= lp.var_ub + 1e-6)
    assert np.array_equal(x, runs[1].primal()) and np.array_equal(sol.dual(), runs[1].dual())
