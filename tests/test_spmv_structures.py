"""Every sparse product of the solver on adversarial row structures.

All SpMVs go through the block-interleaved core (cuopt_b200/csrc/spmv_bicsr.cuh), and several of its branches are
reached only by particular matrix STRUCTURES: rows longer than a block (one warp strides the plain CSR), matrices
without a single interleaved block, empty rows and whole blocks of them, blocks closed by the 256-row limit, rows that
span 2 .. 32 lanes of a block, column blocks without entries, long rows that a column split turns into a short and a
long part.  The generators of the other test files (k entries in every row, 2-3 per column) and the MPS fixtures
reach none of them, so this file builds a zoo of such structures (numpy, seeded), proves on the CPU that each case has
the property it is named for, and runs the setup kernels, K2, K3, the evaluation and full solves on them, unblocked and
with gather blocking forced on.

References.  A row sum is compared COMPONENTWISE with the correctly rounded exact sum (`row_sums_hp`: error-free
products, math.fsum), never norm-wise: a dropped entry of a 6-entry row must not hide behind the magnitude of a dense
row.  The CPU oracle is checked against the same reference on every structure (CPU tests below) before the GPU tests
use it as a witness.

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
from collections import namedtuple
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp

from cuopt_b200 import capi, lpgen
from oracle import pdlp_oracle as po

U53 = 2.0 ** -53
ROW_SUM_FACTOR = 4.0
TINY = 1e-300
ELEMENTWISE, STEPWISE, TRAJECTORY, ACROSS_TRUST_REGION, OBJECTIVE = 1e-12, 1e-11, 1e-7, 1e-6, 1e-6

SLOTS, MAX_ROWS, CH = 256, 256, 8  # the cut rule of spmv_bicsr.cuh: entries per block, rows per block, entries per lane
ENV = "CUOPT_B200_GATHER_BLOCK_BYTES"

Case = namedtuple("Case", "name offsets indices values m n")


# ------------------------------------------------------------------------------------------------------ structure zoo
def from_row_lengths(name, lengths, n, seed, allowed=None, rows_of_columns=None):
    """CSR with the given row lengths: distinct sorted columns drawn from `allowed` (default: all n), values N(0,1).
    rows_of_columns: {row: explicit column array} for rows whose columns are designed, not drawn."""
    rng = np.random.default_rng(seed)
    allowed = np.arange(n) if allowed is None else np.asarray(allowed)
    cols = []
    for r, k in enumerate(lengths):
        if rows_of_columns and r in rows_of_columns:
            cols.append(np.sort(np.asarray(rows_of_columns[r])))
        elif k == len(allowed):
            cols.append(allowed.copy())
        else:
            cols.append(np.sort(rng.choice(allowed, int(k), replace=False)))
    lens = np.array([len(c) for c in cols], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    indices = (np.concatenate(cols) if lens.sum() else np.zeros(0)).astype(np.int32)
    values = rng.standard_normal(len(indices))
    return Case(name, offsets, indices, values, len(lengths), n)


def transposed(case, name):
    A = sp.csr_matrix((case.values, case.indices, case.offsets), shape=(case.m, case.n))
    T = A.T.tocsr()
    T.sort_indices()
    return Case(name, T.indptr.astype(np.int32), T.indices.astype(np.int32), T.data.copy(), case.n, case.m)


def long_row_lengths(rows, n, seed):
    """6-entry rows with rows of 255 .. n entries among them: long rows first, last and adjacent."""
    rng = np.random.default_rng(seed)
    lens = np.full(rows, 6)
    lens[0] = 257
    lens[rows - 1] = 300
    spots = np.sort(rng.choice(np.arange(10, rows - 10, 3), 8, replace=False))
    for r, k in zip(spots, (255, 256, 257, 512, 1000, n, 700, 260)):
        lens[r] = k
    lens[spots[3] + 1] = 513  # two long rows next to each other
    # one row dense on the first 288 columns plus a few elsewhere: every column split of at least 288 columns per block
    # leaves it a long part in block 0 and short parts in later blocks
    designed = {int(spots[6]): np.concatenate([np.arange(288), 288 + rng.choice(n - 288, 40, replace=False)])}
    return lens, designed


def heavy_tail(name, m, n, seed):
    rng = np.random.default_rng(seed)
    lens = np.minimum(rng.zipf(1.5, m), n)
    lens[rng.random(m) < 0.05] = 0
    return from_row_lengths(name, lens, n, seed + 1)


@functools.lru_cache(maxsize=None)
def zoo():
    out = []
    n = 4608  # 16 column blocks of 288 columns: a block can still hold a part of more than 256 entries
    lens, designed = long_row_lengths(n, n, 1)
    out.append(from_row_lengths("long_rows", lens, n, 2, rows_of_columns=designed))
    lens, designed = long_row_lengths(n, n, 3)
    out.append(transposed(from_row_lengths("", lens, n, 4, rows_of_columns=designed), "dense_columns"))
    out.append(from_row_lengths("only_long", [600] * 40, 600, 5))

    # empty rows / columns: [704, 1408) is a whole column block at 3 blocks of 704 and covers blocks 5 .. 7 at 160 columns
    n = 2112
    empty = np.zeros(n, bool)
    empty[[0, n - 1, 50, 52, 54, 1500, 1600]] = True
    empty[704:1408] = True
    lens = np.where(empty, 0, 7)
    lens[[49, 51, 53]] = 200  # full blocks between isolated empty rows
    out.append(from_row_lengths("empty_rows_and_columns", lens, n, 6, allowed=np.flatnonzero(~empty)))

    rng = np.random.default_rng(7)
    lens = np.concatenate([np.ones(1200, np.int64), rng.integers(1, 3, 1500)])
    out.append(from_row_lengths("singleton_runs", lens, 1500, 8))

    rng = np.random.default_rng(9)
    lens = [256, 1, 255, 255, 1, 248, 8, 248, 9, 8, 9, 16, 17, 24, 63, 64, 65, 248, 255, 256]
    lens += list(rng.integers(17, 41, 300)) + list(rng.integers(41, 200, 60)) + [256, 8, 8, 8, 8]
    out.append(from_row_lengths("lane_spans", lens, 600, 10))

    out.append(from_row_lengths("tiny_1x1", [1], 1, 11))
    out.append(from_row_lengths("tiny_1x700", [700], 700, 12))
    out.append(transposed(from_row_lengths("", [700], 700, 13), "tiny_700x1"))
    out.append(from_row_lengths("tiny_few_blocks", [10] * 60, 50, 14))
    out.append(heavy_tail("heavy_tail_1", 1500, 1200, 15))
    out.append(heavy_tail("heavy_tail_2", 1200, 1500, 17))
    return {c.name: c for c in out}


ZOO = ["long_rows", "dense_columns", "only_long", "empty_rows_and_columns", "singleton_runs", "lane_spans", "tiny_1x1",
       "tiny_1x700", "tiny_700x1", "tiny_few_blocks", "heavy_tail_1", "heavy_tail_2"]
BLOCKING = [None, 3, 16]  # unblocked, ~3 column blocks, 16 column blocks (of the smaller side; the other gets <= 16)


def block_bytes(case, blocks):
    """CUOPT_B200_GATHER_BLOCK_BYTES that cuts the gathered vector of the smaller side of `case` into `blocks` pieces."""
    if blocks is None:
        return None
    return max(1, int(8 * min(case.m, case.n) / (2.5 if blocks == 3 else blocks)))


def column_blocks(cols, nnz, nbytes):
    """(number of column blocks, their width) the solver uses for a matrix that gathers from `cols` values: blocking
    starts above 1.5 blocks of gathered vector, at most 16 blocks, widths a multiple of 32 (DESIGN.md section 5)."""
    nbytes = 0 if nbytes is None else int(nbytes)
    if nbytes == 0 or nnz == 0 or 8 * cols <= nbytes + nbytes // 2:
        return 1, cols
    B = min(16, -(-8 * cols // nbytes))
    width = (-(-cols // B) + 31) & ~31
    B = -(-cols // width)
    return (B, width) if B > 1 else (1, cols)


# ------------------------------------------------------------------------- numpy model of the block cut (DESIGN.md section 4)
def cut_blocks(offsets):
    """Whole consecutive rows, at most 256 entries and 256 rows per block; a longer row is a long-row block.
    -> (interleaved blocks [(first row, one past last row)], long rows).  (Cuts never cross a 65536-row segment: this is
    the cut of one segment; test_wide_shapes.py models several.)"""
    off = np.asarray(offsets, np.int64)
    rows = len(off) - 1
    assert rows <= 65536
    std, long_rows, r = [], [], 0
    while r < rows:
        if off[r + 1] - off[r] > SLOTS:
            long_rows.append(r)
            r += 1
            continue
        r1 = r
        while r1 < rows and off[r1 + 1] - off[r] <= SLOTS and r1 - r < MAX_ROWS:
            r1 += 1
        std.append((r, r1))
        r = r1
    return std, long_rows


def structure(offsets):
    """The properties of a matrix that decide which branches of the SpMV core run."""
    off = np.asarray(offsets, np.int64)
    std, long_rows = cut_blocks(off)
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
                two_payload_groups=len(std) > 0 and rows > 40 * len(std),  # fused_npre() == 2
                lanes_spanned=lanes_spanned, empty_rows=int(np.sum(np.diff(off) == 0)))


def split_columns(case, width):
    """Row offsets of the column blocks [b width, (b + 1) width) of a matrix."""
    B = -(-case.n // width)
    row = np.repeat(np.arange(case.m), np.diff(case.offsets))
    counts = np.zeros((B, case.m), np.int64)
    np.add.at(counts, (case.indices // width, row), 1)
    return [np.concatenate([[0], np.cumsum(c)]) for c in counts]


def as_transpose(case):
    return transposed(case, case.name + "^T")


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


# ----------------------------------------------------------------------------------------------------- planted LPs
def planted(case, seed=1):
    """An LP on the structure with a known optimum, built as lpgen.sparse_lp builds one: x* half zero, y* with
    complementary slackness, c = A^T y* + r*, rows E / L / G with half of the inequalities inactive.  Empty rows get
    bounds that contain 0."""
    rng = np.random.default_rng(seed)
    m, n = case.m, case.n
    row = np.repeat(np.arange(m), np.diff(case.offsets))
    x_star = np.where(rng.random(n) < 0.5, 0.0, rng.uniform(0.0, 10.0, n))
    ax = np.bincount(row, weights=case.values * x_star[case.indices], minlength=m)
    kind = rng.random(m)
    is_e, is_l, is_g = kind < 0.5, (kind >= 0.5) & (kind < 0.75), kind >= 0.75
    active = rng.random(m) < 0.5
    y_star = rng.standard_normal(m)
    y_star = np.where(is_l, -np.abs(y_star), np.where(is_g, np.abs(y_star), y_star))
    y_star = np.where(~is_e & ~active, 0.0, y_star)
    slack = rng.uniform(0.0, 1.0, m)
    con_lb = np.where(is_e, ax, np.where(is_g, np.where(active, ax, ax - slack), -np.inf))
    con_ub = np.where(is_e, ax, np.where(is_l, np.where(active, ax, ax + slack), np.inf))
    empty = np.diff(case.offsets) == 0
    y_star[empty] = 0.0
    con_lb[empty] = np.where(is_l[empty], -np.inf, -slack[empty])
    con_ub[empty] = np.where(is_g[empty], np.inf, slack[empty])
    r_star = np.where(x_star > 0.0, 0.0, rng.uniform(0.0, 1.0, n))
    c = np.bincount(case.indices, weights=case.values * y_star[row], minlength=n) + r_star
    return lpgen.LP(case.offsets, case.indices, case.values, c, np.zeros(n), np.full(n, np.inf), con_lb, con_ub,
                    float(c @ x_star), x_star, y_star, name=f"planted({case.name},seed={seed})")


def oracle_of(lp, mode=1, tol=1e-4, **kw):
    return po.Oracle(lp.offsets, lp.indices, lp.values, lp.c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub, mode=mode, tol=tol,
                     **kw)


def rel_err(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b)))) if a.size else 0.0


def transpose_structure(case):
    """(row offsets, column indices, source positions) of A^T: entry k of A^T is entry positions[k] of A (stable order)."""
    T = sp.csr_matrix((np.arange(1, len(case.values) + 1, dtype=np.float64), case.indices, case.offsets),
                      shape=(case.m, case.n)).T.tocsr()
    T.sort_indices()
    return T.indptr, T.indices, T.data.astype(np.int64) - 1


def scaled_transpose(case, scaled_values, scaled_values_t):
    """CSR of the scaled A^T: the structure of the input's transpose with the solver's own scaled values of A^T, after
    checking entry by entry that they are the scaled values of A at the transposed positions.  The two are scaled
    separately, (a Dr) Dc and (a Dc) Dr as the reference does, so they agree to two roundings, not bit for bit."""
    off, idx, pos = transpose_structure(case)
    moved = np.asarray(scaled_values)[pos]
    assert np.all(np.abs(scaled_values_t - moved) <= 4 * U53 * np.abs(moved))
    return off, idx, np.asarray(scaled_values_t)


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


def reduced_cost_reference(lp, y):
    """Reduced costs of the default preset (c - A^T y where the bound it presses against is finite, else 0) from exact row
    sums, and the componentwise tolerance; twice the row-sum bound, since a gradient within that bound of 0 may pick the
    other bound."""
    T = as_transpose(Case("", lp.offsets, lp.indices, lp.values, lp.m, lp.n))
    aty, mag, lens = row_sums_hp(T.offsets, T.indices, T.values, y)
    g = lp.c - aty
    bound = np.where(g > 0.0, lp.var_lb, lp.var_ub)
    rc = np.where((g != 0.0) & np.isfinite(bound), g, 0.0)
    return rc, g, 2.0 * (row_sum_tolerance(mag, lens) + 4 * U53 * (np.abs(lp.c) + np.abs(aty)))


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
    std, _ = cut_blocks(off)
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
            assert any(o[-1] == 0 for o in split_columns(cc, width)), (cc.name, blocks)
    # ... and a long row keeps a long part in one block and a short, non-empty part in another
    for cc in (z["long_rows"], as_transpose(z["dense_columns"])):
        for blocks in (3, 16):
            width = column_blocks(cc.n, 1, block_bytes(cc, blocks))[1]
            parts = np.array([np.diff(o) for o in split_columns(cc, width)])  # blocks x rows
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
@pytest.fixture
def gather_block_bytes(monkeypatch):
    """Force gather blocking on small LPs (normally on only when the gathered vector is several times the block size);
    None: leave it to the solver, which does not block at these sizes."""
    def force(nbytes):
        if nbytes is None:
            monkeypatch.delenv(ENV, raising=False)
        else:
            monkeypatch.setenv(ENV, str(int(nbytes)))
    yield force
    monkeypatch.delenv(ENV, raising=False)


def problem_of(lp):
    return capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)


def settings_of(mode=1, tol=1e-4, **kw):
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=mode, **kw)
    s.set("optimality_tolerance", tol)
    return s


def session(case, blocks, force, mode=1, tol=1e-9, seed=1):
    """(planted LP, initialised GPU session) with the column blocking asked for, which is asserted."""
    lp = planted(case, seed)
    nbytes = block_bytes(case, blocks)
    force(nbytes)
    g = capi.Solver(problem_of(lp), settings_of(mode, tol))
    g.initialise()
    assert g.scalar("eval_blocks") == column_blocks(case.n, len(case.values), nbytes)[0]
    assert g.scalar("eval_blocks_t") == column_blocks(case.m, len(case.values), nbytes)[0]
    return lp, g


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


def check_evaluation(lp, sol, **oracle_settings):
    """stats() and reduced_costs() of a solution against a recomputation from its own primal() and dual()."""
    assert sol.return_code == 0, sol.error_string
    x, y, st = sol.primal(), sol.dual(), sol.stats()
    cv = oracle_of(lp, **oracle_settings).convergence(x, y)
    for v in ("l2_primal_residual", "l2_dual_residual", "primal_objective", "dual_objective", "gap"):
        assert getattr(st, v) == pytest.approx(cv[v], rel=STEPWISE, abs=STEPWISE), v
    rc, _, tol = reduced_cost_reference(lp, y)
    got = sol.reduced_costs()
    bad = np.flatnonzero(~(np.abs(got - rc) <= tol))
    assert bad.size == 0, ("columns", bad[:8].tolist(), got[bad[:8]].tolist(), rc[bad[:8]].tolist())
    ax = row_sums_hp(lp.offsets, lp.indices, lp.values, x)[0]
    viol = np.maximum(lp.con_lb - ax, 0.0) + np.maximum(ax - lp.con_ub, 0.0)
    assert st.l2_primal_residual == pytest.approx(np.linalg.norm(viol), rel=STEPWISE, abs=STEPWISE)


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
    check_evaluation(lp, sol)


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", BLOCKING)
def test_evaluation_with_per_constraint_residual(blocks, gather_block_bytes):
    case = zoo()["long_rows"]
    lp = planted(case)
    gather_block_bytes(block_bytes(case, blocks))
    sol = capi.solve(problem_of(lp), settings_of(tol=1e-12, iteration_limit=40, per_constraint_residual=True))
    assert sol.termination_reason == "IterationLimit"
    check_evaluation(lp, sol, per_constraint_residual=True)


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
