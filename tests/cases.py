"""The seeded structures and LPs of the tests, and the builders of problems, settings and oracles around them (support
module: pytest does not collect it).

  zoo()             adversarial row structures of the SpMV core: rows longer than a block, matrices without a single
                    interleaved block, empty rows and whole blocks of them, blocks closed by the 256-row limit, rows that
                    span 2 .. 32 lanes of a block, column blocks without entries, long rows that a column split turns
                    into a short and a long part; planted() puts an LP with a known optimum on each
  bound_zoo()       LPs with every bound kind in every role of a planted optimum (planted_bounds), and certificates():
                    small LPs infeasible or unbounded because of one bound kind
  wide()            LPs past one launch wave, one 65 536-row cut segment and one staging slot
"""
import functools
import os
from collections import namedtuple

import numpy as np

from conftest import mps_path, problem_arrays
from cuopt_b200 import capi, lpgen
from device_model import SEGMENT
from exact import transpose
from oracle import pdlp_oracle as po

inf = np.inf
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
    toff, tidx, pos = transpose(case.offsets, case.indices, case.n)
    return Case(name, toff.astype(np.int32), tidx.astype(np.int32), case.values[pos], case.n, case.m)


def as_transpose(case):
    return transposed(case, case.name + "^T")


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


# ------------------------------------------------------------------------------------------------------- bound zoo
VAR_ROLES = ["free", "lower_neg_at", "lower_neg_in", "lower_zero_at", "lower_zero_in", "lower_pos_at", "lower_pos_in",
             "upper_neg_at", "upper_pos_at", "upper_in",
             "box_at_l", "box_at_u", "box_in", "box_above_at_l", "box_above_at_u", "box_above_in", "box_below_at_l",
             "box_below_at_u", "box_below_in", "box_thin", "fixed_r_pos", "fixed_r_neg", "fixed_zero"]
ROW_ROLES = ["E", "L_active", "L_inactive", "G_active", "G_inactive", "ranged_at_lc", "ranged_at_uc", "ranged_inside",
             "free", "empty_ranged"]


def roles(count, names, rng):
    """Every role at least once (at random positions), the rest drawn at random."""
    assert count >= len(names)
    r = np.concatenate([np.arange(len(names)), rng.integers(0, len(names), count - len(names))])
    return np.array(names, dtype=object)[rng.permutation(r)]


def planted_bounds(m, n, seed, maximize=False, offset=0.0, per_row=6, heavy_rows=0):
    """An LP with every bound kind in every role of a known optimum (x*, y*, r* = c - A^T y*).
    `heavy_rows` of the m rows (the last ones) get the Zipf row lengths of heavy_tail.
    Returns lpgen.LP with c of the problem to MINIMISE; `user_c` / `maximize` / `offset` describe the problem as posed
    (max -c'x + offset when maximising), `optimal_objective` is its optimum."""
    rng = np.random.default_rng(seed)
    vr, rr = roles(n, VAR_ROLES, rng), roles(m, ROW_ROLES, rng)
    lens = np.where(rr == "empty_ranged", 0, per_row)
    base = from_row_lengths("", lens[:m - heavy_rows], n, seed + 1)
    if heavy_rows:
        h = heavy_tail("", heavy_rows, n, seed + 2)
        off = np.concatenate([base.offsets, base.offsets[-1] + h.offsets[1:]]).astype(np.int32)
        base = Case("", off, np.concatenate([base.indices, h.indices]), np.concatenate([base.values, h.values]), m, n)
        rr[m - heavy_rows:][np.diff(h.offsets) == 0] = "empty_ranged"   # an empty heavy-tail row is an empty row
        rr[m - heavy_rows:][(np.diff(h.offsets) > 0) & (rr[m - heavy_rows:] == "empty_ranged")] = "ranged_inside"
    assert np.all((np.diff(base.offsets) == 0) == (rr == "empty_ranged"))

    # variables: bounds, x*, r*
    l, u, x, r = np.zeros(n), np.full(n, inf), np.zeros(n), np.zeros(n)
    pos = lambda k=n: rng.uniform(0.5, 2.0, k)  # noqa: E731  strictly positive reduced costs / duals / slacks
    for j, role in enumerate(vr):
        a, b = sorted(rng.uniform(-10.0, 10.0, 2))
        lo_, hi_ = -abs(a) - 0.5, abs(b) + 0.5                           # a box that straddles 0
        above, below = (abs(a) + 0.5, abs(a) + abs(b) + 1.0), (-abs(a) - abs(b) - 1.0, -abs(a) - 0.5)
        rp, mid = float(pos(1)[0]), float(rng.uniform(0.2, 0.8))
        if role == "free":
            l[j], u[j], x[j] = -inf, inf, rng.normal(0.0, 3.0)
        elif role.startswith("lower"):
            l[j] = {"neg": -abs(a) - 0.5, "zero": 0.0, "pos": abs(a) + 0.5}[role.split("_")[1]]
            x[j], r[j] = (l[j], rp) if role.endswith("_at") else (l[j] + rng.uniform(0.5, 5.0), 0.0)
        elif role.startswith("upper"):
            l[j], u[j] = -inf, {"upper_neg_at": -abs(b) - 0.5, "upper_pos_at": abs(b) + 0.5}.get(role, b)
            x[j], r[j] = (u[j], -rp) if role.endswith("_at") else (u[j] - rng.uniform(0.5, 5.0), 0.0)
        elif role.startswith("box"):
            l[j], u[j] = above if "above" in role else below if "below" in role else (lo_, hi_)
            if role == "box_thin":
                l[j] = abs(a) + 1.0
                u[j] = l[j] * (1.0 + 1e-6)
            if role.endswith("at_l") or role == "box_thin":
                x[j], r[j] = l[j], rp
            elif role.endswith("at_u"):
                x[j], r[j] = u[j], -rp
            else:
                x[j] = l[j] + mid * (u[j] - l[j])
        else:  # fixed
            l[j] = u[j] = 0.0 if role == "fixed_zero" else a
            x[j], r[j] = l[j], {"fixed_r_pos": rp, "fixed_r_neg": -rp}.get(role, rng.choice([-1.0, 1.0]) * rp)

    # rows: bounds and y*
    row = np.repeat(np.arange(m), np.diff(base.offsets))
    ax = np.bincount(row, weights=base.values * x[base.indices], minlength=m)
    y, s1, s2 = np.zeros(m), pos(m), pos(m)
    lc, uc = ax.copy(), ax.copy()
    for i, role in enumerate(rr):
        if role == "E":
            y[i] = rng.normal() + np.sign(rng.normal()) * 0.5
        elif role == "L_active":
            lc[i], y[i] = -inf, -s1[i]
        elif role == "L_inactive":
            lc[i], uc[i] = -inf, ax[i] + s2[i]
        elif role == "G_active":
            uc[i], y[i] = inf, s1[i]
        elif role == "G_inactive":
            lc[i], uc[i] = ax[i] - s2[i], inf
        elif role == "ranged_at_lc":
            uc[i], y[i] = ax[i] + s2[i], s1[i]
        elif role == "ranged_at_uc":
            lc[i], y[i] = ax[i] - s2[i], -s1[i]
        elif role == "ranged_inside":
            lc[i], uc[i] = ax[i] - s1[i], ax[i] + s2[i]
        elif role == "free":
            lc[i], uc[i] = -inf, inf
        else:  # empty ranged row containing 0 (ax = 0)
            lc[i], uc[i] = -s1[i], s2[i]
    c = np.bincount(base.indices, weights=base.values * y[row], minlength=n) + r
    lp = lpgen.LP(base.offsets, base.indices, base.values, c, l, u, lc, uc, None, x, y,
                  name=f"planted_bounds({m}x{n},seed={seed},max={maximize},offset={offset})")
    lp.r_star, lp.var_role, lp.row_role = r, vr, rr
    lp.maximize, lp.offset = maximize, offset
    lp.user_c = -c if maximize else c
    lp.optimal_objective = float(lp.user_c @ x) + offset
    return lp


BOUND_ZOO = ["tiny", "medium", "heavy", "medium_max", "medium_offset"]


@functools.lru_cache(maxsize=None)
def bound_zoo(name):
    if name == "tiny":
        return planted_bounds(40, 30, 21)
    if name == "heavy":
        return planted_bounds(1600, 1200, 23, heavy_rows=600)
    return planted_bounds(3000, 2500, 22, maximize=name == "medium_max",
                          offset={"medium_offset": 123.25}.get(name, 0.0))


# ------------------------------------------------------------------------------------------------------ certificates
Cert = namedtuple("Cert", "name offsets indices values c l u lc uc status")  # 1 optimal, 2 infeasible, 3 unbounded
HIGHS_STATUS = {1: 0, 2: 2, 3: 3}  # linprog: 0 optimal, 2 infeasible, 3 unbounded


def cert(name, rows, c, l, u, lc, uc, status):
    """rows: list of {column: value}."""
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    idx = np.array([j for r in rows for j in sorted(r)], np.int32)
    val = np.array([r[j] for r in rows for j in sorted(r)], float)
    return Cert(name, off, idx, val, *(np.asarray(v, float) for v in (c, l, u, lc, uc)), status)


@functools.lru_cache(maxsize=None)
def certificates():
    """Small LPs whose infeasibility / unboundedness rests on ONE bound kind (without it they are feasible / bounded).
    A feasible ranged row and a boxed variable ride along in each, so the verdict passes other kinds too."""
    return [
        # x0 fixed at 1, but x0 + x1 <= 0 with x1 >= 0
        cert("infeasible_fixed_var", [{0: 1, 1: 1}, {1: 1, 2: 1}], [1, 1, 1], [1, 0, -1], [1, inf, 1],
             [-inf, -2], [0, 2], 2),
        # x0 <= -1 (upper-only), but x0 - x1 >= 0 with x1 >= 0
        cert("infeasible_upper_only_var", [{0: 1, 1: -1}, {1: 1, 2: 1}], [1, 1, 1], [-inf, 0, -1], [-1, inf, 1],
             [0, -2], [inf, 2], 2),
        # 1 <= x0 + x1 <= 2 (ranged), but x0 + x1 >= 3
        cert("infeasible_ranged_row", [{0: 1, 1: 1}, {0: 1, 1: 1}, {1: 1, 2: 1}], [1, 1, 1], [0, 0, -1], [inf, inf, 1],
             [1, 3, -2], [2, inf, 2], 2),
        # x0 + x1 = -1 with x >= 0
        cert("infeasible_equality_row", [{0: 1, 1: 1}, {1: 1, 2: 1}], [1, 1, 1], [0, 0, -1], [inf, inf, 1],
             [-1, -2], [-1, 2], 2),
        # min x0 with x0 free and x0 + x1 - x3 = 1, x1, x3 >= 0
        cert("unbounded_free_var", [{0: 1, 1: 1, 3: -1}, {2: 1, 3: 1}], [1, 0, 1, 0], [-inf, 0, -1, 0],
             [inf, inf, 1, inf], [1, -2], [1, 2], 3),
        # min -x1 with x0 + x1 = 1 and x0 <= 2 (upper-only): x1 grows as x0 falls
        cert("unbounded_upper_only_var_negative_cost", [{0: 1, 1: 1}, {1: 1, 2: 1}], [0, -1, 1], [-inf, 0, -1],
             [2, inf, 1], [1, -2], [1, inf], 3),
        # min x0 + x2 with -inf < x0 <= 3 (lower bound -inf) and x0 + x1 = -4, x1 >= -2 (negative lower bound)
        cert("unbounded_minus_inf_lower_bound", [{0: 1, 1: 1}, {2: 1, 3: 1}], [1, 0, 1, 0], [-inf, -2, -1, 0],
             [3, inf, 1, inf], [-4, -2], [-4, 2], 3),
        # the control: min -x0 + x1 / 1000 with x0 + x1 >= 100 and 0 <= x0 <= 5 is bounded only by the upper bound
        # of x0; while the iterate is short of the G row (primal infeasible, homogeneous residual 0) the ray test
        # runs, and it is the finite upper bound of x0 that must keep it from reporting Unbounded
        cert("optimal_because_of_upper_bound", [{0: 1, 1: 1}], [-1, 1e-3], [0, 0], [5, inf], [100], [inf], 1),
    ]


MPS_CERTIFICATES = [("good-mps-free-var", 3), ("good-mps-lower-bound-inf-var", 3), ("good-mps-fixed-var", 2),
                    ("good-mps-fixed-ranges", 2), ("good-mps-free-ranges", 2)]


def mps_arrays(name):
    a = problem_arrays(capi.Problem.read(mps_path(f"linear_programming/{name}.mps")))
    assert not a["maximize"]
    return a


def certificate_args(name):
    if name.startswith("good-mps"):
        a = mps_arrays(name)
        return tuple(a[k] for k in ("offsets", "indices", "values", "c", "var_lb", "var_ub", "con_lb", "con_ub"))
    k = next(k for k in certificates() if k.name == name)
    return k.offsets, k.indices, k.values, k.c, k.l, k.u, k.lc, k.uc


CERTIFICATES = [k.name for k in certificates()] + [n for n, _ in MPS_CERTIFICATES]
CERT_STATUS = {**{k.name: k.status for k in certificates()}, **dict(MPS_CERTIFICATES)}


def c_api_infeasible_lp():
    """The LP of the reference's test_infeasible_problem (cpp/tests/linear_programming/c_api_tests/c_api_test.c:625-700)."""
    off = np.array([0, 2, 4, 6, 7, 9, 10, 12, 15, 17], np.int32)
    idx = np.array([0, 1, 0, 1, 0, 1, 3, 2, 3, 2, 0, 3, 0, 1, 2, 1, 2], np.int32)
    val = np.array([-0.5, 1.0, 2.0, -1.0, 3.0, 1.0, 1.0, 3.0, -1.0, 1.0, 1.0, 1.0, 1.0, 2.0, 1.0, 1.0, 1.0])
    rhs = np.array([0.5, 3.0, 6.0, 2.0, 2.0, 5.0, 10.0, 14.0, 1.0])
    sense = "GGLLLGLLG"
    lc = np.array([r if s in "GE" else -inf for r, s in zip(rhs, sense)])
    uc = np.array([r if s in "LE" else inf for r, s in zip(rhs, sense)])
    return off, idx, val, np.zeros(4), np.zeros(4), np.full(4, inf), lc, uc


def unbounded_lp():
    # min -x  s.t.  x - y = 0,  x, y >= 0: the ray (1, 1) improves forever
    off, idx, val = np.array([0, 2], np.int32), np.array([0, 1], np.int32), np.array([1.0, -1.0])
    return off, idx, val, np.array([-1.0, 0.0]), np.zeros(2), np.full(2, np.inf), np.zeros(1), np.zeros(1)


# c_api_test.c:761-790 (test_ranged_problem)
RANGED_LP = dict(offsets=np.array([0, 2, 4, 6], np.int32), indices=np.array([0, 1, 0, 1, 0, 1], np.int32),
                 values=np.array([2.0, 3.0, 3.0, 1.0, 1.0, 2.0]), c=np.array([5.0, 8.0]),
                 con_lb=np.array([-inf, -inf, 2.0]), con_ub=np.array([12.0, 6.0, 8.0]),
                 var_lb=np.array([0.0, 0.0]), var_ub=np.array([10.0, 10.0]))


# ------------------------------------------------------------------------------------------------------- wide shapes
def from_lengths(name, lens, n, seed):
    """CSR with the given row lengths, distinct sorted columns uniform in [0, n), values N(0, 1) (vectorised)."""
    rng = np.random.default_rng(seed)
    lens = np.asarray(lens, np.int64)
    row = np.repeat(np.arange(len(lens)), lens)
    cols = rng.integers(0, n, int(lens.sum()))
    for _ in range(64):
        cols = cols[np.lexsort((cols, row))]
        dup = np.zeros(len(cols), bool)
        dup[1:] = (cols[1:] == cols[:-1]) & (row[1:] == row[:-1])
        if not dup.any():
            break
        cols[dup] = rng.integers(0, n, int(dup.sum()))
    assert not dup.any()
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return Case(name, offsets, cols.astype(np.int32), rng.standard_normal(len(cols)), len(lens), n)


WIDE = ["tall", "short_rows", "segment_edges"]
B1, B2, B3 = SEGMENT, 2 * SEGMENT, 3 * SEGMENT
RUN = (B2 - 300, B2 + 300)         # 1-entry rows across the second boundary
EMPTY = (B3 - 150, B3 + 50)        # empty rows across the third, ordinary rows after them


@functools.lru_cache(maxsize=None)
def wide(name):
    """(Case, planted LP) of the cases test_wide_shapes.py describes."""
    if name == "tall":
        lp = lpgen.sparse_lp(600_000, 400_000, 8, seed=5)
        return Case(name, lp.offsets, lp.indices, lp.values, lp.m, lp.n), lp
    rng = np.random.default_rng({"short_rows": 31, "segment_edges": 32}[name])
    if name == "short_rows":
        case = from_lengths(name, rng.integers(1, 4, 1_100_000), 1_100_000, 33)
    else:
        m = 3 * SEGMENT + 77
        lens = np.full(m, 6)
        lens[rng.choice(m, 6200, replace=False)] = rng.integers(257, 301, 6200)
        lens[B1 - 1], lens[B1] = 280, 290
        lens[RUN[0]:RUN[1]] = 1
        lens[EMPTY[0]:EMPTY[1]] = 0
        case = from_lengths(name, lens, 40_000, 34)
    return case, planted(case, 35)


def host_threads():
    try:
        return max(1, min(32, len(os.sched_getaffinity(0))))
    except Exception:  # noqa: BLE001
        return 8


# ----------------------------------------------------------------------------- problems, settings and oracles
def problem_of(lp):
    """The C-ABI problem of an lpgen.LP."""
    return capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)


def bounds_problem(lp):
    """The C-ABI problem of a planted_bounds() LP, as posed: user_c, maximize, offset."""
    return capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.user_c, lp.var_lb,
                                      lp.var_ub, maximize=lp.maximize, objective_offset=lp.offset)


def oracle_of(lp, mode=1, tol=1e-4, **kw):
    return po.Oracle(lp.offsets, lp.indices, lp.values, lp.c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub, mode=mode, tol=tol,
                     **kw)


def bounds_oracle(lp, mode, tol=1e-9, **kw):
    return po.Oracle(lp.offsets, lp.indices, lp.values, lp.user_c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub,
                     maximize=lp.maximize, objective_offset=lp.offset, mode=mode, tol=tol, **kw)


def settings_of(mode=1, tol=1e-4, **kw):
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=mode, **kw)
    s.set("optimality_tolerance", tol)
    return s


def make_pair(p, **kw):
    """(GPU solver session, oracle) on the same problem and settings."""
    a = problem_arrays(p)
    tol = kw.pop("tol", 1e-4)
    mode = kw.pop("mode", 1)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=mode, **kw)
    s.set("optimality_tolerance", tol)
    g = capi.Solver(p, s)
    o = po.Oracle(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"],
                  maximize=a["maximize"], objective_offset=a["objective_offset"], mode=mode, tol=tol,
                  iteration_limit=kw.get("iteration_limit", 2**31 - 1))
    return g, o, s


def lp_relaxation(rel):
    """Root LP relaxation of an MPS instance (configs[4]): read it, then re-create it with every variable continuous,
    which is what a C-ABI client does (the reference's MIP path calls PDLP on exactly this relaxation,
    cpp/src/mip/relaxed_lp/relaxed_lp.cu:53-127)."""
    p = capi.Problem.read(mps_path(rel))
    if not p.is_mip:
        return p
    a = problem_arrays(p)
    return capi.Problem.create_ranged(a["offsets"], a["indices"], a["values"], a["con_lb"], a["con_ub"], a["c"],
                                      a["var_lb"], a["var_ub"], maximize=a["maximize"],
                                      objective_offset=a["objective_offset"])


# ------------------------------------------------------------------------------------------- recycled device memory
def solve_arrays(sol):
    st = sol.stats()
    stats = {k: getattr(st, k) for k, _ in type(st)._fields_ if not (k == "solve_time" or k.endswith("_seconds"))}
    return sol.primal(), sol.dual(), sol.reduced_costs(), stats


RECYCLE = {"stable2_checks": dict(mode=po.STABLE2, per_constraint_residual=True, infeasibility_detection=True),
           "methodical1": dict(mode=po.METHODICAL1)}


def recycle_lp(seed):
    return lpgen.sparse_lp(600_000, 400_000, 8, seed=seed)


def cache_probe():
    """A small session that stays open: it reads the process's block-cache counter without allocating anything."""
    g = capi.Solver(problem_of(lpgen.sparse_lp(200, 150, 4, seed=1)), settings_of())
    g.initialise()
    return g


def recycle_solve(config, seed):
    kw = dict(RECYCLE[config])
    return capi.solve(problem_of(recycle_lp(seed)), settings_of(tol=1e-12, iteration_limit=300, **kw))
