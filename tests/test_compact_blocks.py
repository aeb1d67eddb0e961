"""Compact column blocks (CUOPT_B200_COMPACT_BLOCKS, spmv_bicsr.cuh): three-byte block-local column indices and the
non-empty-row mask in place of the row-slot table.

CPU: the numpy model of the encoding in device_model.py — local indices, the flags of the high bytes, pad slots, masks
and the ordinals under which the row sums pass through shared memory — round-trips to the plain BICSR arrays of every
column block of the structure zoo of cases.py, and the host rule that chooses the form is checked at the 2^21-column
edge of the three-byte indices.

GPU: the compact form changes where bytes come from, not what is added, so every product of the solver must be
BIT-EQUAL with the switch on and off: K2's y', K3's A^T y', the three dot products of the step rule, the products of
the termination evaluation (through a solve's residuals and objectives) and a 200-iteration trajectory, at forced cuts
of 3 and 16 column blocks.
"""
import numpy as np
import pytest

from cases import ZOO, Case, as_transpose, planted, problem_of, settings_of, zoo
from cuopt_b200 import capi
from device_model import (CH, GATHER, IDX3, IDX3_MAX_WIDTH, MASK, SLOTS, block_bytes, column_blocks, cut, decode_compact,
                          encode_compact, encode_plain, host_form, ordinal_of_row, ordinals_of_ends, split_columns)

SWITCH = "CUOPT_B200_COMPACT_BLOCKS"


def column_block_cases():
    """(case name, side, blocks, b, off, idx, col0) for every column block of the zoo at forced cuts of 3 and 16."""
    for name in ZOO:
        case = zoo()[name]
        sides = [("A", case)]
        if case.m != case.n or name in ("long_rows", "empty_rows_and_columns"):
            sides.append(("AT", as_transpose(case)))
        for side, M in sides:
            for blocks in (3, 16):
                width = column_blocks(M.n, len(M.values), block_bytes(case, blocks))[1]
                for b, (off, idx) in enumerate(split_columns(M, width)):
                    yield name, side, blocks, b, off, idx, b * width


def test_compact_encoding_round_trips_on_the_zoo():
    seen = dict(empty_block=0, empty_rows=0, lane_spans=0, pads=0, blocks=0)
    for name, side, blocks, b, off, idx, col0 in column_block_cases():
        std, _ = cut(off)
        if len(idx) == 0:
            seen["empty_block"] += 1
        for blk in std:
            r0, r1 = blk
            plain_slots, plain_row_slot = encode_plain(off, idx, blk)
            lo16, hi8, mask = encode_compact(off, idx, blk, col0)
            slots, row_slot = decode_compact(lo16, hi8, mask, col0, r1 - r0)
            where = (name, side, blocks, b, blk)
            assert np.array_equal(slots, plain_slots), where
            assert np.array_equal(row_slot, plain_row_slot), where
            # the ordinal a row end's sum is written under is the ordinal its row's epilogue lane reads
            ords = ordinals_of_ends(hi8)
            lo = off[r0]
            for i in range(r1 - r0):
                if off[r0 + i + 1] > off[r0 + i]:
                    assert ords[off[r0 + i + 1] - 1 - lo] == ordinal_of_row(mask, i), where
            assert len(ords) == sum(bin(int(w)).count("1") for w in mask), where
            seen["blocks"] += 1
            seen["empty_rows"] += int((np.diff(off[r0:r1 + 1]) == 0).any())
            seen["lane_spans"] += int((np.diff(off[r0:r1 + 1]) > CH).any())
            seen["pads"] += int(off[r1] - off[r0] < SLOTS)
    assert all(v > 0 for v in seen.values()), seen


def test_three_byte_indices_at_the_width_edge():
    width = IDX3_MAX_WIDTH
    rng = np.random.default_rng(3)
    for b in (0, 1):
        # the first and the last column of the block, in rows of 1 .. 9 entries
        lens = rng.integers(1, 10, 40)
        cols = [np.sort(rng.choice(width, k, replace=False)) for k in lens]
        cols[0][0], cols[-1][-1] = 0, width - 1
        idx = np.concatenate(cols) + b * width
        off = np.concatenate([[0], np.cumsum(lens)])
        for blk in cut(off)[0]:
            lo16, hi8, mask = encode_compact(off, idx, blk, b * width)
            slots, row_slot = decode_compact(lo16, hi8, mask, b * width, blk[1] - blk[0])
            plain = encode_plain(off, idx, blk)
            assert np.array_equal(slots, plain[0]) and np.array_equal(row_slot, plain[1])
    # one column more and the local index no longer fits: the host falls back to 4-byte indices
    with pytest.raises(AssertionError, match="21 bits"):
        encode_compact(np.array([0, 1]), np.array([width]), (0, 1), 0)
    assert host_form(3, width) == 3
    assert host_form(3, width + 32) == MASK
    assert host_form(IDX3, width + 32) == 0
    assert host_form(0, width) == 0
    assert host_form(3, width, sharded=True) == 0 and host_form(3, width, forced_width=True) == 0
    # the cuts the GPU test below asks for land on both sides of the edge
    assert column_blocks(1 << 22, 1, 1 << 24) == (2, width)
    assert column_blocks((1 << 22) + 64, 1, (1 << 24) + 1024) == (2, width + 32)


# ------------------------------------------------------------------------------------------------------ GPU: bit-equal
CASES = ["empty_rows_and_columns", "lane_spans", "singleton_runs", "long_rows", "heavy_tail_1"]


def bits(v):
    return np.asarray(v, np.float64).view(np.uint64)


def trajectory(lp, nbytes, form, monkeypatch, checkpoints=(1, 7, 50, 200), mode=1):
    monkeypatch.setenv(GATHER, str(int(nbytes)))
    monkeypatch.setenv(SWITCH, str(form))
    g = capi.Solver(problem_of(lp), settings_of(mode, 1e-12))
    g.initialise()
    out = {"form_a": g.scalar("blocks_form_a"), "form_at": g.scalar("blocks_form_at")}
    done = 0
    for c in checkpoints:
        g.advance(c - done)
        done = c
        out[c] = {v: g.vector(v) for v in ("x", "y", "aty", "x_bar")}
        out[c].update({s: g.scalar(s) for s in ("interaction", "norm_dx2", "norm_dy2", "step_size", "k_pdhg")})
    g.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", [3, 16])
@pytest.mark.parametrize("name", CASES)
def test_steps_are_bit_equal_with_the_switch_on_and_off(name, blocks, monkeypatch):
    """K2's y' (and the x_bar it reads), K3's A^T y', the step rule's dot products, over 200 iterations."""
    case = zoo()[name]
    lp = planted(case)
    nbytes = block_bytes(case, blocks)
    off = trajectory(lp, nbytes, 0, monkeypatch)
    on = trajectory(lp, nbytes, 3, monkeypatch)
    assert off["form_a"] == 0 and off["form_at"] == 0
    B_a = column_blocks(case.n, len(case.values), nbytes)[0]
    B_at = column_blocks(case.m, len(case.values), nbytes)[0]
    assert on["form_a"] == (3 if B_a > 1 else 0) and on["form_at"] == (3 if B_at > 1 else 0)
    assert B_a > 1 or B_at > 1
    for c in (1, 7, 50, 200):
        for k, v in off[c].items():
            assert np.array_equal(bits(on[c][k]), bits(v)), (c, k)


@pytest.mark.gpu
@pytest.mark.parametrize("form", [IDX3, MASK])
def test_each_item_alone_is_bit_equal(form, monkeypatch):
    case = zoo()["heavy_tail_2"]
    lp = planted(case)
    nbytes = block_bytes(case, 16)
    off = trajectory(lp, nbytes, 0, monkeypatch, checkpoints=(30,))
    on = trajectory(lp, nbytes, form, monkeypatch, checkpoints=(30,))
    assert on["form_a"] == form
    for k, v in off[30].items():
        assert np.array_equal(bits(on[30][k]), bits(v)), k


def solve(lp, nbytes, form, monkeypatch, **kw):
    monkeypatch.setenv(GATHER, str(int(nbytes)))
    monkeypatch.setenv(SWITCH, str(form))
    s = settings_of(1, 1e-6, **kw)
    sol = capi.solve(problem_of(lp), s)
    assert sol.return_code == 0, sol.error_string
    st = sol.stats()
    return sol, {k: getattr(st, k) for k in ("number_of_steps_taken", "primal_objective", "dual_objective", "gap",
                                             "l2_primal_residual", "l2_dual_residual")}


@pytest.mark.gpu
@pytest.mark.parametrize("blocks", [3, 16])
@pytest.mark.parametrize("name", ["empty_rows_and_columns", "lane_spans", "heavy_tail_2"])
def test_evaluation_is_bit_equal_with_the_switch_on_and_off(name, blocks, monkeypatch):
    """The termination evaluation multiplies by the unscaled column blocks (k_spmv_pair): residuals, objectives, gap,
    the iteration it stops at and the solution."""
    case = zoo()[name]
    lp = planted(case)
    nbytes = block_bytes(case, blocks)
    s0, st0 = solve(lp, nbytes, 0, monkeypatch, per_constraint_residual=True, iteration_limit=600)
    s1, st1 = solve(lp, nbytes, 3, monkeypatch, per_constraint_residual=True, iteration_limit=600)
    for k, v in st0.items():
        assert np.array_equal(bits(st1[k]), bits(v)), k
    for f in ("primal", "dual", "reduced_costs"):
        assert np.array_equal(bits(getattr(s1, f)()), bits(getattr(s0, f)())), f


def wide(n, seed=5):
    """4096 rows of 1 .. 9 entries over n columns, the first and the last column of every block included."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 10, 4096)
    cols = [np.sort(rng.choice(n, k, replace=False)) for k in lens]
    cols[0] = np.array([0, (1 << 21) - 1, 1 << 21, n - 1])
    lens[0] = 4
    idx = np.concatenate(cols).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return Case("wide", off, idx, rng.standard_normal(len(idx)), 4096, n)


@pytest.mark.gpu
@pytest.mark.parametrize("n,nbytes,form", [(1 << 22, 1 << 24, IDX3 | MASK), ((1 << 22) + 64, (1 << 24) + 1024, MASK)])
def test_width_edge_of_three_byte_indices(n, nbytes, form, monkeypatch):
    """A column block of exactly 2^21 columns takes three-byte indices; one 32 columns wider falls back to four."""
    lp = planted(wide(n))
    off = trajectory(lp, nbytes, 0, monkeypatch, checkpoints=(5,))
    on = trajectory(lp, nbytes, 3, monkeypatch, checkpoints=(5,))
    assert on["form_a"] == form
    for k, v in off[5].items():
        assert np.array_equal(bits(on[5][k]), bits(v)), k
