"""The host restatement of what the solver builds on the device and launches (support module: pytest does not collect
it).  Every test that reasons about the BICSR cut, the column blocks, their compact encoding or the launch grids uses
this one model; the constants are those of the sources named beside them.

  cut            whole consecutive rows, at most SLOTS entries and MAX_ROWS rows per interleaved block; a longer row is a
                 long-row block; blocks never cross a SEGMENT-row segment (pdlp_solver.cu cuts segments on worker threads)
  column blocks  blocking starts above 1.5 blocks of gathered vector, at most 16 blocks, widths a multiple of 32
                 (DESIGN.md section 5)
  compact form   three-byte block-local column indices and the non-empty-row mask in place of the row-slot table
  grids          SpMV, element-wise and scaling-statistics grids for a device of `sms` SMs, the staging ring's fills
"""
import numpy as np
import pytest

from cuopt_b200 import capi

# spmv_bicsr.cuh: entries per block, rows per block, entries per lane
SLOTS, MAX_ROWS, CH = 256, 256, 8
# compact column blocks (spmv_bicsr.cuh): form bits, widest block of three-byte indices, plain pad slot, row-slot table's
# empty row, high-byte flags of a pad slot and of a row end
IDX3, MASK = 1, 2
IDX3_MAX_WIDTH = 1 << 21
PAD = 0x7FFFFFFF
EMPTY = 0xFFFF
HI_PAD, HI_END = 0x40, 0x80
# pdlp_solver.cu: SCHEDULE_SEGMENT, staging ring (slot bytes, slots; arrays below SLOT / 4 bypass it)
SEGMENT = 1 << 16
SLOT, RING = 32 << 20, 4
# pdlp_kernels.cuh: element-wise CTA size; warps (= blocks in flight) per SpMV CTA; CTAs per SM the launch bounds aim
# at: SpMV kernels, fused K2 with two payload groups
EW_THREADS, WARPS = 256, 8
OCC, OCC2 = 4, 3

GATHER = "CUOPT_B200_GATHER_BLOCK_BYTES"


# -------------------------------------------------------------------------------------------------------- the cut
def cut(offsets, segment=SEGMENT):
    """The BICSR cut of `segment`-row segments joined in order -> (interleaved blocks [(first row, one past last row)],
    long rows)."""
    off = np.asarray(offsets, np.int64)
    rows = len(off) - 1
    std, long_rows = [], []
    for s0 in range(0, rows, segment):
        s1, r = min(rows, s0 + segment), s0
        while r < s1:
            if off[r + 1] - off[r] > SLOTS:
                long_rows.append(r)
                r += 1
                continue
            r1 = min(int(np.searchsorted(off, off[r] + SLOTS, side="right")) - 1, r + MAX_ROWS, s1)
            std.append((r, r1))
            r = r1
    return std, long_rows


def k2_npre(rows, n_std):
    """Payload row groups the fused K2 fetches ahead (fused_npre())."""
    return 2 if n_std and rows > 40 * n_std else 1


# ---------------------------------------------------------------------------------------------- column blocks
def block_bytes(case, blocks):
    """CUOPT_B200_GATHER_BLOCK_BYTES that cuts the gathered vector of the smaller side of `case` into `blocks` pieces
    (None: leave blocking to the solver)."""
    if blocks is None:
        return None
    return max(1, int(8 * min(case.m, case.n) / (2.5 if blocks == 3 else blocks)))


def column_blocks(cols, nnz, nbytes):
    """(number of column blocks, their width) the solver uses for a matrix that gathers from `cols` values."""
    nbytes = 0 if nbytes is None else int(nbytes)
    if nbytes == 0 or nnz == 0 or 8 * cols <= nbytes + nbytes // 2:
        return 1, cols
    B = min(16, -(-8 * cols // nbytes))
    width = (-(-cols // B) + 31) & ~31
    B = -(-cols // width)
    return (B, width) if B > 1 else (1, cols)


def split_columns(case, width):
    """[(row offsets, global column indices)] of the column blocks [b width, (b + 1) width) of a matrix: the entries of
    every row with a column in the block, in row order."""
    off = np.asarray(case.offsets, np.int64)
    idx = np.asarray(case.indices, np.int64)
    row = np.repeat(np.arange(case.m), np.diff(off))
    out = []
    for b in range(-(-case.n // width)):
        keep = (idx >= b * width) & (idx < (b + 1) * width)
        counts = np.bincount(row[keep], minlength=case.m)
        out.append((np.concatenate([[0], np.cumsum(counts)]).astype(np.int64), idx[keep]))
    return out


# ------------------------------------------------------------------------------------------------ compact form
def slot(q):
    return (q % CH) * 32 + q // CH


def encode_plain(off, idx, blk):
    """Slots (bit 31: row end, PAD unused) and row-slot table of one interleaved block (r0, r1)."""
    r0, r1 = blk
    lo, cnt = off[r0], off[r1] - off[r0]
    slots = np.full(SLOTS, PAD, np.int64)
    for q in range(cnt):
        slots[slot(q)] = idx[lo + q]
    row_slot = np.full(r1 - r0, EMPTY, np.int64)
    for r in range(r0, r1):
        if off[r + 1] > off[r]:
            s = slot(off[r + 1] - 1 - lo)
            slots[s] |= 1 << 31
            row_slot[r - r0] = s
    return slots, row_slot


def encode_compact(off, idx, blk, col0):
    """lo16 (lane-major: entry q at position q), hi8 (lane l: one word, byte k = entry 8 l + k) and the 8 mask words."""
    r0, r1 = blk
    lo, cnt = off[r0], off[r1] - off[r0]
    ends = np.zeros(SLOTS, bool)
    mask = np.zeros(8, np.uint64)
    for r in range(r0, r1):
        if off[r + 1] > off[r]:
            ends[off[r + 1] - 1 - lo] = True
            mask[(r - r0) // 32] |= np.uint64(1 << ((r - r0) % 32))
    lo16 = np.zeros(SLOTS, np.uint16)
    hi8 = np.zeros(32, np.uint64)
    for q in range(SLOTS):
        if q < cnt:
            c = int(idx[lo + q]) - col0
            assert 0 <= c < IDX3_MAX_WIDTH, "a three-byte index holds 21 bits"
            lo16[q] = c & 0xFFFF
            hb = (c >> 16) | (HI_END if ends[q] else 0)
        else:
            hb = HI_PAD
        hi8[q // CH] |= np.uint64(hb << (8 * (q % CH)))
    return lo16, hi8, mask.astype(np.uint32)


def decode_compact(lo16, hi8, mask, col0, n_rows):
    """The plain slots and row-slot table back from the compact arrays (what the kernels read, in the kernels' terms)."""
    slots = np.full(SLOTS, PAD, np.int64)
    for l in range(32):
        for k in range(CH):
            q = CH * l + k
            hb = (int(hi8[l]) >> (8 * k)) & 0xFF
            if hb & HI_PAD:
                continue
            col = (((hb & 0x1F) << 16) | int(lo16[q])) + col0
            slots[k * 32 + l] = col | ((1 << 31) if hb & HI_END else 0)
    # the mask says which rows are non-empty; their last entries are the row ends in entry order
    end_entries = [q for q in range(SLOTS) if (int(hi8[q // CH]) >> (8 * (q % CH) + 7)) & 1]
    row_slot = np.full(n_rows, EMPTY, np.int64)
    for i in range(n_rows):
        if (int(mask[i // 32]) >> (i % 32)) & 1:
            row_slot[i] = slot(end_entries[ordinal_of_row(mask, i)])
    return slots, row_slot


def ordinal_of_row(mask, i):
    """Epilogue side: popcount of the mask below row i (bicsr_mask_cursor_t)."""
    below = sum(bin(int(w)).count("1") for w in mask[: i // 32])
    return below + bin(int(mask[i // 32]) & ((1 << (i % 32)) - 1)).count("1")


def ordinals_of_ends(hi8):
    """Row-sum side: the ordinal of every row end from the per-lane end bits, as the ballots form it
    (bicsr_block_row_sums<true>: prefix popcount over the 4 bits of the per-lane counts, then inside the lane)."""
    ends = [sum(((int(hi8[l]) >> (8 * k + 7)) & 1) << k for k in range(CH)) for l in range(32)]
    cnt = [bin(e).count("1") for e in ends]
    out = {}
    for l in range(32):
        ballots = [sum(((cnt[j] >> b) & 1) << j for j in range(32)) for b in range(4)]
        before = sum(bin(ballots[b] & ((1 << l) - 1)).count("1") << b for b in range(4))
        for k in range(CH):
            if (ends[l] >> k) & 1:
                out[CH * l + k] = before + bin(ends[l] & ((1 << k) - 1)).count("1")
    return out


def host_form(compact_blocks, width, sharded=False, forced_width=False):
    """build_gather_blocks: the form of the column blocks of a single-GPU product."""
    if sharded or forced_width:
        return 0
    fmt = compact_blocks & (IDX3 | MASK)
    if width > IDX3_MAX_WIDTH:
        fmt &= ~IDX3
    return fmt


# ----------------------------------------------------------------------------------------------- launch geometry
def ew_grid(count, sms):
    return max(1, min(-(-count // EW_THREADS), 8 * sms))


def spmv_grid(n_blk, sms, occ):
    return max(1, min(-(-n_blk // WARPS), sms * occ))


def row_group_width(rows, nnz):
    avg = nnz / rows if rows else 0.0
    return 4 if avg <= 4 else 8 if avg <= 8 else 16 if avg <= 16 else 32


def scaling_rounds(rows, nnz, sms):
    w = row_group_width(rows, nnz)
    grid = max(1, min(-(-rows * w // 256), 16 * sms))
    return -(-rows // (grid * (256 // w)))


def staged_arrays(lp):
    """Bytes of the host arrays a session uploads (A, bounds, costs)."""
    return [4 * (lp.m + 1), 4 * lp.nnz, 8 * lp.nnz] + [8 * lp.n] * 3 + [8 * lp.m] * 2


def staged_fills(lp):
    return sum(-(-b // SLOT) for b in staged_arrays(lp) if b >= SLOT // 4)


def cut_counts(offsets, offsets_t):
    """Block counts of the cuts of A and A^T."""
    a, at = cut(offsets), cut(offsets_t)
    return dict(n_std_a=len(a[0]), n_blk_a=len(a[0]) + len(a[1]), n_long_a=len(a[1]),
                n_std_at=len(at[0]), n_blk_at=len(at[0]) + len(at[1]), n_long_at=len(at[1]),
                k2_npre=k2_npre(len(offsets) - 1, len(a[0])))


def geometry(counts, lp, sms, occ=OCC, occ2=OCC2):
    """What the solver launches (unblocked) for an LP with the cut_counts() `counts` on `sms` SMs."""
    s = dict(counts)
    s["grid_k2"] = spmv_grid(s["n_blk_a"], sms, occ2 if s["k2_npre"] == 2 else occ)
    s["grid_k3"] = spmv_grid(s["n_blk_at"], sms, occ)
    s["grid_n"], s["grid_m"] = ew_grid(lp.n, sms), ew_grid(lp.m, sms)
    s["grid_k1"] = s["grid_n"]
    s["staged_fills"] = staged_fills(lp)
    return s


# ------------------------------------------------------------------------------------------------- GPU sessions
@pytest.fixture
def gather_block_bytes(monkeypatch):
    """Force gather blocking on small LPs (normally on only when the gathered vector is several times the block size);
    None: leave it to the solver, which does not block at these sizes."""
    def force(nbytes):
        if nbytes is None:
            monkeypatch.delenv(GATHER, raising=False)
        else:
            monkeypatch.setenv(GATHER, str(int(nbytes)))
    yield force
    monkeypatch.delenv(GATHER, raising=False)


def session(case, problem, settings, blocks, force):
    """An initialised GPU session of `problem` (whose matrix is `case`) with the column blocking asked for, which is
    asserted against the model on both sides."""
    nbytes = block_bytes(case, blocks)
    force(nbytes)
    g = capi.Solver(problem, settings)
    g.initialise()
    assert g.scalar("eval_blocks") == column_blocks(case.n, len(case.values), nbytes)[0]
    assert g.scalar("eval_blocks_t") == column_blocks(case.m, len(case.values), nbytes)[0]
    return g
