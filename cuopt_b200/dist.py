"""Host-side helpers for the row-sharded multi-GPU solve (one process per GPU, torch.distributed for the plumbing).

shard_rows      contiguous, nnz-balanced partition of the constraint rows (the unit the path shards on)
local_problem   the rows of one rank as a C-ABI problem (all columns, global column indices)
bootstrap       NCCL communicator of libcuopt.so: rank 0 creates the unique id, torch.distributed broadcasts it
reference_protocol_step   numpy restatement of what ONE distributed PDHG attempt exchanges (used by the gloo CPU tests)
"""
from __future__ import annotations

import numpy as np


def shard_bounds(offsets: np.ndarray, world: int) -> np.ndarray:
    """Row boundaries b[0..world]: rank g owns rows [b[g], b[g+1]).  Balanced on nnz + rows (both cost memory traffic)."""
    m = len(offsets) - 1
    cost = offsets.astype(np.int64) + np.arange(m + 1, dtype=np.int64)  # cumulative (nnz + rows)
    targets = cost[-1] * np.arange(1, world, dtype=np.float64) / world
    cuts = np.searchsorted(cost, targets, side="left")
    b = np.concatenate([[0], cuts, [m]]).astype(np.int64)
    return np.maximum.accumulate(b)


def shard_rows(lp, rank: int, world: int):
    """(row_start, row_end, local CSR offsets, indices, values, con_lb, con_ub) of `rank`."""
    b = shard_bounds(lp.offsets, world)
    r0, r1 = int(b[rank]), int(b[rank + 1])
    lo, hi = int(lp.offsets[r0]), int(lp.offsets[r1])
    off = (lp.offsets[r0:r1 + 1] - lo).astype(np.int32)
    return r0, r1, off, lp.indices[lo:hi], lp.values[lo:hi], lp.con_lb[r0:r1], lp.con_ub[r0:r1]


def local_problem(lp, rank: int, world: int):
    from . import capi
    r0, r1, off, idx, val, clb, cub = shard_rows(lp, rank, world)
    p = capi.Problem.create_ranged(off, idx, val, clb, cub, lp.c, lp.var_lb, lp.var_ub)
    return p, (r0, r1)


def bootstrap(rank: int, world: int, device=None):
    """Create the libcuopt NCCL communicator; the 128-byte unique id travels through torch.distributed."""
    import torch
    import torch.distributed as dist

    from . import capi
    uid = capi.Dist.unique_id() if rank == 0 else bytes(128)
    t = torch.frombuffer(bytearray(uid), dtype=torch.uint8).clone()
    if device is not None:
        t = t.to(device)
    dist.broadcast(t, src=0)
    return capi.Dist(rank, world, bytes(t.cpu().numpy().tobytes()))


def reference_protocol_step(shard, x, x_next, aty, y_local, sigma, lc, uc, allreduce_sum):
    """What one attempt exchanges in the row-sharded scheme, in numpy (float64), for the CPU protocol tests.

    shard = (A_local as scipy.sparse.csr_matrix); vectors of length n are replicated, y / bounds are local rows.
    Returns (y_next_local, aty_next (global, identical on all ranks), interaction, ||dx||^2, ||dy||^2).
    One collective: the all-reduce of [A_g^T y'_g ; ||dy_g||^2]  (n + 1 doubles).
    """
    A = shard
    xbar = x_next - x + x_next
    ybar = y_local - sigma * (A @ xbar)
    y_next = np.maximum(ybar + sigma * lc, np.minimum(ybar + sigma * uc, 0.0))
    dy = y_next - y_local
    buf = np.concatenate([A.T @ y_next, [float(dy @ dy)]])
    buf = allreduce_sum(buf)
    aty_next, dy2 = buf[:-1], float(buf[-1])
    dx = x_next - x
    return y_next, aty_next, float(dx @ (aty_next - aty)), float(dx @ dx), dy2


def slice_bounds(n: int, world: int):
    """Column slices of the primal side in the sliced schemes: nslice = ceil(n / world) rounded up to 32 (the padded
    length world * nslice is what the all-gathers move); rank g owns [g * nslice, min(n, (g + 1) * nslice))."""
    nslice = (((n + world - 1) // world) + 31) & ~31
    return nslice, [(min(n, g * nslice), min(n, (g + 1) * nslice)) for g in range(world)]


def reference_protocol_step_sliced(shard, rank, world, x_slice, x_next_slice, aty_slice, y_local, sigma, lc, uc,
                                   allgather, reduce_scatter_sum, allgather_scalars):
    """One attempt of the column-sliced scheme (DESIGN.md §6, scheme (ii)) in numpy: this rank holds rows R_g of A and
    the slice J_g of x, x', A^T y.  Exchanges: xbar slices -> everyone; partial A_g^T y'_g -> slice owners (summed in
    RANK ORDER); three scalars per rank -> everyone (summed in rank order).
    Returns (y_next_local, aty_next_slice, interaction, ||dx||^2, ||dy||^2) with the scalars identical on all ranks."""
    A = shard
    n = A.shape[1]
    nslice, bounds = slice_bounds(n, world)
    j0, j1 = bounds[rank]
    xbar_slice = np.zeros(nslice)
    xbar_slice[: j1 - j0] = x_next_slice - x_slice + x_next_slice
    xbar = allgather(xbar_slice)[:n]                      # world * nslice doubles, pad dropped
    ybar = y_local - sigma * (A @ xbar)
    y_next = np.maximum(ybar + sigma * lc, np.minimum(ybar + sigma * uc, 0.0))
    dy = y_next - y_local
    partial = np.zeros(world * nslice)
    partial[:n] = A.T @ y_next
    aty_next_slice = reduce_scatter_sum(partial)[: j1 - j0]   # this rank's slice of the rank-ordered sum
    dx = x_next_slice - x_slice
    mine = np.array([float(dx @ (aty_next_slice - aty_slice)), float(dx @ dx), float(dy @ dy)])
    table = allgather_scalars(mine)                      # world x 3, rank order
    tot = np.zeros(3)
    for g in range(world):
        tot += table[g]
    return y_next, aty_next_slice, float(tot[0]), float(tot[1]), float(tot[2])


def slice_of_global_transpose(local_transposes, row_starts, j0, j1):
    """What the gather transport's setup builds on the device (k_slice_row_counts / k_slice_fill): rows [j0, j1) of the
    GLOBAL A^T from the transposes A_g^T (scipy csr, n x m_g) of the row blocks, concatenated per row in rank order with
    the column indices shifted to global constraint rows."""
    import scipy.sparse as sp
    m_total = int(row_starts[-1])
    blocks = [sp.csr_matrix(t[j0:j1]) for t in local_transposes]
    return sp.hstack(blocks, format="csr") if blocks else sp.csr_matrix((j1 - j0, m_total))


def reference_protocol_step_gather(shard, at_slice, rank, world, x_slice, x_next_slice, aty_slice, y_local, sigma, lc, uc,
                                   allgather_x, allgather_y, allgather_scalars):
    """One attempt of the gather transport (the default; DESIGN.md section 6) in numpy: this rank holds rows R_g of A, rows
    J_g of the global A^T (`at_slice`, n_g x m) and the slice J_g of x, x', A^T y.  Exchanges: xbar slices -> everyone,
    y' row blocks -> everyone (`allgather_y` returns the m global rows in rank order), three scalars per rank -> everyone
    (summed in rank order).  No partial products: A^T y' on the slice is a complete row sum."""
    A = shard
    n = A.shape[1]
    nslice, bounds = slice_bounds(n, world)
    j0, j1 = bounds[rank]
    xbar_slice = np.zeros(nslice)
    xbar_slice[: j1 - j0] = x_next_slice - x_slice + x_next_slice
    xbar = allgather_x(xbar_slice)[:n]
    ybar = y_local - sigma * (A @ xbar)
    y_next = np.maximum(ybar + sigma * lc, np.minimum(ybar + sigma * uc, 0.0))
    dy = y_next - y_local
    y_full = allgather_y(y_next)
    aty_next_slice = at_slice @ y_full
    dx = x_next_slice - x_slice
    mine = np.array([float(dx @ (aty_next_slice - aty_slice)), float(dx @ dx), float(dy @ dy)])
    table = allgather_scalars(mine)
    tot = np.zeros(3)
    for g in range(world):
        tot += table[g]
    return y_next, aty_next_slice, float(tot[0]), float(tot[1]), float(tot[2])


# ---- packed exchange of the gather transport (DESIGN.md section 6), restated in numpy for the CPU tests ---------------------------
def packed_layout(needed, starts, halves):
    """What packed_positions (pdlp_solver.cu) builds on the device: `needed` marks the entries of a distributed vector this
    rank reads, owner h holds entries [starts[h], starts[h + 1]) and its first half is the first halves[h] of them.  The needed
    entries of the first halves get slots 0, 1, ... in ascending order, those of the second halves W, W + 1, ...
    (W = the larger count rounded up to 32).  Returns (pos, W): pos[j] = slot of entry j, -1 if never read."""
    needed = np.asarray(needed, bool)
    idx = np.arange(len(needed))
    owner = np.searchsorted(np.asarray(starts)[1:], idx, side="right")
    owner = np.minimum(owner, len(halves) - 1)
    first = (idx - np.asarray(starts)[owner]) < np.asarray(halves)[owner]
    fa, fb = needed & first, needed & ~first
    W = (max(int(fa.sum()), int(fb.sum()), 1) + 31) & ~31
    pos = np.full(len(needed), -1, np.int64)
    pos[fa] = np.arange(int(fa.sum()))
    pos[fb] = W + np.arange(int(fb.sum()))
    return pos, W


def send_list(slots_at_destination, half):
    """Sender side (build_send_lists): from the destination's slots of MY entries (-1: not read) the ascending list of the
    entries to send and how many of them belong to my first half (they are sent, and flagged, first)."""
    lst = np.flatnonzero(np.asarray(slots_at_destination) >= 0)
    return lst, int(np.searchsorted(lst, half))
