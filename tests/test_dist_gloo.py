"""Host-side logic of the row-sharded (N > 1) path, on CPU with the gloo backend, world_size 2 and 3:
  * the row partition tiles the matrix and balances nnz,
  * the ONE collective an attempt needs (all-reduce of [A_g^T y'_g ; ||dy_g||^2]) reproduces the single-process
    quantities of the oracle's attempt (A^T y', interaction, movement terms),
  * every rank derives bit-identical scalars from the all-reduced buffer (=> identical accept/reject decisions).
  * the column-sliced scheme (all-gather of xbar slices, rank-ordered reduce-scatter of the partials, rank-ordered sum
    of three scalars per rank) reproduces the same attempt and the same bits on every rank,
  * the gather transport (rows of A and rows of the global A^T per rank, xbar and y' all-gathered, no partial products)
    reproduces the same attempt, and its slice of A^T assembled from the transposed row blocks equals the real one,
  * twenty accepted steps of the gather transport with the adaptive step-size rule on the rank-ordered scalars follow the
    oracle's own twenty steps (same accept / reject decisions on every rank, iterates to 1e-10),
  * the packed exchange (two halves, slot tables, send lists) delivers exactly what every rank reads,
  * the slice bounds tile [0, n) with 32-aligned slices.
Two of these protocols run in CUDA: the gather transport, and the column-sliced scheme as the nccl transport.
tests/test_gpu_dist.py exercises both on >= 2 GPUs; the one-all-reduce attempt is a CPU model only."""
import os
import socket

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from cuopt_b200 import dist as cdist
from cuopt_b200 import lpgen
from oracle import pdlp_oracle as po


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lp = lpgen.sparse_lp(3000, 2500, 6, seed=11)
        # the oracle provides a realistic scaled state after a few iterations (same on every rank: deterministic)
        o = po.Oracle(lp.offsets, lp.indices, lp.values, lp.c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub)
        o.run(9)
        x, y, aty = o.vector("x"), o.vector("y"), o.vector("aty")
        tau, sigma = o.scalar("tau"), o.scalar("sigma")
        want = o.single_attempt(x, y, aty, tau, sigma)
        dr, dc = o.vector("row_scaling"), o.vector("col_scaling")
        A = sp.csr_matrix((lp.values, lp.indices, lp.offsets), shape=(lp.m, lp.n))
        As = sp.diags(dr) @ A @ sp.diags(dc)
        lcs, ucs = o.vector("scaled_lc"), o.vector("scaled_uc")
        b = cdist.shard_bounds(lp.offsets, world)
        r0, r1 = int(b[rank]), int(b[rank + 1])

        def allreduce_sum(buf):
            t = torch.from_numpy(buf.copy())
            dist.all_reduce(t)
            return t.numpy()

        y_next, aty_next, inter, dx2, dy2 = cdist.reference_protocol_step(
            As[r0:r1].tocsr(), x, want["x_next"], aty, y[r0:r1], sigma, lcs[r0:r1], ucs[r0:r1], allreduce_sum)
        ok = (np.allclose(y_next, want["y_next"][r0:r1], rtol=1e-12, atol=1e-13)
              and np.allclose(aty_next, want["aty_next"], rtol=1e-11, atol=1e-12)
              and abs(dx2 - want["norm_dx2"]) <= 1e-11 * want["norm_dx2"]
              and abs(dy2 - want["norm_dy2"]) <= 1e-11 * want["norm_dy2"]
              and abs(inter - want["interaction"]) <= 1e-9 * max(abs(want["interaction"]), want["norm_dx2"]))
        # identical bits on every rank
        g = [torch.zeros(3, dtype=torch.float64) for _ in range(world)]
        dist.all_gather(g, torch.tensor([inter, dx2, dy2], dtype=torch.float64))
        same = all(torch.equal(g[0], t) for t in g)
        # column-sliced scheme (ii): all-gather of xbar slices, reduce-scatter of the partials in rank order,
        # three scalars per rank summed in rank order
        nslice, bounds = cdist.slice_bounds(lp.n, world)
        j0, j1 = bounds[rank]

        def allgather(buf):
            g = [torch.zeros(len(buf), dtype=torch.float64) for _ in range(world)]
            dist.all_gather(g, torch.from_numpy(buf.copy()))
            return torch.cat(g).numpy()

        def reduce_scatter_sum(buf):  # gloo has no reduce_scatter: gather every rank's piece for me, add in rank order
            full = [torch.zeros(world * nslice, dtype=torch.float64) for _ in range(world)]
            dist.all_gather(full, torch.from_numpy(buf.copy()))
            got = [f[rank * nslice:(rank + 1) * nslice] for f in full]
            out = torch.zeros(nslice, dtype=torch.float64)
            for g in range(world):
                out += got[g]
            return out.numpy()

        def allgather_scalars(v):
            g = [torch.zeros(3, dtype=torch.float64) for _ in range(world)]
            dist.all_gather(g, torch.from_numpy(v.copy()))
            return torch.stack(g).numpy()

        y2, aty2, inter2, dx22, dy22 = cdist.reference_protocol_step_sliced(
            As[r0:r1].tocsr(), rank, world, x[j0:j1], want["x_next"][j0:j1], aty[j0:j1], y[r0:r1], sigma, lcs[r0:r1],
            ucs[r0:r1], allgather, reduce_scatter_sum, allgather_scalars)
        ok2 = (np.allclose(y2, want["y_next"][r0:r1], rtol=1e-12, atol=1e-13)
               and np.allclose(aty2, want["aty_next"][j0:j1], rtol=1e-11, atol=1e-12)
               and abs(dx22 - want["norm_dx2"]) <= 1e-11 * want["norm_dx2"]
               and abs(dy22 - want["norm_dy2"]) <= 1e-11 * want["norm_dy2"]
               and abs(inter2 - want["interaction"]) <= 1e-9 * max(abs(want["interaction"]), want["norm_dx2"]))
        g2 = [torch.zeros(3, dtype=torch.float64) for _ in range(world)]
        dist.all_gather(g2, torch.tensor([inter2, dx22, dy22], dtype=torch.float64))
        same2 = all(torch.equal(g2[0], t) for t in g2)
        # gather transport (default): rows J_g of the global A^T assembled from the transposed row blocks, y' all-gathered
        def allgather_y(v):  # ragged row blocks: pad to the longest, drop the pads
            sizes = [int(b[g + 1] - b[g]) for g in range(world)]
            pad = np.zeros(max(sizes)); pad[: len(v)] = v
            g = [torch.zeros(max(sizes), dtype=torch.float64) for _ in range(world)]
            dist.all_gather(g, torch.from_numpy(pad))
            return np.concatenate([g[k].numpy()[: sizes[k]] for k in range(world)])

        transposes = [As[int(b[g]):int(b[g + 1])].T.tocsr() for g in range(world)]  # what every rank holds: its own A_g^T
        at_slice = cdist.slice_of_global_transpose(transposes, b, j0, j1)
        assert (at_slice != As.T.tocsr()[j0:j1]).nnz == 0
        y3, aty3, inter3, dx23, dy23 = cdist.reference_protocol_step_gather(
            As[r0:r1].tocsr(), at_slice, rank, world, x[j0:j1], want["x_next"][j0:j1], aty[j0:j1], y[r0:r1], sigma,
            lcs[r0:r1], ucs[r0:r1], allgather, allgather_y, allgather_scalars)
        ok3 = (np.allclose(y3, want["y_next"][r0:r1], rtol=1e-12, atol=1e-13)
               and np.allclose(aty3, want["aty_next"][j0:j1], rtol=1e-11, atol=1e-12)
               and abs(dx23 - want["norm_dx2"]) <= 1e-11 * want["norm_dx2"]
               and abs(dy23 - want["norm_dy2"]) <= 1e-11 * want["norm_dy2"]
               and abs(inter3 - want["interaction"]) <= 1e-9 * max(abs(want["interaction"]), want["norm_dx2"]))
        g3 = [torch.zeros(3, dtype=torch.float64) for _ in range(world)]
        dist.all_gather(g3, torch.tensor([inter3, dx23, dy23], dtype=torch.float64))
        same3 = all(torch.equal(g3[0], t) for t in g3)
        q.put((rank, bool(ok and ok2 and ok3), bool(same and same2 and same3), r0, r1))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_attempt_protocol_matches_single_process(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(60)
    assert all(r[1] for r in res), res
    assert all(r[2] for r in res), res
    # the shards tile [0, m)
    assert res[0][3] == 0 and res[-1][4] == 3000 and all(res[i][4] == res[i + 1][3] for i in range(world - 1))


def test_shard_bounds_balance_and_edge_cases():
    lp = lpgen.sparse_lp(10_000, 8_000, 8, seed=3)
    for world in (1, 2, 4, 8):
        b = cdist.shard_bounds(lp.offsets, world)
        assert b[0] == 0 and b[-1] == lp.m and np.all(np.diff(b) >= 0)
        nnz = np.diff(lp.offsets[b])
        assert nnz.max() <= 1.05 * lp.nnz / world + 8
    # ragged: one dense row and many empty ones
    off = np.array([0, 0, 0, 1000, 1000, 1001, 1001], np.int32)
    b = cdist.shard_bounds(off, 3)
    assert b[0] == 0 and b[-1] == 6 and np.all(np.diff(b) >= 0)
    # more ranks than rows: some shards are empty
    b = cdist.shard_bounds(np.array([0, 3, 5], np.int32), 4)
    assert b[0] == 0 and b[-1] == 2 and np.all(np.diff(b) >= 0)


def test_shards_reassemble_the_matrix():
    lp = lpgen.sparse_lp(5000, 4000, 5, seed=9)
    rows = []
    for r in range(4):
        r0, r1, off, idx, val, clb, cub = cdist.shard_rows(lp, r, 4)
        rows.append(sp.csr_matrix((val, idx, off), shape=(r1 - r0, lp.n)))
        assert np.array_equal(clb, lp.con_lb[r0:r1]) and np.array_equal(cub, lp.con_ub[r0:r1])
    A = sp.csr_matrix((lp.values, lp.indices, lp.offsets), shape=(lp.m, lp.n))
    assert (sp.vstack(rows) != A).nnz == 0


def test_slice_bounds_tile_the_columns():
    for n, world in [(1000, 2), (1000, 3), (31, 4), (10_000_000, 8), (64, 8), (5, 8)]:
        nslice, b = cdist.slice_bounds(n, world)
        assert nslice % 32 == 0 and nslice * world >= n
        assert b[0][0] == 0 and b[-1][1] == n
        assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
        assert all(0 <= hi - lo <= nslice for lo, hi in b)


def _packed_worker(rank, world, port, q):
    """The packed exchange end to end with gloo as the wire: every rank marks the columns its rows of A touch, numbers them in
    two halves, learns from every peer where its own entries live in the peer's packed buffer, sends first halves then second
    halves — and its renumbered matrix times the packed buffer must equal A_g times the full vector."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lp = lpgen.sparse_lp(3000, 2500, 2, seed=5)  # 2 entries per row: a rank reads well under all of the columns
        A = sp.csr_matrix((lp.values, lp.indices, lp.offsets), shape=(lp.m, lp.n))
        b = cdist.shard_bounds(lp.offsets, world)
        Ag = A[int(b[rank]):int(b[rank + 1])].tocsr()
        nslice, bounds = cdist.slice_bounds(lp.n, world)
        n_pad = nslice * world
        starts = np.arange(world + 1) * nslice
        halves = np.full(world, nslice // 2)
        needed = np.zeros(n_pad, bool)
        needed[Ag.indices] = True
        pos, W = cdist.packed_layout(needed, starts, halves)
        assert 0.2 < needed[:lp.n].mean() < 0.95  # the packing has something to skip
        # every rank learns every peer's slot table
        tables = [torch.zeros(n_pad, dtype=torch.int64) for _ in range(world)]
        dist.all_gather(tables, torch.from_numpy(pos))
        widths = [torch.zeros(1, dtype=torch.int64) for _ in range(world)]
        dist.all_gather(widths, torch.tensor([W]))
        j0 = rank * nslice
        rng = np.random.default_rng(100)
        x_full = rng.standard_normal(n_pad)  # same on every rank; rank h "produces" x_full[h * nslice:(h + 1) * nslice]
        x_mine = x_full[j0:j0 + nslice]
        # what I send to destination r: (slots, values), first-half entries first
        outgoing = []
        for r in range(world):
            slots = tables[r].numpy()[j0:j0 + nslice]
            lst, count_a = cdist.send_list(slots, nslice // 2)
            assert np.all(np.diff(slots[lst][:count_a]) == 1) and np.all(np.diff(slots[lst][count_a:]) == 1)  # consecutive per half
            assert np.all(slots[lst][:count_a] < int(widths[r])) and np.all(slots[lst][count_a:] >= int(widths[r]))
            outgoing.append((slots[lst], x_mine[lst], count_a))
        # the wire: gather everybody's messages for me (gloo: all_gather of padded arrays)
        buf = np.full(2 * W, np.nan)
        for src in range(world):
            for dst in range(world):
                sl, va, _ = outgoing[dst] if src == rank else (np.zeros(0, np.int64), np.zeros(0), 0)
                n_msg = torch.tensor([len(sl)])
                dist.broadcast(n_msg, src=src)
                t_sl = torch.from_numpy(sl.astype(np.int64)) if src == rank else torch.zeros(int(n_msg), dtype=torch.int64)
                t_va = torch.from_numpy(va.copy()) if src == rank else torch.zeros(int(n_msg), dtype=torch.float64)
                dist.broadcast(t_sl, src=src)
                dist.broadcast(t_va, src=src)
                if dst == rank:
                    buf[t_sl.numpy()] = t_va.numpy()
        remapped = sp.csr_matrix((Ag.data, pos[Ag.indices], Ag.indptr), shape=(Ag.shape[0], 2 * W))
        assert not np.isnan(buf[pos[needed]]).any()
        ok = np.allclose(remapped @ np.nan_to_num(buf), Ag @ x_full[:lp.n], rtol=1e-13, atol=1e-13)
        # block 0 of the column split (slots < W) touches first halves only
        first_half_cols = (np.arange(n_pad) % nslice) < nslice // 2
        ok = ok and bool(np.all(first_half_cols[np.flatnonzero(needed)][pos[needed] < W]))
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_packed_exchange_delivers_what_each_rank_reads(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_packed_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(60)
    assert all(r[1] for r in res), res


def _trajectory_worker(rank, world, port, q):
    """20 accepted PDHG steps of the gather transport (numpy + gloo), with the adaptive step-size rule evaluated on the three
    rank-ordered scalars, against the oracle's own 20 steps from the same state: same accept / reject decisions, same
    iterates.  Started after 12 iterations (the every-iteration major iterations of k <= 10 are over, the next one is at 40)."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lp = lpgen.sparse_lp(3000, 2500, 6, seed=11)
        o = po.Oracle(lp.offsets, lp.indices, lp.values, lp.c, lp.var_lb, lp.var_ub, lp.con_lb, lp.con_ub)
        o.run(12)
        x, y, aty = o.vector("x"), o.vector("y"), o.vector("aty")
        eta, w, kp = o.scalar("step_size"), o.scalar("primal_weight"), int(o.scalar("k_pdhg"))
        dr, dc = o.vector("row_scaling"), o.vector("col_scaling")
        A = sp.csr_matrix((lp.values, lp.indices, lp.offsets), shape=(lp.m, lp.n))
        As = (sp.diags(dr) @ A @ sp.diags(dc)).tocsr()
        cs, ls, us = o.vector("scaled_c"), o.vector("scaled_l"), o.vector("scaled_u")
        lcs, ucs = o.vector("scaled_lc"), o.vector("scaled_uc")
        b = cdist.shard_bounds(lp.offsets, world)
        r0, r1 = int(b[rank]), int(b[rank + 1])
        nslice, bounds = cdist.slice_bounds(lp.n, world)
        j0, j1 = bounds[rank]
        Ag = As[r0:r1].tocsr()
        at_slice = As.T.tocsr()[j0:j1]

        def allgather(buf):
            g = [torch.zeros(len(buf), dtype=torch.float64) for _ in range(world)]
            dist.all_gather(g, torch.from_numpy(buf.copy()))
            return torch.cat(g).numpy()

        def allgather_y(v):
            sizes = [int(b[g + 1] - b[g]) for g in range(world)]
            pad = np.zeros(max(sizes)); pad[: len(v)] = v
            g = [torch.zeros(max(sizes), dtype=torch.float64) for _ in range(world)]
            dist.all_gather(g, torch.from_numpy(pad))
            return np.concatenate([g[k].numpy()[: sizes[k]] for k in range(world)])

        def allgather_scalars(v):
            g = [torch.zeros(3, dtype=torch.float64) for _ in range(world)]
            dist.all_gather(g, torch.from_numpy(v.copy()))
            return torch.stack(g).numpy()

        xs, ys, ats = x[j0:j1].copy(), y[r0:r1].copy(), aty[j0:j1].copy()
        accepted = attempts = 0
        while accepted < 20 and attempts < 200:
            attempts += 1
            tau, sigma = eta / w, eta * w
            xn = np.maximum(np.minimum(xs - tau * (cs[j0:j1] - ats), us[j0:j1]), ls[j0:j1])
            yn, atn, inter, dx2, dy2 = cdist.reference_protocol_step_gather(
                Ag, at_slice, rank, world, xs, xn, ats, ys, sigma, lcs[r0:r1], ucs[r0:r1], allgather, allgather_y,
                allgather_scalars)
            # adaptive_step_size_strategy.cu:92-188 (pdhg_step_rule in pdlp_kernels.cuh), on the rank-ordered sums
            movement = 0.5 * w * dx2 + (0.5 / w) * dy2
            assert 0.0 < movement < 1e100
            kp += 1
            limit = movement / abs(inter) if inter != 0.0 else np.inf
            accept = eta <= limit
            eta = min((1.0 - (kp + 1.0) ** -0.3) * limit, (1.0 + (kp + 1.0) ** -0.6) * eta)
            if accept:
                xs, ys, ats = xn, yn, atn
                accepted += 1
        o.run(20)
        ox, oy = o.vector("x"), o.vector("y")
        ok = (accepted == 20 and kp == int(o.scalar("k_pdhg"))
              and np.allclose(xs, ox[j0:j1], rtol=1e-10, atol=1e-11) and np.allclose(ys, oy[r0:r1], rtol=1e-10, atol=1e-11)
              and abs(eta - o.scalar("step_size")) <= 1e-10 * eta)
        q.put((rank, bool(ok), attempts))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gather_transport_follows_the_oracle_over_twenty_steps(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_trajectory_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(60)
    assert all(r[1] for r in res), res
    assert len({r[2] for r in res}) == 1  # every rank took the same number of attempts (identical accept / reject decisions)
