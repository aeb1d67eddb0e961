"""Row-sharded multi-GPU solve (cuOptB200SolveDistributed) against the single-GPU solve of the same LP.
Needs >= 2 GPUs; skipped otherwise."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q, size, extra_cols, tol, mode, transport, block_bytes, iteration_limit=0, nnz_per_row=8):
    import torch
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      CUOPT_B200_DIST_MODE=transport.split("-")[0])
    if "-nopack" in transport:  # gather transport with identity packing: every entry of xbar / y' travels
        os.environ["CUOPT_B200_DIST_PACK"] = "0"
    if "-kernel" in transport:  # gather transport with k_send_packed on the communication stream instead of the fused peer stores
        os.environ["CUOPT_B200_DIST_SEND"] = "kernel"
    if block_bytes:
        os.environ["CUOPT_B200_GATHER_BLOCK_BYTES"] = str(block_bytes)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from cuopt_b200 import capi, lpgen
        from cuopt_b200 import dist as cdist
        lp = lpgen.sparse_lp(size, size + extra_cols, nnz_per_row, seed=21)
        comm = cdist.bootstrap(rank, world, device=torch.device("cuda", rank))
        p, (r0, r1) = cdist.local_problem(lp, rank, world)
        s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=mode)
        if iteration_limit:
            s.set("iteration_limit", iteration_limit)
        s.set("optimality_tolerance", tol)
        sol = capi.solve_distributed(p, s, comm)
        out = dict(rank=rank, rc=sol.return_code, err=sol.error_string)
        if sol.return_code == 0:
            st = sol.stats()
            out.update(status=sol.termination_status, its=st.number_of_steps_taken, obj=st.primal_objective,
                       dobj=st.dual_objective, x=sol.primal(), y=sol.dual(), rows=(r0, r1), rp=st.l2_primal_residual)
        q.put(out)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _solve_on_gpus(world, size, tol, mode, transport, extra_cols=0, block_bytes=0, iteration_limit=0, nnz_per_row=8,
                   expect_ok=True):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, size, extra_cols, tol, mode, transport, block_bytes,
                                               iteration_limit, nnz_per_row))
             for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = sorted((q.get(timeout=300) for _ in range(world)), key=lambda d: d["rank"])
        for p in procs:
            p.join(60)
    finally:
        for p in procs:  # a rank that trapped or hung must not outlive the test
            if p.is_alive():
                p.kill()
    if not expect_ok:
        return res
    for r in res:
        assert r["rc"] == 0, r["err"]
    # every rank reports the same status / iteration count / objectives / primal vector (identical decisions everywhere)
    for r in res[1:]:
        assert r["status"] == res[0]["status"] and r["its"] == res[0]["its"]
        assert r["obj"] == res[0]["obj"] and r["dobj"] == res[0]["dobj"]
        assert np.array_equal(r["x"], res[0]["x"])
    return res


def _single_gpu(size, tol, mode, iteration_limit=0, nnz_per_row=8, extra_cols=0):
    from cuopt_b200 import capi, lpgen
    lp = lpgen.sparse_lp(size, size + extra_cols, nnz_per_row, seed=21)
    p = capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, pdlp_solver_mode=mode)
    s.set("optimality_tolerance", tol)
    if iteration_limit:
        s.set("iteration_limit", iteration_limit)
    one = capi.solve(p, s)
    assert one.termination_status == (4 if iteration_limit else 1)
    return lp, one


@pytest.mark.parametrize("transport,nnz_per_row", [("gather", 8), ("gather", 2), ("gather-nopack", 2), ("gather-kernel", 8), ("gather-kernel", 2), ("nccl", 8), ("nccl", 2)])
def test_sharded_iterates_track_the_single_gpu_iterates(transport, nnz_per_row):
    """The strongest check of a transport: after the SAME number of iterations (no tolerance involved) the sharded solve holds
    the iterate the single GPU holds, element-wise, up to the summation order of the row sums (block cuts of the row blocks
    differ from those of the whole matrix; nccl also adds the partial A_g^T y' over the ranks).  A stale or torn xbar / y'
    exchange shows up here as an O(1) difference.  The 2-per-row LP makes every rank need only part of the other ranks' slices."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    size, its = 40_000, 120  # crosses the every-iteration major iterations (k <= 10) and the ones at 40, 80, 120
    res = _solve_on_gpus(2, size, 0.0, 1, transport, extra_cols=37, iteration_limit=its, nnz_per_row=nnz_per_row)
    lp, one = _single_gpu(size, 0.0, 1, iteration_limit=its, nnz_per_row=nnz_per_row, extra_cols=37)
    assert res[0]["its"] == one.stats().number_of_steps_taken == its
    x1, y1 = one.primal(), one.dual()
    y = np.concatenate([r["y"] for r in res])
    # fp64 tolerance: 1e-7 of the largest entry after 120 iterations and their restarts (rounding differences of the
    # row sums, amplified by the iteration; DESIGN.md section 3 uses the same bound
    # for 120-iteration trajectories against the oracle)
    scale_x, scale_y = np.abs(x1).max(), np.abs(y1).max()
    assert np.abs(res[0]["x"] - x1).max() <= 1e-7 * scale_x
    assert np.abs(y - y1).max() <= 1e-7 * scale_y
    assert res[0]["obj"] == pytest.approx(one.stats().primal_objective, rel=1e-7, abs=1e-7)


# transport of the sharded attempt: gather = every rank owns rows of A AND rows of the global A^T, both products take inputs
# all-gathered by NVLink peer stores of the producing kernels (default; -kernel: k_send_packed, -nopack: every entry
# travels); nccl = all-gather + reduce-scatter
@pytest.mark.parametrize("mode,transport", [(1, "gather"), (1, "gather-kernel"), (1, "gather-nopack"), (1, "nccl"), (3, "gather"),
                                            (3, "nccl")])
def test_two_gpu_solve_matches_single_gpu(mode, transport):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    size, tol, world = 40_000, 1e-6, 2
    res = _solve_on_gpus(world, size, tol, mode, transport)
    lp, one = _single_gpu(size, tol, mode)
    st1 = one.stats()
    assert res[0]["status"] == 1
    # agrees with the single-GPU run: objective to 1e-5 (planted optimum known; both stop at tolerance 1e-6),
    # the iteration count only loosely: partial sums are added in a different order, and at 1e-6 on this degenerate LP
    # the restart decisions amplify last-bit differences (scripts/dist_iteration_table.py tabulates the counts)
    assert res[0]["obj"] == pytest.approx(lp.optimal_objective, rel=1e-5)
    assert res[0]["obj"] == pytest.approx(st1.primal_objective, rel=1e-5)
    assert res[0]["dobj"] == pytest.approx(st1.dual_objective, rel=1e-5)
    # (the iterates track the single-GPU ones through the first 120 iterations, test_sharded_iterates_track_the_single_gpu_iterates,
    # and then part ways at a restart decision, so the count is only banded)
    assert 0.4 * st1.number_of_steps_taken <= res[0]["its"] <= 2.5 * st1.number_of_steps_taken
    # the dual blocks tile the dual vector.  The vectors themselves are NOT compared with the single-GPU ones: the
    # planted LP is degenerate (half of x* sits on its bound), its optimal dual face is not a point, and two
    # tolerance-1e-6 runs can land on it far apart in norm while agreeing on both objectives to 1e-5.
    y = np.concatenate([r["y"] for r in res])
    assert y.shape[0] == lp.m
    assert res[0]["rp"] <= 1e-6 * (1.0 + np.linalg.norm(np.where(np.isfinite(lp.con_ub), lp.con_ub, lp.con_lb))) * 10


@pytest.mark.parametrize("world", [4, 8])
def test_four_and_eight_gpu_solve_matches_single_gpu(world):
    """The same comparison on 4 and 8 ranks (both transports; slices of 1/4 and 1/8 of the columns): needs 4 / 8 GPUs,
    skipped on smaller machines."""
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    size, tol = 40_000, 1e-6
    lp, one = _single_gpu(size, tol, 1)
    st1 = one.stats()
    for transport in ("gather", "nccl"):
        res = _solve_on_gpus(world, size, tol, 1, transport)
        assert res[0]["status"] == 1
        assert res[0]["obj"] == pytest.approx(lp.optimal_objective, rel=1e-5)
        assert res[0]["obj"] == pytest.approx(st1.primal_objective, rel=1e-5)
        assert res[0]["dobj"] == pytest.approx(st1.dual_objective, rel=1e-5)
        assert 0.4 * st1.number_of_steps_taken <= res[0]["its"] <= 2.5 * st1.number_of_steps_taken
        y = np.concatenate([r["y"] for r in res])
        assert y.shape[0] == lp.m and all(r["rows"][1] - r["rows"][0] == len(r["y"]) for r in res)


@pytest.mark.parametrize("world", [4, 8])
def test_many_gpu_iterates_track_the_single_gpu_iterates(world):
    """The element-wise check on 4 and 8 ranks: at 40 000 x 40 037 with 8 entries per row a rank's rows touch 86 % (4 ranks) /
    63 % (8 ranks) of the columns, so the packed exchange sends different subsets of every slice to every rank."""
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    size, its = 40_000, 120
    res = _solve_on_gpus(world, size, 0.0, 1, "gather", extra_cols=37, iteration_limit=its)
    lp, one = _single_gpu(size, 0.0, 1, iteration_limit=its, extra_cols=37)
    assert res[0]["its"] == one.stats().number_of_steps_taken == its
    x1, y1 = one.primal(), one.dual()
    y = np.concatenate([r["y"] for r in res])
    assert np.abs(res[0]["x"] - x1).max() <= 1e-7 * np.abs(x1).max()
    assert np.abs(y - y1).max() <= 1e-7 * np.abs(y1).max()
    assert res[0]["obj"] == pytest.approx(one.stats().primal_objective, rel=1e-7, abs=1e-7)


def test_nccl_transport_is_deterministic_with_ragged_slices():
    """The NCCL transport reproduces itself bit for bit, also when the last column slice is shorter than the 32-aligned
    slice width."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    size, tol, world = 40_000, 1e-6, 2
    ragged = 37  # n = 40037: the last slice is shorter than the 32-aligned slice width
    a = _solve_on_gpus(world, size, tol, 1, "nccl", ragged)
    b = _solve_on_gpus(world, size, tol, 1, "nccl", ragged)
    assert a[0]["status"] == 1
    assert b[0]["its"] == a[0]["its"] and b[0]["obj"] == a[0]["obj"] and b[0]["dobj"] == a[0]["dobj"]
    assert np.array_equal(b[0]["x"], a[0]["x"])
    assert all(np.array_equal(b[r]["y"], a[r]["y"]) for r in range(world))


def test_gather_transport_is_deterministic_with_ragged_slices():
    """The default transport reproduces itself bit for bit (no race between the peer stores of xbar / y', the flags and the
    consuming kernels), also when the last column slice is shorter than the 32-aligned slice width."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    size, tol, world = 40_000, 1e-6, 2
    a = _solve_on_gpus(world, size, tol, 1, "gather", 37)
    b = _solve_on_gpus(world, size, tol, 1, "gather", 37)
    assert a[0]["status"] == 1
    assert b[0]["its"] == a[0]["its"] and b[0]["obj"] == a[0]["obj"] and b[0]["dobj"] == a[0]["dobj"]
    assert np.array_equal(b[0]["x"], a[0]["x"])
    assert all(np.array_equal(b[r]["y"], a[r]["y"]) for r in range(world))


@pytest.mark.parametrize("transport", ["gather", "gather-nopack", "nccl"])
def test_two_gpu_solve_with_gather_blocking(transport):
    """The large-LP kernels (column-blocked passes + element-wise epilogues / scatter) inside the sharded attempt:
    forced on a small LP (4 blocks for A_g, 2 for A_g^T), they must reach the same optimum as the fused kernels."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    size, tol, world = 40_000, 1e-4, 2
    fused = _solve_on_gpus(world, size, tol, 1, transport)
    blocked = _solve_on_gpus(world, size, tol, 1, transport, block_bytes=100_000)
    assert fused[0]["status"] == blocked[0]["status"] == 1
    assert abs(blocked[0]["its"] - fused[0]["its"]) <= max(40, 0.4 * fused[0]["its"])
    assert blocked[0]["obj"] == pytest.approx(fused[0]["obj"], rel=1e-3)  # both are tolerance-1e-4 points
    lp, one = _single_gpu(size, tol, 1)
    assert blocked[0]["obj"] == pytest.approx(lp.optimal_objective, rel=1e-3)


def test_unknown_transport_is_rejected_on_every_rank():
    """A transport name other than gather or nccl (here "p2p") is an invalid argument on every rank.  Each rank raises it
    while it builds the solver, before the first collective, so no rank is left waiting for the others."""
    import torch
    from cuopt_b200 import capi
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    res = _solve_on_gpus(2, 4_000, 1e-4, 1, "p2p", expect_ok=False)
    assert len(res) == 2
    for r in res:
        assert r["rc"] == capi.CUOPT_INVALID_ARGUMENT
        assert "gather" in r["err"] and "nccl" in r["err"]
