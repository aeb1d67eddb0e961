#!/usr/bin/env python
"""A/B of the compact column blocks (CUOPT_B200_COMPACT_BLOCKS) on the bench LP, in one process on one card.

Rounds alternate the plain form (0) and the compact form (3); after them each item runs alone (1 three-byte
indices, 2 non-empty-row masks).  Each run is `--solves` solves of `--iters` iterations
(optimality tolerance 0, so every solve runs all of them) after one warm-up solve; `value` is iterations over the
device seconds of the PDHG loop and the evaluations, as bench.py reports it, and K1 / K2 / K3 come from profile_kernels.
The primal and dual of the last solve of every run are compared bit for bit with those of the plain form.  The card's
name, power limit and clocks are read in the same call, right after the timed solves of every run.
   python scripts/compact_blocks_ab.py [--rounds 3] [--out profiles/h100/compact_blocks_ab_c4.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cuopt_b200 import capi, lpgen  # noqa: E402

ENV = "CUOPT_B200_COMPACT_BLOCKS"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        return {"name": "unknown"}
    name, power, sm, sm_max = [t.strip() for t in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit_w": float(power), "clocks_sm_mhz": float(sm), "clocks_max_sm_mhz": float(sm_max)}


def run(lp, form, solves, iters, reps):
    os.environ[ENV] = str(form)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, iteration_limit=iters)
    s.set("optimality_tolerance", 0.0)
    p = capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)
    its = 0
    dev_s = 0.0
    out = None
    for i in range(solves + 1):
        sol = capi.solve(p, s)
        if sol.return_code != 0:
            raise RuntimeError(sol.error_string)
        st = sol.stats()
        if i > 0:  # the first solve warms up
            its += st.number_of_steps_taken
            dev_s += st.pdhg_loop_seconds + st.termination_seconds
        out = (sol.primal(), sol.dual())
    gpu = card()  # right after the timed solves, while the clocks are those of the load
    g = capi.Solver(p, s)
    prof = g.profile_kernels(120, reps)
    form_a, form_at = g.scalar("blocks_form_a"), g.scalar("blocks_form_at")
    g.close()
    return {"value": its / dev_s, "iterations": its, "device_seconds": dev_s, "blocks_form_a": int(form_a),
            "blocks_form_at": int(form_at), "blocks_dual": prof.blocks_dual, "blocks_transpose": prof.blocks_transpose,
            "ms_k1": prof.ms_primal_step, "ms_k2": prof.ms_dual_step, "ms_k3": prof.ms_transpose_step,
            "ms_attempt_in_batch": prof.ms_iteration, "gpu": gpu}, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--solves", type=int, default=2)
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--items", default="1,2")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "compact_blocks_ab_c4.jsonl"))
    a = ap.parse_args()
    lp = lpgen.sparse_lp(a.rows, a.rows, 8, seed=1234)
    workload = f"sparse_lp(m={a.rows},n={a.rows},k=8,seed=1234), fp64, {a.iters} iterations per solve"
    plan = [(r + 1, f) for r in range(a.rounds) for f in (0, 3)] + [(0, int(f)) for f in a.items.split(",") if f]
    ref = None
    with open(a.out, "w") as f:
        for rnd, form in plan:
            rec, (x, y) = run(lp, form, a.solves, a.iters, a.reps)
            if ref is None:
                ref = (x, y)  # plan[0] is the plain form
            rec.update({"round": rnd, "compact_blocks": form, "workload": workload,
                        "bit_identical_to_plain": bool(np.array_equal(x.view(np.uint64), ref[0].view(np.uint64))
                                                       and np.array_equal(y.view(np.uint64), ref[1].view(np.uint64)))})
            line = json.dumps(rec)
            print(line, flush=True)
            f.write(line + "\n")
    os.environ.pop(ENV, None)


if __name__ == "__main__":
    main()
