#!/usr/bin/env python
"""In-situ timing of the three PDHG kernels (groups) under environment-selected variants, on ONE generated workload.
Each variant builds a fresh solver session (the switches are read when the solver is built), warms it with real PDLP
iterations and calls cuOptB200SolverProfileKernels (CUDA events on the solver stream).  One JSON line per variant.

  python scripts/exp_kernel_variants.py c4 "CUOPT_B200_L2_WARM=1" "CUOPT_B200_L2_WARM=1,CUOPT_B200_GATHER_BLOCK_BYTES=0" ...
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cuopt_b200 import capi, lpgen  # noqa: E402

SIZES = {"c4": 10_000_000, "c2": 1_000_000}


def main():
    wl = sys.argv[1]
    variants = sys.argv[2:] or [""]
    t0 = time.time()
    n = SIZES[wl]
    lp = lpgen.sparse_lp(n, n, 8, seed=1234)
    print(f"# generated {lp.name} in {time.time() - t0:.1f} s", flush=True)
    p = capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)
    b_iter = lp.algorithmic_bytes_per_iteration()
    touched = set()
    for v in variants:
        for k in touched:
            os.environ.pop(k, None)
        env = dict(kv.split("=", 1) for kv in v.split(",") if kv)
        os.environ.update(env)
        touched |= set(env)
        s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False)
        s.set("optimality_tolerance", 0.0)
        t1 = time.time()
        g = capi.Solver(p, s)
        g.initialise()
        t_setup = time.time() - t1
        reps = 30 if wl == "c4" else 200
        k = g.profile_kernels(warmup_steps=120, reps=reps)
        out = {"workload": wl, "variant": v or "default", "us_k1": 1e3 * k.ms_primal_step, "us_k2": 1e3 * k.ms_dual_step,
               "us_k3": 1e3 * k.ms_transpose_step, "us_attempt_in_batch": 1e3 * k.ms_iteration,
               "blocks": [k.blocks_dual, k.blocks_transpose], "setup_s": round(t_setup, 2),
               "roofline_frac_attempt": b_iter / (k.ms_iteration * 1e-3) / 3350e9}  # H100 SXM data sheet
        print(json.dumps(out), flush=True)
        g.close()


if __name__ == "__main__":
    main()
