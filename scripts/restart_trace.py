"""Major-iteration trace of the bench LP (configs[3], bench.py's workload and settings): where two builds' trajectories part.

    python scripts/restart_trace.py run [--iters 2000] > build_a.jsonl      # one line per sampled major iteration
    python scripts/restart_trace.py compare build_a.jsonl build_b.jsonl

`run` steps one solve major iteration by major iteration (k <= 10, then every 40th) and records the restart count, whether
the last restart went to the average, the KKT scores the restart test compared, step size, primal weight and a fixed
sample of the current x and y.  `compare` prints, per sample, the relative differences between two traces and whether
their x / y samples are bit-identical, so the first step at which two builds differ, and the first restart decision they
take differently, can be read off."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SCALARS = ("n_restarts", "last_restart_was_average", "last_candidate_kkt", "last_restart_kkt", "step_size",
           "primal_weight")


def run(args):
    from cuopt_b200 import capi, lpgen
    lp = lpgen.sparse_lp(10_000_000, 10_000_000, 8, seed=1234, locality=0.0)  # bench.py --workload c4
    p = capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, iteration_limit=args.iters)
    s.set("optimality_tolerance", 0.0)
    g = capi.Solver(p, s)
    g.initialise()
    k = 0
    while k < args.iters:
        if g.advance(1 if k < 10 else 40 - k % 40):
            break
        k = int(g.scalar("k_total"))
        rec = {"k": k, **{name: g.scalar(name) for name in SCALARS}}
        for name in ("x", "y"):
            rec[name] = g.vector(name)[::9973][:1024].tolist()
        print(json.dumps(rec), flush=True)


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b)) / max(1e-300, float(np.max(np.abs(a)))))


def compare(args):
    A = [json.loads(l) for l in open(args.a)]
    B = [json.loads(l) for l in open(args.b)]
    print("k restarts(a,b) to_avg(a,b) | rel diff: cand_kkt restart_kkt step weight x y | x,y bit-identical")
    for a, b in zip(A, B):
        same = np.array_equal(a["x"], b["x"]) and np.array_equal(a["y"], b["y"])
        print(f"{a['k']:5d} {a['n_restarts']:3.0f},{b['n_restarts']:3.0f} {a['last_restart_was_average']},"
              f"{b['last_restart_was_average']} | {rel(a['last_candidate_kkt'], b['last_candidate_kkt']):.1e} "
              f"{rel(a['last_restart_kkt'], b['last_restart_kkt']):.1e} {rel(a['step_size'], b['step_size']):.1e} "
              f"{rel(a['primal_weight'], b['primal_weight']):.1e} {rel(a['x'], b['x']):.1e} {rel(a['y'], b['y']):.1e} | "
              f"{same}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("run")
    r.add_argument("--iters", type=int, default=2000)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    run(args) if args.cmd == "run" else compare(args)
