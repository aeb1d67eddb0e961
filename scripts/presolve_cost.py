#!/usr/bin/env python
"""What the opt-in presolve costs and what it changes (one GPU, one call):
  * configs[3] (the 10M x 10M LP of bench.py, 8 nnz/row): setup_seconds with presolve off and on (alternated, `--reps`
    each), presolve and postsolve device time, what presolve removed;
  * iterations to optimality_tolerance 1e-8 with and without presolve on afiro and the sudoku relaxation.
The card's name and power limit are read in the same run.  No threshold is asserted.
   python scripts/presolve_cost.py [--rows N] [--reps 2] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from cuopt_b200 import capi, lpgen  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(problem, presolve, **params):
    s = capi.Settings(method=capi.CUOPT_METHOD_PDLP, log_to_console=False, presolve=presolve)
    for k, v in params.items():
        s.set(k, v)
    sol = capi.solve(problem, s)
    if sol.return_code != 0:
        raise RuntimeError(sol.error_string)
    st, ps = sol.stats(), sol.presolve_stats()
    return dict(status=sol.termination_reason, iterations=st.number_of_steps_taken, objective=st.primal_objective,
                setup_seconds=st.setup_seconds, solve_time=st.solve_time, presolve_seconds=ps.presolve_seconds,
                postsolve_seconds=ps.postsolve_seconds, reduced=[ps.reduced_m, ps.reduced_n, ps.reduced_nnz],
                removed=dict(fixed_columns=ps.fixed_columns, empty_rows=ps.empty_rows,
                             singleton_rows=ps.singleton_rows, empty_columns=ps.empty_columns), rounds=ps.rounds)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON record to this file")
    a = ap.parse_args()
    out = dict(card=card())
    lp = lpgen.sparse_lp(a.rows, a.rows, 8, seed=1234)
    p = capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)
    big = {"off": [], "on": []}
    run(p, False, iteration_limit=1)  # warm-up: module load, staging ring, device block cache
    for _ in range(a.reps):
        for key, on in (("off", False), ("on", True)):
            big[key].append(run(p, on, iteration_limit=10))
    out["configs[3]"] = dict(rows=a.rows, nnz=int(lp.nnz), **big)
    del p, lp
    from conftest import mps_path, problem_arrays  # noqa: E402
    small = {}
    for name, rel in (("afiro", "linear_programming/afiro_original.mps"), ("sudoku relaxation", "mip/sudoku.mps")):
        d = problem_arrays(capi.Problem.read(mps_path(rel)))
        q = capi.Problem.create_ranged(d["offsets"], d["indices"], d["values"], d["con_lb"], d["con_ub"], d["c"],
                                       d["var_lb"], d["var_ub"], maximize=d["maximize"],
                                       objective_offset=d["objective_offset"])
        small[name] = {key: run(q, on, optimality_tolerance=1e-8) for key, on in (("off", False), ("on", True))}
    out["iterations_to_1e-8"] = small
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
