#!/usr/bin/env python
"""Iteration counts / objectives of the 2-GPU transports next to the single-GPU solve (needs >= 2 GPUs).
usage: python scripts/dist_iteration_table.py [size] [world] [quick]"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

import test_gpu_dist as T  # noqa: E402


def main():
    size = int(sys.argv[1]) if len(sys.argv) > 1 else 40_000
    world = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    quick = len(sys.argv) > 3
    for tol in ((1e-4,) if quick else (1e-4, 1e-6)):
        for mode in ((1,) if quick else (1, 3)):
            lp, one = T._single_gpu(size, tol, mode)
            lp, two = T._single_gpu(size, tol, mode)
            s1, s2 = one.stats(), two.stats()
            print(f"tol {tol:g} mode {mode}: single its {s1.number_of_steps_taken} / {s2.number_of_steps_taken} obj "
                  f"{s1.primal_objective:.9g} planted {lp.optimal_objective:.9g}", flush=True)
            for tr in ("gather", "nccl"):
                r = T._solve_on_gpus(world, size, tol, mode, tr)
                print(f"    {tr:10s} its {r[0]['its']} obj {r[0]['obj']:.9g} dobj {r[0]['dobj']:.9g} status {r[0]['status']}",
                      flush=True)


if __name__ == "__main__":
    main()
