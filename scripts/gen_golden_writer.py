#!/usr/bin/env python
"""Generates tests/golden/writer_golden.json from the REFERENCE ITSELF (oracle/_ref, `make -C oracle ref`):

  written_mps_sha256  the MPS file this repo's writer produces for the LP of
                      tests/test_file_writers.py::test_reference_parser_reads_what_we_write
  reference_parse     digests of what the reference's libmps_parser read from exactly that file (A canonicalised to
                      sorted CSR, so the digests do not depend on the entry order the writer uses)
  verdicts            the reference CPU dual simplex's status on the small LPs of tests/test_oracle_pins.py

The tests compare against these where oracle/_ref is not built.  The output is committed.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_cpu  # noqa: E402


def main():
    from test_file_writers import WRITER_LP, canonical_digests, write_via_solve
    from test_oracle_pins import c_api_infeasible_lp, unbounded_lp
    from cuopt_b200 import capi

    lp = WRITER_LP()
    p = capi.Problem.create_ranged(lp.offsets, lp.indices, lp.values, lp.con_lb, lp.con_ub, lp.c, lp.var_lb, lp.var_ub)
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "written.mps")
        write_via_solve(p, out)
        sha = hashlib.sha256(open(out, "rb").read()).hexdigest()
        r = ref_cpu.parse_mps(out)
    parse = canonical_digests(r.offsets, r.indices, r.values, r.m, r.n, c=r.c, con_lb=r.con_lb, con_ub=r.con_ub,
                              var_lb=r.var_lb, var_ub=r.var_ub)
    off, idx, val, c, l, u, lc, uc = c_api_infeasible_lp()
    verdicts = {"c_api_infeasible_lp": ref_cpu.dual_simplex(off, idx, val, lc, uc, c, l, u)["status"]}
    off, idx, val, c, l, u, lc, uc = unbounded_lp()
    verdicts["unbounded_lp"] = ref_cpu.dual_simplex(off, idx, val, lc, uc, c, l, u)["status"]
    gold = {"_provenance": "scripts/gen_golden_writer.py: the reference's libmps_parser and CPU dual simplex (oracle/_ref)",
            "written_mps_sha256": sha, "reference_parse": {"m": r.m, "n": r.n, "digests": parse}, "verdicts": verdicts}
    with open(os.path.join(ROOT, "tests", "golden", "writer_golden.json"), "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
