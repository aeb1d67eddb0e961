"""The device version of the trust-region solve (cuopt_b200/csrc/trust_region.cuh) does not re-reduce the active range
at every trial threshold like the reference / the oracle: it sorts once, takes prefix sums of the two radius terms and
evaluates every partial radius as a difference of prefix sums inside a single-thread bisection.  exact.py transcribes
exactly that formulation in numpy (device_formulation: same formulas, same search functions, same update rules); this
file checks it against the oracle's direct restatement on real iterates — a CPU check of the reformulation, independent
of CUDA."""
import pytest
import scipy.sparse as sp

from conftest import mps_path, problem_arrays
from cuopt_b200 import capi, lpgen
from exact import device_formulation
from oracle import pdlp_oracle as po


def scaled_problem(o, a):
    dr, dc = o.vector("row_scaling"), o.vector("col_scaling")
    A = sp.csr_matrix((a["values"], a["indices"], a["offsets"]), shape=(len(a["con_lb"]), len(a["c"])))
    As = (sp.diags(dr) @ A @ sp.diags(dc)).tocsr()
    return As, o.vector("scaled_c"), o.vector("scaled_l"), o.vector("scaled_u"), o.vector("scaled_lc"), o.vector("scaled_uc")


CASES = ["afiro", "sparse", "multicommodity"]


@pytest.mark.parametrize("case", CASES)
def test_prefix_sum_bisection_equals_the_direct_restatement(case):
    if case == "afiro":
        a = problem_arrays(capi.Problem.read(mps_path("linear_programming/afiro_original.mps")))
    else:
        lp = lpgen.sparse_lp(400, 300, 5, seed=3) if case == "sparse" else lpgen.multicommodity(30, 90, 3, seed=2)
        a = dict(offsets=lp.offsets, indices=lp.indices, values=lp.values, c=lp.c, var_lb=lp.var_lb, var_ub=lp.var_ub,
                 con_lb=lp.con_lb, con_ub=lp.con_ub)
    o = po.Oracle(a["offsets"], a["indices"], a["values"], a["c"], a["var_lb"], a["var_ub"], a["con_lb"], a["con_ub"],
                  mode=po.METHODICAL1, tol=1e-10)
    o.initialise()
    prob = scaled_problem(o, a)
    for steps in (7, 20, 33):      # between restarts: the last-restart point is the origin / an earlier iterate
        o.run(steps)
        px, py = o.vector("x"), o.vector("y")
        tau, sigma = o.scalar("tau"), o.scalar("sigma")
        for radius in (-1.0, 1e-3, 0.5, 1e3):
            lo_want, up_want, used = o.trust_region_bounds(px, py, radius)
            lo_got, up_got = device_formulation(*prob, tau, sigma, px, py, used)
            scale = max(1.0, abs(lo_want), abs(up_want))
            assert abs(lo_got - lo_want) <= 1e-9 * scale, (case, steps, radius)
            assert abs(up_got - up_want) <= 1e-9 * scale, (case, steps, radius)
