"""A line search that fails leaves the step unchanged, and the trust-region loop then judges the full step,
which the search evaluated first.  The warp-register queue kernel keeps that first evaluation's cost and
norms and takes them back instead of evaluating the full step again.  Only when the step is accepted does
it restage the evaluation at the full step, which the next assembly reads (RegTier::restore_full_step and
accept, csrc/lfr_solve_warp2.cuh).  The other kernels evaluate the full step again.

With the default options such a step is rejected on the benchmark's scenes: a full step that fails the
Armijo test with the default sufficient decrease has too small a gain ratio.  So the restaged path needs
other options.  A sufficient decrease of 0.9 and at most three line-search steps make most searches
contract twice, fail, and leave a full step that the gain ratio accepts.  That happens hundreds of times
on cfg1 (per-bucket warp kernels) and on cfg2 at 5 % (queue kernel).  Every route must then match the
oracle's line-search mode that follows the kernels operation for operation."""
import numpy as np
import pytest

from test_gpu_tier_options import assert_agree, options, oracle_result, scene, start_of

OPTS = dict(line_search_sufficient_function_decrease=0.9, max_num_line_search_step_size_iterations=3)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["default", "tile_from_1", "smem_cholesky"])
@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
def test_failed_search_then_accepted_full_step(b200, oracle, name, route):
    p = scene(name)
    for kind in ("zero", "random"):
        start = start_of(name, kind)
        ref = oracle_result(oracle, (name, "restored_full_step", kind), p, OPTS, start)
        got = b200.solve(p, options(b200, route, **OPTS), positions=start)
        assert ref["fast"][1]["total_line_search_steps"] > 0
        assert_agree(p, start, got, ref, (name, route, kind))
        # the route's own line-search totals equal the oracle's: every restored step was taken as evaluated
        assert got[1]["total_line_search_steps"] == ref["fast"][1]["total_line_search_steps"]
        assert np.all(np.isfinite(got[0]))
