"""CPU: the cases of test_gpu_cta_long_cg are meaningful and make the CTA tier's CG run long.

For every case and slot: kappa_2 of the damped system (lm_step_ref.kappa2) keeps the bound 8 n kappa 2^-53
at or below MAX_BOUND, so the step test can tell a right step from a wrong one; the model of the kernel's
PCG (cta_cg_model) runs at least 1000 iterations on every chain of 1970 or more free nodes, at the default
radius and at 1e16; and it never reaches the cap 8 n + 100.  The components of test_gpu_lm_step's
large_problem(), random spanning trees plus random pairs, stay below a thousand iterations (about a
hundred from a start at zero): that is the gap these cases close.  Each case's kappa, bound and model
count are printed.
"""
import numpy as np

import cta_cg_model as cg
import lm_step_ref as ref
from test_gpu_cta_long_cg import CASES, LONG_ITERATIONS, LONG_KEYS, case, is_long
from test_gpu_lm_step import MAX_BOUND, large_problem, start_point


def test_model_is_the_solve():
    """The model's y solves the statement's system to its own tolerance: it is CG on that system."""
    p, _, _, _, sts, models = case("chains")
    for st, m in zip(sts, models):
        y = st.y.astype(np.float64)
        assert not m.capped and m.true_residual <= 1e-13, (st.n, m.true_residual)
        assert np.linalg.norm(m.y - y) <= ref.step_bound(st.n, st.kappa) * np.linalg.norm(y), st.n


def test_cases_are_meaningful_and_run_long():
    lines = []
    for key in CASES:
        p, opts, _, _, sts, models = case(key)
        for s, (st, m) in enumerate(zip(sts, models)):
            bound = ref.step_bound(st.n, st.kappa)
            lines.append("%-18s slot %d: n %5d, kappa %.2e, bound %.2e, model %5d CG iterations, %d restarts "
                         "(cap %d)" % (key, s, st.n, st.kappa, bound, m.iterations, m.restarts, cg.cg_cap(st.n)))
            assert bound <= MAX_BOUND, (key, s, st.n, st.kappa, bound)
            assert not m.capped and m.iterations < cg.cg_cap(st.n), (key, s, m.iterations)
            if key in LONG_KEYS and is_long(p, s):
                assert m.iterations >= LONG_ITERATIONS, (key, s, st.n, m.iterations)
    print("\n".join(lines))
    # every chain of LONG or more free nodes is checked, at both radii
    assert sum(is_long(case(k)[0], s) for k in ("chains", "chains_radius_1e16")
               for s in range(case(k)[0].n_components)) == 4


def test_random_trees_stay_below_a_thousand_iterations():
    """test_gpu_lm_step's large_problem(), random spanning trees plus random pairs past 1008 free nodes,
    1024 nodes and 1969 free nodes: from a start at zero (every residual an inlier) the model converges in
    about a hundred iterations; from the start test_gpu_lm_step uses, where many Tukey edges are outliers
    and parts of the graph hang by a few links, in under a thousand.  The chains above run 1.8 to 18 times
    longer."""
    from oracle_util import load_oracle
    p = large_problem()
    o = load_oracle().default_options()
    its = {kind: [cg.model_of(ref.first_step(p, s, o, start_point(p, kind, 2), want_kappa=False)).iterations
                  for s in range(p.n_components)] for kind in ("zero", "inside")}
    print("large_problem(): model CG iterations per slot", its)
    assert max(its["zero"]) <= 150 and max(its["inside"]) < LONG_ITERATIONS, its
