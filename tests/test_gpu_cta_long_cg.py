"""The CTA tier's PCG step where CG runs long: chains, a grid and a caterpillar against the
extended-precision step (tests/lm_step_ref.py), with the kernel's CG iteration count next to a model's.

The components of test_gpu_lm_step are random spanning trees plus random pairs: shallow graphs on which
block-Jacobi CG converges in about a hundred iterations from a start at zero and in under a thousand from
the start those tests use (tests/cta_cg_model.py).  Long tracks are not like that.  On a chain of n free nodes held by one root at its end, kappa grows like n^2 and CG takes
thousands of iterations, each with three CTA barriers; the recurrence residual drifts from the true one,
so the restarts run late and share the budget 8 n + 100 with the first pass; and the vectors sit in HBM
past 1969 free nodes.  These cases run there:
  * chains of 250, 1000, 1970 and 8191 free nodes, the root at one end, at the default radius and at
    radius 1e16 (damping changes kappa by about 300x);
  * a chain of 16 383 nodes (the 14-bit local index's limit) with its root at local index 8191, in both
    node orders, so that free nodes sit at local indices 0 and 16 382; a root at one end would put kappa
    beyond a meaningful bound;
  * a 90 x 90 grid with its root at a corner;
  * a caterpillar: a spine of 1500 nodes with legs of two, sims over three decades;
  * chains of 2000 free nodes with duplicated edges and with edges without a twin, which take the
    irregular matrix-free product instead of the block-CSR one.
Tracks are three consecutive nodes (Cauchy inside a track, Tukey across); every edge's flow is a constant
of at most 0.03 (M = I: otherwise the flow gradients bound kappa near 1e4 whatever the length) and the
start is zero, so every residual is an inlier.

Checks on every case and route: the first step to test_gpu_lm_step.check's bar; the line-search probe's
modes A (alpha = 1 and 2^-10), B and C to test_gpu_ls_probe's bounds; and the kernel's CG iterations of
the first step (the diagnostic record's tier word, csrc/lfr_lm.cuh) within 10 % of the model's, at least
1000 on the chains of 1970 or more free nodes, and below the cap.  One whole solve of the 1970- and
8191-node chains and the grid against the oracle.  The module ends by printing, per case, the largest
|dl - dl*| / (n kappa u |dl*|), kappa and the kernel's against the model's CG iterations.
"""
import numpy as np
import pytest

import cta_cg_model as cg
import lm_step_ref as ref
from test_gpu_lm_step import check, counter_of, first_steps, lmstep, problem  # noqa: F401
from test_gpu_ls_probe import check_mode_a, check_mode_b, check_mode_c, lsprobe  # noqa: F401
import test_gpu_ls_probe
from test_gpu_tier_options import ROUTES, TIER_CTA

LONG = 1970        # chains of at least this many free nodes must run at least LONG_ITERATIONS
LONG_ITERATIONS = 1000
# The kernel's CG iteration counts are the model's to within 0.3 % on every case here (H100, 700 W).  A
# solve cut short, by a lower cap for instance, can still land within the step's bound (a cap of 1200
# does on the chains at the default radius), so the count is held to the model's within 10 %.
ITERATION_SPREAD = 0.1


# ---------------------------------------------------------------------------------------------------
# constructed components (pure numpy)
# ---------------------------------------------------------------------------------------------------
def from_pairs(rng, nc, roots, pairs, twins="all", dup=0, sim_decades=0.0):
    """A component of `nc` nodes, roots at local indices `roots`, an edge pair per entry of `pairs`
    (both directions, or only the first for twins="none"), `dup` directed edges duplicated; tracks of
    three consecutive nodes; sims in [0.5, 1], or 10^U(-sim_decades, 0).  Every edge's flow is one
    constant vector of |.| <= 0.03 over its grid: M = I + grad flow = I, so a translation of a part costs
    nothing and a chain's system is a path Laplacian whose kappa grows like n^2 (random grids give M a
    spread of about 0.1 around I, which holds kappa near 1e4 at every length)."""
    is_root = np.zeros(nc, np.uint8)
    is_root[list(roots)] = 1
    src, dst = [], []
    for u, v in pairs:
        src += [u] if twins == "none" else [u, v]
        dst += [v] if twins == "none" else [v, u]
    for k in rng.choice(len(src), dup, replace=False) if dup else []:
        src.append(src[k])
        dst.append(dst[k])
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    flow = np.tile(rng.uniform(-0.03, 0.03, (len(src), 2)), 9).astype(np.float32)   # [E, 3 x 3 x 2]
    if sim_decades:
        sim = (10.0 ** rng.uniform(-sim_decades, 0.0, len(src))).astype(np.float32)
    else:
        sim = rng.uniform(0.5, 1.0, len(src)).astype(np.float32)
    return dict(nc=nc, is_root=is_root, src=src, dst=dst, flow=flow, sim=sim, track=np.arange(nc) // 3)


def chain(rng, nc, root=0, **kw):
    return from_pairs(rng, nc, [root], [(v - 1, v) for v in range(1, nc)], **kw)


def grid(rng, side):
    """A side x side grid in row-major order, its root at a corner."""
    ids = np.arange(side * side).reshape(side, side)
    pairs = list(zip(ids[:, :-1].ravel(), ids[:, 1:].ravel())) + list(zip(ids[:-1].ravel(), ids[1:].ravel()))
    return from_pairs(rng, side * side, [0], [(int(u), int(v)) for u, v in pairs])


def caterpillar(rng, spine, legs=2, sim_decades=3.0):
    """A spine of `spine` nodes, each with a path of `legs` nodes hanging from it (a spine node and its
    legs are consecutive: one track), the root at the spine's first node."""
    k = legs + 1
    pairs = [(k * (s - 1), k * s) for s in range(1, spine)]
    pairs += [(k * s + j, k * s + j + 1) for s in range(spine) for j in range(legs)]
    return from_pairs(rng, k * spine, [0], pairs, sim_decades=sim_decades)


CHAIN_FREE = (250, 1000, 1970, 8191)
BIG_CHAIN = 16383


def chains_problem():
    rng = np.random.default_rng(30)
    return problem([chain(rng, n + 1) for n in CHAIN_FREE])


def big_chain_problem():
    """The same 16 383-node chain twice, its root at local index 8191; slot 1's node list reversed."""
    c = chain(np.random.default_rng(31), BIG_CHAIN, root=BIG_CHAIN // 2)
    return problem([c, c], reverse={1})


def grid_problem():
    return problem([grid(np.random.default_rng(32), 90)])


def caterpillar_problem():
    return problem([caterpillar(np.random.default_rng(33), 1500)])


def irregular_problem():
    rng = np.random.default_rng(34)
    return problem([chain(rng, 2001, dup=40), chain(rng, 2001, twins="none")])


R16 = dict(initial_trust_region_radius=1e16)
# key: (problem, options); every case starts at zero
CASES = {
    "chains": (chains_problem, {}),
    "chains_radius_1e16": (chains_problem, R16),
    "chain_16383": (big_chain_problem, R16),
    "grid_90x90": (grid_problem, R16),
    "caterpillar": (caterpillar_problem, R16),
    "irregular_chains": (irregular_problem, R16),
}

_made = {}


def case(key):
    """(problem, options dict, start, lfr_options, first-step statements, model runs) of one case."""
    if key not in _made:
        from oracle_util import load_oracle
        make, opts = CASES[key]
        p = make()
        x0 = np.zeros((p.graph.n_nodes, 2))
        o = load_oracle().default_options(**opts)
        sts = [ref.first_step(p, s, o, x0) for s in range(p.n_components)]
        _made[key] = (p, opts, x0, o, sts, [cg.model_of(st) for st in sts])
    return _made[key]


def is_long(p, s):
    """A chain slot whose first step must run at least LONG_ITERATIONS: LONG or more free nodes, one root."""
    nodes = p.comp_nodes[p.comp_ptr[s]:p.comp_ptr[s + 1]]
    return int((p.is_root[nodes] == 0).sum()) >= LONG


LONG_KEYS = ("chains", "chains_radius_1e16", "chain_16383", "irregular_chains")


# ---------------------------------------------------------------------------------------------------
# the GPU tests
# ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def report(request):
    """Per case: the largest |dl - dl*| / (n kappa u |dl*|) and kappa over its slots and routes, and per
    slot the kernel's CG iterations (every distinct count over the routes) against the model's; printed at
    the end of the module past output capture."""
    seen = {}
    yield seen
    lines = []
    for key, (ratio, kappa, its) in seen.items():
        lines.append("long CG %-18s largest |dl - dl*| / (n kappa u |dl*|) = %.3e, largest kappa %.2e" % (key, ratio, kappa))
        for s, (n, got, model) in sorted(its.items()):
            lines.append("    slot %d, n %5d: CG iterations GPU %s, model %d, cap %d" % (
                s, n, "/".join(str(g) for g in sorted(got)), model, cg.cg_cap(n)))
    tr = request.config.pluginmanager.getplugin("terminalreporter")
    cm = request.config.pluginmanager.getplugin("capturemanager")
    if tr is None or cm is None:
        print("\n".join(lines))
        return
    with cm.global_and_fixture_disabled():
        tr.write_line("")
        for line in lines:
            tr.write_line(line)


def check_iterations(key, p, rec, sts, models):
    """The kernel's CG iterations of each slot's first step against the model's, the floor and the cap.
    Returns them."""
    got = []
    for s, (st, m) in enumerate(zip(sts, models)):
        g = counter_of(rec[s, 6])
        what = (key, s, st.n, g, m.iterations)
        assert g < cg.cg_cap(st.n), (what, "the kernel's CG reached its cap: an unconverged step")
        assert abs(g - m.iterations) <= ITERATION_SPREAD * m.iterations, (what, "not the model's iteration")
        if key in LONG_KEYS and is_long(p, s):
            assert g >= LONG_ITERATIONS, (what, "a long chain converged too early")
        got.append(g)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("key", list(CASES))
def test_first_step(lmstep, report, key, route):  # noqa: F811
    """test_gpu_lm_step.check's bar on every slot, and the kernel's CG iterations (check_iterations)."""
    import test_gpu_lm_step
    p, opts, x0, o, sts, models = case(key)
    test_gpu_lm_step._statements["long_cg_" + key] = sts      # check() reads its statements from this cache
    worst = {}
    _, rec = check(lmstep, worst, "long_cg_" + key, p, x0, route, opts)
    got = check_iterations(key, p, rec, sts, models)
    ratio, kappa, _ = worst[TIER_CTA]
    r = report.setdefault(key, [0.0, 0.0, {}])
    r[0], r[1] = max(r[0], ratio), max(r[1], kappa)
    for s, g in enumerate(got):
        r[2].setdefault(s, (sts[s].n, set(), models[s].iterations))[1].add(g)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("key", list(CASES))
def test_line_search_probe(lsprobe, lmstep, key, route):  # noqa: F811
    """Modes A (alpha 1 and 2^-10), B and C of the probe build, to test_gpu_ls_probe's bounds; mode A's dl
    bitwise the lmstep build's, and its CG count that build's."""
    p, opts, x0, o, sts, models = case(key)
    test_gpu_ls_probe._made["long_cg_" + key] = (p, opts, x0, o, sts)
    probe_report = {}
    dl_seen, recs = {}, {}
    for alpha in (1.0, 2.0 ** -10):
        _, recs[alpha] = check_mode_a(lsprobe, probe_report, "long_cg_" + key, route, alpha, dl_seen)
    check_mode_b(lsprobe, probe_report, "long_cg_" + key, route, recs[1.0], dl_seen)
    check_mode_c(lsprobe, probe_report, "long_cg_" + key, route)
    pos_l, rec_l = first_steps(lmstep, p, route, x0, **opts)
    for s, st in enumerate(sts):
        assert np.array_equal(pos_l[st.free_nodes], dl_seen[s]), (key, route, s, "not the lmstep build's dl")
        assert counter_of(recs[1.0][s, 7]) == counter_of(rec_l[s, 6]), (key, route, s, "CG iterations differ")


@pytest.mark.gpu
def test_whole_solve_matches_oracle(b200, oracle):
    """The 1970- and 8191-node chains and the 90 x 90 grid through lfr_solve on the default route against
    the oracle: every component within 1e-4 px, the same iterations, terminations and costs."""
    from test_gpu_parity import TOL_UNITS, _per_component_agreement
    rng = np.random.default_rng(35)
    p = problem([chain(rng, 1971), chain(rng, 8192), grid(rng, 90)])
    pos_g, st_g = b200.solve(p)
    pos_o, st_o = oracle.solve(p, oracle.default_options(n_threads=3))
    good, err = _per_component_agreement(p, pos_g, st_g, pos_o, st_o)
    assert good.all(), (err, st_g["iterations"], st_o["iterations"], st_g["termination"], st_o["termination"])
    assert err.max() <= TOL_UNITS
    np.testing.assert_allclose(st_g["initial_cost"], st_o["initial_cost"], rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(st_g["final_cost"], st_o["final_cost"], rtol=1e-8, atol=1e-14)
