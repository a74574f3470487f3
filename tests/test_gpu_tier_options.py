"""Every solve tier against the CPU oracle on non-default options, non-zero start points and every
termination code.

All four tiers run one trust-region driver (csrc/lfr_lm.cuh), but each kernel still brings its own
start-point projection and constant (root) positions, its own use of `bound` in the projected gradient
and the trial point, its own LM diagonal clamp, its own phi' for the line search and its own reductions.
This file runs those per-tier pieces on:

  * four scenes whose components reach every warp2 class (n <= 8 / 16 / 24 / 32 unknowns), every tile
    class (48 / 64 / 80), the shared-memory Cholesky warp kernel (80 < n <= 96) and the CTA tier;
  * five routes (lfr_options.debug_flags / linear_solver) that move the same components to other tiers;
  * option sets that change the trajectory or reach a termination code, from zeros and from a random
    start outside the box;
  * constructed problems that end in FAILURE (the start point is kept), EMPTY (no free node), and a
    launch that mixes both with ordinary components;
  * every API path (pageable / pinned / zero-copy lfr_solve, lfr_solve_multi, plans) from a non-zero start;
  * the per-edge evaluation under non-default loss options.

Acceptance is that of tests/test_gpu_parity.py on every component: positions within 1e-4 px, identical
iteration counts and termination codes, initial / final costs to 1e-10 / 1e-8.  The kernels mirror the
oracle's FAST line-search formulation operation for operation, so the whole bar and the line-search
step totals are held against the oracle in that mode.  Against the literal Ceres restatement (the
default mode) the same bar holds on every component whose trajectory the two oracle modes agree on;
where they do not (a line search contracting towards its minimum step size, where Ceres' own fit is
rank-truncated, decides a termination test differently: see tests/test_linesearch_modes.py), the
positions still agree to 1e-4 px.  One exception to equal step totals: the CTA tier's PCG step under
tolerances of 1e-10 (see test_every_route_matches_oracle).  Roots, singleton components and components
that end in FAILURE or EMPTY keep their start values bitwise.
"""
import copy
import ctypes as C
import os

import numpy as np
import pytest

from oracle_util import LS_FAST, line_search_mode

TOL_UNITS = 1e-4 / 16.0   # 1e-4 px, 1 solver unit = 16 px
N_THREADS = os.cpu_count() or 8
SKIPPED, GRADIENT_TOL, PARAMETER_TOL, FUNCTION_TOL, MIN_RADIUS, NO_CONVERGENCE, FAILURE, EMPTY = range(8)
TIER_WARP2, TIER_TILE, TIER_WARP, TIER_CTA = 1, 2, 3, 4   # LmProfile::Tier (csrc/lfr_lm.cuh)
FAILURE_START = 1.7                                       # projected to 1.0 = bound: every residual is zero

# scene -> keypoint scale.  Components by unknowns n (n <= 8 / 16 / 24 / 32 / 48 / 64 / 80 / 96 / > 96):
#   cfg1    207 /   0 /   0 /   0 /   0 /   0 /   0 /  0 /  0
#   cfg2     11 / 168 /  30 /   0 /   0 /   0 /   0 /  0 /  0
#   cfg4      1 /  68 / 230 / 133 / 521 / 464 / 174 /  0 /  0
#   ring60    0 /   1 /  13 /  27 /  15 /  54 /  28 / 31 / 38
SCENES = {"cfg1": 1.0, "cfg2": 0.05, "cfg4": 0.25, "ring60": 0.3}

# route -> (debug_flags, linear_solver), see include/lfr.h
ROUTES = ("default", "smem_cholesky", "tile_from_1", "no_tile", "cta")

OPTION_SETS = {
    "defaults": {},
    "tukey_variant_2": dict(tukey_variant=2),
    "loss_widths": dict(cauchy_a=0.1, tukey_a=0.2),
    "bound_0.05": dict(bound=0.05),
    "max_iter_0": dict(max_num_iterations=0),
    "max_iter_1": dict(max_num_iterations=1),
    "min_radius_2e4": dict(min_trust_region_radius=2e4),
    "min_radius_1": dict(min_trust_region_radius=1.0),
    "gradient_tol_1e-2": dict(gradient_tolerance=1e-2),
    # tolerances of exactly 0 would make FUNCTION_TOL / PARAMETER_TOL fire when the cost or the step
    # stagnates to the last bit, which depends on the order of the sums; 1e-10 stays above that
    "tight_tolerances": dict(gradient_tolerance=0.0, function_tolerance=1e-10, parameter_tolerance=1e-10),
    "line_search_2_steps": dict(max_num_line_search_step_size_iterations=2),
    "sufficient_decrease_0.5": dict(line_search_sufficient_function_decrease=0.5),
    "lm_diagonal_clamp": dict(min_lm_diagonal=1e2, max_lm_diagonal=1e3),
    "max_radius_1e-2": dict(max_trust_region_radius=1e-2),
    "rejected_steps": dict(max_num_consecutive_invalid_steps=1, min_relative_decrease=0.99,
                           initial_trust_region_radius=1e-3),
}

# termination codes each option set reaches in the oracle, over the four scenes and both starts
REACHES = {
    "defaults": {PARAMETER_TOL, FUNCTION_TOL},
    "bound_0.05": {GRADIENT_TOL},
    "max_iter_0": {NO_CONVERGENCE},
    "max_iter_1": {NO_CONVERGENCE},
    "min_radius_2e4": {MIN_RADIUS},
    "min_radius_1": {MIN_RADIUS},
    "gradient_tol_1e-2": {GRADIENT_TOL},
    "tight_tolerances": {NO_CONVERGENCE},
    "max_radius_1e-2": {NO_CONVERGENCE},
}

# the option sets whose profiled solves fill the tier x termination table (with the FAILURE problems)
TABLE_OPTION_SETS = ("defaults", "gradient_tol_1e-2", "min_radius_2e4", "max_iter_1")


# ---------------------------------------------------------------------------------------------------
# problems, start points and options (built once per module)
# ---------------------------------------------------------------------------------------------------
_cache = {}


def _cached(key, make):
    if key not in _cache:
        _cache[key] = make()
    return _cache[key]


def slot_nodes(p, s):
    return p.comp_nodes[p.comp_ptr[s]:p.comp_ptr[s + 1]].astype(np.int64)


def sizes_of(p):
    return np.diff(p.comp_ptr.astype(np.int64))


def free_count(p):
    """Non-root nodes of every slot."""
    nodes = p.comp_nodes.astype(np.int64)
    free = (p.is_root[nodes] == 0).astype(np.int64)
    return np.add.reduceat(free, p.comp_ptr[:-1].astype(np.int64)) * (sizes_of(p) > 0) if len(nodes) else \
        np.zeros(p.n_components, np.int64)


def per_slot_max(p, v):
    """max of the per-node values `v` over the nodes of every slot (0 for an empty slot)."""
    out = np.zeros(p.n_components)
    nz = sizes_of(p) > 0
    if nz.any():
        out[nz] = np.maximum.reduceat(v[p.comp_nodes.astype(np.int64)], p.comp_ptr[:-1][nz].astype(np.int64))
    return out


def scene(name):
    def make():
        from lfr_b200 import build_problem, synth
        return build_problem(synth.generate(name, scale=SCENES[name]))
    return _cached(("scene", name), make)


def random_start(p, seed):
    """uniform(-1.5, 1.5) on every node: free nodes get projected, roots keep out-of-box values."""
    return np.random.default_rng(seed).uniform(-1.5, 1.5, size=(p.graph.n_nodes, 2))


def start_of(name, kind):
    p = scene(name)
    if kind == "zero":
        return np.zeros((p.graph.n_nodes, 2))
    return _cached(("start", name), lambda: random_start(p, 7 + sum(map(ord, name))))


def failure_problem(name):
    """Zero flows, no roots: from a start of 1.7 (projected to 1.0) every residual and the gradient are
    exactly zero, every LM step has zero model change, and the solve ends in FAILURE after 10 invalid
    steps.  Ceres does not commit that solution, so every node keeps 1.7."""
    def make():
        from lfr_b200 import build_problem, synth
        ms = synth.generate(name, scale=SCENES[name])
        ms.disp1[:] = 0
        ms.disp2[:] = 0
        q = build_problem(ms)
        q.is_root = np.zeros_like(q.is_root)
        return q
    return _cached(("failure", name), make)


def empty_problem(name):
    """Every node a root: every component of more than one node has no free node (EMPTY)."""
    def make():
        q = copy.copy(scene(name))
        q.is_root = np.ones_like(q.is_root)
        return q
    return _cached(("empty", name), make)


def mixed_problem():
    """ring60 at 0.3 with the FAILURE construction applied to every 4th component of more than one node
    (roots cleared, flows of their edges zeroed, nodes started at 1.7); the others keep their roots,
    flows and random start.  Returns (problem, start, chosen slots)."""
    def make():
        p = scene("ring60")
        multi = np.nonzero(sizes_of(p) > 1)[0]
        chosen = multi[::4]
        q = copy.copy(p)
        q.graph = copy.copy(p.graph)
        q.graph.edges = p.graph.edges.copy()
        q.is_root = p.is_root.copy()
        start = random_start(p, 60).copy()
        rp = p.graph.row_ptr.astype(np.int64)
        for s in chosen:
            nodes = slot_nodes(p, s)
            q.is_root[nodes] = 0
            start[nodes] = FAILURE_START
            for v in nodes:
                q.graph.edges["flow"][rp[v]:rp[v + 1]] = 0
        return q, start, chosen
    return _cached(("mixed",), make)


def options(lib, route="default", profile=False, **opts):
    from lfr_b200 import capi
    flags = {"default": 0, "smem_cholesky": capi.DBG_FORCE_SMEM_CHOLESKY, "tile_from_1": 1 << capi.DBG_TILE_FROM_SHIFT,
             "no_tile": capi.DBG_NO_TILE, "cta": 0}[route]
    return lib.default_options(debug_flags=flags | (capi.DBG_PROFILE if profile else 0),
                               linear_solver=2 if route == "cta" else 0, **opts)


def expected_tier(n2, route):
    """The tier lfr_capi.cu's schedule picks for a component of n2 unknowns (small components: every
    staged layout fits in shared memory)."""
    if route == "cta" or n2 > 96:
        return TIER_CTA
    if route == "smem_cholesky":
        return TIER_WARP
    if n2 <= 32:
        return TIER_TILE if route == "tile_from_1" else TIER_WARP2
    if n2 <= 80 and route != "no_tile":
        return TIER_TILE
    return TIER_WARP


# ---------------------------------------------------------------------------------------------------
# the oracle (once per problem, options and start: its result does not depend on the route)
# ---------------------------------------------------------------------------------------------------
def oracle_result(oracle, key, p, opts, start):
    """{"literal": (pos, stats), "fast": (pos, stats)}: the oracle in its default (literal Ceres) and in
    its FAST line-search mode."""
    def make():
        out = {}
        o = oracle.default_options(n_threads=N_THREADS, **opts)
        out["literal"] = oracle.solve(p, o, positions=start)
        with line_search_mode(oracle, LS_FAST):
            out["fast"] = oracle.solve(p, o, positions=start)
        return out
    return _cached(("oracle",) + tuple(key), make)


def scene_oracle(oracle, name, opt_name, start_kind):
    return oracle_result(oracle, (name, opt_name, start_kind), scene(name), OPTION_SETS[opt_name],
                         start_of(name, start_kind))


def untouched_nodes(p, term):
    """Nodes whose positions a solve must leave as they started: roots, nodes of singleton components and
    of components that end in FAILURE or EMPTY."""
    sizes = sizes_of(p)
    per_node = np.zeros(p.graph.n_nodes, bool)
    keep_slot = (sizes <= 1) | (term == FAILURE) | (term == EMPTY)
    per_node[p.comp_nodes.astype(np.int64)] = np.repeat(keep_slot, sizes)
    return per_node | (p.is_root != 0)


def assert_agree(p, start, got, ref, what, exact_line_search=True):
    """The parity bar on every component against the FAST oracle (iteration counts, termination codes,
    positions, costs, line-search step totals); against the literal oracle on every component where the
    two oracle modes agree on the trajectory, positions alone elsewhere; untouched nodes bitwise at the
    start.  Returns (max |dx| against the literal oracle, components where the oracle modes disagree)."""
    pos_g, st_g = got
    (pos_l, st_l), (pos_f, st_f) = ref["literal"], ref["fast"]
    for name, (pos_o, st_o), only in (("fast", (pos_f, st_f), None),
                                     ("literal", (pos_l, st_l), (st_l["iterations"] == st_f["iterations"]) &
                                      (st_l["termination"] == st_f["termination"]))):
        err = per_slot_max(p, np.abs(pos_g - pos_o).max(axis=1))
        bad = (err > TOL_UNITS)
        traj = (st_g["iterations"] != st_o["iterations"]) | (st_g["termination"] != st_o["termination"])
        bad |= traj if only is None else (traj & only)
        sel = np.ones(p.n_components, bool) if only is None else only
        bad = np.nonzero(bad)[0]
        assert bad.size == 0, (what, name, [(int(c), int(sizes_of(p)[c]), float(err[c]), int(st_g["iterations"][c]),
                                             int(st_o["iterations"][c]), int(st_g["termination"][c]),
                                             int(st_o["termination"][c])) for c in bad[:8]])
        np.testing.assert_allclose(st_g["initial_cost"][sel], st_o["initial_cost"][sel], rtol=1e-10, atol=1e-14,
                                   err_msg="%s %s" % (what, name))
        np.testing.assert_allclose(st_g["final_cost"][sel], st_o["final_cost"][sel], rtol=1e-8, atol=1e-14,
                                   err_msg="%s %s" % (what, name))
        if name == "literal":
            err_l, n_ambiguous = float(err.max()), int((~only).sum())
    assert st_g["n_solved"] == st_f["n_solved"] and st_g["total_iterations"] == st_f["total_iterations"], what
    n_ls_g, n_ls_f = st_g["total_line_search_steps"], st_f["total_line_search_steps"]
    assert n_ls_g == n_ls_f if exact_line_search else abs(n_ls_g - n_ls_f) <= 1 + n_ls_f // 100, (what, n_ls_g, n_ls_f)
    keep = untouched_nodes(p, st_g["termination"])
    assert np.array_equal(pos_g[keep], start[keep]), (what, "untouched nodes moved")
    return err_l, n_ambiguous


def profiled_solve(b200, p, opts, start):
    """The solve through a plan created with LFR_DBG_PROFILE and `start` as its initial positions:
    positions, stats, decoded records."""
    from lfr_b200 import capi
    plan = capi.Plan(b200, p, opts, positions=start)
    try:
        plan.solve()
        pos, st = plan.download()
        rec, _ = plan.profile()
    finally:
        plan.close()
    return pos, st, rec


def assert_bitwise(a, b, what):
    (pa, sa), (pb, sb) = a, b
    assert np.array_equal(pa, pb), (what, float(np.abs(pa - pb).max()))
    for k in ("iterations", "termination", "initial_cost", "final_cost"):
        assert np.array_equal(sa[k], sb[k]), (what, k)
    for k in ("total_iterations", "total_line_search_steps", "n_solved"):
        assert sa[k] == sb[k], (what, k, sa[k], sb[k])


# ---------------------------------------------------------------------------------------------------
# CPU: the oracle alone keeps the fixtures meaningful
# ---------------------------------------------------------------------------------------------------
def test_scenes_reach_every_size_class():
    """Together the scenes hold components in every warp2 class, every tile class, the warp tier's
    80 < n <= 96 and the CTA tier (n > 96)."""
    seen = set()
    for name in SCENES:
        n2 = 2 * free_count(scene(name))
        seen |= set(np.digitize(n2[sizes_of(scene(name)) > 1], [0, 9, 17, 25, 33, 49, 65, 81, 97]).tolist())
    assert seen >= set(range(1, 10)), seen


@pytest.mark.parametrize("opt_name", list(OPTION_SETS))
def test_option_set_reaches_its_codes(oracle, opt_name):
    """Each option set reaches, somewhere in the four scenes, the termination codes the GPU tests rely on,
    and every set but the defaults changes a trajectory (iterations, terminations, line-search steps or
    final costs) of at least one scene and start."""
    codes, changed = set(), False
    for name in SCENES:
        for kind in ("zero", "random"):
            st = scene_oracle(oracle, name, opt_name, kind)["literal"][1]
            d = scene_oracle(oracle, name, "defaults", kind)["literal"][1]
            codes |= set(st["termination"].tolist())
            changed |= not (np.array_equal(st["iterations"], d["iterations"]) and
                            np.array_equal(st["termination"], d["termination"]) and
                            st["total_line_search_steps"] == d["total_line_search_steps"] and
                            np.array_equal(st["final_cost"], d["final_cost"]))
            solved = sizes_of(scene(name)) > 1
            if opt_name == "max_iter_0":
                assert np.all(st["iterations"][solved] == 0) and np.all(st["termination"][solved] == NO_CONVERGENCE)
            if opt_name == "max_iter_1":
                assert np.all(st["iterations"][solved] == 1) and np.all(st["termination"][solved] == NO_CONVERGENCE)
            if opt_name == "min_radius_2e4":
                assert np.all(st["iterations"][solved] == 0) and np.all(st["termination"][solved] == MIN_RADIUS)
    assert codes >= REACHES.get(opt_name, set()), (opt_name, codes)
    assert changed or opt_name == "defaults"
    if opt_name == "defaults":
        # line searches from the random start
        assert all(scene_oracle(oracle, n, opt_name, "random")["literal"][1]["total_line_search_steps"] > 0
                   for n in SCENES)


@pytest.mark.parametrize("name", ["cfg1", "ring60"])
def test_failure_construction(oracle, name):
    """Zero flows, no roots, start 1.7, gradient_tolerance = -1: every component of more than one node
    ends in FAILURE after exactly 10 iterations at zero cost, and every node keeps 1.7 bitwise."""
    q = failure_problem(name)
    assert not q.is_root.any() and not q.graph.edges["flow"].any()
    start = np.full((q.graph.n_nodes, 2), FAILURE_START)
    pos, st = oracle_result(oracle, ("failure", name), q, dict(gradient_tolerance=-1.0), start)["literal"]
    solved = sizes_of(q) > 1
    assert solved.sum() > 100
    assert np.all(st["termination"][solved] == FAILURE) and np.all(st["iterations"][solved] == 10)
    assert np.all(st["initial_cost"][solved] == 0) and np.all(st["final_cost"][solved] == 0)
    assert np.array_equal(pos, start)


@pytest.mark.parametrize("name", list(SCENES))
def test_empty_construction(oracle, name):
    """All nodes roots: every component of more than one node ends EMPTY after 0 iterations; nothing moves."""
    q = empty_problem(name)
    start = start_of(name, "random")
    pos, st = oracle_result(oracle, ("empty", name), q, {}, start)["literal"]
    solved = sizes_of(q) > 1
    assert np.all(st["termination"][solved] == EMPTY) and np.all(st["termination"][~solved] == SKIPPED)
    assert np.all(st["iterations"] == 0) and st["total_iterations"] == 0
    assert np.array_equal(pos, start)


def test_mixed_construction(oracle):
    """The mixed problem is valid (every slot holds whole components, the chosen slots have no roots and
    zero flows on every out-edge, nothing else changed) and, under gradient_tolerance = -1, its FAILURE
    components are exactly the chosen ones, at 1.7 bitwise; the others converge as usual."""
    p = scene("ring60")
    q, start, chosen = mixed_problem()
    assert len(chosen) >= 40
    sizes = sizes_of(q)
    in_chosen = np.zeros(q.graph.n_nodes, bool)
    for s in chosen:
        in_chosen[slot_nodes(q, s)] = True
        assert np.all(q.comp[slot_nodes(q, s)] == q.comp[slot_nodes(q, s)[0]])
    assert not q.is_root[in_chosen].any() and np.array_equal(q.is_root[~in_chosen], p.is_root[~in_chosen])
    src = np.repeat(np.arange(q.graph.n_nodes), np.diff(q.graph.row_ptr.astype(np.int64)))
    assert not q.graph.edges["flow"][in_chosen[src]].any()
    assert np.array_equal(q.graph.edges["flow"][~in_chosen[src]], p.graph.edges["flow"][~in_chosen[src]])
    assert np.all(start[in_chosen] == FAILURE_START) and np.all(np.abs(start[~in_chosen]) <= 1.5)
    pos, st = oracle_result(oracle, ("mixed",), q, dict(gradient_tolerance=-1.0), start)["literal"]
    failed = np.nonzero(st["termination"] == FAILURE)[0]
    assert np.array_equal(failed, np.sort(chosen))
    assert np.all(st["iterations"][chosen] == 10)
    assert np.array_equal(pos[in_chosen], start[in_chosen])
    others = (sizes > 1) & ~np.isin(np.arange(q.n_components), chosen)
    assert set(st["termination"][others].tolist()) <= {PARAMETER_TOL, FUNCTION_TOL}
    assert np.all(st["iterations"][others] > 0)


# ---------------------------------------------------------------------------------------------------
# GPU: scenes x routes x option sets x start points
# ---------------------------------------------------------------------------------------------------
_max_dx = [0.0]


@pytest.mark.gpu
@pytest.mark.parametrize("opt_name", list(OPTION_SETS))
@pytest.mark.parametrize("name", list(SCENES))
def test_every_route_matches_oracle(b200, oracle, name, opt_name):
    """One scene and option set, from zeros and from the random start, through every route."""
    p = scene(name)
    worst, ambiguous = 0.0, 0
    for kind in ("zero", "random"):
        start = start_of(name, kind)
        ref = scene_oracle(oracle, name, opt_name, kind)
        for route in ROUTES:
            got = b200.solve(p, options(b200, route, **OPTION_SETS[opt_name]), positions=start)
            # The CTA tier's PCG step equals the Cholesky step to the last few bits.  Under tolerances of
            # 1e-10 components iterate down to that level, where a line search that contracts to its
            # minimum step size can take one step more or fewer (cfg1 from zeros: 10 against 11) with the
            # same iterations, terminations and positions; the step totals are held to 1 % there.
            exact = not (route == "cta" and opt_name == "tight_tolerances")
            dx, amb = assert_agree(p, start, got, ref, (name, opt_name, kind, route), exact)
            worst, ambiguous = max(worst, dx), max(ambiguous, amb)
    _max_dx[0] = max(_max_dx[0], worst)
    print("%s %s: max |dx| %.2e units (largest so far %.2e); %d components where the oracle's modes disagree"
          % (name, opt_name, worst, _max_dx[0], ambiguous))


# ---------------------------------------------------------------------------------------------------
# GPU: proof of route, and every tier at every termination code
# ---------------------------------------------------------------------------------------------------
def _profiled(b200, key, p, route, opts, start):
    return _cached(("profiled", route) + tuple(key), lambda: profiled_solve(b200, p, options(b200, route, True, **opts),
                                                                           start))


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("name", list(SCENES))
def test_profile_proves_the_route(b200, name, route):
    """From the random start, a plan created with LFR_DBG_PROFILE (and the start as its initial positions)
    gives bitwise the plain lfr_solve results, and every solved slot ran on the tier the route sends it
    to: tier 4 under linear_solver = 2, tier 3 for n <= 96 under FORCE_SMEM_CHOLESKY, tier 2 for
    n <= 32 under TILE_FROM = 1; the default route on ring60 reaches all four tiers."""
    p, start = scene(name), start_of(name, "random")
    plain = b200.solve(p, options(b200, route), positions=start)
    pos, st, rec = _profiled(b200, (name, "defaults", "random"), p, route, {}, start)
    assert_bitwise(plain, (pos, st), (name, route, "profiled plan"))
    n2 = 2 * free_count(p)
    solved = (sizes_of(p) > 1) & (n2 > 0)
    want = np.array([expected_tier(int(n), route) for n in n2])
    assert np.array_equal(rec["tier"][solved], want[solved]), \
        (name, route, sorted(set(zip(n2[solved].tolist(), rec["tier"][solved].tolist(), want[solved].tolist()))))
    assert np.all(rec["tier"][~solved] == 0)
    assert int(rec["ls_steps"].sum()) == st["total_line_search_steps"]
    if route == "cta":
        assert np.all(rec["counter"][solved] > 0)   # CG iterations
    if route == "tile_from_1":
        assert (rec["tier"][solved & (n2 <= 32)] == TIER_TILE).sum() > 0
    if name == "ring60" and route == "default":
        assert set(rec["tier"][solved].tolist()) == {TIER_WARP2, TIER_TILE, TIER_WARP, TIER_CTA}
    print("%s %s: tiers %s" % (name, route, dict(zip(*np.unique(rec["tier"][solved], return_counts=True)))))


@pytest.mark.gpu
def test_every_tier_reaches_every_termination_code(b200, oracle):
    """Profiled solves of the four scenes from the random start under the defaults, gradient_tolerance =
    1e-2, min_trust_region_radius = 2e4 and max_num_iterations = 1, and of the FAILURE problems, on every
    route: each tier 1-4 ends components with every code 1-6, and each profiled run ends every
    component as the oracle does."""
    table = np.zeros((5, 8), np.int64)

    def add(p, st, rec, ref_st):
        assert np.array_equal(st["termination"], ref_st["termination"])
        assert np.array_equal(st["iterations"], ref_st["iterations"])
        np.add.at(table, (rec["tier"], st["termination"]), 1)

    for route in ROUTES:
        for name in SCENES:
            p, start = scene(name), start_of(name, "random")
            for opt_name in TABLE_OPTION_SETS:
                pos, st, rec = _profiled(b200, (name, opt_name, "random"), p, route, OPTION_SETS[opt_name], start)
                add(p, st, rec, scene_oracle(oracle, name, opt_name, "random")["fast"][1])
        for name in ("cfg1", "ring60"):
            q = failure_problem(name)
            start = np.full((q.graph.n_nodes, 2), FAILURE_START)
            opts = dict(gradient_tolerance=-1.0)
            pos, st, rec = _profiled(b200, ("failure", name), q, route, opts, start)
            add(q, st, rec, oracle_result(oracle, ("failure", name), q, opts, start)["fast"][1])
    codes = list(range(1, 7))
    print("tier \\ termination  " + " ".join("%14s" % n for n in ("gradient_tol", "parameter_tol", "function_tol",
                                                                 "min_radius", "no_convergence", "failure")))
    for t, tn in ((TIER_WARP2, "warp2"), (TIER_TILE, "tile"), (TIER_WARP, "warp"), (TIER_CTA, "cta")):
        print("%d %-17s " % (t, tn) + " ".join("%14d" % table[t, c] for c in codes))
    assert np.all(table[1:5, 1:7] > 0), table[1:5, 1:7]


# ---------------------------------------------------------------------------------------------------
# GPU: terminations that need a constructed problem
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg1", "ring60"])
def test_failure_keeps_the_start_on_every_tier(b200, oracle, name):
    """The FAILURE construction on every route: every component of more than one node ends in FAILURE
    after 10 iterations, as in the oracle, and every node keeps 1.7 bitwise (a write-back would leave
    1.0).  The profile records FAILURE on all four tiers."""
    q = failure_problem(name)
    start = np.full((q.graph.n_nodes, 2), FAILURE_START)
    opts = dict(gradient_tolerance=-1.0)
    ref = oracle_result(oracle, ("failure", name), q, opts, start)
    solved = sizes_of(q) > 1
    tiers = set()
    for route in ROUTES:
        got = b200.solve(q, options(b200, route, **opts), positions=start)
        assert_agree(q, start, got, ref, ("failure", name, route))
        pos, st = got
        assert np.array_equal(pos, start), route
        assert np.all(st["termination"][solved] == FAILURE) and np.all(st["iterations"][solved] == 10), route
        pos_p, st_p, rec = _profiled(b200, ("failure", name), q, route, opts, start)
        assert_bitwise(got, (pos_p, st_p), ("failure", name, route, "profiled plan"))
        tiers |= set(rec["tier"][solved].tolist())
    assert tiers == {TIER_WARP2, TIER_TILE, TIER_WARP, TIER_CTA}, tiers


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_empty_components_on_every_route(b200, oracle, name):
    """All nodes roots, random start: on every route (linear_solver = 2 goes through the CTA kernel's
    lm_empty) every component of more than one node ends EMPTY after 0 iterations, as in the oracle,
    and every position is the start bitwise.  EMPTY components write no profile record."""
    q, start = empty_problem(name), start_of(name, "random")
    ref = oracle_result(oracle, ("empty", name), q, {}, start)
    solved = sizes_of(q) > 1
    for route in ROUTES:
        got = b200.solve(q, options(b200, route), positions=start)
        assert_agree(q, start, got, ref, ("empty", name, route))
        pos, st = got
        assert np.array_equal(pos, start), route
        assert np.all(st["termination"][solved] == EMPTY) and np.all(st["iterations"] == 0), route
        pos_p, st_p, rec = _profiled(b200, ("empty", name), q, route, {}, start)
        assert_bitwise(got, (pos_p, st_p), ("empty", name, route, "profiled plan"))
        assert np.all(rec["tier"] == 0) and np.all(rec["total"] == 0), route


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_mixed_launch_matches_oracle(b200, oracle, route):
    """FAILURE components next to ordinary ones in the same launches: warps and CTAs end at different
    times with different codes.  Component by component as in the oracle; FAILURE exactly on the chosen
    components, their nodes at 1.7 bitwise."""
    q, start, chosen = mixed_problem()
    opts = dict(gradient_tolerance=-1.0)
    ref = oracle_result(oracle, ("mixed",), q, opts, start)
    got = b200.solve(q, options(b200, route, **opts), positions=start)
    dx, _ = assert_agree(q, start, got, ref, ("mixed", route))
    pos, st = got
    assert np.array_equal(np.nonzero(st["termination"] == FAILURE)[0], np.sort(chosen))
    for s in chosen:
        nodes = slot_nodes(q, s)
        assert np.all(pos[nodes] == FAILURE_START)
    _, _, rec = _profiled(b200, ("mixed",), q, route, opts, start)
    print("mixed %s: max |dx| %.2e units, FAILURE on tiers %s" % (
        route, dx, sorted(set(rec["tier"][chosen].tolist()))))


# ---------------------------------------------------------------------------------------------------
# GPU: API paths from a non-zero start
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_api_paths_from_a_nonzero_start(b200, oracle):
    """The mixed problem from its start (random, and 1.7 on the FAILURE components) through lfr_solve
    with pageable buffers, with pinned buffers through the copy engine and in place (LFR_DBG_ZERO_COPY:
    only free nodes are written, so untouched entries must keep the caller's values), lfr_solve_multi
    on every visible device with pinned and pageable buffers (merged per owner on the host), and a plan
    created with the start as its initial positions, solved twice: bitwise the same positions and
    statistics everywhere, and in agreement with the oracle."""
    import torch
    from lfr_b200 import capi
    q, start, chosen = mixed_problem()
    opts = dict(gradient_tolerance=-1.0)
    ref = oracle_result(oracle, ("mixed",), q, opts, start)
    base = b200.solve(q, options(b200, **opts), positions=start)
    assert_agree(q, start, base, ref, "pageable lfr_solve")
    N = q.graph.n_nodes
    s, keep = b200.marshal(q)
    e_pin = torch.empty(keep["edges"].nbytes, dtype=torch.uint8).pin_memory()
    e_pin.numpy()[:] = keep["edges"].view(np.uint8).reshape(-1)
    s.edges = e_pin.data_ptr()
    for dbg, what in ((0, "pinned lfr_solve"), (capi.DBG_ZERO_COPY, "zero-copy lfr_solve")):
        pos_pin = torch.zeros(2 * N, dtype=torch.float64).pin_memory()
        pos_pin.numpy()[:] = start.reshape(-1)
        st, bufs = b200.make_stats(q.n_components)
        o = b200.default_options(debug_flags=dbg, **opts)
        b200.check(b200.lib.lfr_solve(C.byref(s), C.byref(o), C.c_void_p(pos_pin.data_ptr()), C.byref(st)), what)
        assert_bitwise(base, (pos_pin.numpy().reshape(N, 2).copy(), b200.stats_dict(st, bufs)), what)
    del keep
    n_dev = torch.cuda.device_count()
    for d in range(n_dev):
        for pinned in (True, False):
            got = b200.solve_multi(q, [d], options(b200, **opts), positions=start, pinned=pinned)
            assert_bitwise(base, got, ("lfr_solve_multi", d, pinned))
    plan = capi.Plan(b200, q, options(b200, **opts), positions=start)
    try:
        for k in range(2):
            plan.solve()
            assert_bitwise(base, plan.download(), ("plan", k))
    finally:
        plan.close()


# ---------------------------------------------------------------------------------------------------
# GPU: per-edge evaluation under non-default loss options
# ---------------------------------------------------------------------------------------------------
def _edge_inputs(outliers):
    """test_gpu_parity.py's edge-evaluation inputs; `outliers` makes every edge a Tukey edge with a large
    residual instead (|r|^2 > a^2 for most)."""
    from lfr_b200 import EDGE_DTYPE
    rng = np.random.default_rng(5)
    n = 20000
    e = np.zeros(n, dtype=EDGE_DTYPE)
    e["flow"] = rng.uniform(-0.5, 0.5, size=(n, 18)).astype(np.float32)
    e["sim"] = rng.uniform(0.5, 1.0, size=n).astype(np.float32)
    kind = rng.integers(1, 3, size=n).astype(np.uint8)
    xs = rng.uniform(-0.8, 0.8, size=(n, 2))
    xs[:100] = np.sign(xs[:100]) * 0.5
    xd = rng.uniform(-1, 1, size=(n, 2))
    if outliers:
        kind[:] = 2
    else:
        e["flow"][: n // 2] *= 0.05
        xd[: n // 2] = xs[: n // 2] + rng.normal(0, 0.02, size=(n // 2, 2))
    return e, kind, xs, xd


@pytest.mark.gpu
@pytest.mark.parametrize("case,opts,outliers", [
    ("tukey_variant_2", dict(tukey_variant=2), False),
    ("loss_widths", dict(cauchy_a=0.1, tukey_a=0.2), False),
    ("tukey_outliers", dict(), True),
    ("tukey_outliers_variant_2", dict(tukey_variant=2), True),
])
def test_edge_eval_under_loss_options_matches_oracle(b200, oracle, case, opts, outliers):
    """lfr_debug_edge_eval against the oracle's edge evaluation under the same options: residuals,
    Jacobians, rho and rho' (the kernel leaves rho'' at 0 on purpose: the solve never reads it)."""
    e, kind, xs, xd = _edge_inputs(outliers)
    rg, jg, rhog = b200.edge_eval(e, kind, xs, xd, b200.default_options(**opts))
    ro, jo, rhoo = oracle.edge_eval(e, kind, xs, xd, oracle.default_options(**opts))
    np.testing.assert_allclose(rg, ro, rtol=0, atol=4e-16 * 4)
    np.testing.assert_allclose(jg, jo, rtol=0, atol=1e-14)
    np.testing.assert_allclose(rhog[:, :2], rhoo[:, :2], rtol=1e-13, atol=1e-18)
    tukey_a = opts.get("tukey_a", 0.0625)
    out = (kind == 2) & ((ro ** 2).sum(axis=1) > tukey_a ** 2)
    if outliers:
        assert out.mean() > 0.9
        # the outlier branch: rho = sim * a^2 / 6 (Ceres 1.x) or a^2 / 3 (2.x), rho' = 0
        cap = tukey_a ** 2 / (3.0 if opts.get("tukey_variant", 1) == 2 else 6.0)
        np.testing.assert_allclose(rhog[out, 0], e["sim"][out].astype(np.float64) * cap, rtol=1e-15)
        assert np.all(rhog[out, 1] == 0)
    else:
        assert out.sum() > 1000 and ((kind == 2) & ~out).sum() > 1000
