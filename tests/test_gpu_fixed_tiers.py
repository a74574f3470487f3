"""Fixed images on every solve tier and route, against the reference's create_and_solve_problem and the
CPU checker.

lfr_plan_fix_images ORs the nodes of the fixed images into the constant mask every tier reads as
`is_root` and builds the plan's schedule again: components change tier, warp2 NREG class, or become
EMPTY, and the warp2 tier can switch between its queue launch and per-bucket launches.  This file runs the
mask and start cases of tests/test_fixed_images_ref.py through plans on the five routes of
tests/test_gpu_tier_options.py and checks, on every component:

  * against the checker in its fast line-search mode: positions within 1e-4 px, identical iterations and
    termination codes, initial / final costs to 1e-10 / 1e-8, equal line-search step totals; against its
    literal mode and against the reference function wherever the two modes agree on the trajectory
    (costs against the reference net of its fixed cost); constant nodes keep their start bits.  On the few
    components where the two modes end differently (cfg4, whole_track, joined start: one component whose
    line search hits a near rank-deficient fit), the kernels may follow either mode: positions to 1e-4 px
    against both, iterations and termination of one of them, and the line-search steps of all the other
    components equal to the fast mode's;
  * proof of route (LFR_DBG_PROFILE): the tier each component ran on, with non-root constant nodes in
    every warp2 class, every tile class, the shared-memory Cholesky kernel and the CTA tier;
  * the tier moves the masks make (CTA -> register tiers, tile -> warp2, NREG class to NREG class) and the
    queue / per-bucket switch on cfg2, read from the profile and from lfr_plan_num_launches;
  * the ring1400 components of more than 1024 nodes with a third of the images fixed;
  * lfr_solve through pageable, pinned and zero-copy buffers and lfr_solve_multi on the same mask and
    start: bitwise the plan's solve;
  * sequences of fix / start / solve / encode on one plan: bitwise a fresh plan given only the final
    settings.
"""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import pytest

from lfr_b200 import synth
from lfr_b200 import wire
from lfr_b200.capi import DBG_PROFILE, DBG_ZERO_COPY, Plan
from lfr_b200.graph import host_input_arrays, problem_from_stage
from lfr_b200.solver import assemble_solution
from refsrc_util import ref_solve
from test_fixed_images_ref import (MOVES, SCENES, assert_matches_reference, bits, cases_of, constant_of, joined_start,
                                   mask_cases, moves, planted_solution, unknowns, with_mask)
from test_gpu_cta_limits import natural, ring1400  # noqa: F401  (module fixtures)
from test_gpu_solution_encode import image_facts
from test_gpu_tier_options import (ROUTES, TIER_CTA, TIER_TILE, TIER_WARP, TIER_WARP2, assert_agree, assert_bitwise,
                                   expected_tier, options, oracle_result, profiled_solve)

pytestmark = pytest.mark.gpu

KINDS = ("zero", "joined")
_cache = {}


def cached(key, make):
    if key not in _cache:
        _cache[key] = make()
    return _cache[key]


def scene(b200, name):
    """(MatchSet, the device stage's graph arrays, their Problem, {case: fixed}, {start kind: bytes}) of a scene."""
    def make():
        ms = synth.generate(name, scale=SCENES[name])
        plan = Plan.from_matches(b200, ms)
        g, sizes = plan.export_graph(), plan.sizes
        plan.close()
        skip, _ = host_input_arrays(ms)
        p = problem_from_stage(ms, skip, g, sizes, "device")
        # the zero start as a SolutionFile without entries: every node joins to +0.0
        return ms, g, p, mask_cases(g, len(ms.image_names)), {"zero": b"", "joined": planted_solution(ms, g, 17)}
    return cached(("scene", name), make)


def checkers(oracle, b200, name, case, kind):
    """(Problem with the constant mask, start, {"literal", "fast"} checker results, reference result)."""
    ms, g, p, cases, data = scene(b200, name)
    const = constant_of(g, cases[case])
    x0 = joined_start(ms, g, data[kind])
    q = with_mask(p, const)
    ref = cached(("ref", name, case, kind), lambda: ref_solve(p, const, x0))
    return q, x0, oracle_result(oracle, ("fixed", name, case, kind), q, {}, x0), ref


def plan_solve(plan, ms, fixed, data):
    plan.fix_images(fixed)
    plan.start_from_solution(data, ms.image_names)
    plan.solve()
    return plan.download()


def route_runs(b200, name, route):
    """Profiled plan solves of every case and start on one plan of the route: {(case, kind): (pos, st, rec)},
    plus the profile of the plan's solve before any mask ("roots", "zero")."""
    def make():
        ms, g, p, cases, data = scene(b200, name)
        plan = Plan.from_matches(b200, ms, options=options(b200, route, profile=True))
        try:
            assert np.array_equal(plan.export_graph()["comp_nodes"], g["comp_nodes"])
            plan.solve()
            out = {("roots", "zero"): plan.download() + (plan.profile()[0],)}
            for case in cases_of(name):
                for kind in KINDS:
                    pos, st = plan_solve(plan, ms, cases[case], data[kind])
                    out[(case, kind)] = (pos, st, plan.profile()[0])
        finally:
            plan.close()
        return out
    return cached(("runs", name, route), make)


def assert_agree_where_modes_differ(oracle, q, x0, got, ref_o, ref, agree, what):
    """The bar of test_gpu_tier_options.assert_agree on a solve with components where the checker's two
    line-search modes end differently (a line search whose polynomial fit is near rank-deficient: which
    trial step it takes turns on the last bits of the LM step, so the kernels' linear solvers can follow
    either mode there; tests/test_linesearch_modes.py).  Every other component is held to the full bar
    against the fast mode, the literal mode and the reference function, and its line-search steps (the
    total less the profiled steps of the other components) to the fast mode's.  Those components agree in
    positions to 1e-4 px with both modes and in iterations and termination with one of them."""
    from test_gpu_cta_limits import subset
    from test_gpu_tier_options import TOL_UNITS, per_slot_max, untouched_nodes
    pos, st, rec = got
    (pos_l, st_l), (pos_f, st_f) = ref_o["literal"], ref_o["fast"]
    amb = np.nonzero(~agree)[0]
    assert amb.size <= 2, (what, "components where the checker's modes disagree", amb.tolist())
    for pos_o, st_o in ((pos_f, st_f), (pos_l, st_l)):
        err = per_slot_max(q, np.abs(pos - pos_o).max(axis=1))
        assert err.max() <= TOL_UNITS, (what, int(np.argmax(err)), float(err.max()))
        bad = agree & ((st["iterations"] != st_o["iterations"]) | (st["termination"] != st_o["termination"]))
        assert not bad.any(), (what, np.nonzero(bad)[0].tolist())
        np.testing.assert_allclose(st["initial_cost"], st_o["initial_cost"], rtol=1e-10, atol=1e-14, err_msg=str(what))
        np.testing.assert_allclose(st["final_cost"][agree], st_o["final_cost"][agree], rtol=1e-8, atol=1e-14,
                                   err_msg=str(what))
    for c in amb:
        mine = (int(st["iterations"][c]), int(st["termination"][c]))
        assert mine in {(int(s["iterations"][c]), int(s["termination"][c])) for s in (st_l, st_f)}, (what, int(c), mine)
    fast_amb = sum(oracle_result(oracle, ("one", what, int(c)), subset(q, [c]), {}, x0)["fast"][1]["total_line_search_steps"]
                   for c in amb)
    assert st["total_line_search_steps"] - int(rec["ls_steps"][amb].sum()) == st_f["total_line_search_steps"] - fast_amb, what
    assert st["n_solved"] == st_f["n_solved"]
    keep = untouched_nodes(q, st["termination"])
    assert np.array_equal(pos[keep], x0[keep]), (what, "untouched nodes moved")
    print("%s: components %s end as the checker's %s mode" % (
        what, amb.tolist(), ["literal" if st["termination"][c] == st_l["termination"][c] else "fast" for c in amb]))
    return float(per_slot_max(q, np.abs(pos - pos_l).max(axis=1)).max())


# ---------------------------------------------------------------------------------------------------
# every scene, route, mask case and start
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("name", list(SCENES))
def test_fixed_plans_match_the_checkers_on_every_route(b200, oracle, name, route):
    ms, g, p, cases, data = scene(b200, name)
    runs = route_runs(b200, name, route)
    worst = 0.0
    for case in cases_of(name):
        for kind in KINDS:
            what = (name, route, case, kind)
            q, x0, ref_o, ref = checkers(oracle, b200, name, case, kind)
            pos, st, rec = runs[(case, kind)]
            (_, st_l), (_, st_f) = ref_o["literal"], ref_o["fast"]
            agree = (st_l["iterations"] == st_f["iterations"]) & (st_l["termination"] == st_f["termination"])
            if agree.all():
                dx, _ = assert_agree(q, x0, (pos, st), ref_o, what)
            else:
                dx = assert_agree_where_modes_differ(oracle, q, x0, (pos, st, rec), ref_o, ref, agree, what)
            worst = max(worst, dx, assert_matches_reference(q, (pos, st), ref, what, sel=agree, cost_rtol=(1e-10, 1e-8),
                                                            ls_steps=False))
            c = q.is_root != 0
            assert np.array_equal(bits(pos[c]), bits(x0[c])), (what, "constant nodes moved")
            # proof of route: every solved slot on the tier its unknowns under the mask send it to
            n2 = unknowns(g, q.is_root)
            solved = (np.diff(q.comp_ptr.astype(np.int64)) > 1) & (n2 > 0)
            want = np.array([expected_tier(int(n), route) for n in n2])
            assert np.array_equal(rec["tier"][solved], want[solved]), (what, "tiers")
            assert np.all(rec["tier"][~solved] == 0), (what, "records of EMPTY or skipped slots")
            assert int(rec["ls_steps"].sum()) == st["total_line_search_steps"], what
    print("%s %s: max |dx| %.2e units" % (name, route, worst))


def test_fixed_masks_reach_every_tier(b200):
    """On the default route, slots holding a non-root constant node ran in every warp2 class (8 / 16 / 24 /
    32 unknowns), every tile class (48 / 64 / 80), on the shared-memory Cholesky warp kernel and on the
    CTA tier."""
    reached = set()
    for name in SCENES:
        ms, g, p, cases, data = scene(b200, name)
        runs = route_runs(b200, name, "default")
        root = g["is_root"] != 0
        for case in cases_of(name):
            const = constant_of(g, cases[case]) != 0
            per_node = (const & ~root)[g["comp_nodes"].astype(np.int64)].astype(np.int64)
            sizes = np.diff(g["comp_ptr"].astype(np.int64))
            has_fixed = np.zeros(sizes.shape[0], bool)
            has_fixed[sizes > 0] = np.add.reduceat(per_node, g["comp_ptr"][:-1][sizes > 0].astype(np.int64)) > 0
            n2 = unknowns(g, const)
            for kind in KINDS:
                tier = runs[(case, kind)][2]["tier"]
                for c in np.nonzero(has_fixed & (tier > 0))[0]:
                    t = int(tier[c])
                    cls = {TIER_WARP2: (int(n2[c]) + 7) // 8 * 8, TIER_TILE: 48 if n2[c] <= 48 else (64 if n2[c] <= 64 else 80),
                           TIER_WARP: 96, TIER_CTA: 0}[t]
                    reached.add((t, cls))
    want = {(TIER_WARP2, 8), (TIER_WARP2, 16), (TIER_WARP2, 24), (TIER_WARP2, 32), (TIER_TILE, 48), (TIER_TILE, 64),
            (TIER_TILE, 80), (TIER_WARP, 96), (TIER_CTA, 0)}
    assert reached >= want, sorted(want - reached)
    print("reached with fixed nodes:", sorted(reached))


def test_masks_move_components_between_tiers(b200):
    """The profiled tier of a slot before any mask and under the tier_moves case: some slot leaves the CTA
    tier for a register tier, some leaves the tile tier for warp2, some changes warp2 NREG class — each
    move as the mask's unknown counts predict (and each moved slot matched the checkers above)."""
    seen = set()
    for name in SCENES:
        ms, g, p, cases, data = scene(b200, name)
        if "tier_moves" not in cases:
            continue
        runs = route_runs(b200, name, "default")
        before = runs[("roots", "zero")][2]["tier"]
        const = constant_of(g, cases["tier_moves"])
        predicted = moves(g, const)
        for kind in KINDS:
            after = runs[("tier_moves", kind)][2]["tier"]
            for m, slots in predicted.items():
                if not slots.size:
                    continue
                if m == "cta_to_register":
                    assert np.all(before[slots] == TIER_CTA) and np.all(np.isin(after[slots], [TIER_WARP2, TIER_TILE])), name
                elif m == "tile_to_warp2":
                    assert np.all(before[slots] == TIER_TILE) and np.all(after[slots] == TIER_WARP2), name
                else:
                    assert np.all(before[slots] == TIER_WARP2) and np.all(after[slots] == TIER_WARP2), name
                seen.add(m)
    assert seen == set(MOVES), seen


def test_cfg2_mask_switches_the_queue_for_bucket_launches(b200, oracle):
    """cfg2 holds warp2 components of more than 16 unknowns, which the queue kernel runs; with every third
    image fixed none is left, the schedule goes back to per-bucket launches and lfr_plan_num_launches
    changes.  An all-zero mask restores the first schedule.  Both solves match the checker."""
    ms, g, p, cases, data = scene(b200, "cfg2")
    n0 = unknowns(g, g["is_root"])
    n1 = unknowns(g, constant_of(g, cases["every_third"]))
    assert ((n0 > 16) & (n0 <= 32)).any() and not ((n1 > 16) & (n1 <= 32)).any()
    plan = Plan.from_matches(b200, ms)
    try:
        before = plan.num_launches()
        plan.fix_images(cases["every_third"])
        during = plan.num_launches()
        q, x0, ref_o, _ = checkers(oracle, b200, "cfg2", "every_third", "joined")
        plan.start_from_solution(data["joined"], ms.image_names)
        plan.solve()
        assert_agree(q, x0, plan.download(), ref_o, "cfg2 every_third")
        plan.fix_images(np.zeros(len(ms.image_names), bool))
        after = plan.num_launches()
    finally:
        plan.close()
    assert during != before and after == before, (before, during, after)
    print("cfg2 launches: %d with the reference's roots, %d with every third image fixed" % (before, during))


# ---------------------------------------------------------------------------------------------------
# past 1024 nodes
# ---------------------------------------------------------------------------------------------------
def test_natural_components_over_1024_nodes_with_fixed_images(b200, oracle, natural):  # noqa: F811
    """ring1400's natural components (every one over 1024 nodes and every 8th other), every third image
    fixed, from a random start outside the box: the CTA tier against the checker on every component, and
    the smallest component over 1024 nodes against the reference function too."""
    from test_gpu_cta_limits import ROWS_CACHED, assert_agree as agree_cta, slot_nodes, subset
    q = natural
    node_image = q.graph.node_image.astype(np.int64)
    fixed = np.arange(int(node_image.max()) + 1) % 3 == 0
    const = ((q.is_root != 0) | fixed[node_image]).astype(np.uint8)
    qc = with_mask(q, const)
    x0 = np.random.default_rng(1400).uniform(-1.5, 1.5, (q.graph.n_nodes, 2))
    sizes = np.diff(q.comp_ptr.astype(np.int64))
    n2 = np.array([2 * int((const[slot_nodes(q, s)] == 0).sum()) for s in range(q.n_components)])
    assert ((sizes > ROWS_CACHED) & (n2 > 96)).sum() >= 25
    pos_g, st_g = b200.solve(qc, positions=x0)
    pos_o, st_o = oracle.solve(qc, oracle.default_options(n_threads=os.cpu_count() or 8), positions=x0)
    err = agree_cta(qc, pos_g, st_g, pos_o, st_o)
    c = const != 0
    assert np.array_equal(bits(pos_g[c]), bits(x0[c]))
    # proof of route: a profiled plan from the same start, bitwise the same, the CTA tier above 96 unknowns
    pos_p, st_p, rec = profiled_solve(b200, qc, options(b200, "default", True), x0)
    assert_bitwise((pos_g, st_g), (pos_p, st_p), "ring1400 profiled plan")
    assert np.all(rec["tier"][n2 > 96] == TIER_CTA) and np.all(rec["counter"][n2 > 96] > 0)
    # the smallest component over 1024 nodes against the reference function (and the checker's two
    # line-search modes: iterations and terminations are compared where those agree)
    big = int(np.nonzero(sizes > ROWS_CACHED)[0][-1])
    one = subset(qc, [big])
    ref = ref_solve(one, const, x0)
    got = b200.solve(one, positions=x0)
    ref_o = oracle_result(oracle, ("ring1400", big), one, {}, x0)
    (_, st_l), (_, st_f) = ref_o["literal"], ref_o["fast"]
    agree = (st_l["iterations"] == st_f["iterations"]) & (st_l["termination"] == st_f["termination"])
    assert_agree(one, x0, got, ref_o, ("ring1400", big))
    assert_matches_reference(one, got, ref, ("ring1400", big), sel=agree, cost_rtol=(1e-10, 1e-8), ls_steps=False)
    assert np.abs(got[0] - ref[0]).max() <= 1e-4 / 16
    print("ring1400 with every third image fixed: %d components, max |dx| %.2e units; the %d-node one (%d unknowns) "
          "matches the reference function" % (q.n_components, err.max(), sizes[big], n2[big]))


# ---------------------------------------------------------------------------------------------------
# API routes on the same mask and start
# ---------------------------------------------------------------------------------------------------
def test_solve_routes_agree_with_the_plan(b200):
    """ring60 with every third image fixed, from the joined start: lfr_solve with the mask as is_root
    through pageable, pinned and zero-copy buffers, and lfr_solve_multi([0]), bitwise the plan's solve."""
    import torch
    ms, g, p, cases, data = scene(b200, "ring60")
    const = constant_of(g, cases["every_third"])
    x0 = joined_start(ms, g, data["joined"])
    q = with_mask(p, const)
    plan = Plan.from_matches(b200, ms)
    try:
        base = plan_solve(plan, ms, cases["every_third"], data["joined"])
    finally:
        plan.close()
    assert_bitwise(base, b200.solve(q, positions=x0), "pageable lfr_solve")
    N = q.graph.n_nodes
    s, keep = b200.marshal(q)
    e_pin = torch.empty(keep["edges"].nbytes, dtype=torch.uint8).pin_memory()
    e_pin.numpy()[:] = keep["edges"].view(np.uint8).reshape(-1)
    s.edges = e_pin.data_ptr()
    for dbg, what in ((0, "pinned lfr_solve"), (DBG_ZERO_COPY, "zero-copy lfr_solve")):
        pos_pin = torch.zeros(2 * N, dtype=torch.float64).pin_memory()
        pos_pin.numpy()[:] = x0.reshape(-1)
        st, bufs = b200.make_stats(q.n_components)
        o = b200.default_options(debug_flags=dbg)
        b200.check(b200.lib.lfr_solve(C.byref(s), C.byref(o), C.c_void_p(pos_pin.data_ptr()), C.byref(st)), what)
        assert_bitwise(base, (pos_pin.numpy().reshape(N, 2).copy(), b200.stats_dict(st, bufs)), what)
    del keep
    for pinned in (False, True):
        assert_bitwise(base, b200.solve_multi(q, [0], positions=x0, pinned=pinned), ("lfr_solve_multi", pinned))


# ---------------------------------------------------------------------------------------------------
# plan state sequences
# ---------------------------------------------------------------------------------------------------
def _result(plan, ms, fact):
    pos, st = plan.download()
    return pos, st, plan.encode_solution(ms.image_names, fact)[0]


def _assert_same(a, b, what):
    assert_bitwise(a[:2], b[:2], what)
    assert a[2] == b[2], (what, "encoded bytes")


def test_plan_state_sequences(b200):
    """On cfg4 x 0.25, each sequence of fix / start / solve on one plan gives bitwise the positions, the
    statistics and the encoded SolutionFile of a fresh plan given only its final settings; a start encodes
    before any solve as the host encodes the joined start; a profiled plan refixed reports the tiers of its
    last solve only."""
    import torch
    ms, g, p, cases, data = scene(b200, "cfg4")
    fact = image_facts(ms)
    A, B = cases["every_third"], cases["tier_moves"]
    S1, S2 = data["joined"], planted_solution(ms, g, 29)
    none = np.zeros(len(ms.image_names), bool)

    def fresh(fixed, start, profile=False):
        plan = Plan.from_matches(b200, ms, options=b200.default_options(debug_flags=DBG_PROFILE if profile else 0))
        try:
            if fixed is not None:
                plan.fix_images(fixed)
            if start is not None:
                plan.start_from_solution(start, ms.image_names)
            plan.solve()
            return _result(plan, ms, fact) + ((plan.profile()[0],) if profile else ())
        finally:
            plan.close()

    def sequence(steps, profile=False):
        plan = Plan.from_matches(b200, ms, options=b200.default_options(debug_flags=DBG_PROFILE if profile else 0))
        try:
            for op, arg in steps:
                {"fix": lambda a: plan.fix_images(a), "start": lambda a: plan.start_from_solution(a, ms.image_names),
                 "solve": lambda a: plan.solve()}[op](arg)
            return _result(plan, ms, fact) + ((plan.profile()[0],) if profile else ())
        finally:
            plan.close()

    want_B = fresh(B, None, profile=True)
    got = sequence([("fix", A), ("solve", None), ("fix", B), ("solve", None)], profile=True)
    _assert_same(got, want_B, "fix A, solve, fix B, solve")
    for k in ("tier", "ls_steps"):
        assert np.array_equal(got[3][k], want_B[3][k]), ("profile after a refix", k)
    _assert_same(sequence([("start", S1), ("solve", None), ("start", S2), ("solve", None)]), fresh(None, S2),
                 "start S1, solve, start S2, solve")
    want_AS = fresh(A, S1)
    _assert_same(sequence([("start", S1), ("fix", A), ("solve", None)]), want_AS, "start, fix, solve")
    _assert_same(sequence([("fix", A), ("start", S1), ("solve", None)]), want_AS, "fix, start, solve")
    _assert_same(sequence([("fix", A), ("start", S1), ("solve", None), ("solve", None)]), want_AS, "solve twice")
    _assert_same(sequence([("solve", None), ("solve", None)]), fresh(None, None), "solve twice, no mask or start")
    _assert_same(sequence([("fix", B), ("solve", None), ("fix", none), ("start", S1), ("solve", None)]), fresh(None, S1),
                 "fix B, solve, unfix, start, solve")
    # a start encodes before any solve as the host encodes the joined start
    plan = Plan.from_matches(b200, ms)
    try:
        plan.fix_images(A)
        plan.start_from_solution(S1, ms.image_names)
        x0 = joined_start(ms, g, S1)
        assert plan.download()[0].tobytes() == x0.tobytes()
        graph = SimpleNamespace(n_nodes=plan.n_nodes, node_image=g["node_image"].astype(np.int64), node_feat=g["node_feat"],
                                image_names=ms.image_names, image_fact=fact)
        sol = assemble_solution(SimpleNamespace(graph=graph), x0)
        want = wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj)
        assert plan.encode_solution(ms.image_names, fact)[0] == want
    finally:
        plan.close()
    # start and solve on a non-default stream
    stream = torch.cuda.Stream()
    plan = Plan.from_matches(b200, ms)
    try:
        plan.fix_images(A)
        plan.start_from_solution(S1, ms.image_names, stream=stream.cuda_stream)
        plan.solve(stream=stream.cuda_stream)
        pos, st = plan.download(stream=stream.cuda_stream)
        _assert_same((pos, st, plan.encode_solution(ms.image_names, fact, stream=stream.cuda_stream)[0]), want_AS,
                     "non-default stream")
    finally:
        plan.close()
