"""Keeping an earlier SolutionFile on the GPU: lfr_plan_keep_solution's device join against the host entries
join (bitwise), kept-solution plans against the GPU host route (lfr_solve with the composed mask, bitwise)
and the CPU checker, on every tier the kept set leaves or moves components to (proven by LFR_DBG_PROFILE),
its composition with lfr_plan_fix_images and lfr_plan_start_from_solution, and the incremental scenario with
--keep_initial_solution through both drop-in hosts and both routes."""
import os

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import Plan
from lfr_b200.graph import host_input_arrays, host_stage_export, problem_from_stage
from lfr_b200.solver import assemble_solution
from test_fixed_images import displacement, image, random_solution
from test_fixed_images_ref import bits, moves, sizes_of, unknowns
from test_gpu_fixed_images import EMPTY, TOL, _run, plan_and_graph, scene
from test_gpu_tier_options import TIER_CTA, TIER_TILE, TIER_WARP2, options

pytestmark = pytest.mark.gpu


def any_scene(name):
    if name == "ring60":       # components of more than 96 unknowns (tests/test_gpu_fixed_tiers.py's scale)
        return synth.generate("ring60", scale=0.3), ()
    return scene(name)


def kept_file(ms, g, seed, whole=(0,), frac=0.2):
    """A SolutionFile listing every feature of the images in `whole` and a `frac` share of the others'."""
    rng = np.random.default_rng(seed)
    node_image, node_feat = g["node_image"].astype(np.int64), g["node_feat"]
    msgs = []
    for k, nm in enumerate(ms.image_names):
        feats = node_feat[node_image == k]
        if k not in whole:
            feats = feats[rng.random(feats.shape[0]) < frac]
        vals = rng.uniform(-0.6, 0.6, (feats.shape[0], 2)).astype(np.float32)
        msgs.append(image(nm, [displacement(f, a, b) for f, (a, b) in zip(feats.tolist(), vals)]))
    return b"".join(msgs)


def composed(ms, g, data, fixed_ids=()):
    """(is_const = root OR fixed image OR entry, joined start, has_entry), from the host entries join."""
    start, _, has = wire.join_solution(data, ms.image_names, g["node_image"], g["node_feat"], entries=True)
    fixed = np.zeros(len(ms.image_names), bool)
    fixed[list(fixed_ids)] = True
    const = (g["is_root"] != 0) | fixed[g["node_image"].astype(np.int64)] | has
    return const.astype(np.uint8), start, has


def host_problem(ms, banned, g, sizes, is_const):
    skip, _ = host_input_arrays(ms, banned)
    p = problem_from_stage(ms, skip, g, sizes, "device")
    p.is_root = is_const
    return p


def assert_same(a, b, what):
    assert a[0].tobytes() == b[0].tobytes(), what
    for k in ("iterations", "termination"):
        assert np.array_equal(a[1][k], b[1][k]), (what, k)


# ---------------------------------------------------------------------------------------------------
# the device join
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg1", "cfg2x0.1", "cfg2x0.1-banned", "adv:star_200_descending", "adv:duplicates"])
def test_keep_join_equals_host_entries_join(b200, name):
    ms, banned = scene(name)
    plan, g = plan_and_graph(b200, ms, banned)
    data = random_solution(ms, g, np.random.default_rng(6))
    want, n_want, has = wire.join_solution(data, ms.image_names, g["node_image"], g["node_feat"], entries=True)
    assert plan.keep_solution(data, ms.image_names) == n_want == int(has.sum())
    assert plan.download()[0].tobytes() == want.tobytes()
    assert np.array_equal(plan.export_graph()["is_root"], g["is_root"])       # export keeps the reference roots
    plan.close()


def test_keep_join_of_multi_part_input(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    half = ms.n_pairs // 2
    plan = Plan.from_wire(b200, [wire.encode_matching_file(ms, 0, half), wire.encode_matching_file(ms, half, ms.n_pairs)])
    g = plan.export_graph()
    data = random_solution(ms, g, np.random.default_rng(9))
    want, n_want = wire.join_solution(data, plan.image_names, g["node_image"], g["node_feat"])
    assert plan.keep_solution(data, plan.image_names) == n_want
    assert plan.download()[0].tobytes() == want.tobytes()
    plan.close()


def test_keep_refuses_malformed_bytes_and_leaves_the_plan(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    plan, g = plan_and_graph(b200, ms)
    data = kept_file(ms, g, 1)
    plan.keep_solution(data, ms.image_names)
    with pytest.raises(RuntimeError):
        plan.keep_solution(b"\x0a\xff\xff\xff\xff\x0f not a protobuf", ms.image_names)
    plan.solve()
    got = plan.download()
    ref, _ = plan_and_graph(b200, ms)
    ref.keep_solution(data, ms.image_names)
    ref.solve()
    assert_same(got, ref.download(), "after a refused call")
    plan.close()
    ref.close()


# ---------------------------------------------------------------------------------------------------
# plan solves against the host route and the checker
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg2x0.1", "cfg4x0.25", "adv:star_200_descending", "ring60"])
def test_kept_plan_matches_the_host_route_and_the_checker(b200, oracle, name):
    ms, banned = any_scene(name)
    plan = Plan.from_matches(b200, ms, banned_images=banned, options=options(b200, "default", profile=True))
    g = plan.export_graph()
    data = kept_file(ms, g, 13, whole=(0,), frac=0.05 if name == "ring60" else 0.3)
    const, start, has = composed(ms, g, data)
    assert has.any() and not const.all()
    assert plan.keep_solution(data, ms.image_names) == int(has.sum())
    plan.solve()
    pos, st = plan.download()
    rec = plan.profile()[0]
    p = host_problem(ms, banned, g, plan.sizes, const)
    assert_same((pos, st), b200.solve(p, positions=start), name)
    pos_o, st_o = oracle.solve(p, oracle.default_options(n_threads=8), positions=start)
    assert np.abs(pos - pos_o).max() <= TOL
    assert np.array_equal(st["iterations"], st_o["iterations"]) and np.array_equal(st["termination"], st_o["termination"])
    c = const.astype(bool)
    assert np.array_equal(bits(pos[c]), bits(start[c]))                    # kept nodes: their values in the file
    free = ~c
    assert (pos[free] != start[free]).any()
    # components of more than 96 unknowns under the kept set ran on the CTA tier (ring60 has many; cfg4's
    # are capped at its 38 images)
    n2 = unknowns(g, const)
    assert np.all(rec["tier"][n2 > 96] == TIER_CTA) and np.all(rec["counter"][n2 > 96] > 0)
    if name == "ring60":
        assert (n2 > 96).sum() >= 10
    plan.close()


def test_kept_set_moves_components_between_tiers(b200, oracle):
    """ring60 with image 0 and a fifth of the other keypoints kept: slots leave the CTA tier for a register
    tier, leave the tile tier for warp2 and change warp2 NREG class, as the unknown counts predict (the
    profiled tier of each slot before and after), and the moved plan matches the host route and the checker."""
    ms, _ = any_scene("ring60")
    plan = Plan.from_matches(b200, ms, options=options(b200, "default", profile=True))
    g = plan.export_graph()
    plan.solve()
    before = plan.profile()[0]["tier"].copy()
    data = kept_file(ms, g, 7, whole=(0,), frac=0.2)
    const, start, _ = composed(ms, g, data)
    predicted = moves(g, const)
    assert all(v.size for v in predicted.values()), {k: v.size for k, v in predicted.items()}
    plan.keep_solution(data, ms.image_names)
    plan.solve()
    pos, st = plan.download()
    after = plan.profile()[0]["tier"]
    for m, slots in predicted.items():
        if m == "cta_to_register":
            assert np.all(before[slots] == TIER_CTA) and np.all(np.isin(after[slots], [TIER_WARP2, TIER_TILE]))
        elif m == "tile_to_warp2":
            assert np.all(before[slots] == TIER_TILE) and np.all(after[slots] == TIER_WARP2)
        else:
            assert np.all(before[slots] == TIER_WARP2) and np.all(after[slots] == TIER_WARP2)
    p = host_problem(ms, (), g, plan.sizes, const)
    assert_same((pos, st), b200.solve(p, positions=start), "ring60 moved")
    pos_o, st_o = oracle.solve(p, oracle.default_options(n_threads=8), positions=start)
    assert np.abs(pos - pos_o).max() <= TOL
    assert np.array_equal(st["iterations"], st_o["iterations"]) and np.array_equal(st["termination"], st_o["termination"])
    plan.close()


# ---------------------------------------------------------------------------------------------------
# composition with fix_images and start_from_solution
# ---------------------------------------------------------------------------------------------------
def test_composition(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    plan_a, g = plan_and_graph(b200, ms)
    fixed = np.zeros(len(ms.image_names), bool)
    fixed[[1, 9]] = True
    data = kept_file(ms, g, 3, whole=(4,), frac=0.4)
    const, start, _ = composed(ms, g, data, fixed_ids=(1, 9))
    # fix then keep, keep then fix: the same solve, and the host route's with the composed mask
    plan_a.fix_images(fixed)
    plan_a.keep_solution(data, ms.image_names)
    plan_a.solve()
    a = plan_a.download()
    plan_b, _ = plan_and_graph(b200, ms)
    plan_b.keep_solution(data, ms.image_names)
    plan_b.fix_images(fixed)
    plan_b.solve()
    assert_same(a, plan_b.download(), "fix/keep order")
    assert_same(a, b200.solve(host_problem(ms, (), g, plan_a.sizes, const), positions=start), "host route")
    # a later start_from_solution changes only the start values: the kept set stays
    other = random_solution(ms, g, np.random.default_rng(21))
    plan_b.start_from_solution(other, ms.image_names)
    plan_b.solve()
    start2, _ = wire.join_solution(other, ms.image_names, g["node_image"], g["node_feat"])
    assert_same(plan_b.download(), b200.solve(host_problem(ms, (), g, plan_a.sizes, const), positions=start2),
                "keep then start")
    # an empty SolutionFile clears the kept set (and starts from zeros): the fix_images-only plan, bitwise
    assert plan_a.keep_solution(b"", ms.image_names) == 0
    plan_a.solve()
    ref, _ = plan_and_graph(b200, ms)
    ref.fix_images(fixed)
    ref.solve()
    assert_same(plan_a.download(), ref.download(), "empty keep")
    # a plan that never keeps solves as before: the host route with root OR fixed image
    ref.start_from_solution(data, ms.image_names)
    ref.solve()
    const_f, _, _ = composed(ms, g, b"", fixed_ids=(1, 9))
    assert_same(ref.download(), b200.solve(host_problem(ms, (), g, ref.sizes, const_f), positions=start), "never kept")
    # everything kept: every slot is EMPTY and comes back as it went in
    every = kept_file(ms, g, 5, whole=range(len(ms.image_names)))
    plan_a.keep_solution(every, ms.image_names)
    plan_a.solve()
    pos, st = plan_a.download()
    full, _ = wire.join_solution(every, ms.image_names, g["node_image"], g["node_feat"])
    assert pos.tobytes() == full.tobytes() and (st["termination"][sizes_of(g) > 1] == EMPTY).all()
    for pl in (plan_a, plan_b, ref):
        pl.close()


# ---------------------------------------------------------------------------------------------------
# the incremental scenario through both drop-in hosts and both routes
# ---------------------------------------------------------------------------------------------------
def test_incremental_keep_through_both_hosts_and_routes(oracle, tmp_path):
    """Refine cfg2 without images 8-10 (solution A), then the full scene with --initial_solution A
    --keep_initial_solution: every node A lists comes back bit for bit, the old images' keypoints that A
    never matched are refined with the new images, and the four runs write the same bytes."""
    ms = synth.generate("cfg2")
    m, a = tmp_path / "m.pb", tmp_path / "a.pb"
    m.write_bytes(wire.encode_matching_file(ms))
    args = ["--matches_file", str(m), "--output_file", str(a)]
    for nm in ms.image_names[8:11]:
        args += ["--banned_images", nm]
    r = _run(args)
    assert r.returncode == 0, r.stderr
    A = a.read_bytes()
    outs = []
    for python in (False, True):
        for route in ("host", "device"):
            o = tmp_path / ("o_%d_%s.pb" % (python, route))
            r = _run(["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a),
                      "--keep_initial_solution"], python=python, route=route)
            assert r.returncode == 0, r.stderr
            outs.append(o.read_bytes())
    assert all(x == outs[0] for x in outs[1:])
    got = {nm: dict(zip(fi.tolist(), zip(bits(di).tolist(), bits(dj).tolist())))
           for nm, _, fi, di, dj in wire.decode_solution(outs[0])}
    for nm, _, fi, di, dj in wire.decode_solution(A):
        for f, x, y in zip(fi.tolist(), bits(di).tolist(), bits(dj).tolist()):
            assert got[nm][f] == (x, y), (nm, f)
    # the checker on the composed mask and the joined start
    skip, arrs = host_input_arrays(ms)
    rc, g, sz = host_stage_export(arrs, len(ms.image_names))
    assert rc == 0
    p = problem_from_stage(ms, skip, g, sz, "native")
    q = problem_from_stage(ms, skip, g, sz, "native")
    const, start, _ = composed(ms, g, A)
    q.is_root = const
    pos_o, _ = oracle.solve(q, oracle.default_options(n_threads=os.cpu_count() or 8), positions=start)
    old = (g["node_image"] < 8) & (const == 0)
    assert old.any() and (pos_o[old] != 0).any()       # old keypoints A never listed exist, and some move
    sol = assemble_solution(p, pos_o)
    dec = {nm: (fi, di, dj) for nm, _, fi, di, dj in wire.decode_solution(outs[0])}
    moved = 0
    for k, nm in enumerate(sol.image_names):
        lo, hi = int(sol.img_ptr[k]), int(sol.img_ptr[k + 1])
        gfi, gdi, gdj = dec[nm]
        assert np.array_equal(gfi, sol.feature_idx[lo:hi])
        assert np.abs(gdi.astype(np.float64) - sol.di[lo:hi]).max(initial=0) <= TOL
        assert np.abs(gdj.astype(np.float64) - sol.dj[lo:hi]).max(initial=0) <= TOL
        moved += int((gdi != 0).sum())
    assert moved
