"""Updating an earlier SolutionFile on the GPU: lfr_plan_update_solution against the host update
(lfr_wire_update_solution) and the GPU host route (lfr_solve on the composed mask), bitwise, on every tier —
the warp2 queue, tile (TILE_FROM), the shared-memory Cholesky (FORCE_SMEM_CHOLESKY), the single-warp register
tier (NO_TILE), PCG (linear_solver = 2) and the CTA tier past 1024 nodes — with touched and held components in
the same launch.  Touched components solve as the plan never given a file does; held ones come back with the
file's bits.  Also: composition with fix_images in both orders, replacement by a later keep or update, an
empty file, malformed bytes, the device and carried encoders, and the drop-in through both hosts and routes."""
import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import Plan, load_b200
from lfr_b200.graph import host_input_arrays, problem_from_stage
from lfr_b200.solver import assemble_solution
from test_fixed_images import displacement, image
from test_fixed_images_ref import bits
from test_gpu_carry_solution import host_carried
from test_gpu_fixed_images import _run, scene
from test_gpu_keep_solution import assert_same, kept_file
from test_gpu_solution_encode import image_facts
from test_gpu_tier_options import TIER_CTA, TIER_TILE, TIER_WARP, TIER_WARP2, options

pytestmark = pytest.mark.gpu

EMPTY, SKIPPED = 7, 0
SPECIAL_BITS = [0x80000000, 0x00000001, 0x7FC12345, 0x807FFFFF]


def ring1400():
    """1400 images on a ring at 3 % of 2000 keypoints: components of more than 1024 nodes (the scene of
    tests/test_gpu_cta_limits.py)."""
    cfg = synth.SynthConfig("ring1400", 1400, 2000, "ring", 0.7, match_prob=0.3, window=20, n_random=5,
                            vis_halfwidth=12, seed=1400, outlier_match_ratio=0.125)
    return synth.generate(cfg, scale=0.03)


def any_scene(name):
    if name == "ring60":
        return synth.generate("ring60", scale=0.3), ()
    if name == "ring1400":
        return ring1400(), ()
    return scene(name)


def old_file(ms, g, n_new, seed=0, special=True):
    """A SolutionFile listing every keypoint of the images before the last `n_new`, with random values and,
    when `special`, -0.0, a denormal and a NaN payload on the first ones."""
    data = kept_file(ms, g, seed, whole=range(len(ms.image_names) - n_new), frac=0.0)
    if not special:
        return data
    msgs = wire.decode_solution(data)
    out = []
    j = 0
    for nm, fact, fi, di, dj in msgs:
        di, dj = di.copy(), dj.copy()
        for k in range(min(fi.shape[0], 2)):
            di.view(np.uint32)[k] = SPECIAL_BITS[j % 4]
            dj.view(np.uint32)[k] = SPECIAL_BITS[(j + 1) % 4]
            j += 1
        out.append(image(nm, [displacement(f, a, b) for f, a, b in zip(fi.tolist(), di, dj)], fact=fact))
    return b"".join(out)


def host_update(ms, g, data):
    n_comp = int(g["comp_ptr"].shape[0] - 1)
    return wire.update_solution(data, ms.image_names, g["node_image"], g["node_feat"], g["comp"], n_comp)


def host_problem(ms, banned, g, sizes, is_const):
    skip, _ = host_input_arrays(ms, banned)
    p = problem_from_stage(ms, skip, g, sizes, "device")
    p.is_root = np.ascontiguousarray(is_const, np.uint8)
    return p


def touched_slots(g, held):
    """touched by dispatch slot (the index of the per-component stats): comp is the component id of a node,
    comp_order the component id of a slot."""
    comp = g["comp"].astype(np.int64)
    t = np.zeros(int(g["comp_ptr"].shape[0] - 1), bool)
    t[comp[~held]] = True
    return t[g["comp_order"].astype(np.int64)]


# ---------------------------------------------------------------------------------------------------
# the device update against the host update
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg1", "cfg2x0.1", "cfg2x0.1-banned", "cfg4x0.25", "adv:star_200_descending",
                                  "adv:duplicates", "ring60"])
def test_device_update_equals_the_host_update(b200, name):
    ms, banned = any_scene(name)
    plan = Plan.from_matches(b200, ms, banned_images=banned)
    g = plan.export_graph()
    data = old_file(ms, g, max(1, len(ms.image_names) // 8))
    pos, held, n_held, n_touched = host_update(ms, g, data)
    assert plan.update_solution(data, ms.image_names) == (n_held, n_touched)
    assert plan.download()[0].tobytes() == pos.tobytes()                 # start = working positions, before a solve
    assert np.array_equal(plan.export_graph()["is_root"], g["is_root"])  # export keeps the reference roots
    plan.close()


# ---------------------------------------------------------------------------------------------------
# every tier: the host route on the composed mask, and the plain plan on the touched components
# ---------------------------------------------------------------------------------------------------
ROUTE_TIERS = {"default": (TIER_WARP2,), "tile_from_1": (TIER_TILE,), "smem_cholesky": (TIER_WARP,),
               "no_tile": (TIER_WARP,), "cta": (TIER_CTA,)}


@pytest.mark.parametrize("route", list(ROUTE_TIERS))
@pytest.mark.parametrize("name", ["cfg4x0.25", "ring60"])
def test_update_on_every_route_matches_the_host_route_and_the_plain_plan(b200, name, route):
    ms, banned = any_scene(name)
    opts = options(b200, route, profile=True)
    plan = Plan.from_matches(b200, ms, banned_images=banned, options=opts)
    g = plan.export_graph()
    data = old_file(ms, g, max(2, len(ms.image_names) // 6), seed=3)
    start, held, n_held, n_touched = host_update(ms, g, data)
    assert plan.update_solution(data, ms.image_names) == (n_held, n_touched)
    assert 0 < n_held < held.shape[0] and 0 < n_touched
    plan.solve()
    pos, st = plan.download()
    tier = plan.profile()[0]["tier"].copy()
    const = (g["is_root"] != 0) | held
    assert_same((pos, st), b200.solve(host_problem(ms, banned, g, plan.sizes, const), opts, positions=start),
                (name, route))
    # the touched components: the plan never given a file, bit for bit
    plain = Plan.from_matches(b200, ms, banned_images=banned, options=opts)
    plain.solve()
    pos0, st0 = plain.download()
    t = touched_slots(g, held)
    assert pos[~held].tobytes() == pos0[~held].tobytes()
    for k in ("iterations", "termination"):
        assert np.array_equal(st[k][t], st0[k][t]), k
    # held components: the file's bits, no iteration
    assert bits(pos[held]).tobytes() == bits(start[held]).tobytes()
    size = np.diff(g["comp_ptr"].astype(np.int64))
    assert np.all(st["termination"][~t & (size > 1)] == EMPTY) and np.all(st["termination"][~t & (size == 1)] == SKIPPED)
    # the route's tier ran touched components, in the same launch list as the held ones
    assert np.isin(tier[t & (size > 1)], ROUTE_TIERS[route]).any(), (route, np.unique(tier[t]))
    plain.close()
    plan.close()


def test_update_on_the_cta_tier_past_1024_nodes(b200):
    ms, _ = any_scene("ring1400")
    opts = options(b200, "default", profile=True)
    plan = Plan.from_matches(b200, ms, options=opts)
    g = plan.export_graph()
    data = old_file(ms, g, 200, seed=5)
    start, held, n_held, n_touched = host_update(ms, g, data)
    assert plan.update_solution(data, ms.image_names) == (n_held, n_touched)
    plan.solve()
    pos, st = plan.download()
    tier = plan.profile()[0]["tier"].copy()
    size = np.diff(g["comp_ptr"].astype(np.int64))
    t = touched_slots(g, held)
    assert (t & (size > 1024) & (tier == TIER_CTA)).any() and (~t & (size > 1)).any()
    const = (g["is_root"] != 0) | held
    assert_same((pos, st), b200.solve(host_problem(ms, (), g, plan.sizes, const), opts, positions=start), "ring1400")
    plain = Plan.from_matches(b200, ms, options=opts)
    plain.solve()
    pos0, st0 = plain.download()
    assert pos[~held].tobytes() == pos0[~held].tobytes()
    assert np.array_equal(st["iterations"][t], st0["iterations"][t])
    assert bits(pos[held]).tobytes() == bits(start[held]).tobytes()
    plain.close()
    plan.close()


# ---------------------------------------------------------------------------------------------------
# composition, replacement, the empty file, malformed bytes
# ---------------------------------------------------------------------------------------------------
def test_composition_and_replacement(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    fixed = np.zeros(len(ms.image_names), bool)
    fixed[[1, 9]] = True
    plan_a = Plan.from_matches(b200, ms)
    g = plan_a.export_graph()
    data = old_file(ms, g, 3, seed=2)
    start, held, _, _ = host_update(ms, g, data)
    const = (g["is_root"] != 0) | fixed[g["node_image"].astype(np.int64)] | held
    # fix then update, update then fix: the same solve, and the host route's with the composed mask
    plan_a.fix_images(fixed)
    plan_a.update_solution(data, ms.image_names)
    plan_a.solve()
    a = plan_a.download()
    plan_b = Plan.from_matches(b200, ms)
    plan_b.update_solution(data, ms.image_names)
    plan_b.fix_images(fixed)
    plan_b.solve()
    assert_same(a, plan_b.download(), "fix/update order")
    assert_same(a, b200.solve(host_problem(ms, (), g, plan_a.sizes, const), positions=start), "host route")
    # a later keep replaces the held set: the keep-only plan, bitwise
    keep = kept_file(ms, g, 4, whole=(4,), frac=0.4)
    plan_b.keep_solution(keep, ms.image_names)
    plan_b.solve()
    ref = Plan.from_matches(b200, ms)
    ref.fix_images(fixed)
    ref.keep_solution(keep, ms.image_names)
    ref.solve()
    assert_same(plan_b.download(), ref.download(), "update then keep")
    # a later update replaces the kept set: the update-only plan
    ref.update_solution(data, ms.image_names)
    ref.solve()
    assert_same(ref.download(), a, "keep then update")
    # an empty file clears it: every component touched, the fix_images-only plan
    assert plan_a.update_solution(b"", ms.image_names) == (0, int(g["comp_ptr"].shape[0] - 1))
    plan_a.solve()
    only_fix = Plan.from_matches(b200, ms)
    only_fix.fix_images(fixed)
    only_fix.solve()
    assert_same(plan_a.download(), only_fix.download(), "empty update")
    for pl in (plan_a, plan_b, ref, only_fix):
        pl.close()


def test_malformed_bytes_leave_positions_and_mask(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    plan = Plan.from_matches(b200, ms)
    g = plan.export_graph()
    data = old_file(ms, g, 2, seed=6)
    plan.update_solution(data, ms.image_names)
    before = plan.download()[0].copy()
    for bad in (b"\x0a\xff", b"\x0a\xff\xff\xff\xff\x0f not a protobuf"):
        with pytest.raises(RuntimeError):
            plan.update_solution(bad, ms.image_names)
    assert plan.download()[0].tobytes() == before.tobytes()
    plan.solve()
    ref = Plan.from_matches(b200, ms)
    ref.update_solution(data, ms.image_names)
    ref.solve()
    assert_same(plan.download(), ref.download(), "after a refused call")
    plan.close()
    ref.close()


# ---------------------------------------------------------------------------------------------------
# the device and carried encoders
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg2x0.1", "cfg4x0.25"])
def test_encoders_equal_the_host_assembly(b200, name):
    ms, banned = scene(name)
    plan = Plan.from_matches(b200, ms, banned_images=banned)
    g = plan.export_graph()
    data = old_file(ms, g, 3, seed=7)
    plan.update_solution(data, ms.image_names)
    plan.solve()
    fact = image_facts(ms, banned)
    pos, _ = plan.download()
    skip, _ = host_input_arrays(ms, banned)
    s = assemble_solution(problem_from_stage(ms, skip, g, plan.sizes, "device"), pos)
    got, n_out = plan.encode_solution(ms.image_names, fact)
    assert got == wire.encode_solution(s.image_names, s.fact, s.img_ptr, s.feature_idx, s.di, s.dj) and n_out == s.n_outside
    want = host_carried(plan, ms.image_names, fact, data)
    assert plan.encode_solution_carried(ms.image_names, fact, data) == want
    plan.close()


# ---------------------------------------------------------------------------------------------------
# the drop-in through both hosts and both routes
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [[], ["--carry_initial_solution"], ["--fixed_images", 2]], ids=["update", "carry", "fixed"])
def test_incremental_update_through_both_hosts_and_routes(tmp_path, extra):
    """Refine cfg2 without its last 3 images (A), then every pair with --update_initial_solution A: the four
    runs write the same bytes; the touched keypoints are the plain run's, the held ones A's."""
    ms = synth.generate("cfg2")
    extra = [ms.image_names[x] if isinstance(x, int) else x for x in extra]
    m, a = tmp_path / "m.pb", tmp_path / "a.pb"
    m.write_bytes(wire.encode_matching_file(ms))
    args = ["--matches_file", str(m), "--output_file", str(a)]
    for nm in ms.image_names[-3:]:
        args += ["--banned_images", nm]
    r = _run(args)
    assert r.returncode == 0, r.stderr
    A = a.read_bytes()
    outs = []
    for python in (False, True):
        for route in ("host", "device"):
            o = tmp_path / ("o_%d_%s.pb" % (python, route))
            r = _run(["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a),
                      "--update_initial_solution"] + extra, python=python, route=route)
            assert r.returncode == 0, r.stderr
            outs.append(o.read_bytes())
    assert all(x == outs[0] for x in outs[1:])
    o0 = tmp_path / "plain.pb"
    r = _run(["--matches_file", str(m), "--output_file", str(o0)] + [x for x in extra if x != "--carry_initial_solution"],
             route="device")
    assert r.returncode == 0, r.stderr
    plan = Plan.from_matches(load_b200(), ms)
    g = plan.export_graph()
    plan.close()
    _, held, _, n_touched = host_update(ms, g, A)
    assert 0 < n_touched and held.any() and not held.all()
    got = {}
    for nm, _, fi, di, dj in wire.decode_solution(outs[0]):
        got.update({(nm, f): (x, y) for f, x, y in zip(fi.tolist(), di.view(np.uint32).tolist(), dj.view(np.uint32).tolist())})
    plain = {}
    for nm, _, fi, di, dj in wire.decode_solution(o0.read_bytes()):
        plain.update({(nm, f): (x, y) for f, x, y in zip(fi.tolist(), di.view(np.uint32).tolist(), dj.view(np.uint32).tolist())})
    a_t = {}
    for nm, _, fi, di, dj in wire.decode_solution(A):
        a_t.update({(nm, f): (x, y) for f, x, y in zip(fi.tolist(), di.view(np.uint32).tolist(), dj.view(np.uint32).tolist())})
    for v, (i, f) in enumerate(zip(g["node_image"].tolist(), g["node_feat"].tolist())):
        k = (ms.image_names[i], int(f))
        want = a_t[k] if held[v] else plain.get(k, (0, 0))
        assert got.get(k, (0, 0)) == want, k
