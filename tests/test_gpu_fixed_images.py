"""Fixed images and start solutions on the GPU: the device join of lfr_plan_start_from_solution against the
host join (bitwise), plans with lfr_plan_fix_images against the CPU checker and the GPU host route, the
invariants of constant nodes, and the incremental scenario through both drop-in hosts and both routes."""
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import Plan, TERM_NAMES
from lfr_b200.graph import host_input_arrays, problem_from_stage
from lfr_b200.solver import assemble_solution
from test_fixed_images import random_solution
from test_graph_stage_adversarial import CASES, E2E_CASES
from test_ref_solve import LAUNCHER

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT = os.path.join(ROOT, "multi-view-refinement", "build", "solve_native")
TOL = 1e-4 / 16          # 1e-4 px in units of 16 px
EMPTY = [k for k, v in TERM_NAMES.items() if v == "empty"][0]


def scene(name):
    if name.startswith("adv:"):
        return CASES[name[4:]](), ()
    cfg, scale, banned = {"cfg1": ("cfg1", 1.0, ()), "cfg2x0.1": ("cfg2", 0.1, ()), "cfg2": ("cfg2", 1.0, ()),
                          "cfg4x0.25": ("cfg4", 0.25, ()), "cfg2x0.1-banned": ("cfg2", 0.1, (1, 6))}[name]
    ms = synth.generate(cfg, scale=scale, seed=3 if scale < 1 else None)
    return ms, tuple(ms.image_names[k] for k in banned)


SCENES = ["cfg1", "cfg2x0.1", "cfg2", "cfg4x0.25", "cfg2x0.1-banned"] + ["adv:" + c for c in E2E_CASES]


def plan_and_graph(b200, ms, banned=()):
    plan = Plan.from_matches(b200, ms, banned_images=banned)
    return plan, plan.export_graph()


@pytest.mark.parametrize("name", SCENES)
def test_device_join_equals_host_join(b200, name):
    ms, banned = scene(name)
    plan, g = plan_and_graph(b200, ms, banned)
    data = random_solution(ms, g, np.random.default_rng(5))
    want, n_want = wire.join_solution(data, ms.image_names, g["node_image"], g["node_feat"])
    n = plan.start_from_solution(data, ms.image_names)
    pos, _ = plan.download()                      # before any solve: the start point
    assert n == n_want and pos.tobytes() == want.tobytes()
    plan.close()


def test_device_join_of_multi_part_input(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    half = ms.n_pairs // 2
    parts = [wire.encode_matching_file(ms, 0, half), wire.encode_matching_file(ms, half, ms.n_pairs)]
    plan = Plan.from_wire(b200, parts)
    g = plan.export_graph()
    data = random_solution(ms, g, np.random.default_rng(8))
    want, n_want = wire.join_solution(data, plan.image_names, g["node_image"], g["node_feat"])
    assert plan.start_from_solution(data, plan.image_names) == n_want
    assert plan.download()[0].tobytes() == want.tobytes()
    plan.close()


def constant_arrays(ms, g, fixed_ids, data):
    fixed = np.zeros(len(ms.image_names), bool)
    fixed[list(fixed_ids)] = True
    is_const = ((g["is_root"] != 0) | fixed[g["node_image"].astype(np.int64)]).astype(np.uint8)
    start, _ = wire.join_solution(data, ms.image_names, g["node_image"], g["node_feat"])
    return fixed, is_const, start


def host_problem(ms, banned, g, plan, is_const):
    skip, _ = host_input_arrays(ms, banned)
    p = problem_from_stage(ms, skip, g, plan.sizes, "device")
    p.is_root = is_const
    return p


@pytest.mark.parametrize("name", ["cfg1", "cfg2x0.1", "cfg2", "cfg4x0.25", "adv:star_200_descending"])
def test_fixed_plan_matches_the_checker_and_the_host_route(b200, oracle, name):
    ms, banned = scene(name)
    plan, g = plan_and_graph(b200, ms, banned)
    data = random_solution(ms, g, np.random.default_rng(13))
    fixed, is_const, start = constant_arrays(ms, g, range(0, len(ms.image_names), 3), data)
    plan.fix_images(fixed)
    plan.start_from_solution(data, ms.image_names)
    plan.solve()
    pos, st = plan.download()
    assert (g["is_root"] == plan.export_graph()["is_root"]).all()      # export keeps the reference's roots
    p = host_problem(ms, banned, g, plan, is_const)
    pos_o, st_o = oracle.solve(p, oracle.default_options(n_threads=8), positions=start)
    assert np.abs(pos - pos_o).max() <= TOL
    assert np.array_equal(st["iterations"], st_o["iterations"]) and np.array_equal(st["termination"], st_o["termination"])
    pos_h, st_h = b200.solve(p, positions=start)
    assert pos.tobytes() == pos_h.tobytes()
    assert np.array_equal(st["iterations"], st_h["iterations"])
    c = is_const.astype(bool)
    assert pos[c].tobytes() == start[c].tobytes()                      # constant nodes keep their start bits
    plan.close()


def test_every_image_fixed_and_the_all_zero_mask(b200):
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    plan, g = plan_and_graph(b200, ms)
    data = random_solution(ms, g, np.random.default_rng(2))
    plan.start_from_solution(data, ms.image_names)
    start = plan.download()[0]
    plan.fix_images(np.ones(len(ms.image_names), bool))
    plan.solve()
    pos, st = plan.download()
    assert pos.tobytes() == start.tobytes()
    sizes = np.diff(g["comp_ptr"].astype(np.int64))
    assert (st["termination"][sizes > 1] == EMPTY).all()
    # an all-zero mask solves as a plan never given one
    ref, _ = plan_and_graph(b200, ms)
    ref.start_from_solution(data, ms.image_names)
    ref.solve()
    want, st_want = ref.download()
    plan.fix_images(np.zeros(len(ms.image_names), bool))
    plan.solve()
    got, st_got = plan.download()
    assert got.tobytes() == want.tobytes() and np.array_equal(st_got["iterations"], st_want["iterations"])
    plan.close()
    ref.close()


def _run(args, python=False, route=None):
    env = dict(os.environ)
    if route:
        env["LFR_GRAPH_STAGE"] = route
    if python:
        env["LFR_SOLVE_PYTHON"] = "1"
        return subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=env)
    return subprocess.run([PRODUCT] + args, capture_output=True, env=env)


def test_incremental_scenario_through_both_hosts_and_routes(oracle, tmp_path):
    """Refine cfg2 without images 8-10 (solution A), then the full scene with images 0-7 fixed and A as the
    start: images 0-7 keep A's values bit for bit, the new images match the checker."""
    ms = synth.generate("cfg2")
    m, a, a_file = tmp_path / "m.pb", tmp_path / "a.pb", tmp_path / "a_in.pb"
    m.write_bytes(wire.encode_matching_file(ms))
    banned = ms.image_names[8:11]
    args = ["--matches_file", str(m), "--output_file", str(a)]
    for nm in banned:
        args += ["--banned_images", nm]
    r = _run(args)
    assert r.returncode == 0, r.stderr
    A = a.read_bytes()
    a_file.write_bytes(A)
    outs = []
    for python in (False, True):
        for route in ("host", "device"):
            o = tmp_path / ("o_%d_%s.pb" % (python, route))
            args = ["--matches_file", str(m), "--output_file", str(o), "--initial_solution", str(a_file)]
            for nm in ms.image_names[:8]:
                args += ["--fixed_images", nm]
            r = _run(args, python=python, route=route)
            assert r.returncode == 0, r.stderr
            outs.append(o.read_bytes())
    assert all(x == outs[0] for x in outs[1:])
    got = {nm: (fi, di, dj) for nm, _, fi, di, dj in wire.decode_solution(outs[0])}
    for nm, _, fi, di, dj in wire.decode_solution(A):
        if nm not in ms.image_names[:8]:
            continue
        gfi, gdi, gdj = got[nm]
        at = {int(f): k for k, f in enumerate(gfi.tolist())}
        idx = np.array([at[int(f)] for f in fi.tolist()])
        assert gdi[idx].tobytes() == di.tobytes() and gdj[idx].tobytes() == dj.tobytes()
        rest = np.setdiff1d(np.arange(gfi.shape[0]), idx)
        assert not gdi[rest].any() and not gdj[rest].any()          # not in A: constant at zero
    # the checker on the same arrays
    skip, arrs = host_input_arrays(ms)
    from lfr_b200.graph import host_stage_export
    rc, g, sz = host_stage_export(arrs, len(ms.image_names))
    assert rc == 0
    p = problem_from_stage(ms, skip, g, sz, "native")
    q = problem_from_stage(ms, skip, g, sz, "native")
    _, q.is_root, start = constant_arrays(ms, g, range(8), A)
    pos_o, _ = oracle.solve(q, oracle.default_options(n_threads=8), positions=start)
    sol = assemble_solution(p, pos_o)
    for k, nm in enumerate(sol.image_names):
        lo, hi = int(sol.img_ptr[k]), int(sol.img_ptr[k + 1])
        gfi, gdi, gdj = got[nm]
        assert np.array_equal(gfi, sol.feature_idx[lo:hi])
        assert np.abs(gdi.astype(np.float64) - sol.di[lo:hi]).max(initial=0) <= TOL
        assert np.abs(gdj.astype(np.float64) - sol.dj[lo:hi]).max(initial=0) <= TOL
