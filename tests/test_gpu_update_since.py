"""Updating an earlier SolutionFile since an earlier MatchingFile on the GPU: lfr_plan_update_solution_since
(the compare in csrc/lfr_diff.cuh) against the host form (lfr_wire_update_solution_since) on every case of
tests/test_update_since.py, with the earlier plan built both from the decoded matches and from the wire
bytes; the drop-in's device route against its host route byte for byte; and cfg4 with 20 new images against
the Python statement of the rule."""
import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import Plan
from lfr_b200.graph import problem_from_stage
from test_fixed_images import stage
from test_fixed_images_ref import bits
from test_gpu_fixed_images import _run
from test_update_since import CASES, banned_args, reencode, since_model

pytestmark = pytest.mark.gpu


def gpu_case(tmp_path, name):
    """(OLD, NEW, banned, OLD path, NEW path, A path, A bytes): A.pb is the drop-in's device-route output on OLD."""
    old, new, banned = CASES[name]()
    o, n, a = tmp_path / "old.pb", tmp_path / "new.pb", tmp_path / "a.pb"
    o.write_bytes(wire.encode_matching_file(old))
    n.write_bytes(wire.encode_matching_file(new))
    r = _run(["--matches_file", str(o), "--output_file", str(a)], route="device")
    assert r.returncode == 0, r.stderr
    return old, new, tuple(banned), o, n, a, a.read_bytes()


def device_update(b200, new, banned, old_bytes, A, from_wire):
    """(start positions, held, counts) of lfr_plan_update_solution_since on a plan of NEW."""
    plan = Plan.from_matches(b200, new, banned_images=banned)
    prev = Plan.from_wire(b200, [old_bytes]) if from_wire else Plan.from_matches(b200, wire.decode_matching_file(old_bytes))
    try:
        counts = plan.update_solution(A, new.image_names, previous=prev)
        pos, _ = plan.download()
        g = plan.export_graph()
    finally:
        prev.close()
        plan.close()
    return pos, counts, g


@pytest.mark.parametrize("from_wire", [False, True], ids=["matches", "wire"])
@pytest.mark.parametrize("name", list(CASES))
def test_device_equals_the_host_form(b200, tmp_path, name, from_wire):
    old, new, banned, o, n, a, A = gpu_case(tmp_path, name)
    pos, counts, g = device_update(b200, new, banned, o.read_bytes(), A, from_wire)
    skip, h, sz = stage(new, banned)
    assert all(np.array_equal(g[k], h[k]) for k in ("node_image", "node_feat", "comp"))
    want = wire.update_solution_since(A, problem_from_stage(new, skip, h, sz, "native"), old)
    assert counts == want[2:]
    assert bits(pos[want[1]]).tobytes() == bits(want[0][want[1]]).tobytes()   # held: A's bits
    assert not pos[~want[1]].any()                                             # touched: start at 0


@pytest.mark.parametrize("name", list(CASES))
def test_drop_in_device_route_equals_host_route(tmp_path, name):
    old, new, banned, o, n, a, A = gpu_case(tmp_path, name)
    outs = []
    for python in (False, True):
        for route in ("host", "device"):
            out = tmp_path / ("o_%d_%s.pb" % (python, route))
            r = _run(["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a),
                      "--update_initial_solution", "--previous_matches_file", str(o)] + banned_args(banned),
                     python=python, route=route)
            assert r.returncode == 0, (python, route, r.stderr)
            outs.append(out.read_bytes())
    assert all(x == outs[0] for x in outs[1:])
    if name in ("same", "new-k1", "new-k3"):
        full = tmp_path / "full.pb"
        r = _run(["--matches_file", str(n), "--output_file", str(full)], route="device")
        assert r.returncode == 0, r.stderr
        assert outs[0] == full.read_bytes()


def test_cfg4_twenty_new_images_against_the_model(b200, tmp_path):
    base = synth.generate("cfg4")
    new_img = np.arange(len(base.image_names) - 20, len(base.image_names))
    touch = np.isin(base.pair_img1, new_img) | np.isin(base.pair_img2, new_img)
    old_idx, new_idx = np.nonzero(~touch)[0], np.nonzero(touch)[0]
    old = reencode(base.select_pairs(old_idx))
    new = reencode(base.select_pairs(np.concatenate([old_idx, new_idx])))
    o, a = tmp_path / "old.pb", tmp_path / "a.pb"
    o.write_bytes(wire.encode_matching_file(old))
    r = _run(["--matches_file", str(o), "--output_file", str(a)], route="device")
    assert r.returncode == 0, r.stderr
    A = a.read_bytes()
    pos, counts, g = device_update(b200, new, (), o.read_bytes(), A, True)
    want = since_model(new, (), old, A)
    assert counts == want[2:] and 0 < counts[0] and 0 < counts[2]
    assert bits(pos).tobytes() == bits(want[0]).tobytes()
