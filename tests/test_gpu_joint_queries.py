"""--joint_queries on the GPU: the joint batch through both graph-stage routes (LFR_GRAPH_STAGE=host|device), the
host cut and the device cut (LFR_DEVICE_CUT=1), the host and the GPU match decode, against every group's own run
and against the CPU checker's bytes; the device stage's arrays on a joint grouping against the host stage's."""
import os
import subprocess

import numpy as np
import pytest

from lfr_b200 import wire
from lfr_b200.capi import DBG_DEVICE_CUT, Plan
from lfr_b200.graph import host_input_arrays, host_stage_export
from test_gpu_query_images import ROUTES, _run
from test_joint_queries import batch_args, check_joint_batch, group_own_runs, joint_scene, query_groups
from test_native_exe import PRODUCT, checker_exe, product_exe  # noqa: F401
from test_query_images import MODES, mode_args
from test_ref_solve import untimed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def small(tmp_path_factory, checker_exe, product_exe):  # noqa: F811
    d = tmp_path_factory.mktemp("gpu_joint")
    db, batch, queries, banned = joint_scene()
    wire.write_matching_file(db, str(d / "db.pb"))
    r = subprocess.run([checker_exe, "--matches_file", str(d / "db.pb"), "--output_file", str(d / "A.pb")], capture_output=True)
    assert r.returncode == 0, r.stderr
    wire.write_matching_file(batch, str(d / "batch.pb"), pairs_per_part=7)
    return d, db, batch, queries, banned, query_groups(batch, queries, [banned])


def _route_env(route):
    """The environment of an own run on `route`: the forced device route only where the group holds a match."""
    def env(own):
        e = {k: v for k, v in os.environ.items() if k not in ("LFR_GRAPH_STAGE", "LFR_DEVICE_CUT")}
        if own.n_matches:
            e.update(ROUTES[route])
        return e
    return env


@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("mode", sorted(MODES))
def test_joint_batch_equals_the_checker_and_every_groups_own_run(small, checker_exe, mode, route):  # noqa: F811
    d, db, batch, queries, banned, groups = small
    extra = mode_args(d, db, mode)
    want_o = d / ("checker_%s.pb" % mode)
    rc = subprocess.run([checker_exe] + batch_args(d, want_o, queries, banned, extra), capture_output=True)
    assert rc.returncode == 0, rc.stderr
    o = d / ("gpu_%s_%s.pb" % (mode, route))
    r = _run(batch_args(d, o, queries, banned, extra), ROUTES[route])
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == want_o.read_bytes()
    assert untimed(r.stdout.decode()) == untimed(rc.stdout.decode())
    msgs, vals, _ = group_own_runs(PRODUCT, d, batch, groups, banned, extra, "%s_%s" % (mode, route), _route_env(route))
    check_joint_batch(o.read_bytes(), r.stdout.decode(), msgs, vals, queries)


@pytest.mark.parametrize("route", ["host", "device"])
@pytest.mark.parametrize("mode", ["plain", "keep"])
def test_python_host_equals_the_checker(small, checker_exe, mode, route):  # noqa: F811
    d, db, batch, queries, banned, groups = small
    extra = mode_args(d, db, mode)
    want_o = d / ("checker_py_%s.pb" % mode)
    rc = subprocess.run([checker_exe] + batch_args(d, want_o, queries, banned, extra), capture_output=True)
    assert rc.returncode == 0, rc.stderr
    o = d / ("py_%s_%s.pb" % (mode, route))
    r = _run(batch_args(d, o, queries, banned, extra), ROUTES[route], python=True)
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == want_o.read_bytes()
    assert untimed(r.stdout.decode()) == untimed(rc.stdout.decode())


def _large():
    """A joint batch past the match count at which the device route decodes the matches on the GPU."""
    return joint_scene(seed=8, scale=0.5, long_chain=70)


@pytest.fixture(scope="module")
def large(tmp_path_factory, product_exe):  # noqa: F811
    d = tmp_path_factory.mktemp("gpu_joint_large")
    db, batch, queries, banned = _large()
    wire.write_matching_file(batch, str(d / "batch.pb"))
    return d, db, batch, queries, banned, query_groups(batch, queries, [banned])


def test_large_joint_batch_decoded_on_the_gpu(large, b200):
    d, db, batch, queries, banned, groups = large
    assert batch.n_matches >= 262144 and b200.lib.lfr_wire_decode_on_device(batch.n_matches) == 1
    outs = {}
    for route, env in (("auto", {}), ("host", ROUTES["host"]), ("device_cut", ROUTES["device_cut"])):
        o = d / ("large_%s.pb" % route)
        r = _run(batch_args(d, o, queries, banned, []), env)
        assert r.returncode == 0, r.stderr
        outs[route] = (o.read_bytes(), untimed(r.stdout.decode()))
    assert outs["auto"] == outs["host"] == outs["device_cut"]
    msgs, vals, _ = group_own_runs(PRODUCT, d, batch, groups, banned, [], "large")
    check_joint_batch(outs["host"][0], "\n".join(outs["host"][1]), msgs, vals, queries)


@pytest.mark.parametrize("scene", ["small", "large"])
@pytest.mark.parametrize("device_cut", [False, True], ids=["host_cut", "device_cut"])
def test_device_stage_on_a_joint_grouping_equals_the_host_stage(b200, scene, device_cut):
    db, batch, queries, banned = joint_scene() if scene == "small" else _large()
    sub, group = batch.query_subscenes(queries, [banned], joint=True)
    _, arrs = host_input_arrays(sub, (), group)
    n = len(sub.image_names)
    rc, want, sz = host_stage_export(arrs, n)
    assert rc == 0 and sz["n_oversized_meta_components"] > 0
    opts = b200.default_options(debug_flags=DBG_DEVICE_CUT) if device_cut else None
    plan = Plan.from_matches(b200, arrs, options=opts, n_images=n)
    try:
        got = plan.export_graph()
        for k in ("n_nodes", "n_edges", "n_tracks", "n_components", "n_images_seen", "max_track_size",
                  "max_component_size", "n_meta_components", "n_oversized_meta_components"):
            assert plan.sizes[k] == sz[k], k
    finally:
        plan.close()
    for k, v in want.items():
        if k == "edges":
            assert got[k].tobytes() == v.tobytes()
        else:
            assert np.array_equal(got[k], v), k
