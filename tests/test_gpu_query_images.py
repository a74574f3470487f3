"""--query_images on the GPU: the batch through both graph-stage routes (LFR_GRAPH_STAGE=host|device), the host
cut and the device cut (LFR_DEVICE_CUT=1), the host and the GPU match decode, against every query's own run
and against the CPU checker's bytes; the device stage's arrays with sub-scenes against the host stage's."""
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import wire
from lfr_b200.capi import DBG_DEVICE_CUT, Plan
from lfr_b200.graph import host_input_arrays, host_stage_export
from test_native_exe import PRODUCT, checker_exe, product_exe  # noqa: F401
from test_query_images import MODES, check_batch, localization_scene, messages, mode_args, own_matches, stdout_values
from test_ref_solve import LAUNCHER, untimed

pytestmark = pytest.mark.gpu

ROUTES = {"host": dict(LFR_GRAPH_STAGE="host"), "device": dict(LFR_GRAPH_STAGE="device"),
          "device_cut": dict(LFR_GRAPH_STAGE="device", LFR_DEVICE_CUT="1")}


def _run(cmd, env_extra, python=False):
    env = {k: v for k, v in os.environ.items() if k not in ("LFR_GRAPH_STAGE", "LFR_DEVICE_CUT")}
    env.update(env_extra)
    if python:
        env["LFR_SOLVE_PYTHON"] = "1"
        cmd = [sys.executable, LAUNCHER] + cmd
    else:
        cmd = [PRODUCT] + cmd
    return subprocess.run(cmd, capture_output=True, env=env)


def batch_args(d, name, out, queries, banned, extra):
    args = ["--matches_file", str(d / name), "--output_file", str(out), "--banned_images", banned] + extra
    for q in queries:
        args += ["--query_images", q]
    return args


@pytest.fixture(scope="module")
def small(tmp_path_factory, checker_exe, product_exe):  # noqa: F811
    d = tmp_path_factory.mktemp("gpu_loc")
    db, batch, queries, banned = localization_scene()
    wire.write_matching_file(db, str(d / "db.pb"))
    r = subprocess.run([checker_exe, "--matches_file", str(d / "db.pb"), "--output_file", str(d / "A.pb")], capture_output=True)
    assert r.returncode == 0, r.stderr
    wire.write_matching_file(batch, str(d / "batch.pb"), pairs_per_part=7)
    return d, db, batch, queries, banned


@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("mode", sorted(MODES))
def test_batch_equals_the_checker_and_every_querys_own_run(small, checker_exe, mode, route):  # noqa: F811
    d, db, batch, queries, banned = small
    extra = mode_args(d, db, mode)
    want_o = d / ("checker_%s.pb" % mode)
    rc = subprocess.run([checker_exe] + batch_args(d, "batch.pb", want_o, queries, banned, extra), capture_output=True)
    assert rc.returncode == 0, rc.stderr
    o = d / ("gpu_%s_%s.pb" % (mode, route))
    r = _run(batch_args(d, "batch.pb", o, queries, banned, extra), ROUTES[route])
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == want_o.read_bytes()
    assert untimed(r.stdout.decode()) == untimed(rc.stdout.decode())
    # every query's own run on the same route
    own = {}
    for q in queries:
        mq = d / ("own_%s.pb" % q)
        wire.write_matching_file(own_matches(batch, q, [banned]), str(mq))
        oq = d / ("own_%s_%s_%s.pb" % (q, mode, route))
        rq = _run(["--matches_file", str(mq), "--output_file", str(oq), "--banned_images", banned] + extra,
                  ROUTES[route] if own_matches(batch, q, [banned]).n_matches else {})
        assert rq.returncode == 0, rq.stderr
        mine = [m for nm, m in messages(oq.read_bytes()) if nm == q]
        own[q] = (mine[0] if mine else None, stdout_values(rq.stdout.decode()))
    check_batch(o.read_bytes(), r.stdout.decode(), own, queries)


@pytest.mark.parametrize("route", ["host", "device"])
@pytest.mark.parametrize("mode", ["plain", "keep"])
def test_python_host_equals_the_checker(small, checker_exe, mode, route):  # noqa: F811
    d, db, batch, queries, banned = small
    extra = mode_args(d, db, mode)
    want_o = d / ("checker_py_%s.pb" % mode)
    rc = subprocess.run([checker_exe] + batch_args(d, "batch.pb", want_o, queries, banned, extra), capture_output=True)
    assert rc.returncode == 0, rc.stderr
    o = d / ("py_%s_%s.pb" % (mode, route))
    r = _run(batch_args(d, "batch.pb", o, queries, banned, extra), ROUTES[route], python=True)
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == want_o.read_bytes()
    assert untimed(r.stdout.decode()) == untimed(rc.stdout.decode())


def _large():
    """A batch past the match count at which the device route decodes the matches on the GPU."""
    return localization_scene(seed=7, k=4, scale=4.0)


@pytest.fixture(scope="module")
def large(tmp_path_factory, product_exe):  # noqa: F811
    d = tmp_path_factory.mktemp("gpu_loc_large")
    db, batch, queries, banned = _large()
    wire.write_matching_file(batch, str(d / "batch.pb"))
    return d, db, batch, queries, banned


def test_large_batch_decoded_on_the_gpu(large, b200):
    d, db, batch, queries, banned = large
    assert b200.lib.lfr_wire_decode_on_device(batch.n_matches) == 1
    outs = {}
    for route, env in (("auto", {}), ("host", ROUTES["host"]), ("device_cut", ROUTES["device_cut"])):
        o = d / ("large_%s.pb" % route)
        r = _run(batch_args(d, "batch.pb", o, queries, banned, []), env)
        assert r.returncode == 0, r.stderr
        outs[route] = (o.read_bytes(), untimed(r.stdout.decode()))
    assert outs["auto"] == outs["host"] == outs["device_cut"]
    own = {}
    for q in queries:
        mq = d / ("own_%s.pb" % q)
        wire.write_matching_file(own_matches(batch, q, [banned]), str(mq))
        oq = d / ("own_%s_out.pb" % q)
        rq = _run(["--matches_file", str(mq), "--output_file", str(oq), "--banned_images", banned], {})
        assert rq.returncode == 0, rq.stderr
        mine = [m for nm, m in messages(oq.read_bytes()) if nm == q]
        own[q] = (mine[0] if mine else None, stdout_values(rq.stdout.decode()))
    check_batch(outs["host"][0], "\n".join(outs["host"][1]), own, queries)


@pytest.mark.parametrize("scene", ["small", "large"])
@pytest.mark.parametrize("device_cut", [False, True], ids=["host_cut", "device_cut"])
def test_device_stage_with_sub_scenes_equals_the_host_stage(b200, scene, device_cut):
    db, batch, queries, banned = localization_scene() if scene == "small" else _large()
    sub, group = batch.query_subscenes(queries, [banned])
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

