"""Both `solve` programs route the graph stage by the library's size rule (lfr_graph_stage_on_device,
include/lfr_graph.h): on the device (lfr_plan_create_from_matches, the plan solved in place) or on the
host (lfr_host_stage_create + lfr_solve).  LFR_GRAPH_STAGE=host|device forces a route.

CPU: the rule itself (exported, needs no device), and the hook on builds and hosts that cannot take the
device route: they stop with a message instead of running the host stage.
GPU: the two routes, forced, give byte-identical SolutionFiles and the same untimed stdout lines, through
the native drop-in and through the Python host, on the goldens and on every kind of input the drop-in
reads; the automatic route shows in --stats_json."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import B200_LIB_PATH, GRAPH_SYMBOLS, Library
from lfr_b200.graph import HostInput, host_input_arrays
from lfr_b200.solver import GraphStageRouteError, graph_stage_on_device
from test_native_exe import PRODUCT, checker_exe, product_exe, run  # noqa: F401  (fixtures)
from test_ref_solve import GOLD, LAUNCHER, banned_inputs, untimed

ROUTES = ("host", "device")


@pytest.fixture(scope="module")
def product_lib(product_exe):  # noqa: F811  (built by the product_exe fixture)
    return Library(B200_LIB_PATH)


def rule(lib, pair_ptr, n_images, n_devices=1, pair_skip=None):
    """lfr_graph_stage_on_device on an input that has only its pair list: that is all the rule reads."""
    ptr = np.ascontiguousarray(pair_ptr, dtype=np.uint64)
    skip = None if pair_skip is None else np.ascontiguousarray(pair_skip, dtype=np.uint8)
    inp = HostInput(n_pairs=ptr.shape[0] - 1, n_matches=int(ptr[-1]), n_images=n_images, pair_ptr=ptr.ctypes.data,
                    pair_skip=None if skip is None else skip.ctypes.data)
    return lib.lib.lfr_graph_stage_on_device(C.byref(inp), n_devices)


# ---------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------
def test_route_rule_is_exported_and_decides_from_sizes_alone(product_lib):
    assert "lfr_graph_stage_on_device" in GRAPH_SYMBOLS
    for s in GRAPH_SYMBOLS:
        getattr(product_lib.lib, s)
    cfg5 = np.arange(24787, dtype=np.uint64) * 221          # cfg5's shape: 24 786 pairs, ~11 M directed edges
    assert rule(product_lib, cfg5, 1000) == 1
    assert rule(product_lib, cfg5, 1000, n_devices=2) == 0  # lfr_solve_multi() takes a host problem
    assert rule(product_lib, cfg5, 1000, n_devices=0) == 0
    assert rule(product_lib, cfg5, 1000, pair_skip=np.ones(24786)) == 0   # every pair banned: nothing to build
    assert rule(product_lib, cfg5, 65536) == 0               # more images than either stage takes
    assert rule(product_lib, [0], 0) == 0                    # empty input
    assert rule(product_lib, [0, 1, 2], 3) == 0              # below the threshold
    assert rule(product_lib, [0, 2 ** 30 - 1], 2) == 1       # 2^31 - 2 directed edges
    assert rule(product_lib, [0, 2 ** 30], 2) == 0           # 2^31: the device stage refuses it
    assert rule(product_lib, [0, 5, 3], 2) == 0              # malformed pair list: the host stage reports it
    assert product_lib.lib.lfr_graph_stage_on_device(None, 1) == 0


def test_route_rule_needs_no_device():
    """In a process that sees no device at all."""
    code = ("import sys, numpy as np; sys.path[:0] = %r\n"
            "from test_drop_in_device_stage import rule\n"
            "from lfr_b200.capi import B200_LIB_PATH, Library\n"
            "print(rule(Library(B200_LIB_PATH), np.arange(24787) * 221, 1000))\n") % (
        [os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.dirname(os.path.abspath(__file__))],)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0 and r.stdout == "1\n", r.stderr


def test_checker_build_refuses_a_forced_device_route(checker_exe, tmp_path):  # noqa: F811
    """The CPU checker has no graph stage on the GPU: forcing that route stops with a message and writes
    nothing; forcing the host route (or none) runs as before."""
    m, o = os.path.join(GOLD, "tiny_matches.pb"), tmp_path / "o.pb"
    env = dict(os.environ, LFR_GRAPH_STAGE="device")
    r = subprocess.run([checker_exe, "--matches_file", m, "--output_file", str(o)], capture_output=True, text=True, env=env)
    assert (r.returncode, r.stdout) == (2, "")
    assert r.stderr == "ERROR: LFR_GRAPH_STAGE=device: the solve library has no graph stage on the GPU\n"
    assert not o.exists()
    r = subprocess.run([checker_exe, "--matches_file", m, "--output_file", str(o)], capture_output=True, text=True,
                       env=dict(os.environ, LFR_GRAPH_STAGE="host"))
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read()
    assert untimed(r.stdout) == open(os.path.join(GOLD, "tiny_stdout.txt")).read().splitlines()


@pytest.mark.parametrize("value,gpus,message", [
    ("sideways", "1", "ERROR: LFR_GRAPH_STAGE must be 'host' or 'device'\n"),
    ("device", "2", "ERROR: LFR_GRAPH_STAGE=device: the graph stage on the GPU drives one device (--gpus 1)\n"),
])
def test_both_hosts_refuse_a_route_they_cannot_take(product_exe, tmp_path, value, gpus, message):  # noqa: F811
    """The native drop-in and the Python host: same exit code, same message, no file."""
    m = os.path.join(GOLD, "tiny_matches.pb")
    for cmd, extra in ((product_exe, {}), (sys.executable, {"LFR_SOLVE_PYTHON": "1"})):
        o = tmp_path / "o.pb"
        argv = ([LAUNCHER] if cmd == sys.executable else []) + ["--matches_file", m, "--output_file", str(o), "--gpus", gpus]
        r = subprocess.run([cmd] + argv, capture_output=True, text=True, env=dict(os.environ, LFR_GRAPH_STAGE=value, **extra))
        assert (r.returncode, r.stdout, r.stderr) == (2, "", message)
        assert not o.exists()


def test_python_host_honours_the_hook(product_lib, oracle, monkeypatch):
    # the rule reads the pair list and the match count only (feat1's length; never its content)
    big = {"pair_img1": np.zeros(1, np.uint32), "pair_img2": np.ones(1, np.uint32), "pair_skip": np.zeros(1, np.uint8),
           "pair_ptr": np.array([0, 2 ** 24], np.uint64), "feat1": np.broadcast_to(np.uint32(0), (2 ** 24,))}
    small = dict(big, pair_ptr=np.array([0, 1], np.uint64), feat1=np.zeros(1, np.uint32))
    monkeypatch.delenv("LFR_GRAPH_STAGE", raising=False)
    assert graph_stage_on_device(product_lib, big, 2) and not graph_stage_on_device(product_lib, small, 2)
    assert not graph_stage_on_device(product_lib, big, 2, n_devices=2)
    assert not graph_stage_on_device(oracle, big, 2)        # no graph stage on the GPU: the host route
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    assert not graph_stage_on_device(product_lib, big, 2)
    monkeypatch.setenv("LFR_GRAPH_STAGE", "device")
    assert graph_stage_on_device(product_lib, small, 2)
    with pytest.raises(GraphStageRouteError, match="has no graph stage on the GPU"):
        graph_stage_on_device(oracle, small, 2)
    with pytest.raises(GraphStageRouteError, match="drives one device"):
        graph_stage_on_device(product_lib, small, 2, n_devices=4)


# ---------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------
def solution_close(got, want):
    """Equal float for float, as the goldens are compared elsewhere: byte-identical unless a displacement
    sits within 1e-16 of a float32 rounding boundary (the goldens come from the reference's CPU solve)."""
    if got == want:
        return True
    a, b = wire.decode_solution(got), wire.decode_solution(want)
    if [x[0] for x in a] != [x[0] for x in b]:
        return False
    for (_, fa, ia, dia, dja), (_, fb, ib, dib, djb) in zip(a, b):
        if fa != fb or not np.array_equal(ia, ib):
            return False
        if np.abs(dia - dib).max(initial=0) > 1e-4 / 16 or np.abs(dja - djb).max(initial=0) > 1e-4 / 16:
            return False
    return True


def both_routes(tmp_path, args, python=False):
    """{route: (exit code, untimed stdout, stderr, SolutionFile bytes or None)} of one command line."""
    res = {}
    for route in ROUTES:
        o = tmp_path / ("%s_%s.pb" % ("py" if python else "native", route))
        env = dict(os.environ, LFR_GRAPH_STAGE=route)
        cmd = [PRODUCT] + args
        if python:
            env["LFR_SOLVE_PYTHON"] = "1"
            cmd = [sys.executable, LAUNCHER] + args
        r = subprocess.run(cmd + ["--output_file", str(o)], capture_output=True, env=env)
        res[route] = (r.returncode, untimed(r.stdout.decode("utf-8", "surrogateescape")), r.stderr,
                      o.read_bytes() if o.exists() else None)
    return res


def check_routes_agree(tmp_path, args):
    """Native host route = native device route = Python host route = Python device route."""
    native, py = both_routes(tmp_path, args), both_routes(tmp_path, args, python=True)
    ref = native["host"]
    assert ref[0] == 0, ref[2]
    for got in (native["device"], py["host"], py["device"]):
        assert got == ref
    return ref


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "linesearch", "fountain_2pct"])
def test_gpu_routes_agree_on_the_goldens(product_exe, tmp_path, name):  # noqa: F811
    rc, lines, _, sol = check_routes_agree(tmp_path, ["--matches_file", os.path.join(GOLD, name + "_matches.pb")])
    assert lines == open(os.path.join(GOLD, name + "_stdout.txt")).read().splitlines()
    assert solution_close(sol, open(os.path.join(GOLD, name + "_solution.pb"), "rb").read())


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,scale,seed", [("cfg2", 0.25, 11), ("cfg4", 0.1, 7)])
def test_gpu_routes_agree_on_scaled_workloads(product_exe, tmp_path, cfg, scale, seed):  # noqa: F811
    m = tmp_path / "m.pb"
    wire.write_matching_file(synth.generate(cfg, scale=scale, seed=seed), str(m))
    check_routes_agree(tmp_path, ["--matches_file", str(m)])


@pytest.mark.gpu
def test_gpu_routes_agree_on_banned_images_part_files_and_odd_names(product_exe, tmp_path):  # noqa: F811
    ms, banned, parts = banned_inputs()
    m = tmp_path / "m.pb"
    wire.write_matching_file(ms, str(m))
    check_routes_agree(tmp_path, ["--matches_file", str(m), "--banned_images", banned[0], "--banned_images=" + banned[1]])
    for k, part in enumerate(parts):
        (tmp_path / ("split.pb.part.%d" % k)).write_bytes(wire.encode_matching_file(part))
    check_routes_agree(tmp_path, ["--matches_file", str(tmp_path / "split.pb")])
    # names with spaces, non-ASCII characters and invalid UTF-8, one of them banned by the same bytes
    odd_ms = synth.generate("cfg1", seed=5)
    odd = ["im age 0.png", "bild-äöü.jpg", b"raw-\xff\xfe.png".decode("utf-8", errors="surrogateescape")]
    odd_ms.image_names = odd + odd_ms.image_names[len(odd):]
    (tmp_path / "odd.pb").write_bytes(wire.encode_matching_file(odd_ms))
    check_routes_agree(tmp_path, ["--matches_file", str(tmp_path / "odd.pb")])
    check_routes_agree(tmp_path, ["--matches_file", str(tmp_path / "odd.pb"), "--banned_images", odd[2]])


@pytest.mark.gpu
def test_gpu_routes_agree_on_empty_inputs(product_exe, tmp_path):  # noqa: F811
    ms = synth.generate("cfg1", seed=5)
    m = tmp_path / "m.pb"
    wire.write_matching_file(ms, str(m))
    everything = sum((["--banned_images", n] for n in ms.image_names), [])
    rc, lines, _, sol = check_routes_agree(tmp_path, ["--matches_file", str(m)] + everything)
    assert sol == b"" and lines == ["# graph nodes: 0", "# graph edges: 0", "# points with at least one coordinate > 0.5: 0"]
    rc, lines, _, sol = check_routes_agree(tmp_path, ["--matches_file", str(tmp_path / "absent.pb")])
    assert sol == b"" and lines == ["# graph nodes: 0", "# graph edges: 0", "# points with at least one coordinate > 0.5: 0"]


@pytest.mark.gpu
def test_gpu_routes_reject_a_nan_similarity_alike(product_exe, tmp_path):  # noqa: F811
    ms = synth.generate("cfg2", scale=0.1, seed=3)
    ms.sim[7] = np.nan
    m = tmp_path / "m.pb"
    wire.write_matching_file(ms, str(m))
    res = both_routes(tmp_path, ["--matches_file", str(m)])
    assert res["host"][0] == 2 and res["host"][2] == b"ERROR: the host graph stage rejected the input\n"
    assert (res["device"][0], res["device"][2], res["device"][3]) == (res["host"][0], res["host"][2], None)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,stage", [("cfg1", "native"), ("cfg2", "device")])
def test_gpu_stats_json_reports_the_automatic_route(tmp_path, cfg, stage):
    ms = synth.generate(cfg)
    assert Library(B200_LIB_PATH).graph_stage_on_device(host_input_arrays(ms)[1], len(ms.image_names)) == (stage == "device")
    m, o, js = tmp_path / "m.pb", tmp_path / "o.pb", tmp_path / "st.json"
    wire.write_matching_file(ms, str(m))
    env = {k: v for k, v in os.environ.items() if k not in ("LFR_GRAPH_STAGE", "LFR_HOST_PYTHON")}
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", str(m), "--output_file", str(o), "--stats_json", str(js)],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    st = json.load(open(js))
    assert st["info"]["host_stage"] == stage and st["n_nodes"] > 0 and st["tracks_refined"] > 0
    # the same SolutionFile as the native drop-in's automatic route
    r2 = run(PRODUCT, ["--matches_file", str(m), "--output_file", str(tmp_path / "n.pb")])
    assert r2.returncode == 0 and (tmp_path / "n.pb").read_bytes() == o.read_bytes()
    assert untimed(r2.stdout) == untimed(r.stdout)
