"""Matches decoded on the device (lfr_plan_create_from_wire, include/lfr_graph.h; csrc/lfr_wire.cuh)
against the host decode (lfr_wire_decode_matches) + lfr_plan_create_from_matches: the same plan bit for
bit, every encoding decoded alike, malformed input refused exactly where the host codec refuses it, and
the native drop-in's device route equal to its host route."""
import os
import subprocess

import numpy as np
import pytest

from lfr_b200 import MatchSet, synth, wire
from lfr_b200.capi import Plan
from test_drop_in_device_stage import both_routes
from test_gpu_graph_stage import ARRAYS, COUNTS
from test_graph_stage_adversarial import E2E_CASES, make_case
from test_native_exe import product_exe  # noqa: F401  (fixture)
from test_wire_walk import encodings, malformed_match_files

pytestmark = pytest.mark.gpu

LFR_EINVAL = -1


def _host_matchset(parts):
    """The host decode of the parts, concatenated as the drop-in reads `.part.N` files."""
    got = [wire.decode_matching_file(p) for p in parts]
    return got[0] if len(got) == 1 else MatchSet.concatenate(got)


def assert_same_plan(b200, parts, banned=(), solve=True):
    ms = _host_matchset(parts)
    a = Plan.from_matches(b200, ms, banned_images=banned)
    b = Plan.from_wire(b200, parts, banned_images=banned)
    assert b.image_names == ms.image_names
    ga, gb = a.export_graph(), b.export_graph()
    for k in ARRAYS:
        assert ga[k].dtype == gb[k].dtype and ga[k].shape == gb[k].shape, k
        assert ga[k].tobytes() == gb[k].tobytes(), k
    for k in COUNTS:
        assert a.sizes[k] == b.sizes[k], k
    if solve:
        a.solve()
        b.solve()
        (pa, sa), (pb, sb) = a.download(), b.download()
        assert pa.tobytes() == pb.tobytes()
        for k in ("iterations", "termination", "initial_cost", "final_cost"):
            assert sa[k].tobytes() == sb[k].tobytes(), k
        for k in ("total_iterations", "total_line_search_steps", "n_solved"):
            assert sa[k] == sb[k], k
    a.close()
    b.close()
    return ga


@pytest.mark.parametrize("cfg,scale", [("cfg1", 1.0), ("cfg2", 0.02), ("cfg2", 1.0)])
def test_equal_plans_on_scenes(b200, cfg, scale):
    g = assert_same_plan(b200, [wire.encode_matching_file(synth.generate(cfg, scale=scale))])
    assert g["edges"].shape[0] > 0


@pytest.mark.parametrize("case", E2E_CASES)
def test_equal_plans_on_adversarial_match_graphs(b200, case):
    assert_same_plan(b200, [wire.encode_matching_file(make_case(case))])


def test_equal_plans_on_parts_and_banned_images(b200):
    ms = synth.generate("cfg2", scale=0.25, seed=11)
    step = max(1, ms.n_pairs // 3)
    parts = [wire.encode_matching_file(ms, lo, min(ms.n_pairs, lo + step)) for lo in range(0, ms.n_pairs, step)]
    assert len(parts) > 2
    assert_same_plan(b200, parts)
    assert_same_plan(b200, parts, banned=[ms.image_names[1], ms.image_names[4]])
    assert_same_plan(b200, parts + [b""])                     # an empty part
    # every pair banned: the matches are still decoded (and would be refused if malformed), nothing is built
    assert_same_plan(b200, parts, banned=ms.image_names)


@pytest.mark.parametrize("name", sorted(encodings()))
def test_encodings_decode_on_the_device_as_on_the_host(b200, name):
    """The edge records carry every decoded float (sim, both displacement grids) and the node arrays the
    feature indices, so equal plans mean equal decoded arrays."""
    assert_same_plan(b200, [encodings()[name]], solve=False)


def _host_accepts(data):
    try:
        wire.decode_matching_file(data)
        return True
    except wire.ParseError:
        return False


def _device_accepts(b200, data):
    try:
        Plan.from_wire(b200, [data]).close()
        return True
    except wire.ParseError:          # the pair walk, on the host
        return False
    except RuntimeError as e:
        assert "(%d): malformed Match message" % LFR_EINVAL in str(e), str(e)
        return False


def test_malformed_input_is_refused_exactly_where_the_host_refuses_it(b200):
    """Each input runs once: truncations of a small file at every byte, length prefixes past the end, bad
    wire types and cut fields inside a match.  A valid call on the same device follows."""
    small = wire.encode_matching_file(synth.generate("cfg1", scale=0.1))[:700]
    good = encodings()["non_canonical_displacements"]
    inputs = [good[:k] for k in range(len(good))] + [small[:k] for k in range(len(small))]
    for k in range(len(good)):            # a length byte pushed past its message
        b = bytearray(good)
        if 0 < b[k] < 0x80 and k and b[k - 1] in (0x0A, 0x22, 0x2A, 0x1A):
            b[k] = 0x7F
            inputs.append(bytes(b))
    inputs += list(malformed_match_files().values())
    n_refused_on_device = 0
    for data in inputs:
        host = _host_accepts(data)
        assert _device_accepts(b200, data) == host
        n_refused_on_device += (not host) and _walks(data)
    assert n_refused_on_device >= len(malformed_match_files())
    assert_same_plan(b200, [good])


def _walks(data):
    try:
        wire.walk_matching_file(data)
        return True
    except wire.ParseError:
        return False


def _first_tag(data, off):
    """The index of a match's first tag: past its length prefix (a varint) at `off`."""
    k = int(off)
    while data[k] & 0x80:
        k += 1
    return k + 1


def test_a_corrupt_match_in_a_large_file(b200):
    ms = synth.generate("cfg2", scale=0.25, seed=3)
    data = bytearray(wire.encode_matching_file(ms))
    off = wire.walk_matching_file(bytes(data))["match_off"]
    data[_first_tag(data, off[len(off) // 2])] = 0x0B     # field 1, wire type 3 (a group)
    assert not _host_accepts(bytes(data)) and _walks(bytes(data))
    assert not _device_accepts(b200, bytes(data))
    assert_same_plan(b200, [wire.encode_matching_file(ms)], solve=False)


# ---- the native drop-in -----------------------------------------------------------------------------
def test_drop_in_device_route_equals_host_route(product_exe, b200, tmp_path):  # noqa: F811
    ms = synth.generate("cfg4", scale=0.5)
    assert b200.lib.lfr_wire_decode_on_device(ms.n_matches) == 1   # the device route decodes on the GPU
    m = tmp_path / "m.pb"
    wire.write_matching_file(ms, str(m))
    for args in (["--matches_file", str(m)],
                 ["--matches_file", str(m), "--banned_images", ms.image_names[2], "--banned_images", ms.image_names[5]]):
        res = both_routes(tmp_path, args)
        assert res["host"][0] == 0, res["host"][2]
        assert res["device"] == res["host"]
    files = wire.write_matching_file(ms, str(tmp_path / "split.pb"), pairs_per_part=max(1, ms.n_pairs // 3))
    assert len(files) > 1
    res = both_routes(tmp_path, ["--matches_file", str(tmp_path / "split.pb")])
    assert res["host"][0] == 0 and res["device"] == res["host"]


# the device route's decode on the GPU (cfg4 x 0.5), and on the host below its size (cfg2 x 0.25)
@pytest.mark.parametrize("cfg,scale", [("cfg4", 0.5), ("cfg2", 0.25)])
def test_drop_in_refuses_a_malformed_match_on_both_routes(product_exe, tmp_path, cfg, scale):  # noqa: F811
    ms = synth.generate(cfg, scale=scale, seed=3)
    parts = [wire.encode_matching_file(ms, 0, ms.n_pairs // 2), bytearray(wire.encode_matching_file(ms, ms.n_pairs // 2))]
    off = wire.walk_matching_file(bytes(parts[1]))["match_off"]
    parts[1][_first_tag(parts[1], off[-1])] = 0x0B
    for k, p in enumerate(parts):
        (tmp_path / ("bad.pb.part.%d" % k)).write_bytes(bytes(p))
    res = both_routes(tmp_path, ["--matches_file", str(tmp_path / "bad.pb")])
    for route in ("host", "device"):
        assert res[route] == (255, [], b"Failed to parse proto object.\n", None), route
    # a non-finite similarity still stops in the graph stage, as on the host route
    ms.sim[7] = np.nan
    m = tmp_path / "nan.pb"
    wire.write_matching_file(ms, str(m))
    res = both_routes(tmp_path, ["--matches_file", str(m)])
    assert res["host"][:3] == (2, [], b"ERROR: the host graph stage rejected the input\n")
    assert res["device"] == res["host"]


def test_drop_in_automatic_route_on_cfg4(product_exe, tmp_path):  # noqa: F811
    """Without the hook, cfg4 takes the device route and the decoder on the GPU; its output equals the forced
    host route's."""
    from test_native_exe import PRODUCT
    from test_ref_solve import untimed
    ms = synth.generate("cfg4")
    m = tmp_path / "m.pb"
    wire.write_matching_file(ms, str(m))
    env = {k: v for k, v in os.environ.items() if k != "LFR_GRAPH_STAGE"}
    r = subprocess.run([PRODUCT, "--matches_file", str(m), "--output_file", str(tmp_path / "auto.pb")], capture_output=True,
                       env=env)
    assert r.returncode == 0, r.stderr
    res = both_routes(tmp_path, ["--matches_file", str(m)])
    assert untimed(r.stdout.decode()) == res["host"][1] and (tmp_path / "auto.pb").read_bytes() == res["host"][3]
