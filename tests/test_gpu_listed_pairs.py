"""--listed_pairs on the GPU: the device expand (lfr_plan_create_from_wire_listed) against the host-built match
arrays, both drop-in hosts on every graph-stage route against every list's own run, and a superset the device
route decodes on the GPU."""
import re
import subprocess

import numpy as np
import pytest

import test_listed_pairs as tlp
from lfr_b200 import synth, wire
from lfr_b200.capi import Plan
from lfr_b200.graph import HOST_SIZES_FIELDS
from lfr_b200.matchset import MatchSet
from test_gpu_query_images import ROUTES, _run
from test_native_exe import product_exe  # noqa: F401
from test_fixed_images import checker_exe  # noqa: F401
from test_listed_pairs import batch, own_runs  # noqa: F401
from test_ref_solve import untimed
from test_sass_footprint import LIB, cuobjdump
from test_scene_batch import _wide_scene

pytestmark = pytest.mark.gpu


def host_built(ms, lists, banned):
    """from_matches()'s input for the batch, built on the host: every list's pairs by select_listed_pairs,
    joined as scenes."""
    sets = [ms if l is None else ms.select_listed_pairs(l) for l in lists]
    return MatchSet.join_scenes(sets, banned)


def assert_plans_equal(a, b):
    for k in HOST_SIZES_FIELDS:
        if not k.endswith("_ms"):
            assert a.sizes[k] == b.sizes[k], k
    ea, eb = a.export_graph(), b.export_graph()
    assert set(ea) == set(eb)
    for k in ea:
        assert ea[k].dtype == eb[k].dtype and ea[k].tobytes() == eb[k].tobytes(), k


@pytest.mark.parametrize("case", ["all_lists", "repeated_and_reordered", "empty_entries", "no_entry"])
def test_device_expand_equals_the_host_built_arrays(b200, tmp_path, case):
    d = tmp_path
    path, ms, named = tlp.make_superset(d)
    parts = [(d / ("superset.pb.part.%d" % k)).read_bytes() for k in range(3)]
    parts.append(wire.encode_matching_file(_wide_scene(4, "z")))        # two pairs without matches
    full = MatchSet.concatenate([wire.decode_matching_file(p) for p in parts])
    zero = [("z0.png", "z1.png"), ("z2.png", "z3.png")]
    lists = {"all_lists": [None] + list(named.values()),
             "repeated_and_reordered": [named["repeated"], named["reordered"][::-1], named["repeated"], None],
             "empty_entries": [zero + named["hub_alone"] + zero[::-1], [], zero],
             "no_entry": [[], named["all_banned"]]}[case]
    want_ms, group = host_built(full, lists, tlp.BANNED)
    opts = b200.default_options()
    got = Plan.from_wire_listed(b200, parts, lists, tlp.BANNED, opts)
    want = Plan.from_matches(b200, dict(pair_img1=want_ms.pair_img1, pair_img2=want_ms.pair_img2,
                                        pair_skip=np.zeros(want_ms.n_pairs, np.uint8), pair_ptr=want_ms.pair_ptr,
                                        feat1=want_ms.feat1, feat2=want_ms.feat2, sim=want_ms.sim,
                                        disp1=want_ms.disp1, disp2=want_ms.disp2, image_group=group),
                             options=opts, n_images=len(want_ms.image_names))
    assert got.image_names == want_ms.image_names and np.array_equal(got.image_group, group)
    assert_plans_equal(got, want)
    if got.n_nodes:
        got.solve()
        want.solve()
        assert got.download()[0].tobytes() == want.download()[0].tobytes()
    fact = np.ones(len(want_ms.image_names), np.float32)
    n = max(len(lists), 1)
    assert got.encode_solution_groups(got.image_names, fact, group, n) == want.encode_solution_groups(
        want_ms.image_names, fact, group, n)


def test_device_expand_refuses_inconsistent_entries(b200, tmp_path):
    import ctypes as C
    from lfr_b200.capi import LfrWirePart
    from lfr_b200.graph import HostInput, HostSizes
    data = wire.encode_matching_file(synth.generate("cfg1"))
    a = wire.walk_matching_file(data)
    buf = np.frombuffer(data, np.uint8)
    part = (LfrWirePart * 1)(LfrWirePart(buf=buf.ctypes.data, len=buf.size, match_off=a["match_off"].ctypes.data,
                                         n_matches=a["match_off"].shape[0]))
    sp = np.ascontiguousarray(a["pair_ptr"], np.uint64)
    P = sp.shape[0] - 1
    img = np.zeros(2, np.uint32)
    skip = np.zeros(2, np.uint8)
    for src, ptr, why in (([0, P], None, "out of range"), ([0, 1], [0, 1, 2], "not the scan")):
        src = np.array(src, np.uint64)
        c = (sp[1:] - sp[:-1])[np.minimum(src, P - 1).astype(np.int64)]
        ptr = np.array(ptr if ptr is not None else [0, c[0], c[0] + c[1]], np.uint64)
        inp = HostInput(n_pairs=2, n_matches=int(ptr[-1]), n_images=1, pair_img1=img.ctypes.data, pair_img2=img.ctypes.data,
                        pair_skip=skip.ctypes.data, pair_ptr=ptr.ctypes.data)
        h, sz = C.c_void_p(), HostSizes()
        rc = b200.lib.lfr_plan_create_from_wire_listed(C.byref(inp), part, 1, sp.ctypes.data, P, src.ctypes.data,
                                                        C.byref(b200.default_options()), None, C.byref(h), C.byref(sz))
        assert rc == -1 and why in b200.last_error(), (rc, b200.last_error())


@pytest.fixture(scope="module")
def checker_batch(batch, checker_exe):  # noqa: F811
    d, path, ms, lists = batch
    args, outs = tlp.batch_args(d, path, lists, "checker")
    r = tlp.run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    return r


@pytest.mark.parametrize("python", [False, True], ids=["native", "python"])
@pytest.mark.parametrize("route", sorted(ROUTES))
def test_drop_in_on_every_route_writes_every_lists_own_run(batch, own_runs, checker_batch, product_exe, route,  # noqa: F811
                                                           python):
    d, path, ms, lists = batch
    args, outs = tlp.batch_args(d, path, lists, "%s_%d" % (route, python))
    r = _run(args, ROUTES[route], python=python)
    assert r.returncode == 0, r.stderr
    tlp.check_batch(outs, r.stdout.decode(), own_runs)
    assert untimed(r.stdout.decode()) == untimed(checker_batch.stdout.decode())


def test_superset_decoded_on_the_gpu(b200, tmp_path, product_exe):  # noqa: F811
    """A superset of more than 262 144 matches: the native host decodes it once on the GPU and expands it into
    sequential windows and a retrieval-style subset; every list's bytes are its own run's."""
    ms = synth.generate("cfg2", scale=3.0, seed=21)
    assert ms.n_matches > 262144 and b200.lib.lfr_wire_decode_on_device(ms.n_matches) == 1
    m = str(tmp_path / "super.pb")
    wire.write_matching_file(ms, m)
    lines = tlp.names_of(ms, range(ms.n_pairs))
    order = {n: k for k, n in enumerate(ms.image_names)}
    rng = np.random.default_rng(8)
    lists = [[l for l in lines if abs(order[l[1]] - order[l[0]]) <= w] for w in (1, 3)]
    lists.append([lines[i] for i in rng.permutation(len(lines))[: len(lines) // 3]] + lines[:2])
    own = []
    r = _run(["--matches_file", m, "--output_file", m + ".own"], {})
    assert r.returncode == 0, r.stderr
    own.append((open(m + ".own", "rb").read(), tlp.stdout_values(r.stdout.decode())))
    entries = []
    for k, ls in enumerate(lists):
        lp = tlp.write_list(tmp_path / ("l%d.txt" % k), ls)
        mk = str(tmp_path / ("own%d.pb" % k))
        with open(mk, "wb") as fh:
            fh.write(wire.encode_matching_file(tlp.own_file(ms, ls)))
        r = _run(["--matches_file", mk, "--output_file", mk + ".out"], {})
        assert r.returncode == 0, r.stderr
        own.append((open(mk + ".out", "rb").read(), tlp.stdout_values(r.stdout.decode())))
        entries.append(lp)
    for route, env in (("auto", {}), ("host", ROUTES["host"]), ("device", ROUTES["device"]),
                       ("device_cut", ROUTES["device_cut"])):
        outs = [m + "." + route] + [e + "." + route for e in entries]
        lst = tlp.pair_list(tmp_path / "p.txt", list(zip(entries, outs[1:])))
        r = _run(["--matches_file", m, "--output_file", outs[0], "--listed_pairs", lst], env)
        assert r.returncode == 0, r.stderr
        tlp.check_batch(outs, r.stdout.decode(), own)


def test_expand_kernels_compile_for_sm90a_without_spills():
    out = subprocess.run([cuobjdump(), "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S*listed_(counts|gather)_kernel\S*)", line)
        if m:
            found[m.group(2)] = lines[i + 1]
    assert set(found) == {"counts", "gather"}, out[:2000]
    for usage in found.values():
        assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), usage
