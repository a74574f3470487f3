"""The SolutionFile encoded on the device (lfr_plan_encode_solution, include/lfr_graph.h; csrc/lfr_solution.cuh)
against the host path on the same plan: lfr_plan_download, the output assembly of solve.cc:643-679
(solver.assemble_solution) and lfr_wire_encode_solution.  Bytes and the "> 0.5" count must be equal, for
plans from matches and from MatchingFile bytes, before the first solve and after each solve.

CPU: only the product library exports the encoder.
GPU: scenes, banned images and parts; varint boundaries of names, facts, feature indices and image bodies;
start points that reach the encoder unsolved (signed zeros, denormals, ties, overflow, infinities, NaN
payloads); refusals and the size protocol; the native drop-in's device route."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from lfr_b200 import MatchSet, build_problem, synth, wire
from lfr_b200.capi import B200_LIB_PATH, HOST_LIB_PATH, Plan
from lfr_b200.solver import assemble_solution
from test_drop_in_device_stage import both_routes
from test_graph_stage_adversarial import E2E_CASES, make_case
from test_native_exe import PRODUCT, product_exe  # noqa: F401  (fixture)
from test_ref_solve import GOLD, untimed

LFR_EINVAL = -1


# ---- helpers ------------------------------------------------------------------------------------------
def decoded(parts):
    """The host decode of MatchingFile parts, concatenated as the drop-in reads `.part.N` files: the image
    ids every plan of these parts uses."""
    got = [wire.decode_matching_file(p) for p in parts]
    return got[0] if len(got) == 1 else MatchSet.concatenate(got)


def image_facts(ms, banned=()):
    """fact by image id: the first one seen among the pairs kept (solve.cc:449,451), 0 for the others."""
    banned = set(banned)
    fact = np.zeros(len(ms.image_names), np.float32)
    seen = np.zeros(len(ms.image_names), bool)
    for a, b, fa, fb in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist(), ms.pair_fact1, ms.pair_fact2):
        if ms.image_names[a] in banned or ms.image_names[b] in banned:
            continue
        for i, f in ((a, fa), (b, fb)):
            if not seen[i]:
                seen[i], fact[i] = True, f
    return fact


def host_encoding(plan, names, fact):
    """The host path on the plan's current positions: (bytes, n_outside)."""
    pos, _ = plan.download()
    g = plan.export_graph()
    graph = SimpleNamespace(n_nodes=plan.n_nodes, node_image=g["node_image"].astype(np.int64), node_feat=g["node_feat"],
                            image_names=names, image_fact=fact)
    with np.errstate(all="ignore"):      # float32 of 1e39, NaN: the conversion x86 does, without warnings
        s = assemble_solution(SimpleNamespace(graph=graph), pos)
    return wire.encode_solution(s.image_names, s.fact, s.img_ptr, s.feature_idx, s.di, s.dj), s.n_outside


def assert_same_encoding(plan, names, fact):
    """The plain encoder against the host path; the masked, grouped and carried encoders, on the inputs that make
    them the plain one (every image written, one group of every image, an empty file), against the plain one."""
    got = plan.encode_solution(names, fact)
    want = host_encoding(plan, names, fact)
    assert got[1] == want[1]
    assert got[0] == want[0]
    data, n_outside = got
    blob, off = wire._names_blob(list(names))
    fact32 = np.ascontiguousarray(fact, np.float32)
    args = (plan.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact32.ctypes.data)
    buf = np.empty(max(len(data), 1), np.uint8)
    f = plan.lib.lib.lfr_plan_encode_solution_images
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_uint64, C.POINTER(C.c_uint64)]
    f.restype = C.c_int64
    n = C.c_uint64(7)
    written = np.ones(max(len(names), 1), np.uint8)
    assert f(*args, written.ctypes.data, buf.ctypes.data, buf.size, C.byref(n)) == len(data)
    assert buf[:len(data)].tobytes() == data and n.value == n_outside
    group = np.zeros(max(len(names), 1), np.uint32)
    goff, outside = np.full(2, 7, np.uint64), np.full(1, 7, np.uint64)
    assert plan.lib.lib.lfr_plan_encode_solution_groups(*args, group.ctypes.data, 1, buf.ctypes.data, buf.size,
                                                        goff.ctypes.data, outside.ctypes.data) == len(data)
    assert buf[:len(data)].tobytes() == data and goff.tolist() == [0, len(data)] and outside.tolist() == [n_outside]
    assert plan.encode_solution_carried(names, fact, b"") == (data, n_outside, 0)
    return data


def plans(b200, parts, banned=(), positions=None):
    """A plan from the host decode of `parts` and one from their bytes, with the names and facts by image id."""
    ms = decoded(parts)
    names, fact = ms.image_names, image_facts(ms, banned)
    a = Plan.from_matches(b200, ms, banned_images=banned, positions=positions)
    b = Plan.from_wire(b200, parts, banned_images=banned, positions=positions)
    assert b.image_names == names
    return [a, b], names, fact


def check_states(b200, parts, banned=()):
    """Before the first solve, after it and after a second solve, on both plans; returns the encodings."""
    ps, names, fact = plans(b200, parts, banned)
    out = []
    for p in ps:
        out.append(assert_same_encoding(p, names, fact))
        if p.n_nodes:
            for _ in range(2):
                p.solve()
                out.append(assert_same_encoding(p, names, fact))
        p.close()
    return out


def pair_set(names, feats, facts=(1.0, 1.0)):
    """Two images, one pair, match k between feature feats[k] of both."""
    n = len(feats)
    f = np.asarray(feats, np.uint32)
    return MatchSet(image_names=list(names), pair_img1=np.array([0]), pair_img2=np.array([1]),
                    pair_fact1=np.array([facts[0]], np.float32), pair_fact2=np.array([facts[1]], np.float32),
                    pair_ptr=np.array([0, n]), feat1=f, feat2=f.copy(), sim=np.ones(n, np.float32),
                    disp1=np.zeros((n, 18), np.float32), disp2=np.zeros((n, 18), np.float32))


def image_bodies(data):
    """(body length, length-prefix bytes) of every top-level Image record."""
    out, k = [], 0
    while k < len(data):
        assert data[k] == 0x0A
        k += 1
        v, shift, n = 0, 0, 0
        while True:
            b = data[k + n]
            v |= (b & 0x7F) << shift
            shift += 7
            n += 1
            if not b & 0x80:
                break
        out.append((v, n))
        k += n + v
    return out


# ---------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------
def test_only_the_product_library_exports_the_encoder(oracle):
    from test_native_exe import _csrc_build
    _csrc_build().build()
    assert hasattr(C.CDLL(B200_LIB_PATH), "lfr_plan_encode_solution")
    assert not hasattr(C.CDLL(HOST_LIB_PATH), "lfr_plan_encode_solution")
    assert not hasattr(oracle.lib, "lfr_plan_encode_solution")


# ---------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg,scale", [("cfg1", 1.0), ("cfg2", 1.0), ("cfg3", 1.0), ("cfg4", 1.0), ("cfg5", 0.1),
                                       ("ring60", 1.0)])
def test_scenes(b200, cfg, scale):
    out = check_states(b200, [wire.encode_matching_file(synth.generate(cfg, scale=scale))])
    assert out[0] != out[1]                 # the solve moved something: zeros before, displacements after


@pytest.mark.gpu
@pytest.mark.parametrize("case", E2E_CASES)
def test_adversarial_match_graphs(b200, case):
    """Among them feature indices 0 and 2^32 - 1, and images without nodes (feature_extremes)."""
    check_states(b200, [wire.encode_matching_file(make_case(case))])


@pytest.mark.gpu
def test_banned_images_parts_empty_and_all_banned(b200):
    ms = decoded([wire.encode_matching_file(synth.generate("cfg2", scale=0.25, seed=11))])
    ms = MatchSet.concatenate([ms, pair_set(["lonely.png", "gone.png"], range(40))])
    data = wire.encode_matching_file(ms)
    # lonely.png is named in the input, but its only pair is banned: it has no node and no Image record
    out = check_states(b200, [data], banned=["gone.png", ms.image_names[3]])
    names = [n for n, *_ in wire.decode_solution(out[-1])]
    assert "lonely.png" not in names and ms.image_names[3] not in names and len(names) == len(ms.image_names) - 3
    step = max(1, ms.n_pairs // 3)
    parts = [wire.encode_matching_file(ms, lo, min(ms.n_pairs, lo + step)) for lo in range(0, ms.n_pairs, step)]
    assert len(parts) > 2
    check_states(b200, parts)
    for parts, banned in (([b""], ()), ([data], ms.image_names)):
        ps, names, fact = plans(b200, parts, banned)
        for p in ps:
            assert p.n_nodes == 0 and p.encode_solution(names, fact) == (b"", 0)
            assert host_encoding(p, names, fact) == (b"", 0)
            p.close()


@pytest.mark.gpu
def test_names_facts_and_feature_indices_at_varint_boundaries(b200):
    names = ["", "a", "b" * 127, "c" * 128, "d" * 16384, "e.png"]
    fact = np.array([0.0, -0.0, 1e-40, 1.0, 0.0, 2.5], np.float32)   # 1e-40: a float32 denormal
    rng = np.random.default_rng(5)
    sets = []
    for i in range(len(names) - 1):
        feats = [0, 127, 128, 2 ** 32 - 1] + rng.choice(np.arange(1, 100000), 30, replace=False).tolist()
        s = pair_set([names[i], names[i + 1]], sorted(set(feats)), facts=(fact[i], fact[i + 1]))
        sets.append(s)
    ms = MatchSet.concatenate(sets)
    assert ms.image_names == names
    out = check_states(b200, [wire.encode_matching_file(ms)])
    got = {n: np.float32(f).view(np.uint32) for n, f, *_ in wire.decode_solution(out[0])}
    assert got == dict(zip(names, fact.view(np.uint32)))


def _record(f):
    return 2 + (0 if f == 0 else 1 + (int(f).bit_length() + 6) // 7) + 10   # di, dj non-zero


def _name_for(room):
    """The name length whose string field takes exactly `room` bytes."""
    for nl in range(room, 0, -1):
        if 1 + (nl.bit_length() + 6) // 7 + nl == room:
            return nl
    raise AssertionError(room)


@pytest.mark.gpu
@pytest.mark.parametrize("limit", [128, 16384, 2097152])
def test_image_length_prefixes_of_1_to_4_bytes(b200, limit):
    """Two images of one pair, bodies limit - 1 and limit: their length prefixes differ by one byte.  Before
    the first solve every node sits at (0.25, -0.125), so every record's size is known."""
    sizes = np.cumsum([_record(f) for f in range(200000)])
    M = int(np.searchsorted(sizes, limit - 1 - 5 - 40, side="right"))
    R = int(sizes[M - 1])
    names = ["x" * _name_for(limit - 1 - 5 - R), "y" * _name_for(limit - 5 - R)]
    parts = [wire.encode_matching_file(pair_set(names, range(M)))]
    ps, names, fact = plans(b200, parts, positions=np.tile([0.25, -0.125], (2 * M, 1)))
    k = (limit.bit_length() - 1) // 7
    for p in ps:
        assert p.n_nodes == 2 * M
        got = assert_same_encoding(p, names, fact)
        assert sorted(image_bodies(got)) == [(limit - 1, k), (limit, k + 1)]
        p.close()


def _f64(bits):
    return np.array([bits], np.uint64).view(np.float64)[0]


@pytest.mark.gpu
def test_start_points_through_the_encoder(b200):
    """Roots and the nodes of size-1 components keep their start bitwise through a solve, so these values
    reach the encoder before and after it.  Non-finite values only where no solve reads them."""
    parts = [wire.encode_matching_file(synth.generate("cfg1"))]
    finite = [0.0, -0.0, 1e-46, -1e-46, 1e-40, -3e-42, 0.5, -0.5, np.nextafter(0.5, 1.0), -np.nextafter(0.5, 1.0),
              1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24, -(1 + 2.0 ** -24), 2.0 ** -150, 3 * 2.0 ** -150, 1e39, -1e39,
              np.float32(3.4028235e38).item() * (1 + 2.0 ** -25)]
    nonfinite = [np.inf, -np.inf, _f64(0x7FF8000000000001), _f64(0x7FF0000000000001), _f64(0xFFF4000020000000),
                 _f64(0x7FF123456789ABCD), _f64(0xFFFFFFFFFFFFFFFF), _f64(0xFFF0000000000001)]
    ms = decoded(parts)
    probe = Plan.from_matches(b200, ms)
    g = probe.export_graph()
    probe.close()
    sizes = np.diff(g["comp_ptr"].astype(np.int64))
    single = g["comp_nodes"][g["comp_ptr"][:-1][sizes == 1]]
    roots = np.nonzero(g["is_root"])[0]
    roots = roots[~np.isin(roots, single)]
    assert single.shape[0] * 2 >= len(nonfinite) and roots.shape[0] * 2 >= len(finite)
    pos = np.zeros((g["node_image"].shape[0], 2))
    pos[roots] = np.resize(finite, (roots.shape[0], 2))
    pos[single] = np.resize(nonfinite + finite, (single.shape[0], 2))
    ps, names, fact = plans(b200, parts, positions=pos)
    for p in ps:
        for _ in range(2):
            assert_same_encoding(p, names, fact)
            p.solve()
        after, _ = p.download()
        assert after[single].tobytes() == pos[single].tobytes() and after[roots].tobytes() == pos[roots].tobytes()
        assert_same_encoding(p, names, fact)
        p.close()


@pytest.mark.gpu
def test_refusals_and_the_size_protocol(b200):
    ms = synth.generate("cfg1")
    p = Plan(b200, build_problem(ms))
    with pytest.raises(RuntimeError, match=r"\(%d\)" % LFR_EINVAL):
        p.encode_solution(ms.image_names, image_facts(ms))
    p.close()
    ps, names, fact = plans(b200, [wire.encode_matching_file(ms)])
    blob, off = wire._names_blob(names)
    f = b200.lib.lfr_plan_encode_solution
    for p in ps:
        p.solve()
        want, n_out = p.encode_solution(names, fact)
        buf = np.full(len(want) + 16, 0xA5, np.uint8)
        n = C.c_uint64(7)
        args = (p.handle, None, len(names), blob.ctypes.data, off.ctypes.data, fact.ctypes.data, buf.ctypes.data)
        assert f(*args, len(want) - 1, C.byref(n)) == len(want)
        assert (buf == 0xA5).all() and n.value == n_out
        assert f(*args, len(want), None) == len(want)
        assert buf[:len(want)].tobytes() == want and (buf[len(want):] == 0xA5).all()
        assert f(p.handle, None, len(names) - 1, blob.ctypes.data, off.ctypes.data, fact.ctypes.data, None, 0, None) \
            == LFR_EINVAL
        p.close()


# ---- the native drop-in -----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["linesearch", "fountain_2pct"])
def test_drop_in_device_route_reproduces_the_goldens(product_exe, tmp_path, name):  # noqa: F811
    """As test_native_exe's GPU test, on the device route: the same stdout, and the reference's SolutionFile
    float for float (byte-identical unless a displacement sits within 1e-16 of a float32 rounding boundary)."""
    o = tmp_path / "o.pb"
    r = subprocess.run([PRODUCT, "--matches_file", os.path.join(GOLD, name + "_matches.pb"), "--output_file", str(o)],
                       capture_output=True, text=True, env=dict(os.environ, LFR_GRAPH_STAGE="device"))
    assert r.returncode == 0, r.stderr
    assert untimed(r.stdout) == open(os.path.join(GOLD, name + "_stdout.txt")).read().splitlines()
    got, want = o.read_bytes(), open(os.path.join(GOLD, name + "_solution.pb"), "rb").read()
    if got != want:
        a, b = wire.decode_solution(got), wire.decode_solution(want)
        assert [x[0] for x in a] == [x[0] for x in b]
        for (_, fa, ia, dia, dja), (_, fb, ib, dib, djb) in zip(a, b):
            assert fa == fb and np.array_equal(ia, ib)
            assert np.abs(dia - dib).max() <= 1e-4 / 16 and np.abs(dja - djb).max() <= 1e-4 / 16


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["cfg2", "cfg4"])
def test_drop_in_device_route_writes_the_host_routes_bytes(product_exe, tmp_path, cfg):  # noqa: F811
    m = tmp_path / "m.pb"
    wire.write_matching_file(synth.generate(cfg), str(m))
    res = both_routes(tmp_path, ["--matches_file", str(m)])
    assert res["host"][0] == 0, res["host"][2]
    assert res["device"] == res["host"] and len(res["host"][3]) > 0
