"""The problem record (include/lfr_graph.h states it), on the CPU: lfr_host_problem_record against an independent
numpy statement of SipHash-2-4 and of the record, built from host-stage exports; its invariance and sensitivity;
the update since a record against the update since the earlier MatchingFile, through the host form and the
native drop-in linked against the CPU checker; chains of runs; the Python host; the command line."""
import os
import struct

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import main as cli_main
from lfr_b200.graph import problem_from_stage
from lfr_b200.matchset import MatchSet
from test_fixed_images import checker_exe, run, stage  # noqa: F401
from test_graph_stage_adversarial import E2E_CASES, make_case
from test_update_since import BASE, CASES, banned_args, case, duplicated, reencode

M64 = (1 << 64) - 1
K0, K1 = b"lfr problem rec0", b"lfr problem rec1"
EARLIER_ERROR = b"ERROR: --earlier_record_file needs --update_initial_solution\n"
BOTH_ERROR = b"ERROR: --earlier_record_file and --previous_matches_file exclude each other\n"


# ---- SipHash-2-4, stated twice: Python integers (any message) and numpy (messages of whole words) ----------
def _rotl(x, b):
    return ((x << b) | (x >> (64 - b))) & M64


def _round(v):
    v0, v1, v2, v3 = v
    v0 = (v0 + v1) & M64; v1 = _rotl(v1, 13) ^ v0; v0 = _rotl(v0, 32)
    v2 = (v2 + v3) & M64; v3 = _rotl(v3, 16) ^ v2
    v0 = (v0 + v3) & M64; v3 = _rotl(v3, 21) ^ v0
    v2 = (v2 + v1) & M64; v1 = _rotl(v1, 17) ^ v2; v2 = _rotl(v2, 32)
    return [v0, v1, v2, v3]


def siphash(key: bytes, msg: bytes) -> int:
    k0, k1 = struct.unpack("<QQ", key)
    v = [k0 ^ 0x736F6D6570736575, k1 ^ 0x646F72616E646F6D, k0 ^ 0x6C7967656E657261, k1 ^ 0x7465646279746573]
    n = len(msg)
    blocks = [int.from_bytes(msg[i:i + 8], "little") for i in range(0, n - n % 8, 8)]
    blocks.append(int.from_bytes(msg[n - n % 8:], "little") | ((n & 0xFF) << 56))
    for m in blocks:
        v[3] ^= m
        v = _round(_round(v))
        v[0] ^= m
    v[2] ^= 0xFF
    for _ in range(4):
        v = _round(v)
    return v[0] ^ v[1] ^ v[2] ^ v[3]


def _nrotl(x, b):
    return (x << np.uint64(b)) | (x >> np.uint64(64 - b))


def _nround(v0, v1, v2, v3):
    v0 = v0 + v1; v1 = _nrotl(v1, 13) ^ v0; v0 = _nrotl(v0, 32)
    v2 = v2 + v3; v3 = _nrotl(v3, 16) ^ v2
    v0 = v0 + v3; v3 = _nrotl(v3, 21) ^ v0
    v2 = v2 + v1; v1 = _nrotl(v1, 17) ^ v2; v2 = _nrotl(v2, 32)
    return v0, v1, v2, v3


def siphash_words(key: bytes, words: np.ndarray) -> np.ndarray:
    """S(key, m) of every row of `words` ([M, n] uint64, each row the message of its n little-endian words)."""
    k0, k1 = (np.uint64(x) for x in struct.unpack("<QQ", key))
    M, n = words.shape
    v = [np.full(M, k0 ^ np.uint64(0x736F6D6570736575)), np.full(M, k1 ^ np.uint64(0x646F72616E646F6D)),
         np.full(M, k0 ^ np.uint64(0x6C7967656E657261)), np.full(M, k1 ^ np.uint64(0x7465646279746573))]
    cols = [words[:, i] for i in range(n)] + [np.full(M, np.uint64((8 * n & 0xFF) << 56))]
    for m in cols:
        v[3] = v[3] ^ m
        v = list(_nround(*_nround(*v)))
        v[0] = v[0] ^ m
    v[2] = v[2] ^ np.uint64(0xFF)
    for _ in range(4):
        v = list(_nround(*v))
    return v[0] ^ v[1] ^ v[2] ^ v[3]


# ---- the record, stated from a host-stage export -----------------------------------------------------------
def elements(g, names):
    """(element words [X, 16] uint64 (node elements zero-padded, hashed at their own length), is_node [X], the
    component of each element [X]) of every node and every kept out-edge."""
    ids = np.array([[siphash(K0, n), siphash(K1, n)] for n in
                    [x.encode("utf-8", errors="surrogateescape") for x in names]] or np.zeros((0, 2)), np.uint64)
    img = g["node_image"].astype(np.int64)
    feat = g["node_feat"].astype(np.uint64)
    track, comp = g["track"].astype(np.int64), g["comp"].astype(np.int64)
    N = img.shape[0]
    nodes = np.zeros((N, 4), np.uint64)
    if N:
        nodes[:, 0] = 0x4E
        nodes[:, 1], nodes[:, 2] = ids[img, 0], ids[img, 1]
        nodes[:, 3] = feat | ((g["is_root"] != 0).astype(np.uint64) << np.uint64(32))
    w = g["edges"].view(np.uint32).reshape(-1, 20).astype(np.uint64)
    src = np.repeat(np.arange(N), np.diff(g["row_ptr"].astype(np.int64)))
    dst = w[:, 19].astype(np.int64)
    kind = np.where(track[src] == track[dst], 1, np.where(comp[src] == comp[dst], 2, 0)).astype(np.uint64)
    k = kind != 0
    src, dst, w, kind = src[k], dst[k], w[k], kind[k]
    edges = np.zeros((src.shape[0], 16), np.uint64)
    if src.shape[0]:
        edges[:, 0] = 0x45
        edges[:, 1], edges[:, 2] = ids[img[src], 0], ids[img[src], 1]
        edges[:, 3], edges[:, 4] = ids[img[dst], 0], ids[img[dst], 1]
        edges[:, 5] = feat[src] | (feat[dst] << np.uint64(32))
        edges[:, 6] = kind | (w[:, 18] << np.uint64(32))
        edges[:, 7:16] = w[:, 0:18:2] | (w[:, 1:18:2] << np.uint64(32))
    return nodes, edges, comp, comp[src]


def model_digests(g, names, n_components):
    """[C, 2] uint64: Digest(c) of every component."""
    nodes, edges, ncomp, ecomp = elements(g, names)
    d = np.zeros((n_components, 2), np.uint64)
    for lane, key in enumerate((K0, K1)):
        np.add.at(d[:, lane], ncomp, siphash_words(key, nodes))
        np.add.at(d[:, lane], ecomp, siphash_words(key, edges))
    return d


def model_record(g, names, n_components):
    d = model_digests(g, names, n_components)
    d = d[np.lexsort((d[:, 1], d[:, 0]))]
    return b"LFRPREC1" + struct.pack("<Q", n_components) + d.astype("<u8").tobytes()


def digests_of(record):
    return [tuple(x) for x in np.frombuffer(record, "<u8", offset=16).reshape(-1, 2).tolist()]


def problem(ms, banned=()):
    skip, g, sz = stage(ms, banned)
    return problem_from_stage(ms, skip, g, sz, "native"), g


# ---- scenes --------------------------------------------------------------------------------------------------
def _edited(ms, **arrays):
    return MatchSet(**{k: (arrays[k] if k in arrays else (v.copy() if isinstance(v, np.ndarray) else v))
                       for k, v in vars(ms).items()})


def _signed_zero_and_nan():
    ms = reencode(BASE)
    d1, d2 = ms.disp1.copy(), ms.disp2.copy()
    d1[3, 4] = -0.0
    d1[4, 4] = 0.0
    d2[5, :] = np.frombuffer(struct.pack("<I", 0x7FC12345) * 18, np.float32)   # NaN payloads
    d2[6, 2] = np.frombuffer(struct.pack("<I", 0xFFA00001), np.float32)[0]
    return _edited(ms, disp1=d1, disp2=d2)


def _non_utf8():
    ms = reencode(BASE)
    names = list(ms.image_names)
    names[0] = b"\xff\xfeimg.png".decode("utf-8", errors="surrogateescape")
    names[3] = b"caf\xe9 \x00 \xc3(".decode("utf-8", errors="surrogateescape")
    return _edited(ms, image_names=names)


def _empty():
    return MatchSet([], np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0, np.float32),
                    np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros(0, np.float32),
                    np.zeros((0, 18), np.float32), np.zeros((0, 18), np.float32))


def _slice(lo, hi):
    ms = synth.generate("cfg2", scale=0.25, seed=5)
    return ms.select_pairs(np.arange(ms.n_pairs)[lo:hi])


SCENES = {
    "cfg1": lambda: synth.generate("cfg1"),
    "cfg2-head": lambda: _slice(0, 40),
    "cfg2-tail": lambda: _slice(-60, None),
    "ring60": lambda: synth.generate("ring60", scale=0.3),
    "duplicated-matches": lambda: duplicated(duplicated(reencode(BASE), 9), 30),
    "signed-zero-nan": _signed_zero_and_nan,
    "non-utf8-names": _non_utf8,
    "empty": _empty,
}
for _c in E2E_CASES:
    SCENES["adv-" + _c] = (lambda c=_c: make_case(c))


def test_siphash_published_vectors():
    key = bytes(range(16))
    assert siphash(key, bytes(range(15))) == 0xA129CA6149BE45E5
    assert siphash(key, b"") == 0x726FDB47DD0E0E31
    rng = np.random.default_rng(1)
    w = rng.integers(0, 1 << 63, size=(40, 5), dtype=np.uint64) * np.uint64(3)
    for n in (0, 1, 4, 5):
        got = siphash_words(key, w[:, :n])
        want = [siphash(key, row[:n].astype("<u8").tobytes()) for row in w]
        assert got.tolist() == want


@pytest.mark.parametrize("threads", ["1", "8"])
@pytest.mark.parametrize("name", list(SCENES))
def test_host_record_equals_the_model(name, threads, monkeypatch):
    monkeypatch.setenv("LFR_HOST_THREADS", threads)
    ms = SCENES[name]()
    p, g = problem(ms)
    got = wire.problem_record(p, ms.image_names)
    assert got == model_record(g, ms.image_names, p.n_components)
    assert len(got) == 16 + 16 * p.n_components and wire.record_is_valid(got)
    if name == "ring60":
        assert (np.diff(p.comp_ptr.astype(np.int64)) == 1).any()       # one-node components are in the record


def _relabelled(p, g, rng):
    """The same problem with nodes renumbered by a random permutation and every CSR row shuffled."""
    N = g["node_image"].shape[0]
    perm = rng.permutation(N)            # new id of old node
    inv = np.argsort(perm)               # old node of new id
    rp = g["row_ptr"].astype(np.int64)
    rows = []
    for new in range(N):
        old = inv[new]
        e = g["edges"][rp[old]:rp[old + 1]].copy()
        e["dst"] = perm[e["dst"].astype(np.int64)]
        rows.append(e[rng.permutation(e.shape[0])])
    edges = np.concatenate(rows) if rows else g["edges"][:0]
    row_ptr = np.concatenate([[0], np.cumsum([r.shape[0] for r in rows])]).astype(np.uint32)
    h = dict(g, row_ptr=row_ptr, edges=edges, node_image=g["node_image"][inv], node_feat=g["node_feat"][inv],
             track=g["track"][inv], comp=g["comp"][inv], is_root=g["is_root"][inv])
    return h


def _problem_of(ms, g, h):
    """A Problem over the arrays of `h` (comp_ptr / comp_nodes are not read by the record)."""
    import dataclasses
    p, _ = problem(ms)
    graph = dataclasses.replace(p.graph, node_image=h["node_image"].astype(np.int64), node_feat=h["node_feat"],
                                row_ptr=h["row_ptr"], edges=h["edges"], n_nodes=h["node_image"].shape[0])
    return dataclasses.replace(p, graph=graph, track=h["track"], comp=h["comp"], is_root=h["is_root"])


def test_record_does_not_depend_on_node_or_edge_order():
    ms = synth.generate("ring60", scale=0.3)
    p, g = problem(ms)
    want = wire.problem_record(p, ms.image_names)
    for seed in range(3):
        h = _relabelled(p, g, np.random.default_rng(seed))
        assert wire.problem_record(_problem_of(ms, g, h), ms.image_names) == want


def _flip_flow_bit(g, e):
    w = g["edges"].view(np.uint32).reshape(-1, 20)
    w[e, 7] ^= 1


def _sim_ulp(g, e):
    g["edges"]["sim"][e] = np.nextafter(g["edges"]["sim"][e], np.float32(2))


def _duplicate_edge(g, e):
    v = int(np.searchsorted(g["row_ptr"].astype(np.int64), e, side="right") - 1)
    g["edges"] = np.insert(g["edges"], e, g["edges"][e])
    g["row_ptr"] = g["row_ptr"].copy()
    g["row_ptr"][v + 1:] += 1


def _kept_edge(g):
    """An edge kept inside a component of at least 3 nodes, and its source."""
    w = g["edges"]
    src = np.repeat(np.arange(g["node_image"].shape[0]), np.diff(g["row_ptr"].astype(np.int64)))
    dst = w["dst"].astype(np.int64)
    size = np.bincount(g["comp"].astype(np.int64))
    ok = np.nonzero((g["track"][src] == g["track"][dst]) & (size[g["comp"][src]] >= 3))[0]
    return int(ok[len(ok) // 2]), int(src[ok[len(ok) // 2]])


SENSITIVITY = ["flow-bit", "sim-ulp", "root-flag", "kind", "duplicated-edge", "renamed-image", "moved-feature"]


@pytest.mark.parametrize("change", SENSITIVITY)
def test_each_change_moves_exactly_the_digests_concerned(change):
    ms = synth.generate("ring60", scale=0.3)
    p, g = problem(ms)
    before = wire.problem_record(p, ms.image_names)
    d = model_digests(g, ms.image_names, p.n_components)
    h = {k: v.copy() for k, v in g.items()}
    e, v = _kept_edge(g)
    names = list(ms.image_names)
    comps = {int(g["comp"][v])}
    if change == "flow-bit":
        _flip_flow_bit(h, e)
    elif change == "sim-ulp":
        _sim_ulp(h, e)
    elif change == "root-flag":
        h["is_root"][v] ^= 1
    elif change == "kind":
        h["track"][v] = h["track"].max() + 1            # v's same-track edges become Tukey edges
    elif change == "duplicated-edge":
        _duplicate_edge(h, e)
    elif change == "renamed-image":
        k = int(g["node_image"][v])
        names[k] = names[k] + ".renamed"
        comps = set(g["comp"][g["node_image"] == k].tolist())
    elif change == "moved-feature":
        h["node_feat"][v] = h["node_feat"].max() + 1
    after = wire.problem_record(_problem_of(_edited(ms, image_names=names), g, h), names)
    assert after == model_record(h, names, p.n_components)
    lost = set(digests_of(before)) - set(digests_of(after))
    assert lost == {tuple(d[c].tolist()) for c in comps}
    assert len(set(digests_of(after)) - set(digests_of(before))) == len(comps)


def _record_of_run(exe, matches, tmp_path, tag, extra=()):
    out, rec = tmp_path / (tag + ".pb"), tmp_path / (tag + ".rec")
    r = run(exe, ["--matches_file", str(matches), "--output_file", str(out), "--record_file", str(rec)] + list(extra))
    assert r.returncode == 0, r.stderr
    return out, rec


def _untimed(stdout):
    return [x for x in stdout.splitlines() if b"time:" not in x]


@pytest.mark.parametrize("name", list(CASES))
def test_update_since_record_equals_update_since_matches(checker_exe, tmp_path_factory, tmp_path, name):  # noqa: F811
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, name)
    a2, rec = _record_of_run(checker_exe, o, tmp_path, "a")
    assert a2.read_bytes() == A                                   # --record_file changes nothing else
    record = rec.read_bytes()
    p_old, g_old = problem(old)
    assert record == model_record(g_old, old.image_names, p_old.n_components)
    p, g = problem(new, banned)
    want = wire.update_solution_since(A, p, old)
    got = wire.update_solution_since_record(A, p, record)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]) and got[2:] == want[2:]
    outs = []
    for flag, path in (("--previous_matches_file", o), ("--earlier_record_file", rec)):
        out = tmp_path / ("out%d.pb" % len(outs))
        r = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a),
                              "--update_initial_solution", flag, str(path)] + banned_args(banned))
        assert r.returncode == 0, r.stderr
        outs.append((out.read_bytes(), _untimed(r.stdout)))
    assert outs[0] == outs[1]


@pytest.mark.parametrize("extra", [["--fixed_images", 1], ["--carry_initial_solution"], ["--gpus", "2"], ["parts"]])
def test_native_with_fixed_images_carry_devices_and_parts(checker_exe, tmp_path_factory, tmp_path, extra):  # noqa: F811
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, "banned")
    _, rec = _record_of_run(checker_exe, o, tmp_path, "a")
    if extra == ["parts"]:
        wire.write_matching_file(new, str(tmp_path / "new_split.pb"), pairs_per_part=max(new.n_pairs // 3, 1))
        n, extra = tmp_path / "new_split.pb", []
    extra = [new.image_names[x] if isinstance(x, int) else x for x in extra]
    outs = []
    for flag, path in (("--previous_matches_file", o), ("--earlier_record_file", rec)):
        out = tmp_path / ("out%d.pb" % len(outs))
        r = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a),
                              "--update_initial_solution", flag, str(path)] + banned_args(banned) + extra)
        assert r.returncode == 0, r.stderr
        outs.append((out.read_bytes(), _untimed(r.stdout)))
    assert outs[0] == outs[1]
    # the record of a run does not depend on --fixed_images, a held set or the start point
    _, r1 = _record_of_run(checker_exe, n, tmp_path, "plain", banned_args(banned))
    _, r2 = _record_of_run(checker_exe, n, tmp_path, "upd", ["--initial_solution", str(a), "--update_initial_solution",
                                                             "--earlier_record_file", str(rec)] + banned_args(banned) + extra)
    assert r1.read_bytes() == r2.read_bytes()


def test_chain_with_records_equals_chain_with_matching_files(checker_exe, tmp_path):  # noqa: F811
    names = BASE.image_names
    stages = []
    for k in (3, 1, 0):
        drop = np.arange(len(names) - k, len(names))
        keep = ~(np.isin(BASE.pair_img1, drop) | np.isin(BASE.pair_img2, drop))
        m = tmp_path / ("m%d.pb" % k)
        m.write_bytes(wire.encode_matching_file(reencode(BASE.select_pairs(np.nonzero(keep)[0]))))
        stages.append(m)
    # chain 1: records; chain 2: the earlier MatchingFiles
    a, rec = _record_of_run(checker_exe, stages[0], tmp_path, "A")
    prev_out, prev_rec = a, rec
    prev_out2 = a
    for i, m in enumerate(stages[1:]):
        out, nrec = _record_of_run(checker_exe, m, tmp_path, "R%d" % i,
                                   ["--initial_solution", str(prev_out), "--u", "--earlier_record_file", str(prev_rec)])
        out2 = tmp_path / ("P%d.pb" % i)
        r = run(checker_exe, ["--matches_file", str(m), "--output_file", str(out2), "--initial_solution", str(prev_out2),
                              "--u", "--previous_matches_file", str(stages[i])])
        assert r.returncode == 0, r.stderr
        assert out.read_bytes() == out2.read_bytes()
        prev_out, prev_rec, prev_out2 = out, nrec, out2


def test_python_host_equals_the_native_host(checker_exe, tmp_path_factory, tmp_path, oracle, monkeypatch):  # noqa: F811
    from lfr_b200.solver import refine
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, "banned")
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    _, rec = _record_of_run(checker_exe, o, tmp_path, "a")
    opts = oracle.default_options(n_threads=4)
    out, rec2 = _record_of_run(checker_exe, n, tmp_path, "b", ["--initial_solution", str(a), "--u",
                                                               "--earlier_record_file", str(rec)] + banned_args(banned))
    _, _, _, sol = refine(wire.read_matching_file(str(n)), banned,
                          solve_fn=lambda q, x=None: oracle.solve(q, opts, positions=x), initial_solution=A,
                          update_initial_solution=True, previous_record=rec.read_bytes(), record_problem=True)
    assert wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj) == out.read_bytes()
    assert sol.record == rec2.read_bytes()
    for bad in (dict(previous_record=rec.read_bytes()),                                  # needs the update
                dict(update_initial_solution=True, previous_record=rec.read_bytes(), previous_matches=old),
                dict(update_initial_solution=True, previous_record=rec.read_bytes()[:-1])):
        with pytest.raises(ValueError):
            refine(new, (), initial_solution=A, **bad)


def test_command_line_errors_and_prefixes(checker_exe, tmp_path_factory, tmp_path, capfd):  # noqa: F811
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, "same")
    _, rec = _record_of_run(checker_exe, o, tmp_path, "a")
    out = tmp_path / "out.pb"
    bad = tmp_path / "bad.rec"
    good = rec.read_bytes()
    base = ["--matches_file", str(n), "--output_file", str(out)]
    upd = ["--initial_solution", str(a), "--u"]
    unordered = good[:16] + good[32:48] + good[16:32] + good[48:] if len(good) >= 48 else None
    cases = [
        (["--earlier_record_file", str(rec)], 2, EARLIER_ERROR, None),
        (["--initial_solution", str(a), "--earlier_record_file", str(rec)], 2, EARLIER_ERROR, None),
        (["--update_initial_solution", "--earlier_record_file", str(rec)], 2,
         b"ERROR: --update_initial_solution needs --initial_solution FILE\n", None),
        (["--previous_matches_file", str(o), "--earlier_record_file", str(rec)], 2,
         b"ERROR: --previous_matches_file needs --update_initial_solution\n", None),
        (upd + ["--previous_matches_file", str(o), "--earlier_record_file", str(rec)], 2, BOTH_ERROR, None),
        (upd + ["--earlier_record_file", str(tmp_path / "missing.rec")], 2,
         b"ERROR: cannot read the earlier record file", None),
    ]
    assert unordered is not None and unordered != good
    for blob in (b"", good[:-1], b"LFRPREC2" + good[8:], good + b"\0" * 16, unordered):
        cases.append((upd + ["--earlier_record_file", str(bad)], 2,
                      b"ERROR: '%s' is not a problem record\n" % str(bad).encode(), blob))
    for args, code, line, blob in cases:
        if blob is not None:
            bad.write_bytes(blob)
        r = run(checker_exe, base + args)
        assert r.returncode == code and r.stdout == b"", (args, r.stderr)
        assert r.stderr.count(b"\n") == 1 and r.stderr.startswith(line), r.stderr
        assert not out.exists()
        assert cli_main(base + args) == code
        err = capfd.readouterr()
        assert err.out == "" and err.err.encode().startswith(line), err
        assert not out.exists()
    # a record file that cannot be written: the SolutionFile is written, then one ERROR line and 255
    unwritable = str(tmp_path / "no-such-dir" / "r.rec")
    r = run(checker_exe, base + ["--record_file", unwritable])
    assert r.returncode == 255 and out.exists()
    assert r.stderr == b"ERROR: cannot write the record file '%s'\n" % unwritable.encode()
    # prefixes: --r / --record and --e / --earlier
    recs = []
    for flag in ("--record_file", "--r", "--record"):
        f = tmp_path / ("p%d.rec" % len(recs))
        r = run(checker_exe, base + [flag, str(f)])
        assert r.returncode == 0, r.stderr
        recs.append(f.read_bytes())
    assert recs[0] == recs[1] == recs[2] == good
    outs = []
    for flag in ("--earlier_record_file", "--e", "--earlier"):
        r = run(checker_exe, base + upd + [flag, str(rec)])
        assert r.returncode == 0, r.stderr
        outs.append(out.read_bytes())
    assert outs[0] == outs[1] == outs[2]
    r = run(checker_exe, base + ["--record_file"])
    assert r.returncode == 1 and b"the required argument for option '--record_file' is missing" in r.stderr
    helptext = run(checker_exe, ["--help"]).stdout
    assert b"record" not in helptext and b"earlier" not in helptext
    from lfr_b200.cli import USAGE
    assert helptext == b"Patch Match graph problem solver\n\n" + USAGE.encode()
