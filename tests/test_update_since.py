"""Updating an earlier SolutionFile since an earlier MatchingFile, on the CPU: the host form
(lfr_wire_update_solution_since, include/lfr_host.h) against an independent Python statement of the rule
(include/lfr_graph.h) built from two host-stage exports, and the drop-in's --previous_matches_file through the
native executable linked against the CPU checker (oracle/liblfr_ref.so) and the Python host's path.  Touched
components are the plain run's, bit for bit; held ones carry A.pb's bits."""
import os

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import main as cli_main
from lfr_b200.graph import problem_from_stage
from lfr_b200.matchset import MatchSet
from lfr_b200.solver import constant_problem
from test_fixed_images import checker_exe, run, stage  # noqa: F401
from test_keep_solution import entries_model
from test_update_solution import EMPTY, SKIPPED, assembled, table

PREV_ERROR = b"ERROR: --previous_matches_file needs --update_initial_solution\n"


def reencode(ms):
    """`ms` through the wire: image ids in order of first appearance, only names that have a pair."""
    return wire.decode_matching_file(wire.encode_matching_file(ms))


def kept_out_edges(g, names):
    """{(name, feat): sorted [(dst key, kind, 19 words)]} of every node's kept out-edges."""
    img, feat, comp, track = (g[k].astype(np.int64) for k in ("node_image", "node_feat", "comp", "track"))
    key = [(names[i], int(f)) for i, f in zip(img.tolist(), feat.tolist())]
    words = g["edges"].view(np.uint32).reshape(-1, 20)
    out = {}
    rp = g["row_ptr"].astype(np.int64)
    for v in range(img.shape[0]):
        recs = []
        for e in range(rp[v], rp[v + 1]):
            w = int(words[e, 19])
            kind = 1 if track[v] == track[w] else (2 if comp[v] == comp[w] else 0)
            if kind:
                recs.append((key[w], kind, tuple(words[e, :19].tolist())))
        out[key[v]] = sorted(recs)
    return key, out


def since_model(new_ms, banned, old_ms, data):
    """The rule, independently: (positions, held, n_held, n_touched, n_changed) of this run's nodes."""
    _, g, _ = stage(new_ms, banned)
    _, h, _ = stage(old_ms)
    key, edges = kept_out_edges(g, new_ms.image_names)
    pkey, pedges = kept_out_edges(h, old_ms.image_names)
    comp = g["comp"].astype(np.int64)
    C_ = int(g["comp_ptr"].shape[0] - 1)
    pcomp = dict(zip(pkey, h["comp"].tolist()))
    proot = dict(zip(pkey, h["is_root"].tolist()))
    pmembers = {}
    for k, c in pcomp.items():
        pmembers.setdefault(c, set()).add(k)
    members = {}
    for v, k in enumerate(key):
        members.setdefault(int(comp[v]), []).append(v)
    changed = np.zeros(C_, bool)
    for c, vs in members.items():
        ks = [key[v] for v in vs]
        pcs = {pcomp.get(k) for k in ks}
        ok = None not in pcs and len(pcs) == 1 and pmembers[pcs.pop()] == set(ks)
        ok = ok and all(bool(g["is_root"][v]) == bool(proot[key[v]]) for v in vs)
        ok = ok and all(edges[k] == pedges[k] for k in ks)
        changed[c] = not ok
    pos, _, has = entries_model(data, new_ms.image_names, g["node_image"], g["node_feat"])
    touched = changed.copy()
    touched[comp[~has]] = True
    held = has & ~touched[comp]
    pos = np.where(held[:, None], pos, 0.0)
    return pos, held, int(held.sum()), int(touched.sum()), int(changed.sum())


def with_match(ms, m, sim=None, disp1=None):
    """`ms` with match m's sim or disp1 replaced."""
    out = MatchSet(**{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in vars(ms).items()})
    if sim is not None:
        out.sim[m] = sim
    if disp1 is not None:
        out.disp1[m] = disp1
    return out


def duplicated(ms, m):
    """`ms` with match m repeated right after itself (its pair gains one match)."""
    p = int(np.searchsorted(ms.pair_ptr, m, side="right") - 1)
    idx = np.insert(np.arange(ms.n_matches), m + 1, m)
    ptr = ms.pair_ptr.copy()
    ptr[p + 1:] += 1
    return MatchSet(ms.image_names, ms.pair_img1, ms.pair_img2, ms.pair_fact1, ms.pair_fact2, ptr, ms.feat1[idx],
                    ms.feat2[idx], ms.sim[idx], ms.disp1[idx], ms.disp2[idx])


BASE = synth.generate("cfg2", scale=0.1, seed=3)


def _appended(k):
    """(OLD, NEW): OLD without the pairs of the last k images, NEW = OLD's pairs then those pairs."""
    new_img = np.arange(len(BASE.image_names) - k, len(BASE.image_names))
    touch = np.isin(BASE.pair_img1, new_img) | np.isin(BASE.pair_img2, new_img)
    old_idx, new_idx = np.nonzero(~touch)[0], np.nonzero(touch)[0]
    return reencode(BASE.select_pairs(old_idx)), reencode(BASE.select_pairs(np.concatenate([old_idx, new_idx]))), ()


def _changed_flow():
    old = reencode(BASE)
    d = old.disp1[5].copy()
    d[3] = 0.0
    old = with_match(old, 5, disp1=d)
    d = d.copy()
    d[3] = -0.0
    return old, with_match(old, 5, disp1=d), ()


def _new_pair():
    a, b = int(BASE.pair_img1[7]), int(BASE.pair_img2[7])
    keep = np.nonzero(~((BASE.pair_img1 == a) & (BASE.pair_img2 == b)))[0]
    old = reencode(BASE.select_pairs(keep))
    return old, reencode(BASE.select_pairs(np.concatenate([keep, [7]]))), ()


def _renamed():
    old = reencode(BASE)
    names = list(old.image_names)
    names[2] = names[2] + ".renamed"
    return old, MatchSet(names, *[getattr(old, k) for k in ("pair_img1", "pair_img2", "pair_fact1", "pair_fact2",
                                                           "pair_ptr", "feat1", "feat2", "sim", "disp1", "disp2")]), ()


CASES = {
    "same": lambda: (reencode(BASE), reencode(BASE), ()),
    "new-k1": lambda: _appended(1),
    "new-k3": lambda: _appended(3),
    "banned": lambda: (reencode(BASE), reencode(BASE), (reencode(BASE).image_names[4],)),
    "sim": lambda: (reencode(BASE), with_match(reencode(BASE), 11, sim=np.nextafter(reencode(BASE).sim[11], np.float32(2))),
                    ()),
    "flow-signed-zero": _changed_flow,
    "duplicate-match": lambda: (reencode(BASE), duplicated(reencode(BASE), 9), ()),
    "new-pair": _new_pair,
    "renamed": _renamed,
}
_cases = {}


def case(checker_exe, tmp_path_factory, name):  # noqa: F811
    """(OLD, NEW, banned, OLD path, NEW path, A.pb path, A bytes): A.pb is the checker's output on OLD."""
    if name not in _cases:
        old, new, banned = CASES[name]()
        d = tmp_path_factory.mktemp("since_" + name)
        o, n, a = d / "old.pb", d / "new.pb", d / "a.pb"
        o.write_bytes(wire.encode_matching_file(old))
        n.write_bytes(wire.encode_matching_file(new))
        r = run(checker_exe, ["--matches_file", str(o), "--output_file", str(a)])
        assert r.returncode == 0, r.stderr
        _cases[name] = (old, new, tuple(banned), o, n, a, a.read_bytes())
    return _cases[name]


def banned_args(banned):
    return [x for nm in banned for x in ("--banned_images", nm)]


def held_keys(ms, g, held):
    return [(ms.image_names[i], int(f)) for i, f in zip(g["node_image"][held].tolist(), g["node_feat"][held].tolist())]


@pytest.mark.parametrize("name", list(CASES))
def test_host_form_equals_the_model(checker_exe, tmp_path_factory, name):  # noqa: F811
    old, new, banned, _, _, _, A = case(checker_exe, tmp_path_factory, name)
    skip, g, sz = stage(new, banned)
    p = problem_from_stage(new, skip, g, sz, "native")
    got = wire.update_solution_since(A, p, old)
    want = since_model(new, banned, old, A)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]) and got[2:] == want[2:], (got[2:], want[2:])
    plain = wire.update_solution(A, new.image_names, g["node_image"], g["node_feat"], g["comp"], p.n_components)
    assert got[3] >= plain[3] and not (got[1] & ~plain[1]).any()   # a superset of the plain update's touched set
    n_changed = got[4]
    if name == "same":
        assert n_changed == 0 and got[1].all()
    elif name in ("sim", "flow-signed-zero", "duplicate-match"):
        assert n_changed <= 2 and got[1].any()                        # at most the match's two endpoints' components
    else:
        assert n_changed >= 1
    if name == "banned":
        assert got[3] > plain[3]                                     # the plain update misses the lost keypoints


@pytest.mark.parametrize("name", list(CASES))
def test_native_output_is_the_full_run_on_touched_and_a_on_held(checker_exe, tmp_path_factory, tmp_path, name):  # noqa: F811
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, name)
    out, out0 = tmp_path / "out.pb", tmp_path / "out0.pb"
    r = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a),
                          "--update_initial_solution", "--previous_matches_file", str(o)] + banned_args(banned))
    assert r.returncode == 0, r.stderr
    r0 = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out0)] + banned_args(banned))
    assert r0.returncode == 0, r0.stderr
    _, g, _ = stage(new, banned)
    _, held, _, _, _ = since_model(new, banned, old, A)
    assert out.read_bytes() == assembled(out0.read_bytes(), A, held_keys(new, g, held))
    if name in ("same", "new-k1", "new-k3"):
        # A.pb is this program's output on OLD and NEW appends pairs: the whole output is the full run's
        assert out.read_bytes() == out0.read_bytes()
    if name == "same":
        assert table(out.read_bytes()) == table(A)


@pytest.mark.parametrize("name", ["new-k3", "banned", "sim"])
def test_touched_stats_are_the_plain_runs_and_held_end_empty(checker_exe, tmp_path_factory, oracle, name):  # noqa: F811
    old, new, banned, _, _, _, A = case(checker_exe, tmp_path_factory, name)
    skip, g, sz = stage(new, banned)
    p = problem_from_stage(new, skip, g, sz, "native")
    opts = oracle.default_options(n_threads=4)
    q, start = constant_problem(p, (), A, update_initial_solution=True, previous_matches=old)
    _, held, _, _, _ = since_model(new, banned, old, A)
    assert np.array_equal(q.is_root, ((g["is_root"] != 0) | held).astype(np.uint8))
    pos, st = oracle.solve(q, opts, positions=start)
    pos0, st0 = oracle.solve(p, opts)
    comp = g["comp"].astype(np.int64)
    held_c = np.ones(p.n_components, bool)
    held_c[comp[~held]] = False
    held_c = held_c[p.comp_order.astype(np.int64)]
    assert pos[~held].tobytes() == pos0[~held].tobytes()
    for k in ("iterations", "termination", "initial_cost", "final_cost"):
        assert np.asarray(st[k])[~held_c].tobytes() == np.asarray(st0[k])[~held_c].tobytes(), k
    size = np.diff(p.comp_ptr.astype(np.int64))
    assert np.all(st["termination"][held_c & (size > 1)] == EMPTY)
    assert np.all(st["termination"][held_c & (size == 1)] == SKIPPED)


@pytest.mark.parametrize("extra", [["--fixed_images", 1], ["--carry_initial_solution"], ["--gpus", "2"]])
def test_native_with_fixed_images_carry_and_several_devices(checker_exe, tmp_path_factory, tmp_path, extra):  # noqa: F811
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, "banned")
    extra = [new.image_names[x] if isinstance(x, int) else x for x in extra]
    plain_extra = [x for x in extra if x != "--carry_initial_solution"]
    out, out0 = tmp_path / "out.pb", tmp_path / "out0.pb"
    r = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a),
                          "--update_initial_solution", "--previous_matches_file", str(o)] + banned_args(banned) + extra)
    assert r.returncode == 0, r.stderr
    r0 = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out0)] + banned_args(banned) + plain_extra)
    assert r0.returncode == 0, r0.stderr
    _, g, _ = stage(new, banned)
    _, held, _, _, _ = since_model(new, banned, old, A)
    want = assembled(out0.read_bytes(), A, held_keys(new, g, held))
    if "--carry_initial_solution" in extra:
        sol = wire.decode_solution(want)
        ptr = np.cumsum([0] + [x[2].shape[0] for x in sol]).astype(np.uint64)
        want, _ = wire.encode_solution_carried([x[0] for x in sol], np.array([x[1] for x in sol], np.float32), ptr,
                                               np.concatenate([x[2] for x in sol]), np.concatenate([x[3] for x in sol]),
                                               np.concatenate([x[4] for x in sol]), A)
    assert out.read_bytes() == want


def test_parts_input_and_prefixes(checker_exe, tmp_path_factory, tmp_path):  # noqa: F811
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, "new-k1")
    parts = wire.write_matching_file(old, str(tmp_path / "old_split.pb"), pairs_per_part=max(old.n_pairs // 3, 1))
    assert len(parts) > 1 and not os.path.exists(tmp_path / "old_split.pb")
    outs = []
    for flag, path in (("--previous_matches_file", str(o)), ("--p", str(tmp_path / "old_split.pb")),
                       ("--previous", str(tmp_path / "old_split.pb"))):
        out = tmp_path / ("out%d.pb" % len(outs))
        r = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a), "--u",
                              flag, path])
        assert r.returncode == 0, r.stderr
        outs.append(out.read_bytes())
    assert outs[0] == outs[1] == outs[2]


def test_python_host_path_equals_the_native_host(checker_exe, tmp_path_factory, tmp_path, oracle, monkeypatch):  # noqa: F811
    from lfr_b200.solver import refine
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, "banned")
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    opts = oracle.default_options(n_threads=4)
    out = tmp_path / "out.pb"
    r = run(checker_exe, ["--matches_file", str(n), "--output_file", str(out), "--initial_solution", str(a), "--u",
                          "--previous_matches_file", str(o)] + banned_args(banned))
    assert r.returncode == 0, r.stderr
    for prev in (o.read_bytes(), old):
        _, _, _, sol = refine(wire.read_matching_file(str(n)), banned,
                              solve_fn=lambda q, x=None: oracle.solve(q, opts, positions=x), initial_solution=A,
                              update_initial_solution=True, previous_matches=prev)
        assert wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj) == out.read_bytes()
    with pytest.raises(ValueError):
        refine(new, (), initial_solution=A, previous_matches=old)


def test_command_line_errors(checker_exe, tmp_path_factory, tmp_path, capfd):  # noqa: F811
    old, new, banned, o, n, a, A = case(checker_exe, tmp_path_factory, "same")
    out = tmp_path / "out.pb"
    bad = tmp_path / "bad.pb"
    bad.write_bytes(b"\x0a\xff\xff")
    base = ["--matches_file", str(n), "--output_file", str(out)]
    cases = [
        (["--previous_matches_file", str(o)], 2, [PREV_ERROR]),
        (["--initial_solution", str(a), "--previous_matches_file", str(o)], 2, [PREV_ERROR]),
        (["--keep_initial_solution", "--previous_matches_file", str(o)], 2,
         [b"ERROR: --keep_initial_solution needs --initial_solution FILE\n"]),
        (["--initial_solution", str(a), "--u", "--previous_matches_file", str(tmp_path / "missing.pb")], 2,
         [b"ERROR: cannot read the previous matches file"]),
        (["--initial_solution", str(a), "--u", "--previous_matches_file", str(bad)], 255, [b"Failed to parse proto object.\n"]),
    ]
    for args, code, lines in cases:
        r = run(checker_exe, base + args)
        assert r.returncode == code and r.stdout == b"", (args, r.stderr)
        assert r.stderr.count(b"\n") == 1 and r.stderr.startswith(lines[0]), r.stderr
        assert not out.exists()
        assert cli_main(base + args) == code
        err = capfd.readouterr()
        assert err.out == "" and err.err.encode().startswith(lines[0]), err
        assert not out.exists()
    r = run(checker_exe, base + ["--previous_matches_file"])
    assert r.returncode == 1 and b"the required argument for option '--previous_matches_file' is missing" in r.stderr
    assert run(checker_exe, ["--help"]).stdout == run(checker_exe, ["--help"]).stdout
    assert b"previous" not in run(checker_exe, ["--help"]).stdout
