"""--listed_pairs: the pairs of many match lists refined out of one MatchingFile, one SolutionFile per list (CPU).

A match list (`NAME1 NAME2` per line, as utils/create_*_matching_list.py and retrieval write it) is what the
two-view network runs on; the network's output for a pair depends on that pair alone.  So a list's own run is
`solve --matches_file M_L --output_file O` with the batch's --banned_images, where M_L holds, for every line of
the list in line order, the first pair of the superset file whose image_name1 and image_name2 are exactly the
line's two names.  Every list's output file must be byte for byte that run's, and the stdout counts the sums over
the own runs (the two maxima their maxima).

The superset is one file in three .part.N pieces: an HPatches-shaped exhaustive scene of six images, a hub scene
whose oversized meta-components a list of its pairs cuts at its own 3 images, not at the 9 the superset keeps, and a star whose centre is a
banned image.  The lists are a subset in file order, a reordered subset across the parts, repeated lines, the
hub pairs alone (their cut cap is the list's image count), an all-banned list and an empty one.  The golden
Fountain file gives a second superset with sequential windows."""
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import wire
from lfr_b200.cli import USAGE
from lfr_b200.graph import host_input_arrays, host_stage_export
from lfr_b200.matchset import MatchSet, UnheldPairError
from lfr_b200.solver import refine_lists
from test_fixed_images import checker_exe, run  # noqa: F401
from test_query_images import COUNTS, MAXIMA, REF_SOLVE, stdout_values
from test_ref_solve import GOLD, LAUNCHER, untimed
from test_scene_batch import _wide_scene, hpatches_scene, hub_scene, star_scene

BANNED = ["center.png"]


def own_file(ms, lines):
    """M_L by the plain rule: for every line, the first pair of `ms` with exactly those two names."""
    names = ms.image_names
    idx = []
    for n1, n2 in lines:
        hit = [p for p in range(ms.n_pairs) if names[ms.pair_img1[p]] == n1 and names[ms.pair_img2[p]] == n2]
        assert hit, (n1, n2)
        idx.append(hit[0])
    return ms.select_pairs(np.array(idx, np.int64))


def write_list(path, lines):
    path.write_bytes(b"".join(b"%s %s\n" % (a.encode(), b.encode()) for a, b in lines))
    return str(path)


def pair_list(path, lists):
    path.write_bytes(b"".join(b"%s\t%s\n" % (os.fsencode(m), os.fsencode(o)) for m, o in lists))
    return str(path)


def names_of(ms, pairs):
    return [(ms.image_names[ms.pair_img1[p]], ms.image_names[ms.pair_img2[p]]) for p in pairs]


def make_superset(d):
    """(superset path, MatchSet, {list name: lines}); the superset is written in three .part.N pieces."""
    hp, hub, star = hpatches_scene(7), hub_scene(), star_scene()
    hp.image_names = ["%d.ppm" % (i + 1) for i in range(6)]
    star.image_names = ["center.png", "s1.png", "s2.png", "s3.png"]
    path = str(d / "superset.pb")
    for k, part in enumerate((hp, hub, star)):
        (d / ("superset.pb.part.%d" % k)).write_bytes(wire.encode_matching_file(part))
    ms = wire.read_matching_file(path)
    assert ms.n_pairs == 15 + 3 + 3 and len(ms.image_names) == 6 + 3 + 4
    rng = np.random.default_rng(5)
    hub_pairs = list(range(15, 18))
    lists = {
        "in_file_order": names_of(ms, range(0, 15, 2)),
        "reordered": names_of(ms, rng.permutation([1, 4, 16, 9, 11, 19, 2, 15, 7])),
        "repeated": names_of(ms, [3, 3, 8, 17, 3, 8]),
        "hub_alone": names_of(ms, hub_pairs),
        "all_banned": names_of(ms, [18, 20]),
        "empty": [],
    }
    return path, ms, lists


@pytest.fixture(scope="module")
def batch(tmp_path_factory):
    """(directory, superset path, MatchSet, [(list name, list path, lines)])."""
    d = tmp_path_factory.mktemp("lists")
    path, ms, lists = make_superset(d)
    out = []
    for name, lines in lists.items():
        out.append((name, write_list(d / ("%s list.txt" % name), lines), lines))   # a path with a space
    return d, path, ms, out


def run_args(m, o, extra=()):
    args = ["--matches_file", m, "--output_file", o]
    for b in BANNED:
        args += ["--banned_images", b]
    return args + list(extra)


@pytest.fixture(scope="module")
def own_runs(batch, checker_exe):  # noqa: F811
    """[(bytes, stdout values)] of list 0 (the superset) and of every list's own run, on the CPU checker."""
    d, path, ms, lists = batch
    res = []
    for name, m in [("all", path)] + [(n, None) for n, _, _ in lists]:
        if m is None:
            lines = next(l for n, _, l in lists if n == name)
            m = str(d / ("own_%s.pb" % name))
            with open(m, "wb") as fh:
                fh.write(wire.encode_matching_file(own_file(ms, lines)))
        o = str(d / ("own_%s.out.pb" % name))
        r = run(checker_exe, run_args(m, o))
        assert r.returncode == 0, r.stderr
        res.append((open(o, "rb").read(), stdout_values(r.stdout.decode())))
    return res


def batch_args(d, path, lists, tag, extra=()):
    """The batch's command line; list 0 and every list write `<name>.<tag>`."""
    outs = [str(d / ("all.%s" % tag))] + [str(d / ("%s.%s" % (n, tag))) for n, _, _ in lists]
    lst = pair_list(d / ("pairs_%s.txt" % tag), [(m, o) for (_, m, _), o in zip(lists, outs[1:])])
    return run_args(path, outs[0], ["--listed_pairs", lst] + list(extra)), outs


def check_batch(outs, stdout, own):
    for k, (o, (want, _)) in enumerate(zip(outs, own)):
        assert open(o, "rb").read() == want, k
    v = stdout_values(stdout)
    for key in COUNTS:
        assert v.get(key, 0) == sum(x.get(key, 0) for _, x in own), key
    for key in MAXIMA:
        assert v.get(key, 0) == max(x.get(key, 0) for _, x in own), key


def test_lists_have_the_structure_they_promise(batch, own_runs):
    d, path, ms, lists = batch
    assert not os.path.exists(path) and os.path.exists(path + ".part.2")
    # the hub's meta-components are cut at the list's own 3 images, not at the 9 images the superset keeps
    hub, _ = MatchSet.join_scenes([own_file(ms, next(l for n, _, l in lists if n == "hub_alone"))])
    _, arrs = host_input_arrays(hub)
    _, _, sz = host_stage_export(arrs, len(hub.image_names))
    assert len(hub.image_names) == 3
    assert sz["n_oversized_meta_components"] > 0
    _, sarrs = host_input_arrays(ms, BANNED)
    _, _, ssz = host_stage_export(sarrs, len(ms.image_names))
    assert sz["n_images_seen"] == 3 and ssz["n_images_seen"] == 9     # the two cut caps
    sizes = {n: len(own_runs[k + 1][0]) for k, (n, _, _) in enumerate(lists)}
    assert sizes["all_banned"] == 0 and sizes["empty"] == 0
    assert all(s > 0 for n, s in sizes.items() if n not in ("all_banned", "empty"))
    rep = next(l for n, _, l in lists if n == "repeated")
    assert len(rep) > len(set(rep))


def test_native_batch_writes_every_lists_own_run(batch, own_runs, checker_exe):  # noqa: F811
    d, path, ms, lists = batch
    args, outs = batch_args(d, path, lists, "native")
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    check_batch(outs, r.stdout.decode(), own_runs)
    timed = [l.split(":")[0] for l in r.stdout.decode().splitlines() if " time:" in l]
    assert timed == ["Graph-cut time", "Solver time", "Total time"]


def test_own_runs_are_the_references(batch, own_runs):
    """For the reordered list and the hub list the own run is also the reference's own main()."""
    if not os.path.exists(REF_SOLVE):
        pytest.skip("the reference's main() is not built")
    d, path, ms, lists = batch
    for name in ("reordered", "hub_alone"):
        k = 1 + [n for n, _, _ in lists].index(name)
        m = str(d / ("own_%s.pb" % name))
        r = subprocess.run([REF_SOLVE] + run_args(m, m + ".ref"), capture_output=True)
        assert r.returncode == 0, r.stderr
        assert open(m + ".ref", "rb").read() == own_runs[k][0], name
        assert stdout_values(r.stdout.decode()) == own_runs[k][1], name


def test_gpus_n_takes_list_batches(batch, own_runs, checker_exe):  # noqa: F811
    d, path, ms, lists = batch
    args, outs = batch_args(d, path, lists, "gpus2", ["--gpus", "2"])
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    check_batch(outs, r.stdout.decode(), own_runs)


@pytest.mark.parametrize("numpy_stage", [False, True], ids=["native_stage", "numpy_stage"])
def test_python_api_writes_every_lists_own_run(batch, own_runs, oracle, numpy_stage, monkeypatch):
    d, path, ms, lists = batch
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    if numpy_stage:
        monkeypatch.setenv("LFR_HOST_PYTHON", "1")
    opts = oracle.default_options(n_threads=4)
    lines, sols = [], []
    got = refine_lists(ms, [None] + [l for _, _, l in lists], BANNED, opts, log=lines.append,
                       solve_fn=lambda p, x=None: oracle.solve(p, opts, positions=x), solutions=sols)
    assert got == [b for b, _ in own_runs]
    assert [s.n_outside for s in sols] == [v.get("# points with at least one coordinate > 0.5", 0) for _, v in own_runs]
    v = stdout_values("\n".join(lines))
    for key in ("# graph nodes", "# graph edges", "# tracks", "# components"):
        assert v[key] == sum(x.get(key, 0) for _, x in own_runs), key


def test_golden_superset_with_sequential_windows(checker_exe, tmp_path):  # noqa: F811
    """The golden Fountain file as the superset of windows of 1, 2 and 3 frames (create_sequential_matching_list
    style) and of a retrieval-style subset in a different order."""
    gold = os.path.join(GOLD, "fountain_2pct_matches.pb")
    ms = wire.read_matching_file(gold)
    lines = names_of(ms, range(ms.n_pairs))
    order = {n: k for k, n in enumerate(dict.fromkeys(n for l in lines for n in l))}
    windows = [[l for l in lines if abs(order[l[1]] - order[l[0]]) <= w] for w in (1, 2, 3)]
    rng = np.random.default_rng(3)
    retrieval = [lines[i] for i in rng.permutation(len(lines))[: len(lines) // 2]]
    lists, outs, own = [], [str(tmp_path / "all.out")], []
    r = run(checker_exe, ["--matches_file", gold, "--output_file", str(tmp_path / "all.own")])
    own.append(((tmp_path / "all.own").read_bytes(), stdout_values(r.stdout.decode())))
    for k, ls in enumerate(windows + [retrieval]):
        assert ls
        lp = write_list(tmp_path / ("l%d.txt" % k), ls)
        m = str(tmp_path / ("own%d.pb" % k))
        with open(m, "wb") as fh:
            fh.write(wire.encode_matching_file(own_file(ms, ls)))
        r = run(checker_exe, ["--matches_file", m, "--output_file", m + ".out"])
        assert r.returncode == 0, r.stderr
        own.append((open(m + ".out", "rb").read(), stdout_values(r.stdout.decode())))
        lists.append((lp, str(tmp_path / ("l%d.out" % k))))
        outs.append(lists[-1][1])
    r = run(checker_exe, ["--matches_file", gold, "--output_file", outs[0], "--listed_pairs",
                          pair_list(tmp_path / "p.txt", lists)])
    assert r.returncode == 0, r.stderr
    check_batch(outs, r.stdout.decode(), own)


def test_select_listed_pairs_is_the_plain_rule(batch):
    d, path, ms, lists = batch
    for _, _, lines in lists:
        a, b = ms.select_listed_pairs(lines), own_file(ms, lines)
        for f in ("pair_img1", "pair_img2", "pair_fact1", "pair_ptr", "feat1", "feat2", "sim", "disp1", "disp2"):
            assert np.array_equal(getattr(a, f), getattr(b, f)), f
    # the first pair wins when the file holds a pair twice
    twice = MatchSet.concatenate([ms, ms])
    assert twice.listed_pair_index(names_of(ms, [4, 2])).tolist() == [4, 2]
    with pytest.raises(UnheldPairError, match=r"line 2: the matches file holds no pair '2.ppm' '1.ppm'; it holds only "
                                              r"'1.ppm' '2.ppm'"):
        ms.listed_pair_index([("1.ppm", "2.ppm"), ("2.ppm", "1.ppm")])


# ---------------------------------------------------------------------------------------------------
# exit codes, refusals and their order
# ---------------------------------------------------------------------------------------------------
def _both_hosts(exe, args, env=None):
    a = subprocess.run([exe] + args, capture_output=True, env=env)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=dict(env or os.environ, LFR_SOLVE_PYTHON="1"))
    return a, b


def _refused(exe, args, msg, env=None):
    for r in _both_hosts(exe, args, env):
        assert (r.returncode, r.stdout, r.stderr) == (2, b"", msg), (r.returncode, r.stdout, r.stderr)


@pytest.mark.parametrize("text,why", [
    (b"a\tb\n\nc\td\n", b"line 2 is not MATCH_LIST<TAB>OUTPUT_FILE: it is empty"),
    (b"a\tb\nc d\n", b"line 2 is not MATCH_LIST<TAB>OUTPUT_FILE: it has no TAB"),
    (b"a\tb\tc", b"line 1 is not MATCH_LIST<TAB>OUTPUT_FILE: it has more than one TAB"),
    (b"\tb\n", b"line 1 is not MATCH_LIST<TAB>OUTPUT_FILE: its match list is empty"),
    (b"a\tb\nc\td\ne\t\n", b"line 3 is not MATCH_LIST<TAB>OUTPUT_FILE: its output file is empty"),
    (b"a\x00\tb\n", b"line 1 is not MATCH_LIST<TAB>OUTPUT_FILE: it holds a NUL byte"),
])
def test_malformed_pair_list_lines_are_refused(checker_exe, tmp_path, text, why):  # noqa: F811
    (tmp_path / "l.txt").write_bytes(text)
    _refused(checker_exe, ["--matches_file", "m.pb", "--output_file", str(tmp_path / "o.pb"), "--listed_pairs",
                           str(tmp_path / "l.txt")], b"ERROR: --listed_pairs: " + why + b"\n")
    assert not (tmp_path / "o.pb").exists()


@pytest.mark.parametrize("text,line,n", [
    (b"1.ppm 2.ppm\n1.ppm  3.ppm\n", 2, 3),     # two spaces: an empty third field
    (b"1.ppm\t2.ppm\n", 1, 1),
    (b"1.ppm 2.ppm\n\n1.ppm 3.ppm\n", 2, 1),    # an empty line
    (b"1.ppm 2.ppm 3.ppm", 1, 3),
    (b"1.ppm 2.ppm \n", 1, 3),
])
def test_malformed_match_list_lines_are_refused(batch, checker_exe, tmp_path, text, line, n):  # noqa: F811
    d, path, ms, lists = batch
    (tmp_path / "m.txt").write_bytes(text)
    lst = pair_list(tmp_path / "l.txt", [(lists[0][1], tmp_path / "a.pb"), (tmp_path / "m.txt", tmp_path / "b.pb")])
    _refused(checker_exe, run_args(path, str(tmp_path / "o.pb"), ["--listed_pairs", lst]),
             b"ERROR: --listed_pairs: line %d of the match list '%s' is not NAME1 NAME2: it has %d fields\n"
             % (line, str(tmp_path / "m.txt").encode(), n))
    assert not any((tmp_path / f).exists() for f in ("o.pb", "a.pb", "b.pb"))


def test_list_refusals_and_their_order(batch, checker_exe, tmp_path):  # noqa: F811
    d, path, ms, lists = batch
    o = str(tmp_path / "o b.pb")
    base = run_args(path, o)
    good = lists[1][1]
    missing = str(tmp_path / "missing.txt")
    _refused(checker_exe, base + ["--listed_pairs", missing], b"ERROR: cannot read the pair list file '%s'\n" % missing.encode())
    # an unreadable match list, named by its line
    lst = pair_list(tmp_path / "l1.txt", [(good, tmp_path / "a.pb"), (missing, tmp_path / "b.pb")])
    _refused(checker_exe, base + ["--listed_pairs", lst],
             b"ERROR: --listed_pairs: line 2: cannot read the match list '%s'\n" % missing.encode())
    # two lists with the same output path, list 0's included, come before reading any match list
    lst = pair_list(tmp_path / "l2.txt", [(missing, tmp_path / "p.pb"), (good, tmp_path / "p.pb")])
    _refused(checker_exe, base + ["--listed_pairs", lst],
             b"ERROR: --listed_pairs: two lists write '%s'\n" % str(tmp_path / "p.pb").encode())
    lst = pair_list(tmp_path / "l3.txt", [(good, o)])
    _refused(checker_exe, base + ["--listed_pairs", lst], b"ERROR: --listed_pairs: two lists write '%s'\n" % o.encode())
    # a pair the file does not hold; one it holds only the other way round; one with an unknown name
    unheld = [("1.ppm", "2.ppm"), ("1.ppm", "no.png")]
    reverse = [("1.ppm", "2.ppm"), ("1.ppm", "3.ppm"), ("3.ppm", "1.ppm")]
    for lines, line, tail in ((unheld, 2, b"'1.ppm' 'no.png'"), (reverse, 3, b"'3.ppm' '1.ppm'; it holds only '1.ppm' '3.ppm'")):
        m = write_list(tmp_path / "u.txt", lines)
        lst = pair_list(tmp_path / "l4.txt", [(good, tmp_path / "a.pb"), (m, tmp_path / "b.pb")])
        _refused(checker_exe, base + ["--listed_pairs", lst],
                 b"ERROR: --listed_pairs: line %d of the match list '%s': the matches file holds no pair %s\n"
                 % (line, m.encode(), tail))
    # every list is read and split before any pair is looked up: a malformed line in a later list comes first
    (tmp_path / "bad.txt").write_bytes(b"1.ppm\n")
    lst = pair_list(tmp_path / "l5.txt", [(m, tmp_path / "a.pb"), (tmp_path / "bad.txt", tmp_path / "b.pb")])
    _refused(checker_exe, base + ["--listed_pairs", lst],
             b"ERROR: --listed_pairs: line 1 of the match list '%s' is not NAME1 NAME2: it has 1 fields\n"
             % str(tmp_path / "bad.txt").encode())
    # a missing matches file holds no pair
    _refused(checker_exe, run_args(str(tmp_path / "none.pb"), o, ["--listed_pairs", pair_list(tmp_path / "l6.txt", [(good, tmp_path / "a.pb")])]),
             b"ERROR: --listed_pairs: line 1 of the match list '%s': the matches file holds no pair '%s' '%s'\n"
             % (good.encode(), lists[1][2][0][0].encode(), lists[1][2][0][1].encode()))
    # the existing option errors come first, then the excluded combinations, then the list
    _refused(checker_exe, base + ["--listed_pairs", missing, "--keep_initial_solution"],
             b"ERROR: --keep_initial_solution needs --initial_solution FILE\n")
    _refused(checker_exe, base + ["--listed_pairs", missing, "--additional_scenes", missing],
             b"ERROR: --listed_pairs and --additional_scenes exclude each other\n")
    assert not os.path.exists(o) and not (tmp_path / "a.pb").exists()


def test_a_malformed_superset_writes_no_file(batch, checker_exe, tmp_path):  # noqa: F811
    d, path, ms, lists = batch
    bad = tmp_path / "bad.pb"
    bad.write_bytes(b"\x0a\xff\xff\xff\xff\x0f")
    lst = pair_list(tmp_path / "l.txt", [(lists[0][1], tmp_path / "1.pb")])
    for r in _both_hosts(checker_exe, ["--matches_file", str(bad), "--output_file", str(tmp_path / "0.pb"),
                                       "--listed_pairs", lst]):
        assert (r.returncode, r.stdout, r.stderr) == (255, b"", b"Failed to parse proto object.\n")
        assert not (tmp_path / "0.pb").exists() and not (tmp_path / "1.pb").exists()


def test_an_empty_pair_list_is_the_plain_run(batch, own_runs, checker_exe, tmp_path):  # noqa: F811
    d, path, ms, lists = batch
    (tmp_path / "empty.txt").write_bytes(b"")
    o = tmp_path / "o.pb"
    r = run(checker_exe, run_args(path, str(o), ["--listed_pairs", str(tmp_path / "empty.txt")]))
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == own_runs[0][0] and stdout_values(r.stdout.decode()) == own_runs[0][1]


@pytest.mark.parametrize("extra,opt", [
    (["--fixed_images", "1.ppm"], "--fixed_images"),
    (["--initial_solution", "S"], "--initial_solution"),
    (["--initial_solution", "S", "--carry_initial_solution"], "--initial_solution"),
    (["--record_file", "R"], "--record_file"),
    (["--initial_solution", "S", "--update_initial_solution", "--earlier_record_file", "R"], "--initial_solution"),
    (["--query_images", "1.ppm"], "--query_images"),
    (["--additional_scenes", "A"], "--additional_scenes"),
])
def test_excluded_combinations(batch, checker_exe, extra, opt):  # noqa: F811
    d, path, ms, lists = batch
    sol = os.path.join(GOLD, "tiny_solution.pb")
    extra = [sol if a == "S" else str(d / "rec.bin") if a == "R" else lists[0][1] if a == "A" else a for a in extra]
    args, outs = batch_args(d, path, lists, "refused", extra)
    _refused(checker_exe, args, b"ERROR: --listed_pairs and %s exclude each other\n" % opt.encode())
    assert not any(os.path.exists(o) for o in outs) and not (d / "rec.bin").exists()


def test_65535_ids_are_taken_and_65536_refused(checker_exe, tmp_path):  # noqa: F811
    """Each list's images count separately: list 0 holds 32 767 ids, the wide pairs again 32 766, and every
    listed self-pair one more."""
    wide = _wide_scene(32766)
    ms = MatchSet(wide.image_names + ["x.png"], np.append(wide.pair_img1, 32766), np.append(wide.pair_img2, 32766),
                  np.append(wide.pair_fact1, 1), np.append(wide.pair_fact2, 1), np.append(wide.pair_ptr, 0),
                  wide.feat1, wide.feat2, wide.sim, wide.disp1, wide.disp2)
    m = str(tmp_path / "w.pb")
    wire.write_matching_file(ms, m)
    wl = write_list(tmp_path / "wide.txt", names_of(ms, range(16383)))
    sl = write_list(tmp_path / "self.txt", [("x.png", "x.png")])
    for n_self, code in ((2, 0), (3, 2)):
        lst = pair_list(tmp_path / "l.txt", [(wl, tmp_path / "wide.out")] + [(sl, tmp_path / ("s%d.out" % k)) for k in range(n_self)])
        args = ["--matches_file", m, "--output_file", str(tmp_path / "a.out"), "--listed_pairs", lst]
        for r in _both_hosts(checker_exe, args) if code else [run(checker_exe, args)]:
            assert r.returncode == code, r.stderr
            if code:
                assert r.stdout == b"" and r.stderr == (b"ERROR: --listed_pairs: the lists hold 65536 images, more than "
                                                        b"65535; split the pair list over several runs\n")
                assert not (tmp_path / "a.out").exists()
            else:
                assert r.stdout.decode().startswith("# graph nodes: 0\n") and (tmp_path / "a.out").read_bytes() == b""
                (tmp_path / "a.out").unlink()
    with pytest.raises(ValueError, match="the lists hold 65536 images, more than 65535"):
        refine_lists(ms, [None, names_of(ms, range(16383))] + [[("x.png", "x.png")]] * 3)


def test_torchrun_ranks_refuse_list_batches(tmp_path):
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    (tmp_path / "l.txt").write_bytes(b"")
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", os.path.join(GOLD, "tiny_matches.pb"), "--output_file",
                        str(tmp_path / "o.pb"), "--listed_pairs", str(tmp_path / "l.txt")], capture_output=True, env=env)
    assert (r.returncode, r.stdout) == (2, b"")
    assert r.stderr == b"ERROR: --listed_pairs: torchrun ranks do not refine list batches; use --gpus N\n"
    assert not (tmp_path / "o.pb").exists()


def test_help_is_unchanged_and_prefixes_work(checker_exe, tmp_path):  # noqa: F811
    for r in _both_hosts(checker_exe, ["--help"]):
        assert r.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    tm = wire.read_matching_file(tiny)
    lp = write_list(tmp_path / "m.txt", names_of(tm, range(tm.n_pairs)))
    pair_list(tmp_path / "l.txt", [(lp, tmp_path / "1.pb")])
    outs = []
    for flag in ("--listed_pairs", "--l", "--listed"):
        r = run(checker_exe, ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), flag, str(tmp_path / "l.txt")])
        assert r.returncode == 0, r.stderr
        outs.append(((tmp_path / "0.pb").read_bytes(), (tmp_path / "1.pb").read_bytes(), untimed(r.stdout.decode())))
    assert outs[0] == outs[1] == outs[2]
    want = open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read()
    assert outs[0][0] == outs[0][1] == want
    # the prefixes the other options own still name them
    r = run(checker_exe, ["--matches_file", tiny, "--output_file", str(tmp_path / "b.pb"), "--b", "x.png"])
    assert r.returncode == 0 and (tmp_path / "b.pb").read_bytes() == want
