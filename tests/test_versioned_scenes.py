"""--versioned_scenes: many scenes updated in one run, each from its own SolutionFile and problem record (CPU).

Every scene's output and record file must be byte for byte what the scene's own run writes:

    solve --matches_file M --output_file O [--initial_solution S --update_initial_solution
          [--earlier_record_file E]] [--record_file R] --banned_images ...

Round 0 solves every scene from zeros and writes a record per scene; round 1 starts from round 0's files with
scenes that gained an image, had one pair's flows changed, are unchanged, run without a record, start from zeros,
are listed twice, or are given another scene's record.  Both hosts, the native checker (CPU solve) and the Python
API, with --gpus 2 too."""
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.matchset import MatchSet
from lfr_b200.solver import refine_scenes
from test_fixed_images import checker_exe, run  # noqa: F401
from test_query_images import COUNTS, MAXIMA, stdout_values
from test_ref_solve import GOLD, LAUNCHER
from test_scene_batch import hub_scene, star_scene

BANNED = ["5.ppm", "center.png"]


def hpatches_scene(seed, n_images=6):
    """n_images images named 1.ppm .. n.ppm, every pair matched: one HPatches sequence (the first n images of it)."""
    cfg = synth.SynthConfig("hp", 6, 800, "exhaustive", 0.8, seed=seed)
    ms = synth.generate(cfg, scale=0.05, seed=seed)
    ms.image_names = ["%d.ppm" % (i + 1) for i in range(6)]
    return ms.without_images(["%d.ppm" % (i + 1) for i in range(n_images, 6)])


def changed_flows(ms, seed):
    """`ms` with the flows of its first pair's matches nudged: the same keypoints, another problem."""
    ms = MatchSet(list(ms.image_names), ms.pair_img1, ms.pair_img2, ms.pair_fact1, ms.pair_fact2, ms.pair_ptr,
                  ms.feat1, ms.feat2, ms.sim, ms.disp1.copy(), ms.disp2.copy())
    lo, hi = int(ms.pair_ptr[0]), int(ms.pair_ptr[1])
    ms.disp1[lo:hi] += np.random.default_rng(seed).uniform(-0.05, 0.05, ms.disp1[lo:hi].shape).astype(np.float32)
    return ms


def nudged(data, by=0.01):
    """The SolutionFile `data` with every displacement moved by `by`: the same keys, other values."""
    imgs = wire.decode_solution(data)
    img_ptr = np.concatenate([[0], np.cumsum([len(fi) for _, _, fi, _, _ in imgs])]).astype(np.uint64)
    cat = lambda k, dt: np.concatenate([x[k] for x in imgs]).astype(dt) if imgs else np.zeros(0, dt)  # noqa: E731
    return wire.encode_solution([x[0] for x in imgs], np.array([x[1] for x in imgs], np.float32), img_ptr,
                                cat(2, np.uint32), cat(3, np.float32) + np.float32(by), cat(4, np.float32) - np.float32(by))


def write_list(path, rows):
    path.write_bytes(b"".join(b"\t".join(os.fsencode(str(f)) for f in r) + b"\n" for r in rows))
    return path


def own_args(m, o, init=None, earlier=None, record=None):
    args = ["--matches_file", str(m), "--output_file", str(o)]
    if init:
        args += ["--initial_solution", str(init), "--update_initial_solution"]
    if earlier:
        args += ["--earlier_record_file", str(earlier)]
    if record:
        args += ["--record_file", str(record)]
    for b in BANNED:
        args += ["--banned_images", b]
    return args


def read(path):
    return open(path, "rb").read() if path and os.path.exists(path) else None


@pytest.fixture(scope="module")
def rounds(tmp_path_factory, checker_exe):  # noqa: F811
    """The two rounds: [(dir, rows, own)], rows = [(matches, output, initial, earlier, record)] ('' = none) and
    own = [(output bytes, record bytes or None, stdout values)] of every scene's own run on the CPU checker."""
    d = tmp_path_factory.mktemp("versioned")
    # round 0: no starts, a record per scene
    sets0 = {"hp%d" % k: hpatches_scene(200 + k, 5 if k == 0 else 6) for k in range(6)}
    sets0["hub"] = hub_scene()
    sets0["star"] = star_scene()
    for name, ms in sets0.items():
        wire.write_matching_file(ms, str(d / ("%s.0.pb" % name)))
    parts = synth.generate("cfg2", scale=0.05, seed=9)
    wire.write_matching_file(parts, str(d / "parts.0.pb"), pairs_per_part=4)
    names0 = ["hp0", "hp1", "hub", "parts", "missing", "hp2", "star", "hp3", "hp4", "hp5"]
    rows0 = [(d / ("%s.0.pb" % n), d / ("%s.0.out" % n), "", "", d / ("%s.0.rec" % n)) for n in names0]
    # round 1: hp0 gained an image, hp1 had one pair's flows changed, hub, parts and hp2 are unchanged, hp3 runs
    # without a record, hp4 starts from zeros, and hp5 is given hp1's record.  hp2 is listed twice: first with its
    # own record, then from moved values and hp4's record, so that its digests are in the batch's records but not
    # in its own: the second copy touches every component and solves from zeros (a lookup over every scene's
    # records would hold the moved values)
    wire.write_matching_file(hpatches_scene(200, 6), str(d / "hp0.1.pb"))
    wire.write_matching_file(changed_flows(sets0["hp1"], 5), str(d / "hp1.1.pb"))

    def r1(name, m, init=True, earlier=True, earlier_of=None, out=None):
        return (m, d / ("%s.1.out" % (out or name)), d / ("%s.0.out" % name) if init else "",
                d / ("%s.0.rec" % (earlier_of or name)) if earlier else "", d / ("%s.1.rec" % (out or name)))
    rows1 = [r1("hp0", d / "hp0.1.pb"), r1("hp1", d / "hp1.1.pb"), r1("hub", d / "hub.0.pb"),
             r1("parts", d / "parts.0.pb"), r1("missing", d / "missing.0.pb"), r1("hp2", d / "hp2.0.pb"),
             r1("star", d / "star.0.pb"), r1("hp3", d / "hp3.0.pb", earlier=False),
             r1("hp4", d / "hp4.0.pb", init=False, earlier=False),
             (d / "hp2.0.pb", d / "hp2b.1.out", d / "hp2.0.moved", d / "hp4.0.rec", d / "hp2b.1.rec"),
             r1("hp5", d / "hp5.0.pb", earlier_of="hp1")]
    out = []
    for rows in (rows0, rows1):
        own = []
        for m, o, init, earlier, rec in rows:
            oo, rr = str(o) + ".own", str(rec) + ".own" if rec else None
            r = run(checker_exe, own_args(m, oo, init, earlier, rr))
            assert r.returncode == 0, r.stderr
            own.append((read(oo), read(rr), stdout_values(r.stdout.decode())))
        if rows is rows0:  # round 1 starts from round 0's own files
            for (m, o, _, _, rec), (ob, rb, _) in zip(rows, own):
                open(o, "wb").write(ob)
                open(rec, "wb").write(rb)
            open(d / "hp2.0.moved", "wb").write(nudged(read(d / "hp2.0.out")))
        out.append((d, rows, own))
    return out


def batch_args(d, rows, tag, extra=()):
    """The batch's command line, every scene writing `<output>.<tag>` and `<record>.<tag>`."""
    tagged = [(m, "%s.%s" % (o, tag), init, earlier, "%s.%s" % (rec, tag) if rec else "") for m, o, init, earlier, rec in rows]
    lst = write_list(d / ("list_%s.txt" % tag), tagged[1:])
    m, o, init, earlier, rec = tagged[0]
    return own_args(m, o, init, earlier, rec) + ["--versioned_scenes", str(lst)] + list(extra), tagged


def check(tagged, stdout, own):
    for k, ((_, o, _, _, rec), (ob, rb, _)) in enumerate(zip(tagged, own)):
        assert read(o) == ob, k
        assert read(rec or None) == rb, k
    v = stdout_values(stdout)
    for key in COUNTS:
        assert v.get(key, 0) == sum(x.get(key, 0) for _, _, x in own), key
    for key in MAXIMA:
        assert v.get(key, 0) == max(x.get(key, 0) for _, _, x in own), key


def test_rounds_have_the_structure_they_promise(rounds):
    (_, rows0, own0), (_, rows1, own1) = rounds
    assert own0[4][0] == b"" and own0[6][0] == b""            # the missing and the all-banned scene
    assert all(rb is not None and rb[:8] == b"LFRPREC1" for _, rb, _ in own0)
    assert own1[0][0] != own0[0][0] and own1[1][0] != own0[1][0]   # gained an image; changed flows
    assert own1[2][0] == own0[2][0] and own1[5][0] == own0[5][0]   # unchanged: every component held
    assert own1[9][:2] == own1[5][:2]             # the same scene twice: the second copy solved from zeros again
    assert own1[9][0] != read(rows1[9][2])        # and not held at the moved values
    assert own1[1][1] != own0[1][1] and own1[2][1] == own0[2][1]


@pytest.mark.parametrize("k", [0, 1])
@pytest.mark.parametrize("extra", [[], ["--gpus", "2"]], ids=["gpus1", "gpus2"])
def test_native_batch_writes_every_scenes_own_run(rounds, checker_exe, k, extra):  # noqa: F811
    d, rows, own = rounds[k]
    args, tagged = batch_args(d, rows, "native%d%s" % (k, "".join(extra)), extra)
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    check(tagged, r.stdout.decode(), own)


@pytest.mark.parametrize("k", [0, 1])
@pytest.mark.parametrize("numpy_stage", [False, True], ids=["native_stage", "numpy_stage"])
def test_python_api_updates_every_scene_as_its_own_run(rounds, oracle, monkeypatch, k, numpy_stage):
    d, rows, own = rounds[k]
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    if numpy_stage:
        monkeypatch.setenv("LFR_HOST_PYTHON", "1")
    opts = oracle.default_options(n_threads=4)
    sets = [wire.read_matching_file(str(m)) if wire.matches_files(str(m)) else MatchSet.empty() for m, *_ in rows]
    sols = []
    got = refine_scenes(sets, BANNED, opts, solve_fn=lambda p, x=None: oracle.solve(p, opts, positions=x), solutions=sols,
                        initial_solutions=[read(init or None) for _, _, init, _, _ in rows],
                        previous_records=[read(e or None) for _, _, _, e, _ in rows], record_problem=True)
    assert got == [ob for ob, _, _ in own]
    assert [s.record for s in sols] == [rb for _, rb, _ in own]


def test_a_scene_updates_in_place(rounds, checker_exe, tmp_path):  # noqa: F811
    """OUTPUT_FILE = INITIAL_SOLUTION and RECORD_FILE = EARLIER_RECORD: every input is read before any output."""
    d, rows, own = rounds[1]
    placed = []
    for k, (m, o, init, earlier, rec) in enumerate(rows):
        if init:
            o2, r2 = tmp_path / ("%d.out" % k), tmp_path / ("%d.rec" % k)
            o2.write_bytes(read(init))
            if earlier:
                r2.write_bytes(read(earlier))
            placed.append((m, o2, o2, r2 if earlier else "", r2))
        else:
            placed.append((m, tmp_path / ("%d.out" % k), "", "", tmp_path / ("%d.rec" % k)))
    rows_ip = placed   # every scene in its own pair of files, updated in place
    lst = write_list(tmp_path / "l.txt", rows_ip[1:])
    r = run(checker_exe, own_args(*rows_ip[0]) + ["--versioned_scenes", str(lst)])
    assert r.returncode == 0, r.stderr
    for k, ((_, o, _, _, rec), (ob, rb, _)) in enumerate(zip(rows_ip, own)):
        assert read(o) == ob and read(rec) == rb, k


def test_a_batch_without_starts_is_an_additional_scenes_batch(rounds, checker_exe):  # noqa: F811
    d, rows, _ = rounds[0]
    plain = write_list(d / "plain.txt", [(m, "%s.plain" % o) for m, o, *_ in rows[1:]])
    a = run(checker_exe, ["--matches_file", str(rows[0][0]), "--output_file", "%s.plain" % rows[0][1],
                          "--additional_scenes", str(plain)] + sum((["--banned_images", b] for b in BANNED), []))
    args, tagged = batch_args(d, [(m, o, "", "", "") for m, o, *_ in rows], "nostart")
    b = run(checker_exe, args)
    assert a.returncode == b.returncode == 0
    strip = lambda s: [l for l in s.decode().splitlines() if " time:" not in l]  # noqa: E731
    assert strip(a.stdout) == strip(b.stdout)
    for (m, o, *_), (_, t, *_) in zip(rows, tagged):
        assert read("%s.plain" % o) == read(t)


# ---------------------------------------------------------------------------------------------------
# refusals: both hosts, identical exit code, stdout and stderr, and no file written
# ---------------------------------------------------------------------------------------------------
def _both_hosts(exe, args):
    a = subprocess.run([exe] + args, capture_output=True)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=dict(os.environ, LFR_SOLVE_PYTHON="1"))
    return a, b


def _refused(exe, args, msg, outs=()):
    for r in _both_hosts(exe, args):
        assert (r.returncode, r.stdout, r.stderr) == (2, b"", msg), (r.returncode, r.stdout, r.stderr)
        assert not any(os.path.exists(o) for o in outs)


LINE = b"MATCHES_FILE<TAB>OUTPUT_FILE<TAB>INITIAL_SOLUTION<TAB>EARLIER_RECORD<TAB>RECORD_FILE"


@pytest.mark.parametrize("text,why", [
    (b"a\tb\t\t\t\n\n", b"line 2 is not %s: it is empty" % LINE),
    (b"a\tb\t\t\n", b"line 1 is not %s: it has fewer than four TABs" % LINE),
    (b"a\tb\n", b"line 1 is not %s: it has fewer than four TABs" % LINE),
    (b"a\tb\t\t\t\t\n", b"line 1 is not %s: it has more than four TABs" % LINE),
    (b"\tb\t\t\t\n", b"line 1 is not %s: its matches file is empty" % LINE),
    (b"a\tb\t\t\t\nc\t\t\t\t\n", b"line 2 is not %s: its output file is empty" % LINE),
    (b"a\x00\tb\t\t\t\n", b"line 1 is not %s: it holds a NUL byte" % LINE),
    (b"a\tb\t\tE\t\n", b"line 1 is not %s: it has an earlier record but no initial solution" % LINE),
    (b"a\tb\t\t\tr\nc\td\t\t\tb\n", b"two files written are 'b'"),
    (b"a\tb\t\t\tr\nc\td\t\t\tr\n", b"two files written are 'r'"),
])
def test_malformed_lines_are_refused(checker_exe, tmp_path, text, why):  # noqa: F811
    (tmp_path / "l.txt").write_bytes(text)
    o = str(tmp_path / "o.pb")
    _refused(checker_exe, ["--matches_file", "m.pb", "--output_file", o, "--versioned_scenes", str(tmp_path / "l.txt")],
             b"ERROR: --versioned_scenes: " + why + b"\n", [o])


def test_unreadable_and_malformed_inputs_are_refused(checker_exe, tmp_path):  # noqa: F811
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    sol = os.path.join(GOLD, "tiny_solution.pb")
    o, o1, o2 = str(tmp_path / "o.pb"), str(tmp_path / "1.pb"), str(tmp_path / "2.pb")
    base = ["--matches_file", tiny, "--output_file", o]
    missing = str(tmp_path / "missing.txt")
    _refused(checker_exe, base + ["--versioned_scenes", missing], b"ERROR: cannot read the scene list file '%s'\n" %
             missing.encode(), [o])
    (tmp_path / "bad.pb").write_bytes(b"\x0a\xff\xff\xff\xff\x0f")
    (tmp_path / "bad.rec").write_bytes(b"LFRPREC1\x01" + b"\0" * 7)
    bad, badrec = str(tmp_path / "bad.pb"), str(tmp_path / "bad.rec")
    for row, msg in (((tiny, o2, missing, "", ""), b"line 1: cannot read the initial solution file '%s'" % missing.encode()),
                     ((tiny, o2, bad, "", ""), b"line 1: the initial solution file '%s' does not parse" % bad.encode()),
                     ((tiny, o2, sol, missing, ""), b"line 1: cannot read the earlier record file '%s'" % missing.encode()),
                     ((tiny, o2, sol, badrec, ""), b"line 1: '%s' is not a problem record" % badrec.encode())):
        lst = write_list(tmp_path / "l.txt", [(tiny, o1, "", "", ""), row])
        _refused(checker_exe, base + ["--versioned_scenes", str(lst)],
                 b"ERROR: --versioned_scenes: line 2" + msg[6:] + b"\n", [o, o1, o2])
    # scene 0's start keeps its own messages, and comes before the list's
    lst = write_list(tmp_path / "l.txt", [(tiny, o1, bad, "", "")])
    _refused(checker_exe, base + ["--initial_solution", missing, "--update_initial_solution", "--versioned_scenes", str(lst)],
             b"ERROR: cannot read the initial solution file '%s'\n" % missing.encode(), [o, o1])
    # a malformed scene writes no file
    lst = write_list(tmp_path / "l.txt", [(bad, o1, "", "", "")])
    for r in _both_hosts(checker_exe, base + ["--versioned_scenes", str(lst)]):
        assert (r.returncode, r.stdout, r.stderr) == (255, b"", b"Failed to parse proto object.\n")
        assert not os.path.exists(o) and not os.path.exists(o1)


OPT_IN = {"--fixed_images": ["1.ppm"], "--initial_solution": ["S"], "--keep_initial_solution": [],
          "--carry_initial_solution": [], "--update_initial_solution": [], "--previous_matches_file": ["M"],
          "--record_file": ["R"], "--earlier_record_file": ["R"], "--query_images": ["1.ppm"], "--joint_queries": [],
          "--additional_scenes": ["L"], "--listed_pairs": ["L"]}


@pytest.mark.parametrize("opt", sorted(OPT_IN))
def test_combinations_with_every_opt_in_option_agree(checker_exe, tmp_path, opt):  # noqa: F811
    """--versioned_scenes with each opt-in option, alone and with --initial_solution --update_initial_solution:
    every refusal is the same on both hosts (exit code, stdout and stderr).  Only refusals are compared here: a
    command line the native checker accepts is solved, which the Python host does on the GPU, so the accepted
    combinations are compared in tests/test_gpu_versioned_scenes.py."""
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    sub = {"S": os.path.join(GOLD, "tiny_solution.pb"), "M": tiny, "R": str(tmp_path / "r.rec"),
           "L": str(tmp_path / "l.txt")}
    write_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb", "", "", "")])
    for with_start in (False, True):
        args = ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), "--versioned_scenes",
                str(tmp_path / "l.txt"), opt] + [sub.get(a, a) for a in OPT_IN[opt]]
        if with_start and opt not in ("--initial_solution", "--update_initial_solution"):
            args += ["--initial_solution", sub["S"], "--update_initial_solution"]
        a, b = _both_hosts(checker_exe, args)
        if a.returncode == 0:   # a run, which the Python host solves on the GPU (tests/test_gpu_versioned_scenes.py)
            continue
        assert (a.returncode, a.stdout, a.stderr) == (b.returncode, b.stdout, b.stderr), args
        assert a.returncode == 2 and a.stderr.startswith(b"ERROR: ")


@pytest.mark.parametrize("extra,msg", [
    (["--fixed_images", "1.ppm"], b"ERROR: --versioned_scenes and --fixed_images exclude each other\n"),
    (["--initial_solution", "S"], b"ERROR: --versioned_scenes: --initial_solution needs --update_initial_solution\n"),
    (["--initial_solution", "S", "--keep_initial_solution"], b"ERROR: --versioned_scenes and --keep_initial_solution "
                                                              b"exclude each other\n"),
    (["--initial_solution", "S", "--carry_initial_solution"], b"ERROR: --versioned_scenes and --carry_initial_solution "
                                                               b"exclude each other\n"),
    (["--initial_solution", "S", "--update_initial_solution", "--previous_matches_file", "M"],
     b"ERROR: --versioned_scenes and --previous_matches_file exclude each other\n"),
    (["--query_images", "1.ppm"], b"ERROR: --versioned_scenes and --query_images exclude each other\n"),
    (["--additional_scenes", "L"], b"ERROR: --versioned_scenes and --additional_scenes exclude each other\n"),
    (["--listed_pairs", "L"], b"ERROR: --versioned_scenes and --listed_pairs exclude each other\n"),
])
def test_excluded_combinations(checker_exe, tmp_path, extra, msg):  # noqa: F811
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    sub = {"S": os.path.join(GOLD, "tiny_solution.pb"), "M": tiny, "L": str(tmp_path / "l.txt")}
    write_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb", "", "", "")])
    o = str(tmp_path / "0.pb")
    _refused(checker_exe, ["--matches_file", tiny, "--output_file", o, "--versioned_scenes", str(tmp_path / "l.txt")] +
             [sub.get(a, a) for a in extra], msg, [o, str(tmp_path / "1.pb")])


def test_torchrun_ranks_refuse_versioned_scenes(tmp_path):
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    (tmp_path / "l.txt").write_bytes(b"")
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", os.path.join(GOLD, "tiny_matches.pb"), "--output_file",
                        str(tmp_path / "o.pb"), "--versioned_scenes", str(tmp_path / "l.txt")], capture_output=True, env=env)
    assert (r.returncode, r.stdout) == (2, b"")
    assert r.stderr == b"ERROR: --versioned_scenes: torchrun ranks do not refine scene batches; use --gpus N\n"
    assert not (tmp_path / "o.pb").exists()


def test_the_prefix_v_takes_the_option(checker_exe, tmp_path):  # noqa: F811
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    write_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb", "", "", tmp_path / "1.rec")])
    r = run(checker_exe, ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), "--v", str(tmp_path / "l.txt")])
    assert r.returncode == 0, r.stderr
    want = open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read()
    assert (tmp_path / "0.pb").read_bytes() == (tmp_path / "1.pb").read_bytes() == want
    assert (tmp_path / "1.rec").read_bytes()[:8] == b"LFRPREC1"


@pytest.mark.parametrize("versioned", [False, True], ids=["plain", "versioned"])
def test_an_empty_record_path_still_fails_to_write(checker_exe, tmp_path, versioned):  # noqa: F811
    """`--record_file ''` asks for a record whose file cannot be written: exit 255 after the SolutionFile, as before
    --versioned_scenes existed, with the option too (the GPU test compares the Python host)."""
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    args = ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), "--record_file", ""]
    if versioned:
        write_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb", "", "", tmp_path / "1.rec")])
        args += ["--versioned_scenes", str(tmp_path / "l.txt")]
    r = run(checker_exe, args)
    assert (r.returncode, r.stderr) == (255, b"ERROR: cannot write the record file ''\n")
    assert (tmp_path / "0.pb").read_bytes() == open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read()
    assert not (tmp_path / "1.rec").exists()
