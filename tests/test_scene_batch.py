"""--additional_scenes: many scenes refined in one run, one SolutionFile per scene (CPU).

Every scene's output file must be byte for byte what the scene's own run writes: the same command with
`--matches_file M --output_file O` of that scene alone and the batch's --banned_images.  The stdout counts are
the sums over the own runs, the two maxima their maxima.

The batch holds twenty HPatches-shaped scenes (six images each, all named 1.ppm .. 6.ppm), a scene whose hub
matches make meta-components larger than its own three images (so the cut runs with the scene's own cap, not
the batch's image count), a scene split over .part.N files, a scene whose matches file is missing and a scene
in which every pair is banned.  One banned name, 5.ppm, occurs in every HPatches scene."""
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import USAGE
from lfr_b200.graph import host_input_arrays, host_stage_export
from lfr_b200.matchset import MatchSet
from lfr_b200.solver import refine_scenes
from test_fixed_images import checker_exe, run  # noqa: F401
from test_query_images import COUNTS, MAXIMA, REF_SOLVE, stdout_values
from test_ref_solve import GOLD, LAUNCHER, untimed

BANNED = ["5.ppm", "center.png"]
N_HPATCHES = 20


def hpatches_scene(seed):
    """Six images named 1.ppm .. 6.ppm, every pair matched: one HPatches sequence."""
    cfg = synth.SynthConfig("hp", 6, 800, "exhaustive", 0.8, seed=seed)
    ms = synth.generate(cfg, scale=0.05, seed=seed)
    ms.image_names = ["%d.ppm" % (i + 1) for i in range(6)]
    return ms


def hub_scene(seed=41):
    """Three images; in every pair 8 keypoints of one image match one keypoint of the other.  They cannot share
    a track, so each hub is a meta-component of 9 nodes: past the scene's own 3 images and within the batch's
    image count."""
    cfg = synth.SynthConfig("hub", 3, 1500, "exhaustive", 0.8, seed=seed)
    base = synth.generate(cfg, scale=0.05, seed=seed)
    rng = np.random.default_rng(seed)
    ptr = base.pair_ptr.tolist()
    f1, f2, sim, d1, d2, new_ptr = [], [], [], [], [], [0]
    for p in range(base.n_pairs):
        lo, hi = ptr[p], ptr[p + 1]
        h = 8
        f1 += [base.feat1[lo:hi], np.full(h, 900, np.uint32)]
        f2 += [base.feat2[lo:hi], np.arange(800, 800 + h, dtype=np.uint32)]
        sim += [base.sim[lo:hi], np.full(h, 0.85, np.float32)]
        d1 += [base.disp1[lo:hi], rng.uniform(-0.2, 0.2, (h, 18)).astype(np.float32)]
        d2 += [base.disp2[lo:hi], rng.uniform(-0.2, 0.2, (h, 18)).astype(np.float32)]
        new_ptr.append(new_ptr[-1] + hi - lo + h)
    ms = MatchSet(["a.png", "b.png", "c.png"], base.pair_img1, base.pair_img2, base.pair_fact1, base.pair_fact2,
                  np.array(new_ptr, np.int64), *map(np.concatenate, (f1, f2, sim, d1, d2)))
    ms.validate()
    return ms


def star_scene(seed=43):
    """Every pair names center.png, a banned name: the scene's own run writes an empty solution."""
    cfg = synth.SynthConfig("star", 4, 800, "exhaustive", 0.8, seed=seed)
    ms = synth.generate(cfg, scale=0.05, seed=seed, pairs=[(0, 1), (0, 2), (0, 3)])
    ms.image_names = ["center.png", "1.ppm", "2.ppm", "3.ppm"]
    return ms


def scene_list(path, scenes):
    path.write_bytes(b"".join(b"%s\t%s\n" % (os.fsencode(m), os.fsencode(o)) for m, o in scenes))
    return path


@pytest.fixture(scope="module")
def batch(tmp_path_factory):
    """(directory, [(matches path, output path, MatchSet or None)]); scene 0 is an HPatches scene."""
    d = tmp_path_factory.mktemp("scenes")
    scenes = []
    for k in range(N_HPATCHES):
        m = d / ("hp %02d.pb" % k)                       # a path with a space
        ms = hpatches_scene(100 + k)
        wire.write_matching_file(ms, str(m))
        scenes.append((str(m), str(d / ("hp %02d.out.pb" % k)), ms))
    ms = hub_scene()
    wire.write_matching_file(ms, str(d / "hub.pb"))
    scenes.insert(3, (str(d / "hub.pb"), str(d / "hub.out.pb"), ms))
    ms = synth.generate("cfg2", scale=0.05, seed=9)
    wire.write_matching_file(ms, str(d / "parts.pb"), pairs_per_part=4)
    assert not (d / "parts.pb").exists() and (d / "parts.pb.part.2").exists()
    scenes.insert(7, (str(d / "parts.pb"), str(d / "parts.out.pb"), ms))
    scenes.insert(11, (str(d / "missing.pb"), str(d / "missing.out.pb"), None))
    ms = star_scene()
    wire.write_matching_file(ms, str(d / "star.pb"))
    scenes.insert(15, (str(d / "star.pb"), str(d / "star.out.pb"), ms))
    return d, scenes


def batch_args(d, scenes, tag, extra=()):
    """The batch's command line; every scene writes to `<output>.<tag>`."""
    outs = [o + "." + tag for _, o, _ in scenes]
    lst = scene_list(d / ("list_%s.txt" % tag), [(m, o) for (m, _, _), o in zip(scenes[1:], outs[1:])])
    args = ["--matches_file", scenes[0][0], "--output_file", outs[0], "--additional_scenes", str(lst)]
    for b in BANNED:
        args += ["--banned_images", b]
    return args + list(extra), outs


@pytest.fixture(scope="module")
def own_runs(batch, checker_exe):  # noqa: F811
    """[(bytes, stdout values)] of every scene's own run on the CPU checker."""
    d, scenes = batch
    res = []
    for m, o, _ in scenes:
        args = ["--matches_file", m, "--output_file", o]
        for b in BANNED:
            args += ["--banned_images", b]
        r = run(checker_exe, args)
        assert r.returncode == 0, r.stderr
        res.append((open(o, "rb").read(), stdout_values(r.stdout.decode())))
    return res


def check_batch(outs, stdout, own):
    for k, (o, (want, _)) in enumerate(zip(outs, own)):
        assert open(o, "rb").read() == want, k
    v = stdout_values(stdout)
    for key in COUNTS:
        assert v.get(key, 0) == sum(x.get(key, 0) for _, x in own), key
    for key in MAXIMA:
        assert v.get(key, 0) == max(x.get(key, 0) for _, x in own), key


def test_batch_has_the_structure_it_promises(batch, own_runs):
    d, scenes = batch
    names = [tuple(ms.image_names) for _, _, ms in scenes if ms is not None and len(ms.image_names) == 6]
    assert len(names) == N_HPATCHES and len(set(names)) == 1
    hub = next(ms for m, _, ms in scenes if m.endswith("hub.pb"))
    _, arrs = host_input_arrays(hub)
    _, _, sz = host_stage_export(arrs, len(hub.image_names))
    assert sz["n_oversized_meta_components"] > 0
    # the missing scene and the all-banned one write empty files; every HPatches scene writes 5 images
    sizes = [len(b) for b, _ in own_runs]
    assert sizes[11] == 0 and sizes[15] == 0 and all(s > 0 for k, s in enumerate(sizes) if k not in (11, 15))
    assert all(b"5.ppm" not in own_runs[k][0] for k in range(len(scenes)))


def test_native_batch_writes_every_scenes_own_run(batch, own_runs, checker_exe):  # noqa: F811
    d, scenes = batch
    args, outs = batch_args(d, scenes, "native")
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    check_batch(outs, r.stdout.decode(), own_runs)
    timed = [l.split(":")[0] for l in r.stdout.decode().splitlines() if " time:" in l]
    assert timed == ["Graph-cut time", "Solver time", "Total time"]


def test_own_runs_are_the_references(batch, own_runs):
    """For an HPatches scene and the hub scene the own run is also the reference's own main()."""
    if not os.path.exists(REF_SOLVE):
        pytest.skip("the reference's main() is not built")
    d, scenes = batch
    for k in (0, 3):
        m, o, _ = scenes[k]
        args = [REF_SOLVE, "--matches_file", m, "--output_file", o + ".ref"]
        for b in BANNED:
            args += ["--banned_images", b]
        r = subprocess.run(args, capture_output=True)
        assert r.returncode == 0, r.stderr
        assert open(o + ".ref", "rb").read() == own_runs[k][0], k
        assert stdout_values(r.stdout.decode()) == own_runs[k][1], k


def test_gpus_n_takes_scene_batches(batch, own_runs, checker_exe):  # noqa: F811
    d, scenes = batch
    args, outs = batch_args(d, scenes, "gpus2", ["--gpus", "2"])
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    check_batch(outs, r.stdout.decode(), own_runs)


@pytest.mark.parametrize("numpy_stage", [False, True], ids=["native_stage", "numpy_stage"])
def test_python_api_writes_every_scenes_own_run(batch, own_runs, oracle, numpy_stage, monkeypatch):
    d, scenes = batch
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")
    if numpy_stage:
        monkeypatch.setenv("LFR_HOST_PYTHON", "1")
    opts = oracle.default_options(n_threads=4)
    sets = [wire.read_matching_file(m) if wire.matches_files(m) else MatchSet.empty() for m, _, _ in scenes]
    lines, sols = [], []
    got = refine_scenes(sets, BANNED, opts, log=lines.append, solve_fn=lambda p, x=None: oracle.solve(p, opts, positions=x),
                        solutions=sols)
    assert got == [b for b, _ in own_runs]
    assert [s.n_outside for s in sols] == [v.get("# points with at least one coordinate > 0.5", 0) for _, v in own_runs]
    v = stdout_values("\n".join(lines))
    for key in ("# graph nodes", "# graph edges", "# tracks", "# components"):
        assert v[key] == sum(x.get(key, 0) for _, x in own_runs), key


def test_join_scenes_keys_ids_by_scene_and_name(batch):
    d, scenes = batch
    sets = [ms for _, _, ms in scenes[:3]]
    ms, group = MatchSet.join_scenes(sets, BANNED)
    assert len(ms.image_names) == 15 and group.tolist() == [0] * 5 + [1] * 5 + [2] * 5
    assert ms.image_names[:5] == ms.image_names[5:10] and "5.ppm" not in ms.image_names
    assert ms.n_pairs == 30 and ms.n_matches == sum(s.without_images(BANNED).n_matches for s in sets)


def test_an_empty_list_is_the_plain_run(batch, own_runs, checker_exe, tmp_path):  # noqa: F811
    d, scenes = batch
    (tmp_path / "empty.txt").write_bytes(b"")
    m, _, _ = scenes[7]
    o = tmp_path / "o.pb"
    args = ["--matches_file", m, "--output_file", str(o)] + sum((["--banned_images", b] for b in BANNED), [])
    r = run(checker_exe, args + ["--a", str(tmp_path / "empty.txt")])
    assert r.returncode == 0, r.stderr
    assert o.read_bytes() == own_runs[7][0] and stdout_values(r.stdout.decode()) == own_runs[7][1]


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


def test_a_malformed_scene_writes_no_file(batch, checker_exe, tmp_path):  # noqa: F811
    d, scenes = batch
    bad = tmp_path / "bad.pb"
    bad.write_bytes(b"\x0a\xff\xff\xff\xff\x0f")
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    lst = scene_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb"), (str(bad), tmp_path / "2.pb"), (tiny, tmp_path / "3.pb")])
    for r in _both_hosts(checker_exe, ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"),
                                       "--additional_scenes", str(lst)]):
        assert (r.returncode, r.stdout, r.stderr) == (255, b"", b"Failed to parse proto object.\n")
        assert not any((tmp_path / ("%d.pb" % k)).exists() for k in range(4))


def test_outputs_are_written_in_scene_order(checker_exe, tmp_path):  # noqa: F811
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    lst = scene_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb"), (tiny, tmp_path / "no_dir" / "2.pb"),
                                          (tiny, tmp_path / "3.pb")])
    r = run(checker_exe, ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), "--additional_scenes", str(lst)])
    assert r.returncode == 255 and r.stderr == b"Failed to write proto object.\n"
    want = open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read()
    assert (tmp_path / "0.pb").read_bytes() == want and (tmp_path / "1.pb").read_bytes() == want
    assert not (tmp_path / "3.pb").exists()


@pytest.mark.parametrize("text,why", [
    (b"a\tb\n\nc\td\n", b"line 2 is not MATCHES_FILE<TAB>OUTPUT_FILE: it is empty"),
    (b"a\tb\nc d\n", b"line 2 is not MATCHES_FILE<TAB>OUTPUT_FILE: it has no TAB"),
    (b"a\tb\tc", b"line 1 is not MATCHES_FILE<TAB>OUTPUT_FILE: it has more than one TAB"),
    (b"\tb\n", b"line 1 is not MATCHES_FILE<TAB>OUTPUT_FILE: its matches file is empty"),
    (b"a\tb\nc\td\ne\t\n", b"line 3 is not MATCHES_FILE<TAB>OUTPUT_FILE: its output file is empty"),
    (b"a\x00\tb\n", b"line 1 is not MATCHES_FILE<TAB>OUTPUT_FILE: it holds a NUL byte"),
    (b"\n", b"line 1 is not MATCHES_FILE<TAB>OUTPUT_FILE: it is empty"),
])
def test_malformed_lines_are_refused(checker_exe, tmp_path, text, why):  # noqa: F811
    (tmp_path / "l.txt").write_bytes(text)
    _refused(checker_exe, ["--matches_file", "m.pb", "--output_file", str(tmp_path / "o.pb"), "--additional_scenes",
                           str(tmp_path / "l.txt")], b"ERROR: --additional_scenes: " + why + b"\n")
    assert not (tmp_path / "o.pb").exists()


def test_list_refusals_and_their_order(checker_exe, tmp_path):  # noqa: F811
    o = str(tmp_path / "o b.pb")
    base = ["--matches_file", "m.pb", "--output_file", o]
    missing = str(tmp_path / "missing.txt")
    _refused(checker_exe, base + ["--additional_scenes", missing],
             b"ERROR: cannot read the scene list file '%s'\n" % missing.encode())
    _refused(checker_exe, base + ["--additional_scenes", str(tmp_path)],
             b"ERROR: cannot read the scene list file '%s'\n" % str(tmp_path).encode())
    # two scenes with the same output path, the first scene's included; compared as bytes
    scene_list(tmp_path / "dup.txt", [("x.pb", tmp_path / "p.pb"), ("y.pb", tmp_path / "q.pb"), ("z.pb", tmp_path / "p.pb")])
    _refused(checker_exe, base + ["--additional_scenes", str(tmp_path / "dup.txt")],
             b"ERROR: --additional_scenes: two scenes write '%s'\n" % str(tmp_path / "p.pb").encode())
    scene_list(tmp_path / "dup0.txt", [("x.pb", o)])
    _refused(checker_exe, base + ["--additional_scenes", str(tmp_path / "dup0.txt")],
             b"ERROR: --additional_scenes: two scenes write '%s'\n" % o.encode())
    # the existing option errors come first, then the excluded combinations, then the list
    _refused(checker_exe, base + ["--additional_scenes", missing, "--keep_initial_solution"],
             b"ERROR: --keep_initial_solution needs --initial_solution FILE\n")
    _refused(checker_exe, base + ["--additional_scenes", missing, "--joint_queries"],
             b"ERROR: --joint_queries needs --query_images\n")
    _refused(checker_exe, base + ["--additional_scenes", missing, "--fixed_images", "x"],
             b"ERROR: --additional_scenes and --fixed_images exclude each other\n")
    assert not os.path.exists(o)


@pytest.mark.parametrize("extra,opt", [
    (["--fixed_images", "1.ppm"], "--fixed_images"),
    (["--initial_solution", "S"], "--initial_solution"),
    (["--initial_solution", "S", "--keep_initial_solution"], "--initial_solution"),
    (["--initial_solution", "S", "--carry_initial_solution"], "--initial_solution"),
    (["--initial_solution", "S", "--update_initial_solution", "--previous_matches_file", "M"], "--initial_solution"),
    (["--record_file", "R"], "--record_file"),
    (["--initial_solution", "S", "--update_initial_solution", "--earlier_record_file", "R"], "--initial_solution"),
    (["--query_images", "1.ppm"], "--query_images"),
    (["--query_images", "1.ppm", "--joint_queries"], "--query_images"),
])
def test_excluded_combinations(batch, checker_exe, extra, opt):  # noqa: F811
    d, scenes = batch
    sol = os.path.join(GOLD, "tiny_solution.pb")
    extra = [sol if a == "S" else scenes[1][0] if a == "M" else str(d / "rec.bin") if a == "R" else a for a in extra]
    args, outs = batch_args(d, scenes, "refused", extra)
    _refused(checker_exe, args, b"ERROR: --additional_scenes and %s exclude each other\n" % opt.encode())
    assert not any(os.path.exists(o) for o in outs) and not (d / "rec.bin").exists()


def _wide_scene(n_images, prefix=""):
    """n_images / 2 pairs without matches, each naming two new images."""
    n_pairs = n_images // 2
    z = np.zeros(n_pairs, np.float32)
    return MatchSet(["%s%d.png" % (prefix, i) for i in range(n_images)], np.arange(0, n_images, 2, dtype=np.int64),
                    np.arange(1, n_images, 2, dtype=np.int64), z + 1, z + 1, np.zeros(n_pairs + 1, np.int64),
                    np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros(0, np.float32), np.zeros((0, 18), np.float32),
                    np.zeros((0, 18), np.float32))


def test_65535_ids_are_taken_and_65536_refused(checker_exe, tmp_path):  # noqa: F811
    """Each scene's images count separately: two scenes of the same 32 768 names hold 65 536 ids."""
    wire.write_matching_file(_wide_scene(32768), str(tmp_path / "a.pb"))
    wire.write_matching_file(_wide_scene(32766), str(tmp_path / "b.pb"))
    wire.write_matching_file(_wide_scene(2, "x"), str(tmp_path / "c.pb"))
    one = _wide_scene(2, "x")                              # one image: a self-pair
    one.pair_img2[:] = 0
    wire.write_matching_file(one, str(tmp_path / "d.pb"))
    a, b, c, e = (str(tmp_path / n) for n in ("a.pb", "b.pb", "c.pb", "d.pb"))
    for extra, code in (([(b, tmp_path / "b.out"), (e, tmp_path / "e.out")], 0),
                        ([(b, tmp_path / "b.out"), (c, tmp_path / "c.out")], 2),
                        ([(a, tmp_path / "a2.out")], 2)):
        lst = scene_list(tmp_path / "l.txt", extra)
        r = run(checker_exe, ["--matches_file", a, "--output_file", str(tmp_path / "a.out"), "--additional_scenes", str(lst)])
        assert r.returncode == code, r.stderr
        if code:
            assert r.stdout == b"" and r.stderr == (b"ERROR: --additional_scenes: the scenes hold 65536 images, more than "
                                                    b"65535; split the scene list over several runs\n")
            assert not (tmp_path / "a.out").exists()
        else:
            assert r.stdout.decode().startswith("# graph nodes: 0\n") and (tmp_path / "a.out").read_bytes() == b""
            (tmp_path / "a.out").unlink()
    with pytest.raises(ValueError, match="the scenes hold 65536 images, more than 65535"):
        refine_scenes([_wide_scene(32768), _wide_scene(32768)])


def test_torchrun_ranks_refuse_scene_batches(tmp_path):
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    (tmp_path / "l.txt").write_bytes(b"")
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", os.path.join(GOLD, "tiny_matches.pb"), "--output_file",
                        str(tmp_path / "o.pb"), "--additional_scenes", str(tmp_path / "l.txt")], capture_output=True, env=env)
    assert (r.returncode, r.stdout) == (2, b"")
    assert r.stderr == b"ERROR: --additional_scenes: torchrun ranks do not refine scene batches; use --gpus N\n"
    assert not (tmp_path / "o.pb").exists()


def test_help_is_unchanged_and_prefixes_still_work(batch, checker_exe, tmp_path):  # noqa: F811
    for r in _both_hosts(checker_exe, ["--help"]):
        assert r.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
    tiny = os.path.join(GOLD, "tiny_matches.pb")
    scene_list(tmp_path / "l.txt", [(tiny, tmp_path / "1.pb")])
    outs = []
    for flag in ("--additional_scenes", "--a", "--add"):
        r = run(checker_exe, ["--matches_file", tiny, "--output_file", str(tmp_path / "0.pb"), flag, str(tmp_path / "l.txt")])
        assert r.returncode == 0, r.stderr
        outs.append(((tmp_path / "0.pb").read_bytes(), (tmp_path / "1.pb").read_bytes(), untimed(r.stdout.decode())))
    assert outs[0] == outs[1] == outs[2]
    want = open(os.path.join(GOLD, "tiny_solution.pb"), "rb").read()
    assert outs[0][0] == outs[0][1] == want
    # --b is still --banned_images, and --s still --stats_json in the Python host
    r = run(checker_exe, ["--matches_file", tiny, "--output_file", str(tmp_path / "b.pb"), "--b", "x.png"])
    assert r.returncode == 0 and (tmp_path / "b.pb").read_bytes() == want
