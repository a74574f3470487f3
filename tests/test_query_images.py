"""--query_images: many queries localized against one database in a single run (CPU).

Every query's Image message in the batch output must be byte for byte the one its own run writes: the same
command without --query_images on a MatchingFile holding only the pairs of the query's sub-scene, in file order.
The stdout counts are the sums of the own runs' counts, the maxima their maxima.  The scene is built here from
synth.py: a database refined into A.pb, queries matched to a few database images each, with hub matches that
make meta-components larger than the query's own image count (so the cut runs with a cap that differs from the
batch's), similarities rounded to 1/20 so ties cross queries, a banned query, a query whose pairs hold no match,
and pairs interleaved across queries and split over .part.N files."""
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.cli import USAGE
from lfr_b200.graph import build_problem, host_input_arrays, host_stage_export
from lfr_b200.matchset import MatchSet
from lfr_b200.solver import refine
from test_fixed_images import checker_exe, run  # noqa: F401
from test_ref_solve import GOLD, LAUNCHER, untimed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SOLVE = os.path.join(ROOT, "oracle", "_ref", "solve")
DB = 6          # database images 0..5; queries are the other images
N_IMAGES = 14


def _pairs_of(ms, keep):
    return ms.select_pairs(np.array(keep, dtype=np.int64))


def localization_scene(seed=5, k=3, scale=0.05):
    """(database MatchSet, batch MatchSet, query names, banned query name).  The batch holds the database pairs
    (they name no query, so the batch does not solve them) and every query's pairs, interleaved."""
    cfg = dataclasses.replace(synth.CONFIGS["cfg2"], n_images=N_IMAGES)
    base = synth.generate(cfg, scale=scale, seed=seed)
    base.sim = (np.round(base.sim * 20) / 20).astype(np.float32)   # ties across queries
    rng = np.random.default_rng(seed)
    a1, a2 = base.pair_img1.tolist(), base.pair_img2.tolist()
    db_pairs = [p for p in range(base.n_pairs) if a1[p] < DB and a2[p] < DB]
    q_pairs = []
    for q in range(DB, N_IMAGES):
        ds = set(rng.choice(DB, k, replace=False).tolist())
        q_pairs += [p for p in range(base.n_pairs) if (a1[p] == q and a2[p] in ds) or (a2[p] == q and a1[p] in ds)]
    db = _pairs_of(base, db_pairs)
    order = db_pairs + q_pairs
    perm = rng.permutation(len(order))
    batch = _pairs_of(base, [order[i] for i in perm])
    # hub matches: in every other query pair, twelve query keypoints all match one database keypoint; they
    # cannot share a track, so each hub makes a meta-component larger than the query's k + 1 images
    ptr = batch.pair_ptr.tolist()
    f1, f2, sim, d1, d2, new_ptr = [], [], [], [], [], [0]
    for p in range(batch.n_pairs):
        lo, hi = ptr[p], ptr[p + 1]
        f1.append(batch.feat1[lo:hi]); f2.append(batch.feat2[lo:hi]); sim.append(batch.sim[lo:hi])
        d1.append(batch.disp1[lo:hi]); d2.append(batch.disp2[lo:hi])
        n = hi - lo
        q_side1 = batch.pair_img1[p] >= DB
        if (batch.pair_img1[p] >= DB or batch.pair_img2[p] >= DB) and p % 2 == 0:
            many = np.arange(200, 212, dtype=np.uint32)
            one = np.full(12, 300, dtype=np.uint32)
            f1.append(many if q_side1 else one); f2.append(one if q_side1 else many)
            sim.append(np.full(12, 0.85, np.float32))
            d1.append(rng.uniform(-0.2, 0.2, (12, 18)).astype(np.float32))
            d2.append(rng.uniform(-0.2, 0.2, (12, 18)).astype(np.float32))
            n += 12
        new_ptr.append(new_ptr[-1] + n)
    batch = MatchSet(batch.image_names, batch.pair_img1, batch.pair_img2, batch.pair_fact1, batch.pair_fact2,
                     np.array(new_ptr, np.int64), np.concatenate(f1), np.concatenate(f2), np.concatenate(sim),
                     np.concatenate(d1), np.concatenate(d2))
    # a query whose pairs hold no match, and a query name that is not in the file
    names = list(batch.image_names) + ["nomatch.png"]
    e = len(names) - 1
    batch = MatchSet(names, np.concatenate([batch.pair_img1, [e, 0]]), np.concatenate([batch.pair_img2, [1, e]]),
                     np.concatenate([batch.pair_fact1, [1.0, 1.0]]).astype(np.float32),
                     np.concatenate([batch.pair_fact2, [1.0, 1.0]]).astype(np.float32),
                     np.concatenate([batch.pair_ptr, [batch.n_matches, batch.n_matches]]), batch.feat1, batch.feat2,
                     batch.sim, batch.disp1, batch.disp2)
    batch.validate()
    queries = [base.image_names[q] for q in range(DB, N_IMAGES)] + ["nomatch.png", "absent.png"]
    return db, batch, queries, base.image_names[DB + 1]


def own_matches(batch, q, banned=()):
    """The pairs of query q's sub-scene, in file order."""
    names = batch.image_names
    keep = [p for p, (a, b) in enumerate(zip(batch.pair_img1.tolist(), batch.pair_img2.tolist()))
            if q in (names[a], names[b]) and names[a] not in banned and names[b] not in banned]
    return _pairs_of(batch, keep)


def messages(data):
    """The SolutionFile's Image messages in order: [(name, bytes of the whole field)]."""
    out, i = [], 0
    while i < len(data):
        j = i + 1
        n, s = 0, 0
        while True:
            b = data[j]
            n |= (b & 0x7F) << s
            s += 7
            j += 1
            if b < 0x80:
                break
        assert data[i] == 0x0A
        field = data[i:j + n]
        out.append((wire.decode_solution(field)[0][0], field))
        i = j + n
    return out


COUNTS = ("# graph nodes", "# graph edges", "# tracks", "# components", "# points with at least one coordinate > 0.5")
MAXIMA = ("max track size", "max component size")


def stdout_values(text):
    vals = {}
    for line in text.splitlines():
        key, _, v = line.rpartition(": ")
        if key in COUNTS or key in MAXIMA:
            vals[key] = int(v)
    return vals


@pytest.fixture(scope="module")
def scene(tmp_path_factory, checker_exe):  # noqa: F811
    d = tmp_path_factory.mktemp("loc")
    db, batch, queries, banned = localization_scene()
    wire.write_matching_file(db, str(d / "db.pb"))
    r = run(checker_exe, ["--matches_file", str(d / "db.pb"), "--output_file", str(d / "A.pb")])
    assert r.returncode == 0, r.stderr
    wire.write_matching_file(batch, str(d / "batch.pb"), pairs_per_part=7)   # .part.0, .part.1, ...
    assert not (d / "batch.pb").exists() and (d / "batch.pb.part.3").exists()
    return d, db, batch, queries, banned


MODES = {"plain": [], "fixed": ["--initial_solution", "A.pb", "--fixed_images", "*db*"],
         "keep": ["--initial_solution", "A.pb", "--keep_initial_solution"]}


def mode_args(d, db, mode):
    args = []
    for a in MODES[mode]:
        if a == "A.pb":
            args.append(str(d / "A.pb"))
        elif a == "*db*":
            args += [db.image_names[0]] + sum([["--fixed_images", n] for n in db.image_names[1:DB]], [])
        else:
            args.append(a)
    return args


def own_runs(exe, d, batch, queries, extra, banned):
    """{query: (its Image message or None, stdout values)} of every query's own run."""
    res = {}
    for q in queries:
        mq = d / ("own_%s.pb" % q)
        wire.write_matching_file(own_matches(batch, q, [banned]), str(mq))
        o = d / ("own_%s_out.pb" % q)
        r = run(exe, ["--matches_file", str(mq), "--output_file", str(o), "--banned_images", banned] + extra)
        assert r.returncode == 0, r.stderr
        mine = [m for nm, m in messages(o.read_bytes()) if nm == q]
        assert len(mine) <= 1
        res[q] = (mine[0] if mine else None, stdout_values(r.stdout.decode()))
    return res


def check_batch(out_bytes, stdout, own, queries):
    got = messages(out_bytes)
    names = [nm for nm, _ in got]
    assert len(set(names)) == len(names) and set(names) <= set(queries)
    for q in queries:
        want = own[q][0]
        have = [m for nm, m in got if nm == q]
        assert (have[0] if have else None) == want, q
    vals = stdout_values(stdout)
    for key in COUNTS:
        assert vals.get(key, 0) == sum(v.get(key, 0) for _, v in own.values()), key
    for key in MAXIMA:
        assert vals.get(key, 0) == max(v.get(key, 0) for _, v in own.values()), key
    return got


@pytest.mark.parametrize("mode", sorted(MODES))
def test_native_batch_equals_every_querys_own_run(scene, checker_exe, mode):  # noqa: F811
    d, db, batch, queries, banned = scene
    extra = mode_args(d, db, mode)
    o = d / ("batch_%s.pb" % mode)
    args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(o), "--banned_images", banned] + extra
    for q in queries:
        args += ["--query_images", q]
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    own = own_runs(checker_exe, d, batch, queries, extra, banned)
    got = check_batch(o.read_bytes(), r.stdout.decode(), own, queries)
    # the banned query, the query without matches and the absent name write nothing; the others all do
    assert [nm for nm, _ in got if nm in (banned, "nomatch.png", "absent.png")] == []
    assert len(got) == N_IMAGES - DB - 1
    # the order is the encoder's: lowest node index, i.e. first kept pair with a match
    first = []
    for p in range(batch.n_pairs):
        a, b = batch.image_names[batch.pair_img1[p]], batch.image_names[batch.pair_img2[p]]
        for nm in (a, b):
            if nm in queries and nm != banned and banned not in (a, b) and batch.pair_ptr[p + 1] > batch.pair_ptr[p] \
                    and nm not in first:
                first.append(nm)
    assert [nm for nm, _ in got] == first
    if mode == "plain" and os.path.exists(REF_SOLVE):
        # the reference's own main() on every query's own file that holds a match (on an empty graph it
        # dereferences the end of an empty track list)
        for q in queries:
            if own_matches(batch, q, [banned]).n_matches == 0:
                continue
            o2 = d / ("ref_%s.pb" % q)
            r2 = subprocess.run([REF_SOLVE, "--matches_file", str(d / ("own_%s.pb" % q)), "--output_file", str(o2),
                                 "--banned_images", banned], capture_output=True)
            assert r2.returncode == 0, r2.stderr
            mine = [m for nm, m in messages(o2.read_bytes()) if nm == q]
            assert (mine[0] if mine else None) == own[q][0], q


def test_cuts_run_with_the_sub_scene_cap(scene):
    """Some query's meta-components exceed its own image count but not the batch's: the cut must use the
    sub-scene's cap, and does (the previous test compares the bytes)."""
    d, db, batch, queries, banned = scene
    n_cut = 0
    for q in queries:
        own = own_matches(batch, q, [banned])
        if not own.n_pairs:
            continue
        _, arrs = host_input_arrays(own)
        rc, _, sz = host_stage_export(arrs, len(own.image_names))
        assert rc == 0
        n_cut += sz["n_oversized_meta_components"]
    assert n_cut > 0


def assert_stages_agree_by_sub_scene(batch, queries, banned, grouped=None):
    """The C++ and numpy stages on the grouped input give, sub-scene by sub-scene, the arrays of the stage on that
    sub-scene's pairs alone, under the renumbering that keeps relative order.  `grouped` (sub MatchSet, image_group)
    replaces batch.query_subscenes(queries, [banned]) as the grouped input: the same sub-scenes, their images
    numbered otherwise."""
    sub, group = grouped if grouped is not None else batch.query_subscenes(queries, [banned])
    _, arrs = host_input_arrays(sub, (), group)
    rc, out, sz = host_stage_export(arrs, len(sub.image_names))
    assert rc == 0
    np_p = build_problem(sub, native=False, image_group=group)
    for k in ("track", "comp", "is_root", "comp_nodes", "comp_ptr"):
        assert np.array_equal(np.asarray(getattr(np_p, k)).astype(np.int64), out[k].astype(np.int64)), k
    assert np.array_equal(np_p.graph.node_image, out["node_image"])
    node_q = group[out["node_image"]]
    for q in queries:
        own = own_matches(batch, q, [banned])
        if own.n_matches == 0:
            continue
        _, oa = host_input_arrays(own)
        rc, o, _ = host_stage_export(oa, len(own.image_names))
        assert rc == 0
        qi = batch.image_names.index(q)
        nodes = np.nonzero(node_q == qi)[0]                      # ascending: the renumbering keeps order
        assert nodes.shape[0] == o["node_feat"].shape[0]
        assert np.array_equal(out["node_feat"][nodes], o["node_feat"])
        names_b = [sub.image_names[i] for i in out["node_image"][nodes].tolist()]
        names_o = [own.image_names[i] for i in o["node_image"].tolist()]
        assert names_b == names_o
        remap = np.full(out["node_feat"].shape[0], -1, np.int64)
        remap[nodes] = np.arange(nodes.shape[0])
        assert np.array_equal(out["is_root"][nodes], o["is_root"])
        for key in ("track", "comp"):                            # the same partition, numbered in node order
            _, inv_b = np.unique(out[key][nodes], return_inverse=True)
            _, inv_o = np.unique(o[key], return_inverse=True)
            assert np.array_equal(inv_b, inv_o), key
        rb, ro = out["row_ptr"].astype(np.int64), o["row_ptr"].astype(np.int64)
        eb = np.concatenate([out["edges"][rb[v]:rb[v + 1]] for v in nodes.tolist()])
        assert np.array_equal(remap[eb["dst"].astype(np.int64)], o["edges"]["dst"].astype(np.int64))
        assert eb["flow"].tobytes() == o["edges"]["flow"].tobytes() and eb["sim"].tobytes() == o["edges"]["sim"].tobytes()
    return out, sz


def test_stage_with_groups_equals_the_per_group_stages(scene):
    d, db, batch, queries, banned = scene
    assert_stages_agree_by_sub_scene(batch, queries, banned)


@pytest.mark.parametrize("mode", sorted(MODES))
def test_python_api_equals_the_native_batch(scene, checker_exe, oracle, mode):  # noqa: F811
    """refine(query_images=...) on the host route writes the native batch's bytes (the checker solves)."""
    d, db, batch, queries, banned = scene
    extra = mode_args(d, db, mode)
    o = d / ("py_native_%s.pb" % mode)
    args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(o), "--banned_images", banned] + extra
    for q in queries:
        args += ["--query_images", q]
    r = run(checker_exe, args)
    assert r.returncode == 0, r.stderr
    opts = oracle.default_options(n_threads=4)
    start = (d / "A.pb").read_bytes() if mode != "plain" else None
    fixed = db.image_names[:DB] if mode == "fixed" else ()
    ms = wire.read_matching_file(str(d / "batch.pb"))
    _, _, _, sol = refine(ms, [banned], opts, solve_fn=lambda p, x=None: oracle.solve(p, opts, positions=x),
                          fixed_images=fixed, initial_solution=start, keep_initial_solution=mode == "keep",
                          query_images=queries)
    assert wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj) == o.read_bytes()
    assert sol.n_outside == stdout_values(r.stdout.decode())["# points with at least one coordinate > 0.5"]


# ---------------------------------------------------------------------------------------------------
# the command line: refusals, the two-query pair, prefixes
# ---------------------------------------------------------------------------------------------------
def _both_hosts(exe, args, env=None):
    a = subprocess.run([exe] + args, capture_output=True, env=env)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=dict(env or os.environ, LFR_SOLVE_PYTHON="1"))
    return a, b


@pytest.mark.parametrize("extra,opt", [
    (["--update_initial_solution"], "--update_initial_solution"),
    (["--update_initial_solution", "--previous_matches_file", "M"], "--update_initial_solution"),
    (["--record_file", "R"], "--record_file"),
    (["--carry_initial_solution"], "--carry_initial_solution"),
])
def test_refused_combinations(scene, checker_exe, extra, opt):  # noqa: F811
    d, db, batch, queries, banned = scene
    o = d / "refused.pb"
    extra = [str(d / "A.pb") if a == "M" else str(d / "rec.bin") if a == "R" else a for a in extra]
    args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(o), "--initial_solution", str(d / "A.pb"),
            "--q", queries[0]] + extra
    for r in _both_hosts(checker_exe, args):
        assert (r.returncode, r.stdout) == (2, b""), r.stderr
        assert r.stderr == ("ERROR: --query_images and %s exclude each other\n" % opt).encode()
    assert not o.exists() and not (d / "rec.bin").exists()


def test_earlier_record_is_refused(scene, checker_exe):  # noqa: F811
    d, db, batch, queries, banned = scene
    rec = d / "earlier.bin"
    rec.write_bytes(b"LFRPREC1" + bytes(8))
    args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(d / "o.pb"), "--initial_solution", str(d / "A.pb"),
            "--update_initial_solution", "--earlier_record_file", str(rec), "--query_images", queries[0]]
    for r in _both_hosts(checker_exe, args):
        assert (r.returncode, r.stdout) == (2, b"")
        assert r.stderr == b"ERROR: --query_images and --update_initial_solution exclude each other\n"


def test_a_pair_of_two_queries_is_an_error_before_any_output(scene, checker_exe):  # noqa: F811
    d, db, batch, queries, banned = scene
    names = batch.image_names
    two = [p for p in range(batch.n_pairs) if batch.pair_img1[p] >= DB and batch.pair_img2[p] < DB]
    a, b = names[batch.pair_img1[two[0]]], names[batch.pair_img2[two[0]]]
    o = d / "two.pb"
    args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(o), "--query_images", a, "--query_images", b]
    ra, rb = _both_hosts(checker_exe, args)
    assert ra.returncode == 2 and ra.stdout == b"" and ra.stderr.startswith(b"ERROR: the pair '")
    assert ra.stderr.count(b"\n") == 1 and b"names two query images" in ra.stderr
    assert (rb.returncode, rb.stdout, rb.stderr) == (ra.returncode, ra.stdout, ra.stderr)
    assert not o.exists()
    # banned, the same pair is no error
    r = run(checker_exe, args + ["--banned_images", b])
    assert r.returncode == 0, r.stderr


def test_torchrun_ranks_refuse_queries(tmp_path):
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, LAUNCHER, "--matches_file", os.path.join(GOLD, "tiny_matches.pb"),
                        "--output_file", str(tmp_path / "o.pb"), "--query_images", "x.png"], capture_output=True, env=env)
    assert (r.returncode, r.stdout) == (2, b"")
    assert r.stderr == b"ERROR: --query_images: torchrun ranks do not localize queries; use --gpus N\n"


def test_help_is_unchanged_and_q_is_a_prefix(scene, checker_exe, tmp_path):  # noqa: F811
    d, db, batch, queries, banned = scene
    for r in _both_hosts(checker_exe, ["--help"]):
        assert r.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
    outs = []
    for flag in ("--query_images", "--q", "--query"):
        o = tmp_path / ("o%s.pb" % flag)
        r = run(checker_exe, ["--matches_file", str(d / "batch.pb"), "--output_file", str(o), flag, queries[0],
                              "--q=" + queries[2]])
        assert r.returncode == 0, r.stderr
        outs.append(o.read_bytes())
    assert outs[0] == outs[1] == outs[2] and outs[0]
    # no query named: nothing is solved and the file is empty
    r = run(checker_exe, ["--matches_file", str(d / "batch.pb"), "--output_file", str(tmp_path / "none.pb"),
                          "--query_images", "absent.png"])
    assert r.returncode == 0 and (tmp_path / "none.pb").read_bytes() == b""
    assert untimed(r.stdout.decode())[:2] == ["# graph nodes: 0", "# graph edges: 0"]


# ---------------------------------------------------------------------------------------------------
# memory: union-find image sets follow the largest sub-scene, not the batch
# ---------------------------------------------------------------------------------------------------
_MEM_CHILD = r"""
import resource, sys
import numpy as np
from lfr_b200.graph import host_input_arrays, host_stage_export
from lfr_b200.matchset import MatchSet
Q, D, F = 1000, 40, 20
# query q has images (q, 0) .. (q, D) in its own group; track f of query q: query keypoint f matched in 12 of the
# database images (so every track crosses the 12-image list limit of the sets)
n_img = Q * (D + 1)
p1, p2, ptr, f1, f2 = [], [], [0], [], []
for q in range(Q):
    base = q * (D + 1)
    for d in range(D):
        feats = [f for f in range(F) if (f + d) % D < 12]
        p1.append(base); p2.append(base + 1 + d)
        f1 += feats; f2 += feats
        ptr.append(ptr[-1] + len(feats))
M = len(f1)
ms = MatchSet(["i%d" % i for i in range(n_img)], np.array(p1), np.array(p2), np.ones(len(p1), np.float32),
              np.ones(len(p1), np.float32), np.array(ptr), np.array(f1, np.uint32), np.array(f2, np.uint32),
              np.full(M, 0.9, np.float32), np.zeros((M, 18), np.float32), np.zeros((M, 18), np.float32))
group = np.repeat(np.arange(Q), D + 1).astype(np.uint32)
_, arrs = host_input_arrays(ms, (), group)
before = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
rc, out, sz = host_stage_export(arrs, n_img)
after = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
assert rc == 0 and sz["max_track_size"] == 13 and sz["n_tracks"] == Q * F, sz
print(Q * F, (after - before) * 1024, M)
"""


def test_host_stage_memory_at_1000_queries_of_40_images():
    """1000 queries x 40 database images (41 000 image ids): 20 000 tracks of 13 images.  Image sets n_images
    wide take a 641-word bitset for every track (about 100 MB) on top of everything else the stage holds; sets
    inside the sub-scene fit one 64-bit mask per node.  The stage's whole peak growth must stay below what the
    wide sets alone would need."""
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", _MEM_CHILD], capture_output=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    n_tracks, grown, m = map(int, r.stdout.split())
    wide_sets = n_tracks * ((1000 * 41 + 63) // 64) * 8
    assert grown < wide_sets, (grown, wide_sets)


def test_gpus_n_takes_batches(scene, checker_exe, tmp_path):  # noqa: F811
    """--gpus N (lfr_solve_multi on the host route) writes the one-device batch's bytes and lines."""
    d, db, batch, queries, banned = scene
    outs = []
    for extra in ([], ["--gpus", "2"]):
        o = tmp_path / ("g%d.pb" % len(extra))
        args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(o), "--banned_images", banned,
                "--initial_solution", str(d / "A.pb"), "--keep_initial_solution"] + extra
        for q in queries:
            args += ["--query_images", q]
        r = run(checker_exe, args)
        assert r.returncode == 0, r.stderr
        outs.append((o.read_bytes(), untimed(r.stdout.decode())))
    assert outs[0] == outs[1] and outs[0][0]
