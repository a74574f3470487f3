"""--joint_queries: query sequences and camera rigs localized in one run (CPU).

With --joint_queries, queries that a kept pair names together are one group: a connected component of the
queries under such pairs, zero-match pairs included.  Every query's Image message in the batch output must be
byte for byte the one its group's own run writes: the same command without --query_images and --joint_queries on
a MatchingFile holding only the pairs of the group's sub-scene, in file order.  The stdout counts are the sums of
the own runs' counts, the maxima their maxima.

The scene extends test_query_images' localization scene: a database refined into A.pb; a 62-frame sequence (a
group of 68 images, whose tracks outgrow the 12-entry image lists and the one-word mask), a 4-frame sequence, a
5-frame sequence broken in two by a banned middle frame, a sequence joined only by a pair without matches, rigs
of 2, 3 and 4 cameras, single queries, a self-pair, a query whose pairs hold no match and an absent name.  Hub
matches make meta-components larger than a query's own image count, some within their group's and some past it;
similarities are rounded to 1/20 so that ties cross groups; half the pairs put the query on side 1; the pairs
are shuffled and split over .part.N files."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

import test_query_images as tq
from lfr_b200 import synth, wire
from lfr_b200.cli import USAGE
from lfr_b200.graph import host_input_arrays, host_stage_export
from lfr_b200.matchset import MatchSet
from lfr_b200.solver import refine
from test_fixed_images import checker_exe, run  # noqa: F401
from test_query_images import COUNTS, MAXIMA, MODES, REF_SOLVE, messages, mode_args, stdout_values
from test_ref_solve import GOLD, LAUNCHER, untimed

DB = tq.DB
LONG = 62


def _layout(rng, long_chain):
    """(pairs, query-query pairs, zero-match pair, self-pair query, banned query, n_images) of the joint scene;
    database images are 0..DB-1, queries the ids after them."""
    ids = itertools.count(DB)
    qq = []

    def chain(n):
        qs = [next(ids) for _ in range(n)]
        qq.extend(zip(qs[:-1], qs[1:]))
        return qs

    chain(long_chain)
    chain(4)
    broken = chain(5)
    zero = chain(4)
    rigs = []
    for n in (2, 3, 4):
        qs = [next(ids) for _ in range(n)]
        qq.extend(itertools.combinations(qs, 2))
        rigs.append(qs)
    singles = [next(ids) for _ in range(3)]
    n_images = next(ids)
    qd = []
    for q in range(DB, n_images):
        ds = [0, 1, 2] if q in zero else rng.choice(DB, 3 if q in singles else 2, replace=False).tolist()
        qd += [(d, q) for d in ds]
    db = list(itertools.combinations(range(DB), 2))
    return db + qd + qq, qq, (zero[1], zero[2]), rigs[1][0], broken[2], n_images


def joint_scene(seed=3, scale=0.05, long_chain=LONG):
    """(database MatchSet, batch MatchSet, query names, banned query name)."""
    rng = np.random.default_rng(seed)
    pairs, qq, zero_pair, self_q, banned_q, n_images = _layout(rng, long_chain)
    cfg = synth.SynthConfig("joint", n_images, 3000, "exhaustive", 0.7, seed=seed)
    base = synth.generate(cfg, scale=scale, seed=seed, pairs=pairs)
    base.sim = (np.round(base.sim * 20) / 20).astype(np.float32)   # ties across groups
    a1, a2 = base.pair_img1.tolist(), base.pair_img2.tolist()
    db_pairs = [p for p in range(base.n_pairs) if a2[p] < DB]
    db = base.select_pairs(np.array(db_pairs, np.int64))
    perm = rng.permutation(base.n_pairs)
    ptr = base.pair_ptr.tolist()
    img1, img2, f1, f2, sim, d1, d2, new_ptr = [], [], [], [], [], [], [], [0]
    hub = itertools.cycle((4, 8, 12))
    for k, p in enumerate(perm.tolist()):
        lo, hi = ptr[p], ptr[p + 1]
        a, b = a1[p], a2[p]
        if (a, b) == zero_pair:
            lo = hi
        pf1, pf2, ps, pd1, pd2 = [base.feat1[lo:hi]], [base.feat2[lo:hi]], [base.sim[lo:hi]], [base.disp1[lo:hi]], [base.disp2[lo:hi]]
        if a < DB <= b and k % 2 == 0:
            # hub: h query keypoints all match one database keypoint; they cannot share a track, so the hub is
            # a meta-component of at least h + 1 nodes
            h = next(hub)
            pf1.append(np.full(h, 300, np.uint32)); pf2.append(np.arange(200, 200 + h, dtype=np.uint32))
            ps.append(np.full(h, 0.85, np.float32))
            pd1.append(rng.uniform(-0.2, 0.2, (h, 18)).astype(np.float32))
            pd2.append(rng.uniform(-0.2, 0.2, (h, 18)).astype(np.float32))
        pf1, pf2, ps, pd1, pd2 = map(np.concatenate, (pf1, pf2, ps, pd1, pd2))
        if b >= DB and k % 2 == 1:                                  # the query on side 1
            a, b, pf1, pf2, pd1, pd2 = b, a, pf2, pf1, pd2, pd1
        img1.append(a); img2.append(b); f1.append(pf1); f2.append(pf2); sim.append(ps); d1.append(pd1); d2.append(pd2)
        new_ptr.append(new_ptr[-1] + pf1.shape[0])
        if k == base.n_pairs // 2:
            # a self-pair: keypoints of one query matched to other keypoints of the same query
            img1.append(self_q); img2.append(self_q)
            f1.append(np.arange(0, 12, 2, dtype=np.uint32)); f2.append(np.arange(1, 13, 2, dtype=np.uint32))
            sim.append(np.full(6, 0.9, np.float32))
            d1.append(rng.uniform(-0.2, 0.2, (6, 18)).astype(np.float32))
            d2.append(rng.uniform(-0.2, 0.2, (6, 18)).astype(np.float32))
            new_ptr.append(new_ptr[-1] + 6)
    names = list(base.image_names) + ["nomatch.png"]
    e = len(names) - 1
    img1 += [e, 0]; img2 += [1, e]
    new_ptr += [new_ptr[-1], new_ptr[-1]]
    n_p = len(img1)
    batch = MatchSet(names, np.array(img1, np.int64), np.array(img2, np.int64), np.ones(n_p, np.float32),
                     np.ones(n_p, np.float32), np.array(new_ptr, np.int64), np.concatenate(f1), np.concatenate(f2),
                     np.concatenate(sim), np.concatenate(d1), np.concatenate(d2))
    batch.validate()
    queries = [names[q] for q in range(DB, n_images)] + ["nomatch.png", "absent.png"]
    return db, batch, queries, names[banned_q]


def kept_pairs(batch, banned):
    names = batch.image_names
    return [(p, names[a], names[b]) for p, (a, b) in enumerate(zip(batch.pair_img1.tolist(), batch.pair_img2.tolist()))
            if names[a] not in banned and names[b] not in banned]


def query_groups(batch, queries, banned, joint=True):
    """The query groups the contract defines, computed here with scipy: [[query names in batch id order]] for
    the queries that a kept pair names."""
    qs = set(queries)
    kept = kept_pairs(batch, banned)
    present = sorted({n for _, a, b in kept for n in (a, b) if n in qs}, key=batch.image_names.index)
    ix = {n: i for i, n in enumerate(present)}
    e = [(ix[a], ix[b]) for _, a, b in kept if joint and a in qs and b in qs]
    m = coo_matrix((np.ones(len(e)), ([x for x, _ in e], [y for _, y in e])), shape=(len(present),) * 2)
    _, lab = connected_components(m, directed=False)
    return [[n for n in present if lab[ix[n]] == g] for g in sorted(set(lab.tolist()), key=lab.tolist().index)]


def group_matches(batch, group, banned=()):
    """The pairs of a group's sub-scene, in file order."""
    g = set(group)
    return batch.select_pairs(np.array([p for p, a, b in kept_pairs(batch, banned) if a in g or b in g], np.int64))


@pytest.fixture(scope="module")
def scene(tmp_path_factory, checker_exe):  # noqa: F811
    d = tmp_path_factory.mktemp("joint")
    db, batch, queries, banned = joint_scene()
    wire.write_matching_file(db, str(d / "db.pb"))
    r = run(checker_exe, ["--matches_file", str(d / "db.pb"), "--output_file", str(d / "A.pb")])
    assert r.returncode == 0, r.stderr
    wire.write_matching_file(batch, str(d / "batch.pb"), pairs_per_part=7)   # .part.0, .part.1, ...
    assert not (d / "batch.pb").exists() and (d / "batch.pb.part.3").exists()
    return d, db, batch, queries, banned, query_groups(batch, queries, [banned])


def batch_args(d, out, queries, banned, extra, joint=True):
    args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(out), "--banned_images", banned] + extra
    for q in queries:
        args += ["--query_images", q]
    return args + (["--joint_queries"] if joint else [])


def group_own_runs(exe, d, batch, groups, banned, extra, tag="", env=None):
    """({query: its Image message in its group's own run, or None}, [stdout values of every own run], [own files])."""
    msgs, vals, files = {}, [], []
    for i, g in enumerate(groups):
        mg = d / ("group_%d.pb" % i)
        own = group_matches(batch, g, [banned])
        wire.write_matching_file(own, str(mg))
        o = d / ("group_%d_%s.pb" % (i, tag))
        r = subprocess.run([exe, "--matches_file", str(mg), "--output_file", str(o), "--banned_images", banned] + extra,
                           capture_output=True, env=env(own) if env else None)
        assert r.returncode == 0, r.stderr
        got = messages(o.read_bytes())
        for q in g:
            mine = [m for nm, m in got if nm == q]
            assert len(mine) <= 1
            msgs[q] = mine[0] if mine else None
        vals.append(stdout_values(r.stdout.decode()))
        files.append((mg, own))
    return msgs, vals, files


def check_joint_batch(out_bytes, stdout, msgs, vals, queries):
    got = messages(out_bytes)
    names = [nm for nm, _ in got]
    assert len(set(names)) == len(names) and set(names) <= set(queries)
    for q in queries:
        have = [m for nm, m in got if nm == q]
        assert (have[0] if have else None) == msgs.get(q), q
    v = stdout_values(stdout)
    for key in COUNTS:
        assert v.get(key, 0) == sum(x.get(key, 0) for x in vals), key
    for key in MAXIMA:
        assert v.get(key, 0) == max(x.get(key, 0) for x in vals), key
    return got


def test_scene_has_the_structure_it_promises(scene):
    d, db, batch, queries, banned, groups = scene
    sizes = sorted(len(g) for g in groups)
    # the long sequence; the 4-frame one and the one joined by a zero-match pair; rigs; the broken sequence
    # (2 + 2, its banned middle frame gone); singles, the self-pair's rig and the query without matches
    assert sizes[-1] == LONG and sizes.count(4) == 3 and 3 in sizes and sizes.count(2) == 3
    assert len(query_groups(batch, queries, [banned], joint=False)) == sum(sizes)
    # without the zero-match pair the sequence it joins falls in two
    zero = [p for p in range(batch.n_pairs) if batch.pair_ptr[p] == batch.pair_ptr[p + 1]
            and batch.pair_img1[p] >= DB and batch.pair_img2[p] >= DB and batch.pair_img1[p] != batch.pair_img2[p]
            and batch.image_names[batch.pair_img1[p]] != "nomatch.png"]
    assert len(zero) == 1
    drop = np.array([p for p in range(batch.n_pairs) if p != zero[0]], np.int64)
    assert len(query_groups(batch.select_pairs(drop), queries, [banned])) == len(groups) + 1
    assert any(batch.pair_img1[p] == batch.pair_img2[p] for p in range(batch.n_pairs))
    # meta-components (connected components of the match graph) against the caps
    n_inside = n_past = 0
    batch_seen = len({n for _, a, b in kept_pairs(batch, [banned]) for n in (a, b)})
    for g in groups:
        own = group_matches(batch, g, [banned])
        _, arrs = host_input_arrays(own)
        rc, out, sz = host_stage_export(arrs, len(own.image_names))
        assert rc == 0
        n = sz["n_nodes"]
        if not n:
            continue
        src = np.repeat(np.arange(n), np.diff(out["row_ptr"].astype(np.int64)))
        _, cc = connected_components(coo_matrix((np.ones(src.shape[0]), (src, out["edges"]["dst"].astype(np.int64))),
                                                shape=(n, n)), directed=False)
        meta = np.bincount(cc)
        group_seen = sz["n_images_seen"]
        one_query = max(len({n_ for _, a, b in kept_pairs(own, [banned]) if q in (a, b) for n_ in (a, b)}) for q in g)
        n_inside += int(((meta > one_query) & (meta <= group_seen)).sum()) if len(g) > 1 else 0
        n_past += int(((meta > group_seen) & (meta <= batch_seen)).sum())
        if len(g) == LONG:
            assert group_seen > 64 and sz["max_track_size"] > 12
    assert n_inside > 0 and n_past > 0


@pytest.mark.parametrize("mode", sorted(MODES))
def test_native_batch_equals_every_groups_own_run(scene, checker_exe, mode):  # noqa: F811
    d, db, batch, queries, banned, groups = scene
    extra = mode_args(d, db, mode)
    o = d / ("batch_%s.pb" % mode)
    r = run(checker_exe, batch_args(d, o, queries, banned, extra))
    assert r.returncode == 0, r.stderr
    msgs, vals, files = group_own_runs(checker_exe, d, batch, groups, banned, extra, mode)
    got = check_joint_batch(o.read_bytes(), r.stdout.decode(), msgs, vals, queries)
    assert [nm for nm, _ in got if nm in (banned, "nomatch.png", "absent.png")] == []
    assert len(got) == sum(len(g) for g in groups) - 1
    # the order is the encoder's: lowest node index, i.e. first kept pair with a match
    first = []
    for p, a, b in kept_pairs(batch, [banned]):
        for nm in (a, b):
            if nm in queries and batch.pair_ptr[p + 1] > batch.pair_ptr[p] and nm not in first:
                first.append(nm)
    assert [nm for nm, _ in got] == first
    if mode == "plain" and os.path.exists(REF_SOLVE):
        # the reference's own main() on every group's own file that holds a match
        for i, (mg, own) in enumerate(files):
            if own.n_matches == 0:
                continue
            o2 = d / ("ref_group_%d.pb" % i)
            r2 = subprocess.run([REF_SOLVE, "--matches_file", str(mg), "--output_file", str(o2), "--banned_images", banned],
                                capture_output=True)
            assert r2.returncode == 0, r2.stderr
            for nm, m in messages(o2.read_bytes()):
                if nm in groups[i]:
                    assert m == msgs[nm], nm


def test_stage_with_groups_equals_the_per_group_stages(scene, monkeypatch):
    """test_query_images' sub-scene check, each group standing as its lowest query: the group's label."""
    d, db, batch, queries, banned, groups = scene
    rep = {g[0]: g for g in groups}
    monkeypatch.setattr(tq, "own_matches", lambda b, q, bn=(): group_matches(b, rep[q], bn))
    out, sz = tq.assert_stages_agree_by_sub_scene(batch, list(rep), banned,
                                                  grouped=batch.query_subscenes(queries, [banned], joint=True))
    assert sz["n_oversized_meta_components"] > 0


def test_grouping_of_both_hosts(scene):
    """query_subscenes' groups are the contract's: every id's label is its group's lowest query id."""
    d, db, batch, queries, banned, groups = scene
    sub, group = batch.query_subscenes(queries, [banned], joint=True)
    label = {}
    for g in groups:
        for q in g:
            label[q] = min(batch.image_names.index(x) for x in g)
    for i, nm in enumerate(sub.image_names):
        if nm in label:
            assert group[i] == label[nm], nm
    assert sorted(set(group.tolist())) == sorted(set(label.values()))


@pytest.mark.parametrize("mode", sorted(MODES))
def test_python_api_equals_the_native_batch(scene, checker_exe, oracle, mode, monkeypatch):  # noqa: F811
    """refine(joint_queries=True) on the host route writes the native batch's bytes (the checker solves)."""
    d, db, batch, queries, banned, groups = scene
    monkeypatch.setenv("LFR_GRAPH_STAGE", "host")   # the batch is past the size rule's device threshold
    extra = mode_args(d, db, mode)
    o = d / ("py_native_%s.pb" % mode)
    r = run(checker_exe, batch_args(d, o, queries, banned, extra))
    assert r.returncode == 0, r.stderr
    opts = oracle.default_options(n_threads=4)
    start = (d / "A.pb").read_bytes() if mode != "plain" else None
    fixed = db.image_names[:DB] if mode == "fixed" else ()
    ms = wire.read_matching_file(str(d / "batch.pb"))
    _, _, _, sol = refine(ms, [banned], opts, solve_fn=lambda p, x=None: oracle.solve(p, opts, positions=x),
                          fixed_images=fixed, initial_solution=start, keep_initial_solution=mode == "keep",
                          query_images=queries, joint_queries=True)
    assert wire.encode_solution(sol.image_names, sol.fact, sol.img_ptr, sol.feature_idx, sol.di, sol.dj) == o.read_bytes()
    assert sol.n_outside == stdout_values(r.stdout.decode())["# points with at least one coordinate > 0.5"]


def test_the_flag_is_the_identity_without_query_pairs(checker_exe, tmp_path):  # noqa: F811
    """test_query_images' scene names no two queries in a pair: the flag changes no byte and no line."""
    db, batch, queries, banned = tq.localization_scene()
    wire.write_matching_file(batch, str(tmp_path / "batch.pb"), pairs_per_part=7)
    outs = []
    for joint in (False, True):
        o = tmp_path / ("o%d.pb" % joint)
        r = run(checker_exe, batch_args(tmp_path, o, queries, banned, [], joint))
        assert r.returncode == 0, r.stderr
        outs.append((o.read_bytes(), untimed(r.stdout.decode())))
    assert outs[0] == outs[1] and outs[0][0]
    a, g = batch.query_subscenes(queries, [banned])
    b, h = batch.query_subscenes(queries, [banned], joint=True)
    assert a.image_names == b.image_names and np.array_equal(g, h)
    assert np.array_equal(a.pair_img1, b.pair_img1) and np.array_equal(a.pair_img2, b.pair_img2)


def test_gpus_n_takes_joint_batches(scene, checker_exe, tmp_path):  # noqa: F811
    d, db, batch, queries, banned, groups = scene
    outs = []
    for extra in ([], ["--gpus", "2"]):
        o = tmp_path / ("g%d.pb" % len(extra))
        r = run(checker_exe, batch_args(d, o, queries, banned, ["--initial_solution", str(d / "A.pb"),
                                                                "--keep_initial_solution"] + extra))
        assert r.returncode == 0, r.stderr
        outs.append((o.read_bytes(), untimed(r.stdout.decode())))
    assert outs[0] == outs[1] and outs[0][0]


# ---------------------------------------------------------------------------------------------------
# the command line: refusals and their order, prefixes, --help
# ---------------------------------------------------------------------------------------------------
def _both_hosts(exe, args, env=None):
    a = subprocess.run([exe] + args, capture_output=True, env=env)
    b = subprocess.run([sys.executable, LAUNCHER] + args, capture_output=True, env=dict(env or os.environ, LFR_SOLVE_PYTHON="1"))
    return a, b


def _refused(exe, args, msg, env=None):
    for r in _both_hosts(exe, args, env):
        assert (r.returncode, r.stdout, r.stderr) == (2, b"", msg.encode())


def test_joint_needs_query_images(scene, checker_exe):  # noqa: F811
    d, db, batch, queries, banned, groups = scene
    base = ["--matches_file", str(d / "batch.pb"), "--output_file", str(d / "refused.pb")]
    _refused(checker_exe, base + ["--joint_queries"], "ERROR: --joint_queries needs --query_images\n")
    # before the start solution is read
    _refused(checker_exe, base + ["--j", "--initial_solution", str(d / "missing.pb")],
             "ERROR: --joint_queries needs --query_images\n")
    # after the existing option errors
    _refused(checker_exe, base + ["--joint_queries", "--keep_initial_solution"],
             "ERROR: --keep_initial_solution needs --initial_solution FILE\n")
    _refused(checker_exe, base + ["--joint_queries", "--initial_solution", str(d / "A.pb"), "--previous_matches_file",
                                  str(d / "db.pb")], "ERROR: --previous_matches_file needs --update_initial_solution\n")
    assert not (d / "refused.pb").exists()
    with pytest.raises(ValueError, match="joint_queries needs query_images"):
        refine(batch, [banned], joint_queries=True)


@pytest.mark.parametrize("extra,opt", [
    (["--update_initial_solution"], "--update_initial_solution"),
    (["--update_initial_solution", "--previous_matches_file", "M"], "--update_initial_solution"),
    (["--record_file", "R"], "--record_file"),
    (["--carry_initial_solution"], "--carry_initial_solution"),
])
def test_refused_combinations(scene, checker_exe, extra, opt):  # noqa: F811
    d, db, batch, queries, banned, groups = scene
    extra = [str(d / "A.pb") if a == "M" else str(d / "rec.bin") if a == "R" else a for a in extra]
    args = ["--matches_file", str(d / "batch.pb"), "--output_file", str(d / "refused.pb"), "--initial_solution",
            str(d / "A.pb"), "--joint_queries", "--q", queries[0]] + extra
    _refused(checker_exe, args, "ERROR: --query_images and %s exclude each other\n" % opt)
    assert not (d / "refused.pb").exists() and not (d / "rec.bin").exists()


def test_torchrun_ranks_refuse_the_flag(tmp_path):
    env = dict(os.environ, LFR_SOLVE_PYTHON="1", RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    base = [sys.executable, LAUNCHER, "--matches_file", os.path.join(GOLD, "tiny_matches.pb"), "--output_file",
            str(tmp_path / "o.pb"), "--joint_queries"]
    r = subprocess.run(base + ["--query_images", "x.png"], capture_output=True, env=env)
    assert (r.returncode, r.stdout) == (2, b"")
    assert r.stderr == b"ERROR: --query_images: torchrun ranks do not localize queries; use --gpus N\n"
    r = subprocess.run(base, capture_output=True, env=env)
    assert (r.returncode, r.stdout, r.stderr) == (2, b"", b"ERROR: --joint_queries needs --query_images\n")
    assert not (tmp_path / "o.pb").exists()


def test_a_pair_of_two_queries_needs_the_flag(scene, checker_exe, tmp_path):  # noqa: F811
    d, db, batch, queries, banned, groups = scene
    o = tmp_path / "two.pb"
    args = batch_args(d, o, queries, banned, [], joint=False)
    for r in _both_hosts(checker_exe, args):
        assert r.returncode == 2 and r.stdout == b"" and r.stderr.startswith(b"ERROR: the pair '")
        assert r.stderr.count(b"\n") == 1 and r.stderr.endswith(b"names two query images\n")
    assert not o.exists()
    r = run(checker_exe, args + ["--joint_queries"])
    assert r.returncode == 0 and o.read_bytes(), r.stderr


def test_help_is_unchanged_and_j_is_a_prefix(scene, checker_exe, tmp_path):  # noqa: F811
    d, db, batch, queries, banned, groups = scene
    for r in _both_hosts(checker_exe, ["--help"]):
        assert r.stdout == ("Patch Match graph problem solver\n\n" + USAGE).encode()
    g = max(groups, key=len)
    outs = []
    for flag in ("--joint_queries", "--j", "--joint"):
        o = tmp_path / ("o%s.pb" % flag)
        r = run(checker_exe, ["--matches_file", str(d / "batch.pb"), "--output_file", str(o), flag,
                              "--q=" + g[0], "--q", g[1]])
        assert r.returncode == 0, r.stderr
        outs.append(o.read_bytes())
    assert outs[0] == outs[1] == outs[2] and outs[0]
    for r in _both_hosts(checker_exe, ["--matches_file", str(d / "batch.pb"), "--output_file", str(tmp_path / "x.pb"),
                                       "--joint_queries=1"]):
        assert r.returncode == 1 and r.stderr.startswith(b"ERROR: option '--joint_queries' does not take any arguments\n")
