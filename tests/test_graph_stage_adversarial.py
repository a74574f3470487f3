"""The graph stage on match graphs built to break it, against the host stage, graph.py and the reference.

Scenes from synth.py have one structure.  The cases here are built pair by pair to force what the
stages' data structures and the device's reservation rounds were written for: many edges on one root
in a round (stars), long runs of image-clash refusals, image sets crossing the 64-bit mask, the
12-entry lists and the pool bitsets at their word edges, the pool at its N / 13 bound, 65 535 images,
equal-size unions at every level, duplicated pairs and matches, meta-components far over the
image-count cap, saturating cut weights, extreme feature indices, and similarities of -0.0 (equal to
+0.0 in the reference's (sim, n1, n2) sort, solve.cc:489).

CPU: the native host stage (csrc/lfr_host.cc) equals graph.py's stage array for array, and the host
pipeline (native stage + CPU oracle + assemble_solution) writes the SolutionFile and the untimed stdout
lines the reference's own main() wrote, recorded in tests/golden/ref_record_graph.json
(tests/golden/make_ref_graph_record.py).
GPU: the device stage (csrc/lfr_graph.cuh) equals the host stage bitwise at every Kruskal window, its
plan solves bitwise like lfr_solve() on the host-stage problem, and the native drop-in on the device
route reproduces the reference's committed SolutionFiles (tests/golden/adv_<case>_solution.pb).
"""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from lfr_b200 import build_problem, synth, wire
from lfr_b200.graph import host_input_arrays, host_stage_export
from lfr_b200.matchset import MatchSet
from test_native_exe import PRODUCT, product_exe  # noqa: F401  (fixture)
from test_ref_solve import oracle_pipeline, untimed

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECORD = os.path.join(GOLD, "ref_record_graph.json")
LFR_EUNSUPPORTED = -5


# ---------------------------------------------------------------------------------------------------
# case constructors
# ---------------------------------------------------------------------------------------------------
def _offset(img, feat):
    """A keypoint's localisation error (units of 16 px), a fixed function of (image, feature index)."""
    x = np.asarray(img, np.float64) * 12.9898 + np.asarray(feat, np.float64) * 78.233
    return 0.3 * np.stack([np.sin(x), np.cos(1.7 * x)], axis=-1)


class Scene:
    """A MatchSet built pair by pair.  Displacements follow the keypoints' errors plus seeded noise."""

    def __init__(self, n_images, seed):
        self.n_images = n_images
        self.rng = np.random.default_rng(seed)
        self.pairs = []

    def pair(self, a, b, f1, f2, sim):
        """One listing of the image pair (a, b) with its matches (feature indices f1 in a, f2 in b)."""
        f1 = np.atleast_1d(np.asarray(f1, np.int64)).astype(np.uint32)
        f2 = np.atleast_1d(np.asarray(f2, np.int64)).astype(np.uint32)
        sim = np.broadcast_to(np.asarray(sim, np.float32), f1.shape).copy()
        self.pairs.append((int(a), int(b), f1, f2, sim))

    def matches(self, a, f1, b, f2, sim):
        """Single matches grouped into one listing per (a, b), pairs and matches in order of first use."""
        a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
        f1, f2 = np.asarray(f1, np.int64), np.asarray(f2, np.int64)
        sim = np.broadcast_to(np.asarray(sim, np.float32), a.shape)
        _, first, inv = np.unique(a * self.n_images + b, return_index=True, return_inverse=True)
        for g in np.argsort(first, kind="stable"):
            sel = np.nonzero(inv == g)[0]
            self.pair(a[sel[0]], b[sel[0]], f1[sel], f2[sel], sim[sel])

    def chain(self, images, feat, sims):
        """A path through one keypoint (`feat`) of each image of `images`, in that order."""
        images = np.asarray(images, np.int64)
        self.matches(images[:-1], np.full(len(images) - 1, feat), images[1:], np.full(len(images) - 1, feat), sims)

    def build(self) -> MatchSet:
        ptr = np.zeros(len(self.pairs) + 1, np.int64)
        np.cumsum([len(p[2]) for p in self.pairs], out=ptr[1:])
        cat = lambda i, dt: (np.concatenate([p[i] for p in self.pairs]).astype(dt) if self.pairs else np.zeros(0, dt))
        img1 = np.repeat([p[0] for p in self.pairs], np.diff(ptr)).astype(np.int64)
        img2 = np.repeat([p[1] for p in self.pairs], np.diff(ptr)).astype(np.int64)
        f1, f2 = cat(2, np.uint32), cat(3, np.uint32)
        dt = _offset(img2, f2) - _offset(img1, f1)                                   # t_b - t_a
        M = f1.shape[0]
        d12 = dt[:, None, :] + self.rng.normal(0, 0.01, size=(M, 9, 2))
        d21 = -dt[:, None, :] + self.rng.normal(0, 0.01, size=(M, 9, 2))
        ms = MatchSet(image_names=["%05d.png" % i for i in range(self.n_images)],
                      pair_img1=np.array([p[0] for p in self.pairs], np.int64),
                      pair_img2=np.array([p[1] for p in self.pairs], np.int64),
                      pair_fact1=np.ones(len(self.pairs), np.float32), pair_fact2=np.ones(len(self.pairs), np.float32),
                      pair_ptr=ptr, feat1=f1, feat2=f2, sim=cat(4, np.float32),
                      disp1=d21.reshape(M, 18).astype(np.float32), disp2=d12.reshape(M, 18).astype(np.float32))
        ms.validate()
        return ms


def _signed_zero(k):
    """cfg1 (synth seed None, 2, 3, 4) with 20 % of the similarities negated and 40 % set to -0.0 or +0.0."""
    ms = synth.generate("cfg1", seed=(None, 2, 3, 4)[k])
    M = ms.sim.shape[0]
    rng = np.random.default_rng(k)
    z = rng.random(M) < 0.4
    neg = rng.random(M) < 0.2
    ms.sim[neg] = -ms.sim[neg]
    ms.sim[z] = np.where(rng.random(z.sum()) < 0.5, np.float32(-0.0), np.float32(0.0))
    return ms


def _signed_zero_all():
    ms = synth.generate("cfg1", seed=3)
    ms.sim[:] = np.where(np.random.default_rng(7).random(ms.sim.shape[0]) < 0.5, np.float32(-0.0), np.float32(0.0))
    return ms


def _denormal():
    """Similarities of +-0.0 and the smallest denormals: distinct in the reference's double sort."""
    ms = synth.generate("cfg1", seed=5)
    tiny = np.array([0.0, -0.0, 1e-45, -1e-45, 3e-45, -3e-45, 1.1754942e-38], np.float32)
    ms.sim[:] = tiny[np.random.default_rng(8).integers(0, tiny.shape[0], ms.sim.shape[0])]
    return ms


def _star(K, order):
    """Hub keypoint 0 of image 0 matched to keypoint 0 of each of K images; hub keypoint 1 matched to the
    same partners just below (or, for `equal`, at) the same similarity: every edge touches the hub's
    root, and every edge of the losing hub is refused by an image clash."""
    sc = Scene(K + 1, seed=K)
    s = {"equal": np.full(K, 0.9, np.float32), "ascending": np.linspace(0.5, 0.99, K, dtype=np.float32),
         "descending": np.linspace(0.99, 0.5, K, dtype=np.float32)}[order]
    s2 = s if order == "equal" else np.nextafter(s, np.float32(0))
    for i in range(1, K + 1):
        sc.pair(0, i, [0, 1], [0, 0], [s[i - 1], s2[i - 1]])
    return sc.build()


def _edge_images(n):
    """Image ids on the 64-bit word edges and the last image."""
    return sorted({i for i in (0, 63, 64, 127, 128, n - 1) if i < n})


def _images(n):
    """Chains through n images: three tracks each of exactly 12, 13, 25, 64 and 65 images (those that
    fit), the first of each length through the word-edge image ids; a chain that revisits an image; and
    low-similarity edges between tracks that share an image (refused, but meta-edges)."""
    sc = Scene(n, seed=n)
    rng = sc.rng
    tracks, feat = [], 0
    for L in (12, 13, 25, 64, 65):
        if L > n:
            continue
        for rep in range(3):
            imgs = rng.choice(n, L, replace=False)
            if rep == 0:
                extra = [i for i in _edge_images(n) if i not in imgs][:L]
                imgs[:len(extra)] = extra
                rng.shuffle(imgs)
            sc.chain(imgs, feat, rng.uniform(0.5, 1.0, L - 1))
            tracks.append((imgs, feat))
            feat += 1
    imgs = rng.choice(n, 14, replace=False)
    imgs[-1] = imgs[0]                                            # revisits its first image: one union refused
    sc.chain(imgs, feat, rng.uniform(0.5, 1.0, 13))
    for (ia, fa), (ib, fb) in zip(tracks[:-1], tracks[1:]):
        if np.intersect1d(ia, ib).shape[0]:
            x, y = rng.integers(0, len(ia)), rng.integers(0, len(ib))
            if ia[x] != ib[y]:
                sc.matches([ia[x]], [fa], [ib[y]], [fb], [0.05])
    return sc.build()


def _pool_bound(n, k):
    """k disjoint chains of exactly 13 images: every set crosses the 12-entry lists once (N = 13 k)."""
    sc = Scene(n, seed=1000 + n)
    for t in range(k):
        sc.chain(sc.rng.choice(n, 13, replace=False), t, sc.rng.uniform(0.5, 1.0, 12))
    return sc.build()


def _many_images(n=65535, top=None):
    """A sparse scene over n images: 8 chains of 20 images spread up to id n - 1 (or `top`)."""
    top = n - 1 if top is None else top
    sc = Scene(n, seed=65535)
    edges = [0, 63, 64, 64 * 1023 - 1, 64 * 1023, top]
    for t in range(8):
        imgs = sc.rng.choice(top, 20, replace=False)
        if t < 2:
            extra = [i for i in edges if i not in imgs]
            imgs[:len(extra)] = extra
            sc.rng.shuffle(imgs)
        sc.chain(imgs, t, sc.rng.uniform(0.5, 1.0, 19))
    return sc.build()


def _balanced(N, n_trees=4):
    """n_trees trees of N = 2^L nodes, one node per image in each: pairs, then pairs of pairs, ...  Every
    union joins two sets of equal size (the "root2 under root1" tie), all edges of one level at one
    similarity, random orientation.  The trees' pairs are listed interleaved, so their node ids are too,
    and which node ends as a root shows in the track numbering (track ids follow the roots' node order)."""
    sc = Scene(N, seed=N)
    rng = sc.rng
    listing = []
    for t in range(n_trees):
        img = rng.permutation(N)
        feat = 1000 * t + rng.integers(0, 1000, N)
        level, half = 1, 1
        while half < N:
            for g in range(0, N, 2 * half):
                u, v = g + rng.integers(0, half), g + half + rng.integers(0, half)
                if rng.random() < 0.5:
                    u, v = v, u
                listing.append((img[u], img[v], feat[u], feat[v], 1.0 - 0.05 * level))
            level, half = level + 1, 2 * half
    for e in rng.permutation(len(listing)):
        a, b, fa, fb, s = listing[e]
        sc.pair(a, b, [fa], [fb], [s])
    return sc.build()


def _duplicates():
    """The same pair listed twice, a pair listed both as (A, B) and (B, A), every match of a pair twice in
    a row; all similarities equal."""
    sc = Scene(6, seed=6)
    rng = sc.rng
    base = []
    for a in range(6):
        for b in range(a + 1, 6):
            base.append((a, b, rng.integers(0, 40, 25), rng.integers(0, 40, 25)))
    for a, b, f1, f2 in base:
        sc.pair(a, b, f1, f2, 0.75)
    a, b, f1, f2 = base[0]
    sc.pair(a, b, f1, f2, 0.75)                       # listed again, identical
    a, b, f1, f2 = base[6]
    sc.pair(b, a, f2, f1, 0.75)                       # reversed
    a, b, f1, f2 = base[11]
    sc.pair(a, b, np.repeat(f1, 2), np.repeat(f2, 2), 0.75)
    return sc.build()


def _giant_meta(n_images=4, n_kpts=200, per_pair=400, lo=0.5, hi=1.0, repeat=1, seed=44):
    """Random matches between few images: many small tracks in one meta-component far over the
    image-count cap, cut recursively into many groups."""
    sc = Scene(n_images, seed=seed)
    rng = sc.rng
    for a in range(n_images):
        for b in range(a + 1, n_images):
            f1, f2 = rng.integers(0, n_kpts, per_pair), rng.integers(0, n_kpts, per_pair)
            sc.pair(a, b, np.repeat(f1, repeat), np.repeat(f2, repeat), np.repeat(rng.uniform(lo, hi, per_pair), repeat))
    return sc.build()


def _saturating_cut():
    """Similarities of 1e8 and more, each match three times: int(100 * sum) of every meta-edge is
    outside the int range (lfr::cut_weight saturates)."""
    return _giant_meta(n_images=3, n_kpts=150, per_pair=300, lo=1e8, hi=2e8, repeat=3, seed=45)


def _feature_extremes():
    """Feature indices 0 and 2^32 - 1 in one image; a pair without matches lists image 6 (counted in
    the image cap, no node); image 7 is never listed."""
    sc = Scene(8, seed=8)
    rng = sc.rng
    top = 2 ** 32 - 1
    for a in range(6):
        for b in range(a + 1, 6):
            f1, f2 = rng.integers(0, 30, 12), rng.integers(0, 30, 12)
            if a == 0:
                f1[:2] = [0, top]
            if b == 2:
                f2[0] = top
            sc.pair(a, b, f1, f2, rng.uniform(0.5, 1.0, 12))
    sc.pair(6, 0, [], [], [])
    return sc.build()


CASES = {}
for _k in range(4):
    CASES["signed_zero_%d" % _k] = (lambda k=_k: _signed_zero(k))
CASES["signed_zero_all"] = _signed_zero_all
CASES["signed_zero_denormal"] = _denormal
for _K in (63, 64, 200, 1500):
    for _o in ("equal", "ascending", "descending"):
        CASES["star_%d_%s" % (_K, _o)] = (lambda K=_K, o=_o: _star(K, o))
for _n in (64, 65, 128, 129, 1000):
    CASES["images_%d" % _n] = (lambda n=_n: _images(n))
CASES["pool_bound_65"] = lambda: _pool_bound(65, 40)
CASES["pool_bound_1000"] = lambda: _pool_bound(1000, 150)
CASES["images_65535"] = _many_images
CASES["balanced_unions_64"] = lambda: _balanced(64)
CASES["balanced_unions_256"] = lambda: _balanced(256)
CASES["duplicates"] = _duplicates
CASES["giant_meta"] = _giant_meta
CASES["saturating_cut"] = _saturating_cut
CASES["feature_extremes"] = _feature_extremes

#: not compared with the reference: its int(100 * sum) cast is undefined there (and graph.py does not saturate)
STAGE_ONLY = ("saturating_cut",)
REF_CASES = [c for c in CASES if c not in STAGE_ONLY]
#: the reference's SolutionFile is committed for these, so the device route can be compared with a tolerance
E2E_CASES = ["signed_zero_2", "signed_zero_all", "signed_zero_denormal", "star_64_equal", "star_200_descending",
             "images_129", "pool_bound_65", "balanced_unions_256", "duplicates", "giant_meta", "feature_extremes"]

_cache = {}


def make_case(name) -> MatchSet:
    if name not in _cache:
        _cache[name] = CASES[name]()
    return _cache[name]


def case_arrays(name):
    """(flat lfr_host_input arrays, private copies; n_images) of a case."""
    ms = make_case(name)
    return {k: v.copy() for k, v in host_input_arrays(ms)[1].items()}, len(ms.image_names)


def solution_path(name):
    return os.path.join(GOLD, "adv_%s_solution.pb" % name)


def _record():
    with open(RECORD) as fh:
        return json.load(fh)


def _sha(b):
    return hashlib.sha256(b).hexdigest()


# ---------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------
def test_cases_have_the_structure_they_are_named_for():
    """The constructors build what the case names promise (checked on graph.py's stage)."""
    for K in (63, 64, 200, 1500):
        for o in ("equal", "ascending", "descending"):
            p = build_problem(make_case("star_%d_%s" % (K, o)), native=False)
            assert sorted(np.bincount(p.track).tolist()) == [1, K + 1]
    for n in (64, 65, 128, 129, 1000):
        p = build_problem(make_case("images_%d" % n), native=False)
        sizes = set(np.bincount(p.track).tolist())
        assert {L for L in (12, 13, 25, 64, 65) if L <= n} <= sizes
        assert set(_edge_images(n)) <= set(p.graph.node_image.tolist())
    for name, k in (("pool_bound_65", 40), ("pool_bound_1000", 150)):
        p = build_problem(make_case(name), native=False)
        assert np.bincount(p.track).tolist() == [13] * k and p.graph.n_nodes == 13 * k
    p = build_problem(make_case("images_65535"), native=False)
    assert p.graph.node_image.max() == 65534 and np.bincount(p.track).min() == 20
    for N in (64, 256):
        p = build_problem(make_case("balanced_unions_%d" % N), native=False)
        assert np.bincount(p.track).tolist() == [N] * 4
    p = build_problem(make_case("giant_meta"), native=False)
    assert p.info["n_oversized_meta_components"] == 1 and p.info["n_cut_groups"] > 50
    p = build_problem(make_case("feature_extremes"), native=False)
    assert {0, 2 ** 32 - 1} <= set(p.graph.node_feat[p.graph.node_image == 0].tolist()) and p.graph.n_images == 7


@pytest.mark.parametrize("case", REF_CASES)
def test_native_host_stage_equals_numpy_stage(case):
    """csrc/lfr_host.cc (include/lfr_host.h) against graph.py, array for array."""
    ms = make_case(case)
    a = build_problem(ms, native=True)
    b = build_problem(ms, native=False)
    for k in ("track", "comp", "is_root", "comp_ptr", "comp_nodes", "comp_order"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert np.array_equal(a.graph.row_ptr, b.graph.row_ptr) and a.graph.edges.tobytes() == b.graph.edges.tobytes()
    assert np.array_equal(a.graph.node_image, b.graph.node_image) and np.array_equal(a.graph.node_feat, b.graph.node_feat)
    assert a.graph.n_images == b.graph.n_images
    for k in ("n_tracks", "n_components", "max_component_size", "n_meta_components", "n_oversized_meta_components",
              "n_cut_groups"):
        assert a.info[k] == b.info[k], k


@pytest.mark.parametrize("case", REF_CASES)
def test_host_pipeline_reproduces_the_reference_binary(oracle, case):
    """Native host stage + CPU oracle + assemble_solution on the encoded case: the SolutionFile bytes and
    the untimed stdout lines of the reference's own main()."""
    want = _record()[case]
    mine, _, _, lines = oracle_pipeline(oracle, wire.encode_matching_file(make_case(case)))
    assert _sha(mine) == want["solution_sha256"]
    assert [l for l in lines if " time:" not in l] == want["stdout"]


def test_committed_solution_files_are_the_reference_binarys_output():
    rec = _record()
    assert sorted(rec) == sorted(REF_CASES)
    for case in E2E_CASES:
        assert _sha(open(solution_path(case), "rb").read()) == rec[case]["solution_sha256"], case


def test_host_stage_refuses_65536_images():
    """65 535 images are taken (16-bit image ids in the lists); one more is refused."""
    arrs, n = case_arrays("images_65535")
    assert n == 65535 and host_stage_export(arrs, n)[0] == 0
    ms = _many_images(65536)
    _, arrs = host_input_arrays(ms)
    assert int(arrs["pair_img1"].max()) == 65535 or int(arrs["pair_img2"].max()) == 65535
    assert host_stage_export(arrs, 65536)[0] == LFR_EUNSUPPORTED


# ---------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_device_stage_equals_host_stage_at_every_window(b200, case, monkeypatch):
    """Every lfr_plan_export_graph array and every lfr_host_sizes count, with the Kruskal window unset
    and at 1, 2, 31, 32, 33 and more than the match count."""
    from test_gpu_graph_stage import ARRAYS, COUNTS, device_stage
    arrs, n = case_arrays(case)
    rc, a, sa = host_stage_export(arrs, n)
    assert rc == 0
    M = arrs["feat1"].shape[0]
    for window in (None, 1, 2, 31, 32, 33, M + 1):
        if window is None:
            monkeypatch.delenv("LFR_KRUSKAL_WINDOW", raising=False)
        else:
            monkeypatch.setenv("LFR_KRUSKAL_WINDOW", str(window))
        rc, b, sb, plan = device_stage(b200, arrs, n)
        assert rc == 0, window
        for k in ARRAYS:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, (window, k)
            assert a[k].tobytes() == b[k].tobytes(), (window, k)
        for k in COUNTS:
            assert sa[k] == sb[k], (window, k, sa[k], sb[k])
        plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_plan_from_matches_solves_like_lfr_solve(b200, case):
    """Positions, per-slot iterations, terminations and costs of the device-built plan equal lfr_solve()
    on the host-stage problem."""
    from lfr_b200.capi import Plan
    ms = make_case(case)
    p = build_problem(ms, native=True)
    want_pos, want = b200.solve(p)
    plan = Plan.from_matches(b200, ms)
    plan.solve()
    got_pos, got = plan.download()
    plan.close()
    assert got_pos.tobytes() == want_pos.tobytes()
    for k in ("iterations", "termination", "initial_cost", "final_cost"):
        assert got[k].tobytes() == want[k].tobytes(), k
    for k in ("total_iterations", "total_line_search_steps", "n_solved"):
        assert got[k] == want[k], k


@pytest.mark.gpu
@pytest.mark.parametrize("case", E2E_CASES)
def test_device_route_reproduces_the_reference_solution_file(product_exe, tmp_path, case):  # noqa: F811
    """The native drop-in with LFR_GRAPH_STAGE=device against the reference's committed SolutionFile:
    the same untimed stdout lines, and the SolutionFile equal float for float (fp32 on the wire) —
    byte-identical unless a displacement sits within 1e-16 of a float32 rounding boundary."""
    m, o = tmp_path / "m.pb", tmp_path / "o.pb"
    m.write_bytes(wire.encode_matching_file(make_case(case)))
    r = subprocess.run([PRODUCT, "--matches_file", str(m), "--output_file", str(o)], capture_output=True, text=True,
                       env=dict(os.environ, LFR_GRAPH_STAGE="device"))
    assert r.returncode == 0, r.stderr
    assert untimed(r.stdout) == _record()[case]["stdout"]
    got, want = o.read_bytes(), open(solution_path(case), "rb").read()
    if got != want:
        a, b = wire.decode_solution(got), wire.decode_solution(want)
        assert [x[0] for x in a] == [x[0] for x in b]
        n_diff = 0
        for (_, fa, ia, dia, dja), (_, fb, ib, dib, djb) in zip(a, b):
            assert fa == fb and np.array_equal(ia, ib)
            assert np.abs(dia - dib).max() <= 1e-4 / 16 and np.abs(dja - djb).max() <= 1e-4 / 16
            n_diff += int((dia != dib).sum() + (dja != djb).sum())
        assert n_diff <= 2


@pytest.mark.gpu
def test_device_stage_takes_65535_images_and_refuses_65536(b200):
    from test_gpu_graph_stage import device_stage
    arrs, n = case_arrays("images_65535")
    rc, _, sizes, plan = device_stage(b200, arrs, n)
    assert rc == 0 and sizes["max_track_size"] == 20
    plan.close()
    _, arrs = host_input_arrays(_many_images(65536))
    assert host_stage_export(arrs, 65536)[0] == LFR_EUNSUPPORTED
    assert device_stage(b200, arrs, 65536)[0] == LFR_EUNSUPPORTED
