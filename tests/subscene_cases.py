"""Query batches whose sub-scenes outgrow the 64-bit image mask (--query_images, MatchSet.query_subscenes).

Every case is a function returning (batch MatchSet, query names, banned image name).  Every kept pair names a
query, so a track is a star around one query keypoint: a track of L images is one query keypoint matched to
L - 1 database images.  MatchSet.query_subscenes numbers each sub-scene's ids by first appearance, and the
union-find image sets index an image by its id inside its sub-scene (its "local id"), so the sets are as wide
as the largest sub-scene.  The cases put those local ids on the 64-bit word edges (63 / 64, 127 / 128), make
image sets cross the 12-entry lists into 2- and 3-word bitsets, refuse unions on a clash between two bitsets,
fill the bitset pool to its N / 13 bound, cut meta-components at sub-scene caps of 2, 3, 65 and 129, and
reach the 65 535-id limit.  `check_structure(name)` asserts, on the host stage's export, what a name promises.

`grouped(name)` gives the grouped stage input of a case.  A name "<case>@q<K>" swaps the query of the
case's largest sub-scene with the image at local id K: the stages take any grouping, and their result does
not depend on how images are numbered, but only this way does a clash fall on the query's image at K alone
(every track of a sub-scene holds the query image, and hosts number the query first).
"""
import numpy as np

from lfr_b200.graph import host_input_arrays, host_stage_export
from test_graph_stage_adversarial import Scene

LFR_EUNSUPPORTED = -5


class Batch:
    """Links (query image, query keypoint, database image, database keypoint, similarity), listed in the
    order of `build(order)`: the order of first use of each (query, database) pair is the pair order."""

    def __init__(self, n_db, n_q, seed):
        self.n_db, self.n_q = n_db, n_q
        self.rng = np.random.default_rng(seed)
        self.links = []

    def q(self, i):
        return self.n_db + i

    def star(self, qi, f, dbs, sims=None, dfeat=None):
        """Query keypoint f of query qi matched to keypoint dfeat (default f) of each of `dbs`."""
        dbs = list(dbs)
        sims = self.rng.uniform(0.5, 1.0, len(dbs)) if sims is None else np.broadcast_to(sims, (len(dbs),))
        for d, s in zip(dbs, sims):
            self.links.append((self.q(qi), f, int(d), f if dfeat is None else dfeat, float(s)))

    def link(self, qi, f, d, df, s):
        self.links.append((self.q(qi), f, int(d), df, float(s)))

    def build(self, shuffle=True, round_sims=None):
        links = list(self.links)
        if shuffle:
            links = [links[i] for i in self.rng.permutation(len(links))]
        sc = Scene(self.n_db + self.n_q, seed=int(self.rng.integers(1 << 30)))
        a, f1, b, f2, s = [], [], [], [], []
        for q, fq, d, fd, sim in links:
            if (q * 7 + d) % 3 == 0:                 # the query on side 2 of a third of the pairs
                a.append(d); f1.append(fd); b.append(q); f2.append(fq)
            else:
                a.append(q); f1.append(fq); b.append(d); f2.append(fd)
            s.append(sim)
        s = np.asarray(s, np.float32)
        if round_sims:
            s = (np.round(s * round_sims) / round_sims).astype(np.float32)
        sc.matches(a, f1, b, f2, s)
        return sc

    def queries(self):
        return ["%05d.png" % self.q(i) for i in range(self.n_q)]


def _name(i):
    return "%05d.png" % i


def _with_empty_pair(ms, a, b):
    """A listing of (a, b) without matches, appended."""
    from lfr_b200.matchset import MatchSet
    out = MatchSet(ms.image_names, np.concatenate([ms.pair_img1, [a]]), np.concatenate([ms.pair_img2, [b]]),
                   np.concatenate([ms.pair_fact1, [1.0]]).astype(np.float32),
                   np.concatenate([ms.pair_fact2, [1.0]]).astype(np.float32),
                   np.concatenate([ms.pair_ptr, [ms.n_matches]]), ms.feat1, ms.feat2, ms.sim, ms.disp1, ms.disp2)
    out.validate()
    return out


def _tracks(B, qi, dbs, sizes, f0, linked=3):
    """Stars of the given image counts over `dbs`, keypoints f0, f0 + 1, ...; `linked` low-similarity
    matches between consecutive tracks (refused: both hold the query image) make meta-edges."""
    feats = []
    for j, L in enumerate(sizes):
        f = f0 + j
        B.star(qi, f, B.rng.choice(dbs, L - 1, replace=False) if L - 1 < len(dbs) else dbs)
        feats.append(f)
    for j in range(min(linked, len(feats) - 1)):
        d = [l[2] for l in B.links if l[0] == B.q(qi) and l[1] == feats[j + 1]][0]
        B.link(qi, feats[j], d, feats[j + 1], 0.1)
    return feats


def _clash_pair(B, qi, dbs, f, n=20):
    """Two tracks of n + 1 images on disjoint database images; query keypoint f + 1 also matches a
    database keypoint of the first, below both tracks' similarities: a union refused by a clash of two
    bitsets on the query's image alone."""
    da = B.rng.choice(dbs, 2 * n, replace=False)
    B.star(qi, f, da[:n], 0.9)
    B.star(qi, f + 1, da[n:], 0.85)
    B.link(qi, f + 1, da[0], f, 0.3)


def mask64():
    """Three queries, each matched to the same 63 database images: sub-scenes of 64 images (local ids up
    to 63, the mask path) in a batch of 192 ids.  Track 0 of each query spans its whole sub-scene."""
    B = Batch(63, 3, seed=64)
    dbs = np.arange(63)
    for qi in range(3):
        B.star(qi, 0, dbs)
        _tracks(B, qi, dbs, [5, 12, 13, 30, 50], 1)
    return B.build().build(), B.queries(), "none.png"


def _big(seed, n_db, sizes, n_small=2):
    """Query 0 on n_db database images (tracks of `sizes` images, one clash pair), next to n_small queries
    of 1 .. 2 database images each (sub-scenes of 2 - 3 images)."""
    B = Batch(n_db + 2, 1 + n_small, seed=seed)
    dbs = np.arange(n_db)
    B.star(0, 0, dbs)                                                  # every image of the sub-scene
    f = _tracks(B, 0, dbs, sizes, 1)
    _clash_pair(B, 0, dbs, f[-1] + 1)
    for qi in range(1, 1 + n_small):
        extra = [n_db, n_db + 1][:qi]
        B.star(qi, 0, extra)
        B.star(qi, 1, extra[:1])
    return B


def bitset65():
    B = _big(65, 64, [64, 13, 12, 65, 13, 12, 40])
    return B.build().build(), B.queries(), "none.png"


def bitset129():
    B = _big(129, 128, [12, 13, 64, 65, 129, 100, 13])
    return B.build().build(), B.queries(), "none.png"


def pool_bound(k=40, n_db=80):
    """One sub-scene of n_db + 1 images; k query keypoints of exactly 13 images each (N = 13 k): every
    set crosses the 12-entry list once."""
    B = Batch(n_db, 1, seed=13)
    for f in range(k):
        B.star(0, f, B.rng.choice(n_db, 12, replace=False))
    return B.build().build(), B.queries(), "none.png"


def interleaved():
    """Four sub-scenes of 70, 100, 129 and 90 images over one pool of database images, their pairs
    interleaved in file order; similarities rounded to 1/20, so ties cross sub-scenes."""
    n_db = 140
    B = Batch(n_db, 4, seed=4)
    for qi, D in enumerate((69, 99, 128, 89)):
        dbs = B.rng.choice(n_db, D, replace=False)
        B.star(qi, 0, dbs)
        sizes = B.rng.integers(2, D, 12).tolist() + [12, 13, 65]
        _tracks(B, qi, dbs, sizes, 1, linked=6)
        _clash_pair(B, qi, dbs, 100, n=min(20, D // 2))
    return B.build(round_sims=20).build(), B.queries(), "none.png"


CAP_HUBS = {0: (1, [12]), 1: (2, [12]), 2: (64, [64, 65]), 3: (128, [128, 129])}


def caps():
    """Sub-scenes seen with 2, 3, 65 and 129 images.  Hub matches (many query keypoints on one database
    keypoint: one track of two, the rest refused) make meta-components of h + 1 nodes: over the cap of the
    small sub-scenes, and in the large ones one exactly at the cap (not cut) and one above it.  In the
    65-image sub-scene one database image is listed only in a pair without matches (it counts towards the
    cap and has no node); in the 129-image sub-scene a banned database image drops a pair of its own."""
    n_db = 130
    B = Batch(n_db + 1, 4, seed=2)
    banned = n_db
    first = {}
    for qi, (D, hubs) in CAP_HUBS.items():
        dbs = np.arange(D) if qi != 1 else np.array([5, 9])
        with_matches = dbs[:-1] if qi == 2 else dbs
        B.star(qi, 0, with_matches)
        if D > 2:
            _tracks(B, qi, with_matches, [13, 30, 12], 1)
        for j, h in enumerate(hubs):
            d = int(with_matches[j])
            for f in range(h):
                B.link(qi, 1000 * (j + 1) + f, d, 5000 + j, 0.8 - 0.001 * (f % 7))
        first[qi] = dbs
    B.star(3, 7, [banned], 0.95)
    ms = B.build().build()
    ms = _with_empty_pair(ms, B.q(2), 63)
    return ms, B.queries(), _name(banned)


def ids(n_q=4369, n_db=14, extra=False):
    """n_q queries x n_db database images: n_q (n_db + 1) ids (65 535 at the defaults); `extra` adds one more
    database image to the last query (65 536).  Two matches per pair."""
    from lfr_b200.matchset import MatchSet
    n_img = n_db + 1 + n_q
    rng = np.random.default_rng(65535)
    p1, p2 = [], []
    for q in range(n_q):
        for d in range(n_db):
            p1.append(n_db + 1 + q); p2.append(d)
    if extra:
        p1.append(n_db + 1 + n_q - 1); p2.append(n_db)
    P = len(p1)
    M = 2 * P
    f = np.tile(np.array([0, 1], np.uint32), P)
    ms = MatchSet(["%05d.png" % i for i in range(n_img)], np.array(p1, np.int64), np.array(p2, np.int64),
                  np.ones(P, np.float32), np.ones(P, np.float32), np.arange(0, M + 1, 2, dtype=np.int64), f, f.copy(),
                  rng.uniform(0.5, 1.0, M).astype(np.float32), rng.normal(0, 0.01, (M, 18)).astype(np.float32),
                  rng.normal(0, 0.01, (M, 18)).astype(np.float32))
    ms.validate()
    return ms, ["%05d.png" % (n_db + 1 + q) for q in range(n_q)], "none.png"


def wide(n_db=1100):
    """One sub-scene of n_db + 1 images whose whole-scene track is one component of n_db + 1 nodes (the CTA
    tier, past 1024 nodes; image sets of 18 words), next to a sub-scene of 3 images."""
    B = Batch(n_db + 2, 2, seed=1101)
    dbs = np.arange(n_db)
    B.star(0, 0, dbs)
    _tracks(B, 0, dbs, [13, 200, 12], 1)
    B.star(1, 0, [n_db, n_db + 1])
    return B.build().build(), B.queries(), "none.png"


def decoded_on_device(n_q=6, n_db=100, k=700):
    """n_q sub-scenes of n_db + 1 images, each with k query keypoints on 40 - 100 database images: about
    300 000 matches, past the count from which the drop-in decodes the matches on the GPU."""
    B = Batch(n_db, n_q, seed=262144)
    for qi in range(n_q):
        for f in range(k):
            B.star(qi, f, B.rng.choice(n_db, int(B.rng.integers(40, n_db + 1)), replace=False))
    return B.build(round_sims=20).build(), B.queries(), "none.png"


CASES = {"mask64": mask64, "bitset65": bitset65, "bitset129": bitset129, "pool_bound": pool_bound,
         "interleaved": interleaved, "caps": caps, "wide1101": wide, "decoded_on_device": decoded_on_device,
         "ids_65535": ids, "ids_65536": lambda: ids(extra=True)}
#: the stage-only variants: the query of the largest sub-scene at local id K
SWAPS = {"bitset65@q63": ("bitset65", 63), "bitset65@q64": ("bitset65", 64),
         "bitset129@q127": ("bitset129", 127), "bitset129@q128": ("bitset129", 128)}
#: the cases the drop-in runs end to end (the id-limit cases have their own tests)
SOLVED = ["mask64", "bitset65", "bitset129", "pool_bound", "interleaved", "caps"]
#: every case the graph stages take
STAGED = SOLVED + list(SWAPS) + ["wide1101", "ids_65535"]

_cache = {}


def make(name):
    """(batch, queries, banned) of a case (cached; do not modify)."""
    base = SWAPS[name][0] if name in SWAPS else name
    if base not in _cache:
        _cache[base] = CASES[base]()
    return _cache[base]


def local_ids(group):
    """The index of every id inside its sub-scene (lfr_host.cc's local_image)."""
    group = np.asarray(group, np.int64)
    loc = np.zeros(group.shape[0], np.int64)
    for g in np.unique(group):
        ids_g = np.nonzero(group == g)[0]
        loc[ids_g] = np.arange(ids_g.shape[0])
    return loc


def grouped(name):
    """(sub MatchSet, image_group) of a case: MatchSet.query_subscenes, with the swap of a "@q" variant."""
    batch, queries, banned = make(name)
    sub, group = batch.query_subscenes(queries, [banned])
    if name not in SWAPS:
        return sub, group
    k = SWAPS[name][1]
    g = np.bincount(group).argmax()
    ids_g = np.nonzero(group == g)[0]
    qid = [i for i in ids_g.tolist() if sub.image_names[i] in set(queries)][0]
    tid = int(ids_g[k])
    perm = np.arange(len(sub.image_names))
    perm[qid], perm[tid] = tid, qid
    names = list(sub.image_names)
    names[qid], names[tid] = names[tid], names[qid]
    sub = sub.select_pairs(np.arange(sub.n_pairs))
    sub.image_names = names
    sub.pair_img1 = perm[sub.pair_img1]
    sub.pair_img2 = perm[sub.pair_img2]
    return sub, group


def stage(name, threads=None):
    """The host stage's export of the grouped case: (arrays, sizes, sub, group)."""
    sub, group = grouped(name)
    _, arrs = host_input_arrays(sub, (), group)
    rc, out, sz = host_stage_export(arrs, len(sub.image_names))
    assert rc == 0, (name, rc)
    return out, sz, sub, group


def refused_clashes(out, group, sub):
    """Local ids of the images on which a union of two sets of more than 12 images each is refused: for
    every match whose two nodes end in different tracks, both tracks hold more than 12 nodes and share
    exactly one image, that image's local id."""
    loc = local_ids(group)
    track = out["track"].astype(np.int64)
    size = np.bincount(track)
    nimg = out["node_image"].astype(np.int64)
    images_of = {}
    for v in range(track.shape[0]):
        images_of.setdefault(track[v], set()).add(int(nimg[v]))
    found = set()
    rp = out["row_ptr"].astype(np.int64)
    for v in range(track.shape[0]):
        for e in range(rp[v], rp[v + 1]):
            w = int(out["edges"]["dst"][e])
            a, b = track[v], track[w]
            if a != b and size[a] > 12 and size[b] > 12:
                common = images_of[a] & images_of[b]
                if len(common) == 1:
                    found.add(int(loc[next(iter(common))]))
    return found


def check_structure(name):
    """Assert, on the host stage's export of the grouped case, what the case's name promises."""
    out, sz, sub, group = stage(name)
    counts = np.unique(group, return_counts=True)[1].tolist()        # images of each sub-scene
    width = max(counts)
    loc = local_ids(group)
    nimg = out["node_image"].astype(np.int64)
    node_group = group[nimg]
    sizes = np.bincount(out["track"].astype(np.int64))
    # track sizes inside the largest sub-scene
    big = np.bincount(group).argmax()
    big_sizes = set(np.bincount(out["track"][node_group == big].astype(np.int64)).tolist()) - {0}
    if name == "mask64":
        assert width == 64 and len(sub.image_names) == 192 and counts == [64] * 3
        assert 63 in set(loc[nimg].tolist()) and 64 in set(sizes.tolist())
    elif name.startswith("bitset65"):
        assert width == 65 and sorted(counts) == [2, 3, 65]
        assert {12, 13, 64, 65} <= big_sizes
    elif name.startswith("bitset129"):
        assert width == 129 and {12, 13, 64, 65, 129} <= big_sizes
        assert {127, 128} <= set(loc[nimg[node_group == big]].tolist())
    elif name == "pool_bound":
        assert width > 64 and sizes.tolist() == [13] * 40 and sz["n_nodes"] == 13 * 40
    elif name == "interleaved":
        assert sorted(counts) == [70, 90, 100, 129]
        assert (loc % 64 != np.arange(loc.shape[0]) % 64).any()
        # pairs of different sub-scenes alternate in file order
        pg = group[sub.pair_img1]
        assert (pg[1:] != pg[:-1]).sum() > 100
        # tied similarities across sub-scenes
        s = sub.sim
        mg = np.repeat(pg, np.diff(sub.pair_ptr))
        assert any(len(set(mg[s == v].tolist())) > 1 for v in np.unique(s)[:5])
    elif name == "caps":
        seen = np.zeros(len(sub.image_names), bool)
        seen[sub.pair_img1] = True
        seen[sub.pair_img2] = True
        assert sorted(np.unique(group[seen], return_counts=True)[1].tolist()) == [2, 3, 65, 129]
        assert _name(130) not in sub.image_names
        assert sz["n_oversized_meta_components"] == 4
    elif name == "wide1101":
        assert width == 1101 and sz["max_component_size"] == 1101
    elif name == "ids_65535":
        assert len(sub.image_names) == 65535 and width == 15
    if "@q" in name:
        k = SWAPS[name][1]
        qid = [i for i in range(len(sub.image_names)) if sub.image_names[i] in set(make(name)[1])
               and group[i] == big][0]
        assert loc[qid] == k
        assert k in refused_clashes(out, group, sub)
    return out, sz, sub, group
