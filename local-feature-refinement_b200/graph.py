"""Host graph stage of `solve` (multi-view-refinement/solve.cc:405-606).

Everything between the parsed MatchingFile and the per-component solves:

  H1  node interning + directed edge lists            solve.cc:53-65, 474-478
  H2  constrained Kruskal -> tracks                   solve.cc:489-549, 67-77
  H3  root node of each track                         solve.cc:552-582
  H4  meta-graph of tracks, connected components,
      size-capped recursive 2-way cut                 solve.cc:252-373, 162-250
  H5  dispatch list (components, largest first)       solve.cc:594-606

The output is the `lfr_problem` of include/lfr.h: CSR-by-source edge records
(80 B each) plus per-node track / component / root arrays and the component
dispatch list.  Tie-breaks follow the reference (descending lexicographic sorts
done as sort+reverse, union-find merge direction, first-appearance numbering).

The one piece that cannot follow the reference is the 2-way normalized cut:
the reference calls colmap::ComputeNormalizedMinGraphCut (Graclus inside
COLMAP, solve.cc:192), which is not in the reference repository nor in this
image.  `two_way_cut` below is a deterministic replacement (BFS region growing
balanced on volume; like the COLMAP call it sees only the edge list and the integer weights,
csrc/lfr_cut.h is the same definition); it only matters for meta-components larger than
#images nodes, and the GPU path and every checker share it.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from .matchset import MatchSet

#: numpy mirror of `lfr_edge` (include/lfr.h): 80 bytes
EDGE_DTYPE = np.dtype([("flow", "<f4", (18,)), ("sim", "<f4"), ("dst", "<u4")])
assert EDGE_DTYPE.itemsize == 80


@dataclass
class MatchGraph:
    """H1: the reference's Graph (graph.h:33-41) in CSR form."""
    n_nodes: int
    node_image: np.ndarray      # [N] image id (index into image_names)
    node_feat: np.ndarray       # [N] uint32 feature_idx
    und_sim: np.ndarray         # [M] float64 (widened from float, solve.cc:458)
    und_n1: np.ndarray          # [M]
    und_n2: np.ndarray          # [M]
    row_ptr: np.ndarray         # [N+1] uint32
    edges: np.ndarray           # [E] EDGE_DTYPE, out-edges in insertion order
    image_names: List[str]
    image_fact: Dict[int, float]  # first sighting (solve.cc:449,451)
    n_images: int               # images_set.size() (solve.cc:448,450,586)

    @property
    def n_edges(self) -> int:
        return int(self.edges.shape[0])


def build_graph(ms: MatchSet, banned_images=()) -> MatchGraph:
    """H1 — solve.cc:438-481."""
    ms = ms.without_images(banned_images)
    M = ms.n_matches
    counts = (ms.pair_ptr[1:] - ms.pair_ptr[:-1]).astype(np.int64)
    img1 = np.repeat(ms.pair_img1.astype(np.int64), counts)
    img2 = np.repeat(ms.pair_img2.astype(np.int64), counts)
    # keys in order of find_or_create_node calls: side 1 then side 2 of every match
    keys = np.empty(2 * M, dtype=np.int64)
    keys[0::2] = (img1 << 32) | ms.feat1.astype(np.int64)
    keys[1::2] = (img2 << 32) | ms.feat2.astype(np.int64)
    uniq, first, inverse = np.unique(keys, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")          # unique ids by first appearance
    rank = np.empty_like(order)
    rank[order] = np.arange(order.shape[0])
    node_of = rank[inverse]
    n1 = node_of[0::2].astype(np.int64)
    n2 = node_of[1::2].astype(np.int64)
    N = int(uniq.shape[0])
    node_key = uniq[order]
    node_image = (node_key >> 32).astype(np.int64)
    node_feat = (node_key & 0xFFFFFFFF).astype(np.uint32)

    # directed edges in add_edge order: n1->n2 carries disp2, n2->n1 carries disp1 (solve.cc:477-478)
    src = np.empty(2 * M, dtype=np.int64)
    src[0::2] = n1
    src[1::2] = n2
    rec = np.zeros(2 * M, dtype=EDGE_DTYPE)
    rec["flow"][0::2] = ms.disp2
    rec["flow"][1::2] = ms.disp1
    rec["sim"][0::2] = ms.sim
    rec["sim"][1::2] = ms.sim
    rec["dst"][0::2] = n2
    rec["dst"][1::2] = n1
    perm = np.argsort(src, kind="stable")
    edges = np.ascontiguousarray(rec[perm])
    row_ptr = np.zeros(N + 1, dtype=np.uint32)
    np.cumsum(np.bincount(src, minlength=N), out=row_ptr[1:])

    image_fact: Dict[int, float] = {}
    seen_images = set()
    for a, b, fa, fb in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist(),
                            ms.pair_fact1.tolist(), ms.pair_fact2.tolist()):
        seen_images.add(ms.image_names[a])
        seen_images.add(ms.image_names[b])
        image_fact.setdefault(a, fa)
        image_fact.setdefault(b, fb)
    return MatchGraph(
        n_nodes=N, node_image=node_image, node_feat=node_feat,
        und_sim=ms.sim.astype(np.float64), und_n1=n1, und_n2=n2,
        row_ptr=row_ptr, edges=edges, image_names=ms.image_names,
        image_fact=image_fact, n_images=len(seen_images),
    )


def compute_tracks(g: MatchGraph) -> np.ndarray:
    """H2 — maximum spanning forest with the "one node per image" constraint
    (solve.cc:489-541).  Returns track_idx[N]."""
    N = g.n_nodes
    # std::sort + std::reverse on (sim, n1, n2)  (solve.cc:489-490)
    order = np.lexsort((g.und_n2, g.und_n1, g.und_sim))[::-1]
    parent = [-1] * N
    # image set of each union-find root as a Python-int bitset
    imgs = [1 << int(i) for i in g.node_image.tolist()]
    size = [1] * N
    a1 = g.und_n1[order].tolist()
    a2 = g.und_n2[order].tolist()
    for u, v in zip(a1, a2):
        r1 = u
        while parent[r1] != -1:
            r1 = parent[r1]
        while parent[u] != -1:            # path compression (solve.cc:74-76)
            nxt = parent[u]
            parent[u] = r1
            u = nxt
        r2 = v
        while parent[r2] != -1:
            r2 = parent[r2]
        while parent[v] != -1:
            nxt = parent[v]
            parent[v] = r2
            v = nxt
        if r1 == r2:
            continue
        if imgs[r1] & imgs[r2]:           # solve.cc:507-511
            continue
        if size[r1] < size[r2]:           # solve.cc:513-521
            parent[r1] = r2
            imgs[r2] |= imgs[r1]
            size[r2] += size[r1]
            imgs[r1] = 0
            size[r1] = 0
        else:
            parent[r2] = r1
            imgs[r1] |= imgs[r2]
            size[r1] += size[r2]
            imgs[r2] = 0
            size[r2] = 0
    par = np.array(parent, dtype=np.int64)
    # full compression, then ids in node order of the roots (solve.cc:526-541)
    root = np.arange(N, dtype=np.int64)
    has_parent = par >= 0
    root[has_parent] = par[has_parent]
    while True:
        nxt = root.copy()
        hp = par[root] >= 0
        nxt[hp] = par[root[hp]]
        if np.array_equal(nxt, root):
            break
        root = nxt
    is_rep = par < 0
    track_of_rep = np.cumsum(is_rep) - 1
    return track_of_rep[root].astype(np.int64)


def edge_sources(g: MatchGraph) -> np.ndarray:
    deg = (g.row_ptr[1:].astype(np.int64) - g.row_ptr[:-1].astype(np.int64))
    return np.repeat(np.arange(g.n_nodes, dtype=np.int64), deg)


def select_roots(g: MatchGraph, track: np.ndarray) -> np.ndarray:
    """H3 — root of a track = node with the largest sum of intra-track out-edge
    similarities; sort+reverse on (score, node_idx) (solve.cc:552-582)."""
    N = g.n_nodes
    src = edge_sources(g)
    dst = g.edges["dst"].astype(np.int64)
    intra = track[src] == track[dst]
    # double accumulation in out-edge insertion order (np.bincount adds sequentially)
    score = np.bincount(src[intra], weights=g.edges["sim"][intra].astype(np.float64), minlength=N)
    order = np.lexsort((np.arange(N), score))[::-1]
    _, first = np.unique(track[order], return_index=True)
    is_root = np.zeros(N, dtype=np.uint8)
    is_root[order[first]] = 1
    return is_root


# ---------------------------------------------------------------------------
# H4 — meta-graph partition
# ---------------------------------------------------------------------------
def _connected_components(n: int, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Labels in order of the lowest member index (= the BFS order of
    solve.cc:291-300: components are numbered by their first meta-node)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    mat = coo_matrix((np.ones(a.shape[0], dtype=np.int8), (a, b)), shape=(n, n))
    _, lab = connected_components(mat, directed=False)
    _, first = np.unique(lab, return_index=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(order.shape[0])
    return rank[lab].astype(np.int64)


def two_way_cut(nodes: List[int], adj: Dict[int, Dict[int, int]]) -> Dict[int, int]:
    """Deterministic stand-in for colmap::ComputeNormalizedMinGraphCut(edges,
    weights, 2) (solve.cc:192) — like the COLMAP call a function of the edge list and the integer
    edge weights only; balance is on volume (weighted degree).  Same definition as
    csrc/lfr_cut.h (the two are tested to agree).  `nodes` all have >= 1 edge inside `adj`.
    Returns node -> {0, 1} with both sides non-empty (when len(nodes) >= 2)."""
    nodes = sorted(nodes)
    vol = {x: sum(adj[x].values()) for x in nodes}
    # connected pieces of this sub-graph
    seen = set()
    pieces = []
    for s in nodes:
        if s in seen:
            continue
        comp = [s]
        seen.add(s)
        head = 0
        while head < len(comp):
            u = comp[head]
            head += 1
            for v in sorted(adj[u]):
                if v not in seen:
                    seen.add(v)
                    comp.append(v)
        pieces.append(comp)
    if len(pieces) > 1:
        # free cut: balance the pieces over the two sides, heaviest first
        pieces.sort(key=lambda c: (-sum(vol[x] for x in c), c[0]))
        w = [0, 0]
        out = {}
        for c in pieces:
            side = 0 if w[0] <= w[1] else 1
            w[side] += sum(vol[x] for x in c)
            for x in c:
                out[x] = side
        return out
    # one connected piece: grow side 0 breadth-first from a pseudo-peripheral
    # node until it holds half the volume.
    def bfs_last(start):
        order = [start]
        mark = {start}
        head = 0
        while head < len(order):
            u = order[head]
            head += 1
            for v in sorted(adj[u]):
                if v not in mark:
                    mark.add(v)
                    order.append(v)
        return order
    start = bfs_last(nodes[0])[-1]
    order = bfs_last(start)
    total = sum(vol[x] for x in nodes)
    out = {}
    acc = 0
    for i, x in enumerate(order):
        if i > 0 and (acc * 2 >= total or i == len(order) - 1):
            break
        out[x] = 0
        acc += vol[x]
    for x in order:
        out.setdefault(x, 1)
    # one refinement sweep: move a node across if that lowers the cut and keeps both sides non-empty
    cnt = [sum(1 for x in out.values() if x == 0), sum(1 for x in out.values() if x == 1)]
    for x in order:
        s = out[x]
        if cnt[s] <= 1:
            continue
        inside = sum(w for v, w in adj[x].items() if out[v] == s)
        outside = sum(w for v, w in adj[x].items() if out[v] != s)
        if outside > inside:
            out[x] = 1 - s
            cnt[s] -= 1
            cnt[1 - s] += 1
    return out


def recursive_cut(edge_a, edge_b, edge_w, node_weight, max_weight) -> List[List[int]]:
    """recursive_graph_cut (solve.cc:185-250) as a work list: split until every
    group weighs <= max_weight or has no internal edge (then its nodes become
    singleton groups, solve.cc:240-246).  Returns the groups."""
    groups: List[List[int]] = []
    work = [list(zip(edge_a, edge_b, edge_w))]
    while work:
        edges = work.pop()
        adj: Dict[int, Dict[int, int]] = {}
        for a, b, w in edges:
            adj.setdefault(a, {})[b] = adj.setdefault(a, {}).get(b, 0) + w
            adj.setdefault(b, {})[a] = adj.setdefault(b, {}).get(a, 0) + w
        nodes = list(adj.keys())
        side = two_way_cut(nodes, adj)
        for s in (0, 1):
            members = sorted(x for x in nodes if side[x] == s)
            if not members:
                continue
            if sum(node_weight[x] for x in members) <= max_weight:
                groups.append(members)            # solve.cc:205-211
                continue
            mset = set(members)
            sub = [(a, b, w) for a, b, w in edges if a in mset and b in mset]
            if sub:
                covered = set()
                for a, b, _ in sub:
                    covered.add(a)
                    covered.add(b)
                work.append(sub)
                for x in members:                  # no edge left inside the subset
                    if x not in covered:
                        groups.append([x])
            else:
                for x in members:
                    groups.append([x])
    return groups


def separate_meta_graph(g: MatchGraph, track: np.ndarray, max_nodes: int,
                        stats: Optional[dict] = None) -> np.ndarray:
    """H4 — solve.cc:252-373.  Returns component_idx[N]."""
    N = g.n_nodes
    T = int(track.max()) + 1 if N else 0
    nodes_in_track = np.bincount(track, minlength=T)
    src = edge_sources(g)
    dst = g.edges["dst"].astype(np.int64)
    ts, tt = track[src], track[dst]
    inter = ts != tt
    key = ts[inter] * T + tt[inter]
    ukey, inv = np.unique(key, return_inverse=True)
    # meta_edges[ts][tt] += sim in node / out-edge order (solve.cc:270-289)
    wsum = np.bincount(inv, weights=g.edges["sim"][inter].astype(np.float64), minlength=ukey.shape[0])
    ma, mb = ukey // T, ukey % T
    cc = _connected_components(T, ma, mb)
    n_cc = int(cc.max()) + 1 if T else 0
    cc_nodes = np.bincount(cc, weights=nodes_in_track, minlength=n_cc).astype(np.int64)
    gc = cc.copy()                 # gc_component_idx_container: start from the CC label
    next_label = n_cc
    big = np.nonzero(cc_nodes > max_nodes)[0]
    n_cut_groups = 0
    if big.shape[0]:
        und = ma < mb              # undirected edge list, weight int(100 * sum sim) (solve.cc:327-330)
        ua, ub = ma[und], mb[und]
        uw = (100.0 * wsum[und]).astype(np.int64)
        ucc = cc[ua]
        nw = nodes_in_track.tolist()
        for c in big.tolist():
            sel = ucc == c
            groups = recursive_cut(ua[sel].tolist(), ub[sel].tolist(), uw[sel].tolist(), nw, max_nodes)
            for grp in groups:
                gc[np.array(grp, dtype=np.int64)] = next_label
                next_label += 1
            n_cut_groups += len(groups)
    # keep meta-edges inside one cut group, re-split into connected components (solve.cc:345-364)
    keep = gc[ma] == gc[mb]
    final = _connected_components(T, ma[keep], mb[keep])
    if stats is not None:
        stats["n_meta_components"] = n_cc
        stats["n_oversized_meta_components"] = int(big.shape[0])
        stats["n_cut_groups"] = n_cut_groups
    return final[track]


@dataclass
class Problem:
    """The arrays of `lfr_problem` (include/lfr.h) + the bookkeeping needed to
    write the SolutionFile."""
    graph: MatchGraph
    track: np.ndarray       # [N] uint32
    comp: np.ndarray        # [N] uint32
    is_root: np.ndarray     # [N] uint8
    comp_ptr: np.ndarray    # [C+1] uint32, dispatch order (largest first)
    comp_nodes: np.ndarray  # [N] uint32
    comp_order: np.ndarray  # [C] component id of each dispatch slot
    info: dict = field(default_factory=dict)

    @property
    def n_components(self) -> int:
        return int(self.comp_ptr.shape[0] - 1)


class HostInput(C.Structure):
    """lfr_host_input (include/lfr_host.h)"""
    _fields_ = [("n_pairs", C.c_uint64), ("n_matches", C.c_uint64), ("n_images", C.c_uint32),
                ("pair_img1", C.c_void_p), ("pair_img2", C.c_void_p), ("pair_skip", C.c_void_p),
                ("pair_ptr", C.c_void_p), ("feat1", C.c_void_p), ("feat2", C.c_void_p), ("sim", C.c_void_p),
                ("disp1", C.c_void_p), ("disp2", C.c_void_p), ("edges_out", C.c_void_p),
                ("edges_out_capacity", C.c_uint64)]


class HostSizes(C.Structure):
    """lfr_host_sizes (include/lfr_host.h)"""
    _fields_ = [("n_nodes", C.c_uint32), ("n_tracks", C.c_uint32), ("n_components", C.c_uint32),
                ("n_images_seen", C.c_uint32), ("max_track_size", C.c_uint32), ("max_component_size", C.c_uint32),
                ("n_meta_components", C.c_uint32), ("n_oversized_meta_components", C.c_uint32),
                ("n_cut_groups", C.c_uint32), ("reserved", C.c_uint32), ("n_edges", C.c_uint64),
                ("tracks_ms", C.c_double), ("graph_cut_ms", C.c_double), ("graph_ms", C.c_double),
                ("dispatch_ms", C.c_double)]


def host_input_arrays(ms: MatchSet, banned_images=()):
    """The flat arrays of lfr_host_input for `ms`: (pair_skip, dict of contiguous arrays by field name)."""
    banned = set(banned_images)
    skip = np.array([(ms.image_names[a] in banned) or (ms.image_names[b] in banned)
                     for a, b in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist())], dtype=np.uint8) \
        if banned else np.zeros(ms.n_pairs, dtype=np.uint8)
    arrs = dict(
        pair_img1=np.ascontiguousarray(ms.pair_img1, dtype=np.uint32), pair_img2=np.ascontiguousarray(ms.pair_img2, dtype=np.uint32),
        pair_skip=skip, pair_ptr=np.ascontiguousarray(ms.pair_ptr, dtype=np.uint64),
        feat1=np.ascontiguousarray(ms.feat1, dtype=np.uint32), feat2=np.ascontiguousarray(ms.feat2, dtype=np.uint32),
        sim=np.ascontiguousarray(ms.sim, dtype=np.float32), disp1=np.ascontiguousarray(ms.disp1, dtype=np.float32),
        disp2=np.ascontiguousarray(ms.disp2, dtype=np.float32))
    return skip, arrs


HOST_SIZES_FIELDS = ("n_nodes", "n_tracks", "n_components", "n_images_seen", "max_track_size", "max_component_size",
                     "n_meta_components", "n_oversized_meta_components", "n_cut_groups", "n_edges",
                     "tracks_ms", "graph_cut_ms", "graph_ms", "dispatch_ms")


def stage_outputs(n_nodes: int, n_components: int, n_edges: int) -> dict:
    """Empty output arrays of lfr_host_stage_export / lfr_plan_export_graph, in argument order."""
    N, Cn = n_nodes, n_components
    return dict(row_ptr=np.zeros(N + 1, np.uint32), edges=np.empty(n_edges, EDGE_DTYPE), track=np.empty(N, np.uint32),
                comp=np.empty(N, np.uint32), is_root=np.empty(N, np.uint8), comp_ptr=np.zeros(Cn + 1, np.uint32),
                comp_nodes=np.empty(N, np.uint32), comp_order=np.empty(Cn, np.uint32),
                node_image=np.empty(N, np.uint32), node_feat=np.empty(N, np.uint32))


def host_stage_export(arrs: dict, n_images: int):
    """The native host stage on the flat lfr_host_input arrays `arrs` (host_input_arrays), run as the
    native drop-in runs it: the edge records are written in place into the output array (edges_out).
    Returns (rc, arrays as stage_outputs, lfr_host_sizes as a dict); arrays and sizes are None when rc != 0."""
    from .capi import load_host
    L = load_host()
    L.lfr_host_stage_create.argtypes = [C.POINTER(HostInput), C.POINTER(C.c_void_p), C.POINTER(HostSizes)]
    L.lfr_host_stage_create.restype = C.c_int
    L.lfr_host_stage_export.argtypes = [C.c_void_p] * 11
    L.lfr_host_stage_export.restype = C.c_int
    L.lfr_host_stage_destroy.argtypes = [C.c_void_p]
    L.lfr_host_stage_destroy.restype = None
    ptr, skip = arrs["pair_ptr"].astype(np.int64), arrs["pair_skip"]
    counts = np.maximum(ptr[1:] - ptr[:-1], 0)
    e_cap = 2 * int(counts[skip == 0].sum()) if skip.size else 0
    edges = np.empty(e_cap, EDGE_DTYPE)
    inp = HostInput(n_pairs=arrs["pair_img1"].shape[0], n_matches=arrs["feat1"].shape[0], n_images=n_images,
                    edges_out=(edges.ctypes.data if e_cap else None), edges_out_capacity=e_cap,
                    **{k: (v.ctypes.data if v.size else None) for k, v in arrs.items()})
    h, sz = C.c_void_p(), HostSizes()
    rc = L.lfr_host_stage_create(C.byref(inp), C.byref(h), C.byref(sz))
    if rc != 0:
        return rc, None, None
    try:
        out = stage_outputs(int(sz.n_nodes), int(sz.n_components), 0)
        out["edges"] = edges
        rc = L.lfr_host_stage_export(h, *[(a.ctypes.data if a.size else None) for a in out.values()])
    finally:
        L.lfr_host_stage_destroy(h)
    if rc != 0:
        return rc, None, None
    return 0, out, {k: getattr(sz, k) for k in HOST_SIZES_FIELDS}


def build_problem_native(ms: MatchSet, banned_images=(), log=None) -> Problem:
    """solve.cc:405-606 through the native host stage (csrc/lfr_host.cc, include/lfr_host.h)."""
    from .capi import load_host

    L = load_host()
    L.lfr_host_stage_create.argtypes = [C.POINTER(HostInput), C.POINTER(C.c_void_p), C.POINTER(HostSizes)]
    L.lfr_host_stage_create.restype = C.c_int
    L.lfr_host_stage_export.argtypes = [C.c_void_p] * 11
    L.lfr_host_stage_export.restype = C.c_int
    L.lfr_host_stage_destroy.argtypes = [C.c_void_p]
    L.lfr_host_stage_destroy.restype = None
    say = log if log is not None else (lambda s: None)
    skip, arrs = host_input_arrays(ms, banned_images)
    # the edge records (80 B each) are written straight into the array handed to lfr_solve
    counts = (arrs["pair_ptr"][1:] - arrs["pair_ptr"][:-1]).astype(np.int64)
    e_cap = 2 * int(counts[skip == 0].sum()) if ms.n_pairs else 0
    edges = np.empty(e_cap, EDGE_DTYPE)
    inp = HostInput(n_pairs=ms.n_pairs, n_matches=ms.n_matches, n_images=len(ms.image_names),
                    edges_out=(edges.ctypes.data if e_cap else None), edges_out_capacity=e_cap,
                    **{k: (v.ctypes.data if v.size else None) for k, v in arrs.items()})
    h = C.c_void_p()
    sz = HostSizes()
    rc = L.lfr_host_stage_create(C.byref(inp), C.byref(h), C.byref(sz))
    if rc != 0:
        raise RuntimeError("lfr_host_stage_create failed (%d)" % rc)
    try:
        N, E, Cn = int(sz.n_nodes), int(sz.n_edges), int(sz.n_components)
        # np.empty: every array is overwritten by the export (the edge records alone are 80 B x E)
        assert E == e_cap
        row_ptr = np.empty(N + 1, np.uint32)
        track = np.empty(N, np.uint32); comp = np.empty(N, np.uint32); is_root = np.empty(N, np.uint8)
        comp_ptr = np.empty(Cn + 1, np.uint32); comp_nodes = np.empty(N, np.uint32); comp_order = np.empty(Cn, np.uint32)
        node_image = np.empty(N, np.uint32); node_feat = np.empty(N, np.uint32)
        if N == 0:
            row_ptr[:] = 0
            comp_ptr[:] = 0
        outs = [row_ptr, edges, track, comp, is_root, comp_ptr, comp_nodes, comp_order, node_image, node_feat]
        rc = L.lfr_host_stage_export(h, *[(a.ctypes.data if a.size else None) for a in outs])
        if rc != 0:
            raise RuntimeError("lfr_host_stage_export failed (%d)" % rc)
    finally:
        L.lfr_host_stage_destroy(h)
    image_fact: Dict[int, float] = {}
    for a, b, fa, fb, sk in zip(ms.pair_img1.tolist(), ms.pair_img2.tolist(), ms.pair_fact1.tolist(),
                                ms.pair_fact2.tolist(), skip.tolist()):
        if sk:
            continue
        image_fact.setdefault(a, fa)
        image_fact.setdefault(b, fb)
    g = MatchGraph(n_nodes=N, node_image=node_image.astype(np.int64), node_feat=node_feat,
                   und_sim=np.zeros(0), und_n1=np.zeros(0, np.int64), und_n2=np.zeros(0, np.int64),
                   row_ptr=row_ptr, edges=edges, image_names=ms.image_names, image_fact=image_fact,
                   n_images=int(sz.n_images_seen))
    say("# graph nodes: %d" % N)
    say("# graph edges: %d" % E)
    info: dict = {}
    if N == 0:
        z32 = np.zeros(0, dtype=np.uint32)
        return Problem(g, z32, z32, np.zeros(0, np.uint8), np.zeros(1, np.uint32), z32, z32, info)
    say("# tracks: %d" % sz.n_tracks)
    say("max track size: %d" % sz.max_track_size)
    say("Graph-cut time: %dms" % int(sz.graph_cut_ms))
    say("# components: %d" % Cn)
    say("max component size: %d" % sz.max_component_size)
    info.update(n_tracks=int(sz.n_tracks), n_components=Cn, max_component_size=int(sz.max_component_size),
                tracks_ms=float(sz.tracks_ms), graph_cut_ms=float(sz.graph_cut_ms), graph_ms=float(sz.graph_ms),
                dispatch_ms=float(sz.dispatch_ms),
                n_meta_components=int(sz.n_meta_components),
                n_oversized_meta_components=int(sz.n_oversized_meta_components), n_cut_groups=int(sz.n_cut_groups),
                host_stage="native")
    return Problem(graph=g, track=track, comp=comp, is_root=is_root, comp_ptr=comp_ptr, comp_nodes=comp_nodes,
                   comp_order=comp_order.astype(np.int64), info=info)


def build_problem(ms: MatchSet, banned_images=(), log=None, native: Optional[bool] = None) -> Problem:
    """solve.cc:405-606 end to end.  Uses the native host stage (csrc/lfr_host.cc)
    unless native=False or LFR_HOST_PYTHON=1 selects the numpy implementation below
    (the two are tested to agree exactly)."""
    import os
    import time
    if native is None:
        native = not os.environ.get("LFR_HOST_PYTHON")
    if native:
        return build_problem_native(ms, banned_images, log)
    g = build_graph(ms, banned_images)
    say = log if log is not None else (lambda s: None)
    say("# graph nodes: %d" % g.n_nodes)                       # solve.cc:484
    say("# graph edges: %d" % (2 * g.und_n1.shape[0]))         # solve.cc:485
    info: dict = {}
    if g.n_nodes == 0:
        z32 = np.zeros(0, dtype=np.uint32)
        return Problem(g, z32, z32, np.zeros(0, np.uint8), np.zeros(1, np.uint32), z32, z32, info)
    t0 = time.perf_counter()
    track = compute_tracks(g)
    n_tracks = int(track.max()) + 1
    say("# tracks: %d" % n_tracks)                             # solve.cc:534
    say("max track size: %d" % int(np.bincount(track).max()))  # solve.cc:549
    is_root = select_roots(g, track)
    t1 = time.perf_counter()
    comp = separate_meta_graph(g, track, g.n_images, info)
    t2 = time.perf_counter()
    say("Graph-cut time: %dms" % int((t2 - t1) * 1e3))         # solve.cc:589
    n_comp = int(comp.max()) + 1
    say("# components: %d" % n_comp)                           # solve.cc:591
    # nodes_in_component ascending node index; dispatch order = sort+reverse on (size, idx)
    sizes = np.bincount(comp, minlength=n_comp)
    comp_order = np.lexsort((np.arange(n_comp), sizes))[::-1]
    say("max component size: %d" % int(sizes[comp_order[0]]))  # solve.cc:606
    slot_of_comp = np.empty(n_comp, dtype=np.int64)
    slot_of_comp[comp_order] = np.arange(n_comp)
    node_slot = slot_of_comp[comp]
    comp_nodes = np.argsort(node_slot, kind="stable").astype(np.uint32)
    comp_ptr = np.zeros(n_comp + 1, dtype=np.uint32)
    np.cumsum(sizes[comp_order], out=comp_ptr[1:])
    info.update(n_tracks=n_tracks, n_components=n_comp, max_component_size=int(sizes[comp_order[0]]),
                tracks_ms=(t1 - t0) * 1e3, graph_cut_ms=(t2 - t1) * 1e3, host_stage="numpy")
    return Problem(
        graph=g, track=track.astype(np.uint32), comp=comp.astype(np.uint32), is_root=is_root,
        comp_ptr=comp_ptr, comp_nodes=comp_nodes, comp_order=comp_order.astype(np.int64), info=info,
    )


def refined_track_count(p: Problem) -> int:
    """Tracks with >= 1 node in a solved (size > 1) component — the unit of the
    tracks-refined/s metric (SURVEY 8d)."""
    if p.graph.n_nodes == 0:
        return 0
    sizes = np.bincount(p.comp.astype(np.int64))
    solved_node = sizes[p.comp.astype(np.int64)] > 1
    return int(np.unique(p.track[solved_node]).shape[0])
