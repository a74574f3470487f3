"""The recursive 2-way cut of oversized meta-components on the device (csrc/lfr_cut.cuh) against the host
cut (csrc/lfr_cut.h, its numpy twin graph.py::recursive_cut): the same groups, group for group.

The CPU tests run a numpy model of the device algorithm — all sub-problems of a recursion level at once,
the BFS order rebuilt level by level from claims (lowest frontier position wins, neighbours ascending),
pieces dealt after a sort on (volume desc, piece asc), side 0 grown to the first order prefix holding half
the volume, then the refinement sweep walked in order as one warp walks it — against graph.py.
The GPU tests run lfr_debug_recursive_cut (exported, not in the headers) on hand-built edge lists, and
the whole graph stage with the device cut (LFR_DBG_DEVICE_CUT) against the host stage.
"""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.capi import DBG_DEVICE_CUT, Plan
from lfr_b200.graph import host_stage_export, recursive_cut, two_way_cut
from test_native_exe import PRODUCT, product_exe  # noqa: F401  (fixture)

INT_MAX = 2 ** 31 - 1
CUT_EDGE = np.dtype([("a", "<u4"), ("b", "<u4"), ("w", "<i8")])
LFR_EINVAL = -1


def host_groups(a, b, w, node_weight, max_weight):
    """graph.py::recursive_cut as group_of[x] = the lowest node of x's group (x for an untouched node)."""
    n = len(node_weight)
    out = np.arange(n, dtype=np.int64)
    if len(a):
        for g in recursive_cut([int(x) for x in a], [int(x) for x in b], [int(x) for x in w], list(node_weight), max_weight):
            out[g] = min(g)
    return out


# ---------------------------------------------------------------------------------------------------
# CPU: the device algorithm in numpy
# ---------------------------------------------------------------------------------------------------
def _adjacency(edges):
    """Merged parallel edges, neighbours ascending (the level's sort by (node, neighbour) + reduce)."""
    adj = {}
    for a, b, w in edges:
        for x, y in ((a, b), (b, a)):
            adj.setdefault(x, {})
            adj[x][y] = adj[x].get(y, 0) + w
    return {x: sorted(r.items()) for x, r in adj.items()}


def _level_bfs(adj, start, visited, order):
    """block_bfs: per frontier, every node claims its unvisited neighbours (lowest frontier position wins),
    then each frontier node appends the neighbours it won, ascending, at its scanned offset."""
    head = len(order)
    order.append(start)
    visited.add(start)
    tail = len(order)
    while head < tail:
        claim = {}
        for p in range(head, tail):
            for v, _ in adj[order[p]]:
                if v not in visited:
                    claim[v] = min(claim.get(v, p), p)
        won = [[v for v, _ in adj[order[p]] if v not in visited and claim[v] == p] for p in range(head, tail)]
        for lst in won:
            order.extend(lst)
        visited.update(order[tail:])
        head, tail = tail, len(order)


def _model_two_way_cut(edges):
    adj = _adjacency(edges)
    nodes = sorted(adj)
    n = len(nodes)
    vol = {x: sum(w for _, w in adj[x]) for x in nodes}
    if n == 2:
        return {nodes[0]: 0, nodes[1]: 1}
    visited, order, starts = set(), [], [0]
    _level_bfs(adj, nodes[0], visited, order)
    if len(order) < n:
        for s in nodes:
            if s not in visited:
                starts.append(len(order))
                _level_bfs(adj, s, visited, order)
        bounds = starts + [n]
        pv = [sum(vol[x] for x in order[bounds[j]:bounds[j + 1]]) for j in range(len(starts))]
        keys = sorted(range(len(starts)), key=lambda j: (-pv[j], j))   # the bitonic sort's order
        w, pside = [0, 0], {}
        for j in keys:
            s = 0 if w[0] <= w[1] else 1
            w[s] += pv[j]
            pside[j] = s
        return {x: pside[j] for j in range(len(starts)) for x in order[bounds[j]:bounds[j + 1]]}
    start = order[-1]
    order = []
    _level_bfs(adj, start, set(), order)
    total = sum(vol.values())
    prefix = np.cumsum([vol[x] for x in order[:-1]])
    hit = np.nonzero(prefix * 2 >= total)[0]
    cut = int(hit[0]) + 1 if len(hit) else n - 1
    side = {x: (0 if q < cut else 1) for q, x in enumerate(order)}
    cnt = [cut, n - cut]
    for x in order:                                                    # the warp's walk
        s = side[x]
        if cnt[s] <= 1:
            continue
        inside = sum(w for v, w in adj[x] if side[v] == s)
        if sum(w for v, w in adj[x]) - inside > inside:
            side[x] = 1 - s
            cnt[s] -= 1
            cnt[1 - s] += 1
    return side


def model_groups(a, b, w, node_weight, max_weight):
    """recursive_cut_on_device: one level at a time, every sub-problem of the level cut independently."""
    n = len(node_weight)
    out = np.arange(n, dtype=np.int64)
    level = [list(zip(map(int, a), map(int, b), map(int, w)))] if len(a) else []
    while level:
        nxt = []
        for edges in level:
            side = _model_two_way_cut(edges)
            for s in (0, 1):
                members = sorted(x for x in side if side[x] == s)
                if not members:
                    continue
                if len(side) == 2 or sum(node_weight[x] for x in members) <= max_weight:
                    out[members] = members[0]
                    continue
                sub = [e for e in edges if side[e[0]] == s and side[e[1]] == s]
                if sub:
                    nxt.append(sub)
        level = nxt
    return out


def random_graph(rng, n, m, kind, wmax=50):
    if kind == "random":
        a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    elif kind == "pieces":           # several pieces of equal volume: the dealing ties
        k = 6
        a = rng.integers(0, max(n // k, 1), m) * k + np.arange(m) % k
        b = rng.integers(0, max(n // k, 1), m) * k + np.arange(m) % k
    elif kind == "path":
        a = np.arange(n - 1)
        b = a + 1
    elif kind == "cycle":
        a = np.arange(n)
        b = (a + 1) % n
    elif kind == "star":
        a = np.zeros(n - 1, np.int64)
        b = np.arange(1, n)
    else:                            # "grid": long BFS orders, many sweep moves
        s = int(np.sqrt(n))
        idx = np.arange(s * s).reshape(s, s)
        a = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
        b = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    keep = a != b
    a, b = a[keep], b[keep]
    w = rng.integers(1, wmax, len(a)) if kind != "pieces" else np.full(len(a), 7)
    return a.astype(np.uint32), b.astype(np.uint32), w.astype(np.int64)


@pytest.mark.parametrize("kind", ["random", "pieces", "path", "cycle", "star", "grid"])
def test_level_model_equals_the_host_cut(kind):
    rng = np.random.default_rng(zlib.crc32(kind.encode()))
    for trial in range(4):
        n = 60 + 40 * trial
        a, b, w = random_graph(rng, n, 3 * n, kind)
        nw = rng.integers(1, 4, n)
        for max_weight in (3, 10, int(nw.sum()) // 3):
            want = host_groups(a, b, w, nw, max_weight)
            assert np.array_equal(model_groups(a, b, w, nw, max_weight), want), (trial, max_weight)


def test_level_bfs_is_the_queue_order():
    """The claim rule reproduces the queue BFS of graph.py::two_way_cut on random graphs."""
    rng = np.random.default_rng(7)
    for _ in range(20):
        a, b, w = random_graph(rng, 80, 200, "random")
        adj = _adjacency(zip(a.tolist(), b.tolist(), w.tolist()))
        start = min(adj)
        got = []
        _level_bfs(adj, start, set(), got)
        want, seen, head = [start], {start}, 0
        while head < len(want):
            for v, _ in adj[want[head]]:
                if v not in seen:
                    seen.add(v)
                    want.append(v)
            head += 1
        assert got == want


def test_host_two_way_cut_agrees_with_the_model_side_for_side():
    rng = np.random.default_rng(11)
    for kind in ("random", "path", "grid", "star"):
        a, b, w = random_graph(rng, 100, 300, kind)
        edges = list(zip(a.tolist(), b.tolist(), w.tolist()))
        adj = {}
        for x, y, ww in edges:
            adj.setdefault(x, {})[y] = adj.setdefault(x, {}).get(y, 0) + ww
            adj.setdefault(y, {})[x] = adj.setdefault(y, {}).get(x, 0) + ww
        want = two_way_cut(list(adj), adj)
        got = _model_two_way_cut(edges)
        if len(adj) == 2:
            continue
        assert got == want, kind


# ---------------------------------------------------------------------------------------------------
# GPU: lfr_debug_recursive_cut against the host cut
# ---------------------------------------------------------------------------------------------------
def device_groups(b200, a, b, w, node_weight, max_weight):
    f = b200.lib.lfr_debug_recursive_cut
    f.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
    f.restype = C.c_int
    e = np.zeros(len(a), CUT_EDGE)
    e["a"], e["b"], e["w"] = a, b, w
    nw = np.ascontiguousarray(node_weight, np.uint32)
    out = np.zeros(len(nw), np.uint32)
    rc = f(e.ctypes.data, len(e), nw.ctypes.data, len(nw), max_weight, out.ctypes.data)
    return rc, out.astype(np.int64)


def check(b200, a, b, w, nw, max_weight):
    a, b, w = np.asarray(a, np.uint32), np.asarray(b, np.uint32), np.asarray(w, np.int64)
    want = host_groups(a, b, w, nw, max_weight)
    rc, got = device_groups(b200, a, b, w, nw, max_weight)
    assert rc == 0
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "pieces", "path", "cycle", "star", "grid"])
def test_device_cut_equals_host_cut(b200, kind):
    rng = np.random.default_rng(zlib.crc32(("dev/" + kind).encode()))
    for n in (3, 17, 300, 2000):
        a, b, w = random_graph(rng, n, 3 * n, kind)
        if not len(a):
            continue
        nw = rng.integers(1, 4, n)
        for max_weight in (1, 4, 25, int(nw.sum()) - 1):
            check(b200, a, b, w, nw, max_weight)


@pytest.mark.gpu
def test_device_cut_edge_cases(b200):
    # two-node sub-problems with parallel and duplicate edges, in both directions
    check(b200, [0, 1, 0, 0], [1, 0, 1, 1], [5, 7, 0, 3], [5, 5], 1)
    # paths: the half-volume stop at the last node; cycles: the pseudo-peripheral restart
    for n in (3, 4, 5, 9):
        check(b200, np.arange(n - 1), np.arange(1, n), np.ones(n - 1), np.ones(n), 1)
        check(b200, np.arange(n), (np.arange(n) + 1) % n, np.arange(n) + 1, np.ones(n), 2)
    # a star: one side must never be emptied by the sweep
    check(b200, np.zeros(40), np.arange(1, 41), np.full(40, 9), np.ones(41), 3)
    # zero and saturated weights (a sub-problem whose pieces all have zero volume is never split, on the host
    # either: all-zero weights stop after the first cut here)
    rng = np.random.default_rng(3)
    a, b, _ = random_graph(rng, 200, 600, "random")
    check(b200, a, b, np.zeros(len(a)), np.ones(200), 199)
    for w in (np.full(len(a), INT_MAX), rng.choice([1, INT_MAX], len(a))):
        check(b200, a, b, w, np.ones(200), 7)
    # max_weight reached exactly: a side of weight == max_weight is a group
    check(b200, [0, 1, 2, 3], [1, 2, 3, 0], [1, 1, 1, 1], [1, 1, 1, 1], 2)
    check(b200, [0, 1, 2, 3], [1, 2, 3, 0], [1, 1, 1, 1], [1, 1, 1, 1], 1)
    # a sweep that moves many nodes: a grid with heavy weights across the BFS levels
    a, b, w = random_graph(rng, 1600, 0, "grid", wmax=1000)
    check(b200, a, b, w, np.ones(1600), 5)
    # pieces whose next start lies more than a CTA's width past the last one: two 1000-node paths, then
    # 50 two-node pieces
    pa = np.concatenate([np.arange(999), 1000 + np.arange(999), 2000 + 2 * np.arange(50)])
    pb = np.concatenate([np.arange(1, 1000), 1001 + np.arange(999), 2001 + 2 * np.arange(50)])
    check(b200, pa, pb, np.ones(len(pa)), np.ones(2100), 500)
    # untouched nodes keep their own id; bad edges are refused
    got = check(b200, [2, 3], [3, 4], [1, 1], np.ones(8), 1)
    assert got[[0, 1, 5, 6, 7]].tolist() == [0, 1, 5, 6, 7]
    assert device_groups(b200, np.array([1]), np.array([1]), np.array([1]), np.ones(3), 1)[0] == LFR_EINVAL
    # two pieces of zero volume both go to side 0 and are cut again forever by lfr_cut.h: refused instead
    assert device_groups(b200, np.array([0, 2]), np.array([1, 3]), np.array([0, 0]), np.ones(4), 1)[0] == LFR_EINVAL
    # two pieces dealt one per side, every edge kept: progress, not a refusal
    check(b200, [0, 0, 2, 2], [1, 1, 3, 3], [4, 1, 2, 3], [1, 1, 1, 1], 1)
    assert device_groups(b200, np.array([0]), np.array([3]), np.array([1]), np.ones(3), 1)[0] == LFR_EINVAL


@pytest.mark.gpu
def test_device_cut_larger_than_shared_memory(b200):
    """One sub-problem of 50 K nodes and 150 K edges: its per-node arrays alone are several times a CTA's
    shared memory, so they live in global memory."""
    rng = np.random.default_rng(5)
    a, b, w = random_graph(rng, 50000, 150000, "random")
    check(b200, a, b, w, np.ones(50000), 2000)


# ---------------------------------------------------------------------------------------------------
# GPU: the whole graph stage with the device cut
# ---------------------------------------------------------------------------------------------------
def assert_stage_with_device_cut(b200, arrs, n_images):
    """lfr_plan_create_from_matches with LFR_DBG_DEVICE_CUT against lfr_host_stage_export: every exported
    array and every count, n_cut_groups included."""
    from test_gpu_graph_stage import ARRAYS, COUNTS
    rc, a, sa = host_stage_export(arrs, n_images)
    assert rc == 0
    plan = Plan.from_matches(b200, arrs, options=b200.default_options(debug_flags=DBG_DEVICE_CUT), n_images=n_images)
    b, sb = plan.export_graph(), plan.sizes
    plan.close()
    for k in ARRAYS:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert a[k].tobytes() == b[k].tobytes(), k
    for k in COUNTS:
        assert sa[k] == sb[k], (k, sa[k], sb[k])
    return sa


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["cfg2", "cfg4", "cfg5"])
def test_stage_with_device_cut_equals_host_stage(b200, cfg):
    from test_gpu_graph_stage import _arrs
    ms = synth.generate(cfg)
    sizes = assert_stage_with_device_cut(b200, _arrs(ms), len(ms.image_names))
    assert sizes["n_oversized_meta_components"] > 0 and sizes["n_cut_groups"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["giant_meta", "saturating_cut", "balanced_unions_64", "balanced_unions_256"])
def test_stage_with_device_cut_on_adversarial_cuts(b200, case):
    from test_graph_stage_adversarial import case_arrays
    arrs, n = case_arrays(case)
    sizes = assert_stage_with_device_cut(b200, arrs, n)
    if case in ("giant_meta", "saturating_cut"):  # the balanced unions stop just at the size limit: nothing to cut
        assert sizes["n_oversized_meta_components"] > 0 and sizes["n_cut_groups"] > 0


@pytest.mark.gpu
def test_drop_in_with_device_cut_reproduces_giant_meta(product_exe, tmp_path):  # noqa: F811
    """The native drop-in on giant_meta (one oversized meta-component), device route with LFR_DEVICE_CUT=1:
    the same stdout lines and bytes as its host route, and the reference's committed SolutionFile."""
    from test_drop_in_device_stage import solution_close
    from test_graph_stage_adversarial import make_case, solution_path
    from test_ref_solve import untimed
    m = tmp_path / "m.pb"
    m.write_bytes(wire.encode_matching_file(make_case("giant_meta")))
    out = {}
    for route, env in (("host", dict(LFR_GRAPH_STAGE="host")), ("device", dict(LFR_GRAPH_STAGE="device", LFR_DEVICE_CUT="1"))):
        o = tmp_path / (route + ".pb")
        r = subprocess.run([PRODUCT, "--matches_file", str(m), "--output_file", str(o)], capture_output=True, text=True,
                           env=dict(os.environ, **env))
        assert r.returncode == 0, r.stderr
        out[route] = (untimed(r.stdout), o.read_bytes())
    assert out["device"] == out["host"]
    assert solution_close(out["device"][1], open(solution_path("giant_meta"), "rb").read())
