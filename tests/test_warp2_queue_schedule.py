"""The register warp tier's queue launches as the host schedule lays them out (lfr_debug_time_schedule
with LFR_SCHED_DUMP: host-only, no device involved): which scenes get a queue, how many launches, how
many warps per SM, and the LFR_DBG_WARP2_WARPS_SHIFT override.

The helpers below are shared with tests/test_gpu_warp2_queue.py: `warp2_layout_bytes` states the
`RegLayout` of lfr_solve_warp2.cuh at 32 threads in Python, `with_need` builds a component whose own layout is an
exact byte count, and `schedule_of` reads the dump of any problem."""
import ctypes as C
import re

import numpy as np
import pytest

from lfr_b200.capi import DBG_TILE_FROM_SHIFT, DBG_WARP2_WARPS_SHIFT
from test_gpu_cta_limits import internal_out_degree, merge, promote_to_roots, sizes_of, slot_nodes, subset

SMEM = 227 * 1024      # kMaxSmemPerBlock (lfr_capi.cu)
MAX_WARPS = 8          # kWarp2QueueMaxWarps (lfr_solve_warp2.cuh)


def cap_of(w):
    """The queue's first-launch slot cap at `w` warps per SM (build_schedule)."""
    return (SMEM // w) & ~15


def warp2_layout_bytes(e, nc, n2):
    """Shared-memory bytes of one warp2 slot laid out for `e` candidate out-edges, `nc` nodes and `n2`
    unknowns: `RegLayout(e, nc, n2, 32).total`, field by field."""
    def up16(o):
        return (o + 15) // 16 * 16
    ldh = n2 | 1
    o = 80 * e + 16                       # staged records, mbarrier
    o += 16 * nc + 16 * nc                # x, xc
    o += 3 * 8 * n2 + 8 * n2 * ldh        # g, S, dl, H
    o += 8 * 7 * e + 8 * 5 * e            # scr, tup
    o = up16(o)
    o += 8 * 2 * 72                       # prow
    o += 4 * e + 4 * e                    # eidx, meta
    o += 4 * nc + 4 * nc + 4 * (nc + 1) + 4 * 2 * nc   # node, rowstart, candptr, cnt
    o += 2 * e + 2 * (nc + 1) + 2 * nc + 2 * (n2 // 2 + 1)   # twin, outptr, freeof, lof
    return up16(o)


def host_dims(p, s):
    """The host's layout sizes of dispatch slot `s`: candidate out-edges (row_ptr sum, at least 1), nodes,
    and unknowns (2 x non-root nodes, at least 2)."""
    nodes = slot_nodes(p, s)
    rp = p.graph.row_ptr.astype(np.int64)
    return max(1, int((rp[nodes + 1] - rp[nodes]).sum())), len(nodes), max(2, 2 * int((p.is_root[nodes] == 0).sum()))


def need_of(p, s):
    return warp2_layout_bytes(*host_dims(p, s))


def schedule_of(b200, capfd, monkeypatch, p, dbg=0):
    """(launches, queue launches [(n, slot, warps)], per-bucket launches [dict]) of `p` as the host lays
    them out with debug flags `dbg`."""
    f = b200.lib.lfr_debug_time_schedule
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    s, keep = b200.marshal(p)
    o = b200.default_options(debug_flags=dbg)
    monkeypatch.setenv("LFR_SCHED_DUMP", "1")
    capfd.readouterr()
    us, nl, dg = C.c_double(), C.c_int(), C.c_uint64()
    assert f(C.byref(s), C.byref(o), 1, C.byref(us), C.byref(nl), C.byref(dg)) == 0
    err = capfd.readouterr().err
    queues = [(int(n), int(slot), int(w)) for n, slot, w in
              re.findall(r"warp2 queue\s+n\s+(\d+)\s+slot\s+(\d+)\s+warps/SM (\d+)", err)]
    keys = ("variant", "n", "emax", "ncmax", "n2max", "smem", "warps")
    buckets = [dict(zip(keys, map(int, m))) for m in re.findall(
        r"bucket variant\s+(\d+)\s+n\s+(\d+)\s+emax\s+(\d+)\s+ncmax\s+(\d+)\s+n2max\s+(\d+)\s+smem/warp\s+(\d+)\s+warps (\d+)", err)]
    # every launch has its line: the buckets, the queue launches and the CTA tier's size classes
    assert nl.value == len(buckets) + len(queues) + len(re.findall(r"^cta group ", err, re.M)), err
    return nl.value, queues, buckets


def schedule(b200, capfd, monkeypatch, name, warps=0):
    from lfr_b200 import build_problem, synth
    n, queues, buckets = schedule_of(b200, capfd, monkeypatch, build_problem(synth.generate(name)),
                                     warps << DBG_WARP2_WARPS_SHIFT)
    return n, queues, [b["variant"] for b in buckets]


def expected_queues(needs, n2s, w):
    """The queue launches build_schedule makes of four-warp register-tier members with layouts `needs`
    and unknowns `n2s` at `w` warps per SM (None: no member above 16 unknowns, no queue)."""
    if max(n2s) <= 16:
        return []
    out = []
    for first in (True, False):
        m = [b for b in needs if (b <= cap_of(w)) == first]
        if m:
            out.append((len(m), max(m), w if first else min(w, SMEM // max(m))))
    return out


# ---------------------------------------------------------------------------------------------------
# constructed components (shared with the GPU tests)
# ---------------------------------------------------------------------------------------------------
def with_need(p, target, n2, seed=0, avoid=()):
    """A one-slot problem made of whole components of `p` (merge, none of the slots `avoid`) with `n2`
    unknowns (promote_to_roots) whose own layout is exactly `target` bytes, and the slots it merged.
    A seeded greedy fill, then an exhaustive last pair."""
    sizes = sizes_of(p)
    avoid = set(avoid)
    pool = [s for s in range(p.n_components) if sizes[s] >= 2 and s not in avoid]
    dims = {s: host_dims(p, s)[:2] for s in pool}
    rng = np.random.default_rng(seed)
    for attempt in range(200):
        order = [pool[i] for i in rng.permutation(len(pool))]
        picked, e, nc = [], 0, 0
        for s in order:
            de, dn = dims[s]
            if warp2_layout_bytes(e + de, nc + dn, n2) > target - 6000:
                continue
            picked.append(s)
            e, nc = e + de, nc + dn
            if warp2_layout_bytes(e, nc, n2) > target - 14000:
                break
        rest = [s for s in order if s not in picked][:400]
        by_sum = {}
        for i, a in enumerate(rest):
            by_sum.setdefault(dims[a], [a])
            for b in rest[i + 1:]:
                by_sum.setdefault((dims[a][0] + dims[b][0], dims[a][1] + dims[b][1]), [a, b])
        for (de, dn), extra in sorted(by_sum.items()):
            if warp2_layout_bytes(e + de, nc + dn, n2) == target:
                q = merge(p, picked + extra)
                nodes = slot_nodes(q, 0)
                if (internal_out_degree(q, nodes) > 0).sum() < n2 // 2:
                    continue
                q = promote_to_roots(q, 0, n2 // 2, list(range(n2 // 2)), seed=seed)
                assert need_of(q, 0) == target
                return q, picked + extra
    raise AssertionError("no component of %d bytes with %d unknowns" % (target, n2))


def combine(parts):
    """One problem holding the dispatch slots of several problems over the same graph (each slot's
    is_root / comp / track taken from the problem it comes from; the slots must be disjoint)."""
    q = subset(parts[0], [])
    q.is_root, q.comp, q.track = parts[0].is_root.copy(), parts[0].comp.copy(), parts[0].track.copy()
    lists, order = [], []
    for r in parts:
        for s in range(r.n_components):
            nodes = slot_nodes(r, s)
            q.is_root[nodes], q.comp[nodes], q.track[nodes] = r.is_root[nodes], r.comp[nodes], r.track[nodes]
            lists.append(nodes)
            order.append(int(np.asarray(r.comp_order)[s]))
    allnodes = np.concatenate(lists)
    assert len(np.unique(allnodes)) == len(allnodes), "overlapping slots"
    q.comp_ptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint32)
    q.comp_nodes = allnodes.astype(np.uint32)
    q.comp_order = np.asarray(order)
    return q


def cap_boundary_problem(p, w, every=97):
    """Slot 0 exactly at the cap of `w` warps (18 unknowns), slot 1 16 bytes past it (24 unknowns), then
    every `every`-th component of `p` of at least two nodes that neither of them merged."""
    at, used = with_need(p, cap_of(w), 18, seed=w)
    past, used2 = with_need(p, cap_of(w) + 16, 24, seed=w + 100, avoid=used)
    used = set(used) | set(used2)
    sizes = sizes_of(p)
    small = [s for s in range(0, p.n_components, every) if s not in used and sizes[s] >= 2]
    return combine([at, past, subset(p, small)])


@pytest.fixture(scope="module")
def cfg2():
    from conftest import get_problem
    return get_problem("cfg2")[1]


@pytest.fixture(scope="module")
def cfg4s():
    """cfg4 at a tenth of its keypoints: 199 queue members, two queue launches at 8 warps per SM."""
    from conftest import get_problem
    return get_problem("cfg4", 0.1)[1]


@pytest.fixture(scope="module")
def cfg5s():
    """cfg5 at a twentieth of its keypoints: CTA-tier components in three size classes."""
    from conftest import get_problem
    return get_problem("cfg5", 0.05)[1]


# ---------------------------------------------------------------------------------------------------
# the existing scene-level checks
# ---------------------------------------------------------------------------------------------------
def test_cfg2_is_one_queue_launch(b200, capfd, monkeypatch):
    n, queues, buckets = schedule(b200, capfd, monkeypatch, "cfg2")
    assert n == 1 and buckets == []
    assert len(queues) == 1 and queues[0][0] == 4218 and queues[0][2] == 8


def test_members_past_the_slot_go_to_a_second_queue(b200, capfd, monkeypatch):
    """cfg4: the members whose own slot does not fit 8 to an SM form a second queue at fewer warps;
    at 4 warps per SM every member fits one slot and one queue takes them all."""
    n8, q8, b8 = schedule(b200, capfd, monkeypatch, "cfg4")
    n4, q4, b4 = schedule(b200, capfd, monkeypatch, "cfg4", warps=4)
    assert len(q8) == 2 and q8[0][2] == 8 and 4 <= q8[1][2] < 8
    assert q8[0][1] <= 227 * 1024 // 8 < q8[1][1] and q8[1][1] * q8[1][2] <= 227 * 1024
    assert len(q4) == 1 and q4[0][2] == 4 and q4[0][0] == q8[0][0] + q8[1][0]
    assert b4 == b8 and n8 == n4 + 1


@pytest.mark.parametrize("warps", [1, 6, 8, 12, 15])
def test_warps_override_is_clamped_to_the_kernel(b200, capfd, monkeypatch, warps):
    n, queues, _ = schedule(b200, capfd, monkeypatch, "cfg2", warps)
    assert n == 1 and queues[0][2] == min(warps, 8)


def test_scenes_without_wide_members_keep_the_bucket_launches(b200, capfd, monkeypatch):
    """cfg3 (no register-tier component above 16 unknowns): the 12-warp per-bucket kernels stay."""
    n, queues, buckets = schedule(b200, capfd, monkeypatch, "cfg3")
    assert queues == [] and buckets and set(buckets) <= {8, 16} and n == len(buckets)


# ---------------------------------------------------------------------------------------------------
# the layout formula, the slot cap, the "wide" rule and the order
# ---------------------------------------------------------------------------------------------------
def _shape_grid(p):
    """One-slot problems over a grid of (e, nc, n2): cfg4 x 0.1 components of 2 to 38 nodes, each
    as it is and with 1, 4, 8, 9, 12 and 16 free nodes."""
    sizes = sizes_of(p)
    out = []
    for target in (2, 3, 5, 8, 12, 17, 23, 30, 38):
        s = int(np.argmin(np.abs(sizes - target) + 1000 * (sizes < 2)))
        q = subset(p, [s])
        if host_dims(q, 0)[2] <= 32:   # (above: the tile tier)
            out.append(q)
        nodes = slot_nodes(q, 0)
        n_cand = int((internal_out_degree(q, nodes) > 0).sum())
        for k in (1, 4, 8, 9, 12, 16):
            if k <= n_cand:
                out.append(promote_to_roots(q, 0, k, list(range(len(nodes) - k, len(nodes))), seed=k))
    return out


def test_layout_formula_matches_the_schedule(b200, capfd, monkeypatch, cfg4s):
    """warp2_layout_bytes is RegLayout at 32 threads: a one-component problem's slot (queue) or smem/warp (four-warp
    bucket) is the layout of its own sizes; a few components share the maximum of theirs (queue) or
    the layout of their maxima (bucket).  Every layout is a multiple of 16 bytes."""
    shapes = _shape_grid(cfg4s)
    seen = set()
    for q in shapes:
        e, nc, n2 = host_dims(q, 0)
        seen.add((nc, n2))
        _, queues, buckets = schedule_of(b200, capfd, monkeypatch, q)
        want = warp2_layout_bytes(e, nc, n2)
        assert want % 16 == 0
        four = 4 * want <= SMEM
        if n2 > 16 and four:
            assert queues == [(1, want, 8 if want <= cap_of(8) else min(8, SMEM // want))] and buckets == [], (e, nc, n2)
        else:   # a four-warp bucket, or a single-warp one for a slot that does not fit four to an SM
            assert queues == [] and len(buckets) == 1, (e, nc, n2)
            b = buckets[0]
            assert (b["emax"], b["ncmax"], b["n2max"], b["smem"], b["warps"]) == (e, nc, n2, want, 4 if four else 1), b
    assert len(seen) >= 30 and {n2 for _, n2 in seen} >= {2, 8, 16, 18, 24, 32}
    # a few components at once: three slots of cfg4 x 0.1 with 8, 12 and 20 unknowns
    sizes = sizes_of(cfg4s)
    trio = [int(np.nonzero(sizes == k)[0][0]) for k in (6, 12, 24)]
    parts = []
    for i, (s, k) in enumerate(zip(trio, (4, 6, 10))):
        r = promote_to_roots(subset(cfg4s, [s]), 0, k, list(range(k)), seed=i)
        parts.append(r)
    q = combine(parts)
    dims = [host_dims(q, s) for s in range(3)]
    _, queues, buckets = schedule_of(b200, capfd, monkeypatch, q)
    assert buckets == [] and queues == expected_queues([warp2_layout_bytes(*d) for d in dims], [d[2] for d in dims], 8)
    # without the 20-unknown member: per-bucket launches sized by the maxima of their members
    q2 = subset(q, [0, 1])
    _, queues, buckets = schedule_of(b200, capfd, monkeypatch, q2)
    assert queues == []
    for b in buckets:
        mem = [d for d in dims[:2] if (d[2] <= 8) == (b["variant"] == 8)]
        mx = [max(d[i] for d in mem) for i in range(3)]
        assert (b["emax"], b["ncmax"], b["n2max"], b["smem"]) == (*mx, warp2_layout_bytes(*mx))


@pytest.mark.parametrize("w", [8, 5, 6])
def test_slot_cap_boundary(b200, capfd, monkeypatch, cfg2, w):
    """Members whose own layout is exactly the cap (227 KB / W, rounded down to 16 bytes) go to the first
    queue launch at W warps; 16 bytes more go to the second, at min(W, 227 KB // slot) warps.  The
    boundary members are built at those exact byte counts, with 18 and 24 unknowns, next to a few
    ordinary cfg2 members."""
    q = cap_boundary_problem(cfg2, w)
    cap = cap_of(w)
    needs = [need_of(q, s) for s in range(q.n_components)]
    assert needs[0] == cap and needs[1] == cap + 16 and max(needs[2:]) <= cap
    n, queues, buckets = schedule_of(b200, capfd, monkeypatch, q, w << DBG_WARP2_WARPS_SHIFT)
    assert buckets == [] and n == 2
    assert queues == [(q.n_components - 1, cap, w), (1, cap + 16, min(w, SMEM // (cap + 16)))]
    # the second launch runs fewer warps than W wherever W slots of cap + 16 bytes do not fit an SM
    assert queues[1][2] < w and queues[1][1] * queues[1][2] <= SMEM
    # every layout is a multiple of 16, so the rounding of the cap moves no member between launches
    assert cap + 16 > SMEM // w
    # without the member past the cap: one launch
    n, queues, _ = schedule_of(b200, capfd, monkeypatch, subset(q, [0] + list(range(2, q.n_components))),
                               w << DBG_WARP2_WARPS_SHIFT)
    assert n == 1 and queues == [(q.n_components - 1, cap, w)]


def test_one_wide_member_moves_the_four_warp_buckets_into_the_queue(b200, capfd, monkeypatch, cfg2):
    """The queue exists only where some four-warp register member has more than 16 unknowns: cfg2's
    members of at most 16 unknowns run the per-bucket kernels alone, and all of them join the queue
    next to one member of 18 unknowns.  TILE_FROM = 16 moves cfg2's wider members to the tile kernel,
    which leaves no queue launch."""
    n2 = np.array([host_dims(cfg2, s)[2] for s in range(cfg2.n_components)])
    narrow = [int(s) for s in np.nonzero((n2 <= 16) & (sizes_of(cfg2) >= 2))[0][::8]]
    wide = int(np.nonzero(n2 == 18)[0][0])
    n, queues, buckets = schedule_of(b200, capfd, monkeypatch, subset(cfg2, narrow))
    assert queues == [] and buckets and n == len(buckets)
    assert all(b["variant"] in (8, 16) and b["warps"] == 4 for b in buckets)
    assert sum(b["n"] for b in buckets) == len(narrow)
    q = subset(cfg2, narrow + [wide])
    n, queues, buckets = schedule_of(b200, capfd, monkeypatch, q)
    assert buckets == [] and n == 1
    assert queues == expected_queues([need_of(q, s) for s in range(q.n_components)], n2[narrow + [wide]].tolist(), 8)
    assert queues[0][0] == len(narrow) + 1
    n, queues, buckets = schedule_of(b200, capfd, monkeypatch, cfg2, 16 << DBG_TILE_FROM_SHIFT)
    assert queues == [] and n == len(buckets)
    assert {b["variant"] for b in buckets} >= {8, 16, 132}
    assert sum(b["n"] for b in buckets if b["variant"] in (8, 16)) == int(((n2 <= 16) & (sizes_of(cfg2) >= 2)).sum())


@pytest.mark.parametrize("scene", ["cfg2", "cfg4s", "cfg5s"])
def test_dispatch_order_does_not_change_the_groups(b200, capfd, monkeypatch, request, scene):
    """The ABI takes comp_ptr in any order: reversed, ascending-size and random dispatch orders give the
    same queue launches (n, slot, warps) as the largest-first order, at 8, 5 and 1 warps per SM.
    cfg5 x 0.05 also has the CTA tier: one launch for each of its three size classes."""
    p = request.getfixturevalue(scene)
    sizes = sizes_of(p)
    orders = {"reversed": list(range(p.n_components))[::-1],
              "ascending": np.argsort(sizes, kind="stable").tolist(),
              "random": np.random.default_rng(7).permutation(p.n_components).tolist()}
    for w in (8, 5, 1):
        dbg = w << DBG_WARP2_WARPS_SHIFT
        ref = schedule_of(b200, capfd, monkeypatch, p, dbg)
        assert ref[1]
        assert ref[0] - len(ref[1]) - len(ref[2]) == (3 if scene == "cfg5s" else 0)   # the CTA groups
        for name, order in orders.items():
            got = schedule_of(b200, capfd, monkeypatch, subset(p, order), dbg)
            assert got[0] == ref[0] and got[1] == ref[1], (name, w)
            assert sorted(map(sorted, (b.items() for b in got[2]))) == sorted(map(sorted, (b.items() for b in ref[2])))
