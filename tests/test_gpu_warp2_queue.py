"""The warp-register tier's queue kernel (solve_warp2_queue_kernel, csrc/lfr_solve_warp2.cuh) on the GPU.

One persistent launch of W warps per SM takes components from one device ticket counter and solves
them in turn, each in the same shared-memory slot laid out from the component's own sizes, on the NREG
path its packed dims word names.  Results must not depend on any of that: every width (W = 1..8), any
dispatch order, the per-bucket kernels, re-entry, concurrent plans and every solve route give the same
bits, and constructed components at the NREG class and slot-cap boundaries agree with the CPU oracle.

Two bars:
  * bitwise: positions, per-component iterations / termination / initial and final cost, and the
    totals, compared as bytes (per-component stats through the permutation where the order changes);
  * parity: test_gpu_parity._compare's bar against the oracle (1e-4 px, identical iterations and
    termination codes, costs to 1e-10 / 1e-8), per component as test_gpu_cta_limits.assert_agree states it.
"""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import get_problem
from lfr_b200.capi import DBG_PROFILE, DBG_TILE_FROM_SHIFT, DBG_WARP2_WARPS_SHIFT, DBG_ZERO_COPY, Plan
from test_gpu_cta_limits import (assert_agree, assert_bitwise, internal_out_degree, merge, numpy_cost,
                                 promote_to_roots, sizes_of, slot_nodes, subset)
from test_warp2_queue_schedule import (MAX_WARPS, cap_boundary_problem, cap_of, combine, host_dims, need_of,
                                       schedule_of)

pytestmark = pytest.mark.gpu

TIER_WARP2 = 1   # LmProfile::kWarp2 (csrc/lfr_lm.cuh)


def wflags(w):
    return w << DBG_WARP2_WARPS_SHIFT


def solve(b200, p, dbg=0):
    return b200.solve(p, b200.default_options(debug_flags=dbg))


def assert_same(a, b, what, perm=None):
    """Bitwise bar.  With `perm`, `b` solved subset(p_a, perm): b's slot k is a's slot perm[k]."""
    (pa, sa), (pb, sb) = a, b
    if perm is None:
        assert_bitwise(a, b, what)
    else:
        assert np.array_equal(pa, pb), (what, float(np.abs(pa - pb).max()))
        for k in ("iterations", "termination", "initial_cost", "final_cost"):
            assert np.array_equal(np.asarray(sa[k])[perm], sb[k]), (what, k)
    for k in ("total_iterations", "total_line_search_steps", "n_solved"):
        assert sa[k] == sb[k], (what, k, sa[k], sb[k])


def oracle_solve(oracle, p):
    return oracle.solve(p, oracle.default_options(n_threads=min(8, os.cpu_count() or 8)))


def nreg_class(n2):
    return 8 if n2 <= 8 else (16 if n2 <= 16 else (24 if n2 <= 24 else 32))


@pytest.fixture(scope="module")
def cfg2():
    return get_problem("cfg2")[1]


@pytest.fixture(scope="module")
def cfg4s():
    """cfg4 at a tenth of its keypoints: two queue launches at W = 5, 6 and 8."""
    return get_problem("cfg4", 0.1)[1]


@pytest.fixture(scope="module")
def ring60():
    return get_problem("ring60")[1]


# ---------------------------------------------------------------------------------------------------
# 1. widths
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["cfg2", "cfg4s", "ring60"])
def test_every_width_is_bitwise_the_default(b200, oracle, capfd, monkeypatch, request, scene):
    """W = 1..8 warps per SM (each warp solves up to C / n_SMs components in sequence at W = 1): bitwise
    the default solve, which agrees with the oracle."""
    p = request.getfixturevalue(scene)
    default = solve(b200, p)
    assert_agree(p, *default, *oracle_solve(oracle, p))
    log = []
    for w in range(1, MAX_WARPS + 1):
        assert_same(default, solve(b200, p, wflags(w)), "%s W=%d" % (scene, w))
        _, queues, _ = schedule_of(b200, capfd, monkeypatch, p, wflags(w))
        assert queues and queues[0][2] == w
        log.append("W=%d %s" % (w, queues))
    with capfd.disabled():
        print("\n%s queue launches (n, slot, warps): %s" % (scene, "; ".join(log)))


# ---------------------------------------------------------------------------------------------------
# 2. the queue against the per-bucket kernels
# ---------------------------------------------------------------------------------------------------
def test_queue_is_bitwise_the_per_bucket_kernels(b200, capfd, monkeypatch, cfg2):
    """cfg2 runs every component in the queue; with TILE_FROM = 16 its components of at most 16 unknowns
    run the 12-warp per-bucket kernels instead (the wider ones go to the tile kernel).  Those components
    are bitwise equal between the two runs.  Likewise a cfg2 subset of such components alone (per-bucket
    launches) and next to one member of 18 unknowns (one queue launch)."""
    n2 = np.array([host_dims(cfg2, s)[2] for s in range(cfg2.n_components)])
    narrow = (n2 <= 16) & (sizes_of(cfg2) >= 2)
    _, q_def, b_def = schedule_of(b200, capfd, monkeypatch, cfg2)
    _, q_tf, b_tf = schedule_of(b200, capfd, monkeypatch, cfg2, 16 << DBG_TILE_FROM_SHIFT)
    assert len(q_def) == 1 and b_def == [] and q_tf == []
    assert sum(b["n"] for b in b_tf if b["variant"] in (8, 16) and b["warps"] == 4) == int(narrow.sum())
    (pa, sa), (pb, sb) = solve(b200, cfg2), solve(b200, cfg2, 16 << DBG_TILE_FROM_SHIFT)
    nodes = np.concatenate([slot_nodes(cfg2, s) for s in np.nonzero(narrow)[0]])
    assert np.array_equal(pa[nodes], pb[nodes])
    for k in ("iterations", "termination", "initial_cost", "final_cost"):
        assert np.array_equal(sa[k][narrow], sb[k][narrow]), k

    few = [int(s) for s in np.nonzero(narrow)[0][::8]]
    wide = int(np.nonzero(n2 == 18)[0][0])
    alone, with_wide = subset(cfg2, few), subset(cfg2, few + [wide])
    _, q1, b1 = schedule_of(b200, capfd, monkeypatch, alone)
    _, q2, b2 = schedule_of(b200, capfd, monkeypatch, with_wide)
    assert q1 == [] and sum(b["n"] for b in b1) == len(few) and b2 == [] and q2[0][0] == len(few) + 1
    (pa, sa), (pb, sb) = solve(b200, alone), solve(b200, with_wide)
    nodes = np.concatenate([slot_nodes(alone, s) for s in range(len(few))])
    assert np.array_equal(pa[nodes], pb[nodes])
    for k in ("iterations", "termination", "initial_cost", "final_cost"):
        assert np.array_equal(sa[k], sb[k][:len(few)]), k
    with capfd.disabled():
        print("\ncfg2: queue %s vs TILE_FROM=16 buckets %s; subset of %d: buckets %s vs queue %s" % (
            q_def, [(b["variant"], b["n"], b["warps"]) for b in b_tf], len(few),
            [(b["variant"], b["n"], b["warps"]) for b in b1], q2))


# ---------------------------------------------------------------------------------------------------
# 3. slot reuse across layouts: dispatch orders
# ---------------------------------------------------------------------------------------------------
def interleaved(p):
    """Slots taken round-robin from the NREG classes in the order 8, 32, 16, 24 (other tiers last)."""
    by = {c: [] for c in (8, 32, 16, 24, 0)}
    for s in range(p.n_components):
        n2 = host_dims(p, s)[2]
        by[nreg_class(n2) if n2 <= 32 else 0].append(s)
    out = []
    while any(by[c] for c in (8, 32, 16, 24)):
        for c in (8, 32, 16, 24):
            if by[c]:
                out.append(by[c].pop(0))
    return out + by[0]


@pytest.mark.parametrize("scene", ["cfg2", "cfg4s"])
def test_dispatch_orders_are_bitwise_the_canonical_order(b200, capfd, monkeypatch, request, scene):
    """Classes interleaved (8, 32, 16, 24, ...), ascending size and random orders, each at W = 1 (a warp
    goes through ~C / n_SMs components of changing layouts and NREG paths in one slot) and at W = 8:
    every component bitwise its result in the canonical, largest-first order."""
    p = request.getfixturevalue(scene)
    if scene == "cfg2":
        p = subset(p, list(range(0, p.n_components, 3)))
    ref = solve(b200, p)
    orders = {"interleaved": interleaved(p), "ascending": np.argsort(sizes_of(p), kind="stable").tolist(),
              "random": np.random.default_rng(11).permutation(p.n_components).tolist()}
    log = []
    for name, order in orders.items():
        assert sorted(order) == list(range(p.n_components))
        q = subset(p, order)
        for w in (1, 8):
            assert_same(ref, solve(b200, q, wflags(w)), "%s %s W=%d" % (scene, name, w), perm=order)
            log.append("%s W=%d %s" % (name, w, schedule_of(b200, capfd, monkeypatch, q, wflags(w))[1]))
    with capfd.disabled():
        print("\n%s (%d components): %s" % (scene, p.n_components, "; ".join(log)))


# ---------------------------------------------------------------------------------------------------
# 4. class and slot boundaries against the oracle
# ---------------------------------------------------------------------------------------------------
def classes_problem(p):
    """One component of `p` per unknown count 2, 8, 10, 16, 18, 24, 26, 32 (promote_to_roots on the
    smallest component with enough candidates that fits a four-warp slot)."""
    parts, used = [], set()
    sizes = sizes_of(p)
    for n2 in (2, 8, 10, 16, 18, 24, 26, 32):
        for s in np.argsort(sizes, kind="stable"):
            s = int(s)
            if s in used or sizes[s] < max(2, n2 // 2):
                continue
            q = subset(p, [s])
            nodes = slot_nodes(q, 0)
            if (internal_out_degree(q, nodes) > 0).sum() < n2 // 2:
                continue
            q = promote_to_roots(q, 0, n2 // 2, list(range(len(nodes) - n2 // 2, len(nodes))), seed=n2)
            if 4 * need_of(q, 0) > 227 * 1024:
                continue
            parts.append(q)
            used.add(s)
            break
    assert [host_dims(r, 0)[2] for r in parts] == [2, 8, 10, 16, 18, 24, 26, 32]
    return combine(parts)


def root_heavy_problem(p):
    """Two components of 140 nodes each, merged from two-node components of `p` (the ones with the fewest
    candidate edges, dealt alternately), all roots but 1 and 4 nodes; and one of 18 unknowns (two
    eight-node components merged) that keeps them in the queue."""
    sizes = sizes_of(p)
    two = sorted((int(s) for s in np.nonzero(sizes == 2)[0]), key=lambda s: host_dims(p, s)[0])
    heavy = [promote_to_roots(merge(p, two[i:140:2]), 0, k, list(range(0, 2 * k, 2)), seed=k)
             for i, k in ((0, 1), (1, 4))]
    big = [int(s) for s in np.nonzero(sizes == 8)[0]][:2]
    wide = promote_to_roots(merge(p, big), 0, 9, list(range(9)), seed=9)
    return combine(heavy + [wide])


def unkept_node_problem(p):
    """Components whose host bound on unknowns is above the device's free count: a node of another
    component (own track, made non-root) is moved into a component of 4 and one of 8 free nodes.  None
    of its edges is kept (they end in its old component, on other tracks), so the device does not
    number it and the NREG path (16, 24) is wider than the device's 8 / 16 unknowns.  One ordinary
    component of 20 unknowns keeps the others in the queue."""
    sizes = sizes_of(p)
    mid = [int(s) for s in np.nonzero((sizes >= 12) & (sizes <= 16))[0]]
    a, b, c = mid[:3]
    donors = [int(s) for s in np.nonzero((sizes >= 3) & (sizes <= 10))[0]][:2]
    q = subset(p, [a, b, c] + donors)
    for s, k in ((0, 4), (1, 8), (2, 10)):
        q = promote_to_roots(q, s, k, list(range(k)), seed=k)
    q.is_root, q.comp, q.track = q.is_root.copy(), p.comp.copy(), p.track.copy()
    lists = [slot_nodes(q, s) for s in range(q.n_components)]
    fresh = int(p.track.max()) + 1
    for i, d in enumerate((3, 4)):
        v = lists[d][-1]
        lists[d] = lists[d][:-1]
        q.comp[v] = q.comp[lists[i][0]]
        q.track[v] = fresh + i
        q.is_root[v] = 0
        lists[i] = np.append(lists[i], v)
    q.comp_ptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint32)
    q.comp_nodes = np.concatenate(lists).astype(np.uint32)
    return q


def check_against_oracle(b200, oracle, capfd, monkeypatch, p, name, widths=(8,)):
    """Parity with the oracle at each width (bitwise across widths), warp2 in every profile record of a
    component with a free node, every register-tier member in a queue launch, and the costs equal to
    numpy_cost at the start and returned positions."""
    pos_o, st_o = oracle_solve(oracle, p)
    first = None
    log = []
    for w in widths:
        got = solve(b200, p, wflags(w))
        assert_agree(p, *got, pos_o, st_o)
        if first is None:
            first = got
        assert_same(first, got, "%s W=%d" % (name, w))
        n, queues, buckets = schedule_of(b200, capfd, monkeypatch, p, wflags(w))
        assert buckets == [] and sum(q[0] for q in queues) == got[1]["n_solved"] == n_solved_of(p), (queues, buckets)
        log.append("W=%d %s" % (w, queues))
        plan = Plan(b200, p, b200.default_options(debug_flags=DBG_PROFILE | wflags(w)))
        try:
            plan.solve()
            prof = plan.download()
            rec, _ = plan.profile()
        finally:
            plan.close()
        assert_same(got, prof, "%s profiled W=%d" % (name, w))
    pos, st = first
    zero = np.zeros_like(pos)
    for s in range(p.n_components):
        if sizes_of(p)[s] < 2:
            continue
        assert rec["tier"][s] in (TIER_WARP2, 0), (name, s, rec["tier"][s])
        for k, x in (("initial_cost", zero), ("final_cost", pos)):
            c = numpy_cost(p, s, x)
            assert abs(c - st[k][s]) <= 1e-12 * max(1.0, abs(c)), (name, s, k, c, st[k][s])
    assert (rec["tier"] == TIER_WARP2).sum() >= 1
    classes = sorted({nreg_class(host_dims(p, s)[2]) for s in range(p.n_components) if sizes_of(p)[s] >= 2})
    with capfd.disabled():
        print("\n%s: %d components, NREG classes %s, host n2 %s; %s" % (
            name, p.n_components, classes, sorted({host_dims(p, s)[2] for s in range(p.n_components)}), "; ".join(log)))
    return first


def n_solved_of(p):
    return int((sizes_of(p) >= 2).sum())


def test_nreg_classes_match_oracle(b200, oracle, capfd, monkeypatch, cfg4s):
    """n2 = 2, 8, 10, 16, 18, 24, 26, 32 in one scene: every NREG path, both sides of each class border."""
    q = classes_problem(cfg4s)
    check_against_oracle(b200, oracle, capfd, monkeypatch, q, "classes", widths=(8, 1, 3))


def test_root_heavy_components_match_oracle(b200, oracle, capfd, monkeypatch):
    """140 nodes in one component with 2 and with 8 unknowns (kept edges only where a free node is an
    end), in the queue next to one member of 18 unknowns."""
    q = root_heavy_problem(get_problem("cfg3")[1])
    dims = [host_dims(q, s) for s in range(3)]
    assert dims[0][1] == dims[1][1] == 140 and (dims[0][2], dims[1][2], dims[2][2]) == (2, 8, 18), dims
    check_against_oracle(b200, oracle, capfd, monkeypatch, q, "root-heavy %s" % dims, widths=(8, 1))


@pytest.mark.parametrize("w", [8, 5, 6])
def test_slot_cap_members_match_oracle(b200, oracle, capfd, monkeypatch, cfg2, w):
    """A member exactly at the cap of W warps (first launch) and one 16 bytes past it (second launch, at
    min(W, 227 KB // slot) warps), with cfg2 members around them."""
    q = cap_boundary_problem(cfg2, w, every=37)
    assert need_of(q, 0) == cap_of(w) and need_of(q, 1) == cap_of(w) + 16
    _, queues, _ = schedule_of(b200, capfd, monkeypatch, q, wflags(w))
    assert len(queues) == 2 and queues[0][1] == cap_of(w) and queues[1] == (1, cap_of(w) + 16, min(w, 227 * 1024 // (cap_of(w) + 16)))
    check_against_oracle(b200, oracle, capfd, monkeypatch, q, "cap W=%d" % w, widths=(w, 8, 1))


def test_host_bound_above_device_free_count_matches_oracle(b200, oracle, capfd, monkeypatch, cfg4s):
    """A non-root node with no kept edge: counted by the host (NREG 16 / 24 path), not by the device."""
    q = unkept_node_problem(cfg4s)
    assert [host_dims(q, s)[2] for s in range(2)] == [10, 18]
    check_against_oracle(b200, oracle, capfd, monkeypatch, q, "unkept node", widths=(8, 1))


# ---------------------------------------------------------------------------------------------------
# 5. re-entry and concurrency
# ---------------------------------------------------------------------------------------------------
def plan_solve(b200, p, dbg=0, times=1):
    plan = Plan(b200, p, b200.default_options(debug_flags=dbg))
    try:
        for _ in range(times):
            plan.solve()
        out = plan.download()
        n = plan.num_launches()
    finally:
        plan.close()
    return out, n


def test_plan_solved_back_to_back_and_launch_counts(b200, capfd, monkeypatch, cfg2, cfg4s):
    """One plan solved three times with no download between (the ticket reset by the last warp of each
    launch) is bitwise its first solve; lfr_stats.n_kernel_launches = Plan.num_launches() = the dump's.
    cfg5 x 0.05 adds the CTA tier, one launch per size class."""
    for name, p in (("cfg4s", cfg4s), ("cfg2", cfg2), ("cfg5s", get_problem("cfg5", 0.05)[1])):
        plan = Plan(b200, p)
        try:
            plan.solve()
            first = plan.download()
            for _ in range(3):
                plan.solve()
            assert_same(first, plan.download(), name + " x3")
            plan.solve()
            assert_same(first, plan.download(), name + " again")
            n_plan = plan.num_launches()
        finally:
            plan.close()
        n_dump, queues, _ = schedule_of(b200, capfd, monkeypatch, p)
        assert first[1]["n_kernel_launches"] == n_plan == n_dump, (name, first[1]["n_kernel_launches"], n_plan, n_dump)
        _, st = solve(b200, p)
        assert st["n_kernel_launches"] == n_plan
        with capfd.disabled():
            print("\n%s: %d launches, queues %s" % (name, n_plan, queues))


def test_two_plans_on_two_streams(b200, cfg2, cfg4s):
    """A cfg4 plan (two queue launches) and a cfg2 plan (one) solved at the same time on two torch
    streams, interleaved three times: each bitwise its solo solve."""
    import torch
    solo4, _ = plan_solve(b200, cfg4s)
    solo2, _ = plan_solve(b200, cfg2)
    p4, p2 = Plan(b200, cfg4s), Plan(b200, cfg2)
    s4, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        for _ in range(3):
            p4.solve(s4.cuda_stream)
            p2.solve(s2.cuda_stream)
        assert_same(solo4, p4.download(s4.cuda_stream), "cfg4 concurrent")
        assert_same(solo2, p2.download(s2.cuda_stream), "cfg2 concurrent")
    finally:
        torch.cuda.synchronize()
        p4.close()
        p2.close()


def test_solve_workspace_across_scenes(b200, cfg2, cfg4s):
    """lfr_solve's cached plan goes cfg4 (two queue launches) -> cfg3 (none) -> cfg2 (one) -> cfg4: each
    bitwise a fresh plan's solve."""
    cfg3 = get_problem("cfg3")[1]
    for name, p in (("cfg4s", cfg4s), ("cfg3", cfg3), ("cfg2", cfg2), ("cfg4s again", cfg4s)):
        fresh, _ = plan_solve(b200, p)
        assert_same(fresh, solve(b200, p), name)


# ---------------------------------------------------------------------------------------------------
# 6. routes
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w", [1, 8])
def test_routes_are_bitwise_the_plan_solve(b200, capfd, monkeypatch, cfg4s, w):
    """At W warps: lfr_solve from page-locked buffers with DBG_ZERO_COPY (paced zero-copy pulls under the
    queue's dispatch), the pinned lfr_solve_multi on [0] and a DBG_PROFILE plan are bitwise the plan."""
    import torch
    p = cfg4s
    ref, _ = plan_solve(b200, p, wflags(w))
    # zero-copy lfr_solve
    s, keep = b200.marshal(p)
    e_pin = torch.empty(keep["edges"].nbytes, dtype=torch.uint8).pin_memory()
    e_pin.numpy()[:] = keep["edges"].view(np.uint8).reshape(-1)
    s.edges = e_pin.data_ptr()
    N = p.graph.n_nodes
    pos_pin = torch.zeros(2 * N, dtype=torch.float64).pin_memory()
    st, bufs = b200.make_stats(p.n_components)
    o = b200.default_options(debug_flags=DBG_ZERO_COPY | wflags(w))
    b200.check(b200.lib.lfr_solve(C.byref(s), C.byref(o), C.c_void_p(pos_pin.data_ptr()), C.byref(st)), "lfr_solve")
    assert_same(ref, (pos_pin.numpy().reshape(N, 2).copy(), b200.stats_dict(st, bufs)), "zero-copy W=%d" % w)
    # pinned multi-device call on [0]
    assert_same(ref, b200.solve_multi(p, [0], b200.default_options(debug_flags=wflags(w)), pinned=True),
                "multi W=%d" % w)
    # profiled plan
    prof, _ = plan_solve(b200, p, DBG_PROFILE | wflags(w))
    assert_same(ref, prof, "profile W=%d" % w)
    queues = schedule_of(b200, capfd, monkeypatch, p, wflags(w))[1]
    assert queues and queues[0][2] == w
    with capfd.disabled():
        print("\nroutes W=%d: queues %s" % (w, queues))
