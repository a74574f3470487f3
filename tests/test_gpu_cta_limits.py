"""The CTA tier (csrc/lfr_solve_cta.cuh) at its size limits, against the CPU oracle.

A component is capped at #images nodes (solve.cc:586), and large scenes have well over 1024 images.
So the CTA tier meets:
  * components of more than 1024 nodes, whose block rows beyond 4 x 256 are walked by the uncached
    row loop of `cta_matvec_bcsr`;
  * more than 1008 free nodes: size class 0, `solve_cta_kernel<256, 2>`, up to 200 KB of CG vectors;
  * CG vectors that do not fit in that shared memory and stay in HBM (more than 1969 free nodes);
  * the 14-bit local indices of `meta` / `fdstE` / the in-list keys: up to 16 383 nodes, 16 384 refused;
  * components of more than 4095 nodes with few unknowns, which the warp tiers cannot index.

The ring1400 scene (1400 images on a ring, 3 % of the keypoints) has 30 natural components of more
than 1024 nodes.  The rest are built from it with three helpers that only rewrite `Problem` arrays:
`subset` keeps chosen dispatch slots, `merge` makes several components one (edges between them become
Tukey edges), `promote_to_roots` makes every node of a component a root but a few, placed at chosen
local indices.  The oracle's dense solve costs O(free nodes^3), so promoting keeps it cheap at any
node count.

Acceptance is that of tests/test_gpu_parity.py, on every compared component: positions within
1e-4 px, identical iteration counts and termination codes, initial / final costs to 1e-10 / 1e-8.
"""
import copy
import os
import time

import numpy as np
import pytest

TOL_UNITS = 1e-4 / 16.0   # 1e-4 px, 1 solver unit = 16 px
ROWS_CACHED = 4 * 256     # kCtaRowsCached x threads of solve_cta_kernel: rows beyond take the uncached loop
MAX_CTA_NODES = 16383     # 14-bit local indices (lfr_capi.cu, to_cta_tier)
CLASS_MAX_FREE = (0xFFFFFFFF, 1008, 504, 250)   # prepare_large's kClassMaxFree
SMEM_VEC_DOUBLES = 200 * 1024 // 8               # CG-vector shared memory of one CTA, in doubles
# free-node local indices around the cached rows, the warp tiers' 12-bit limit and the 13th bit
EDGE_INDICES = (0, 1, 255, 256, 1023, 1024, 1025, 2047, 2048, 4095, 4096, 8191, 8192)
LFR_EUNSUPPORTED = -5
TIER_CTA = 4


# ---------------------------------------------------------------------------------------------------
# problem construction (pure numpy, on copies)
# ---------------------------------------------------------------------------------------------------
def slot_nodes(p, s):
    return p.comp_nodes[p.comp_ptr[s]:p.comp_ptr[s + 1]].astype(np.int64)


def sizes_of(p):
    return np.diff(p.comp_ptr.astype(np.int64))


def non_roots(p):
    """Non-root nodes per slot: the host's free-node count, which picks the CTA size class."""
    return np.array([int((p.is_root[slot_nodes(p, s)] == 0).sum()) for s in range(p.n_components)], np.int64)


def class_of(nfree):
    """prepare_large's size class (lfr_capi.cu): 0 = more than 1008 free nodes, `<256, 2>`."""
    return 0 if nfree > CLASS_MAX_FREE[1] else (1 if nfree > CLASS_MAX_FREE[2] else (2 if nfree > CLASS_MAX_FREE[3] else 3))


def subset(p, slots):
    """A problem holding only the dispatch slots `slots` (in that order)."""
    q = copy.copy(p)
    parts = [slot_nodes(p, s) for s in slots]
    q.comp_ptr = np.concatenate([[0], np.cumsum([len(x) for x in parts])]).astype(np.uint32)
    q.comp_nodes = (np.concatenate(parts) if parts else np.zeros(0)).astype(np.uint32)
    q.comp_order = np.asarray(p.comp_order)[list(slots)]
    return q


def merge(p, slots):
    """A one-slot problem: the components of `slots` made one.  All their nodes get the first one's
    component id, so the edges between them (different tracks, now the same component) are Tukey edges."""
    q = subset(p, [slots[0]])
    nodes = np.concatenate([slot_nodes(p, s) for s in slots])
    q.comp = p.comp.copy()
    q.comp[nodes] = p.comp[nodes[0]]
    q.comp_ptr = np.array([0, len(nodes)], np.uint32)
    q.comp_nodes = nodes.astype(np.uint32)
    return q


def internal_out_degree(p, nodes, within=None):
    """Out-edges of each of `nodes` that end at a node of `within` (default: `nodes`)."""
    g = p.graph
    inside = np.zeros(g.n_nodes, bool)
    inside[nodes if within is None else within] = True
    rp = g.row_ptr.astype(np.int64)
    deg = rp[nodes + 1] - rp[nodes]
    src = np.repeat(np.arange(len(nodes)), deg)
    eidx = np.concatenate([np.arange(rp[v], rp[v + 1]) for v in nodes]) if len(nodes) else np.zeros(0, np.int64)
    return np.bincount(src, weights=inside[g.edges["dst"][eidx].astype(np.int64)], minlength=len(nodes))


def promote_to_roots(p, slot, n_free, place, seed=0):
    """Every node of `slot` becomes a root except `n_free` nodes that have at least one out-edge inside
    the component; the slot's comp_nodes are then permuted so that those free nodes sit at the local
    indices `place` (n_free distinct indices), the others keeping their relative order."""
    rng = np.random.default_rng(seed)
    nodes = slot_nodes(p, slot)
    place = np.asarray(sorted(place), np.int64)
    assert len(place) == n_free == len(set(place.tolist())) and place.min() >= 0 and place.max() < len(nodes)
    cand = nodes[internal_out_degree(p, nodes) > 0]
    assert len(cand) >= n_free
    free = rng.permutation(cand)[:n_free]
    q = copy.copy(p)
    q.is_root = p.is_root.copy()
    q.is_root[nodes] = 1
    q.is_root[free] = 0
    order = np.empty(len(nodes), np.int64)
    at_free = np.zeros(len(nodes), bool)
    at_free[place] = True
    order[place] = free
    order[~at_free] = nodes[~np.isin(nodes, free)]
    q.comp_nodes = p.comp_nodes.copy()
    q.comp_nodes[p.comp_ptr[slot]:p.comp_ptr[slot + 1]] = order.astype(np.uint32)
    return q


def reverse_slot(p, slot):
    """The same problem with the slot's nodes listed in reverse order (local index l -> Nc - 1 - l)."""
    q = copy.copy(p)
    q.comp_nodes = p.comp_nodes.copy()
    b, e = int(p.comp_ptr[slot]), int(p.comp_ptr[slot + 1])
    q.comp_nodes[b:e] = p.comp_nodes[b:e][::-1]
    return q


def spread(nc, n_free, seed=0):
    """n_free distinct local indices in [0, nc): every EDGE_INDICES entry below nc, nc - 1, the rest random."""
    rng = np.random.default_rng(seed)
    must = sorted({i for i in EDGE_INDICES if i < nc} | {nc - 1})
    rest = np.setdiff1d(np.arange(nc), must)
    return sorted(must + rng.choice(rest, n_free - len(must), replace=False).tolist())


def slots_summing_to(p, target):
    """Dispatch slots whose sizes add up to exactly `target` (subset sum, largest slots preferred)."""
    sizes = sizes_of(p)
    items = list(range(p.n_components))
    reach = [1]                                  # reach[i]: bitset of the sums of items[:i]
    mask = (1 << (target + 1)) - 1
    for s in items:
        reach.append((reach[-1] | (reach[-1] << int(sizes[s]))) & mask)
    if not (reach[-1] >> target) & 1:
        return None
    out, t = [], target
    for i in range(len(items), 0, -1):
        if not (reach[i - 1] >> t) & 1:          # items[i-1] is needed for t
            out.append(items[i - 1])
            t -= int(sizes[items[i - 1]])
    assert t == 0
    return sorted(out)


def numpy_cost(p, slot, pos):
    """0.5 * sum rho over the kept edges of one slot at positions `pos` [N, 2] (numpy restatement of
    the robust cost, cost.cc / solve.cc:98-143): an edge is kept when its ends share a track (Cauchy)
    or a component (Tukey) and not both are roots."""
    g = p.graph
    nodes = slot_nodes(p, slot)
    rp = g.row_ptr.astype(np.int64)
    src = np.repeat(nodes, rp[nodes + 1] - rp[nodes])
    eidx = np.concatenate([np.arange(rp[v], rp[v + 1]) for v in nodes])
    dst = g.edges["dst"][eidx].astype(np.int64)
    cauchy = p.track[src] == p.track[dst]
    tukey = ~cauchy & (p.comp[src] == p.comp[dst])
    keep = (cauchy | tukey) & ~((p.is_root[src] != 0) & (p.is_root[dst] != 0))
    src, dst, eidx, cauchy = src[keep], dst[keep], eidx[keep], cauchy[keep]

    def lag(t):
        return np.stack([2 * t * (t - .5), -4 * (t - .5) * (t + .5), 2 * t * (t + .5)], axis=-1)

    D = g.edges["flow"][eidx].astype(np.float64).reshape(-1, 3, 3, 2)
    xs = np.clip(pos[src], -.5, .5)
    f = np.einsum("ei,ej,eijk->ek", lag(xs[:, 0]), lag(xs[:, 1]), D)
    r = pos[dst] - pos[src] - f
    s = (r * r).sum(axis=1)
    sim = g.edges["sim"][eidx].astype(np.float64)
    a2 = 0.0625 ** 2
    rho = np.where(cauchy, 0.0625 * np.log1p(s / 0.0625),
                   np.where(s <= a2, a2 / 6 * (1 - (1 - np.minimum(s, a2) / a2) ** 3), a2 / 6))
    return float(0.5 * (sim * rho).sum())


# ---------------------------------------------------------------------------------------------------
# the scene and the constructed shapes (built once per module)
# ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ring1400():
    """1400 images on a ring (+ 5 random partners each) at 3 % of 2000 keypoints: ~84 000 nodes, 132
    components, 30 of them over 1024 nodes (largest 1385), 28 with more than 1008 free nodes."""
    from lfr_b200 import build_problem, synth
    cfg = synth.SynthConfig("ring1400", 1400, 2000, "ring", 0.7, match_prob=0.3, window=20, n_random=5,
                            vis_halfwidth=12, seed=1400, outlier_match_ratio=0.125)
    return build_problem(synth.generate(cfg, scale=0.03))


@pytest.fixture(scope="module")
def natural(ring1400):
    """Every component of more than 1024 nodes, plus every 8th of the others (the dispatch list is
    size-descending)."""
    sizes = sizes_of(ring1400)
    n_big = int((sizes > ROWS_CACHED).sum())
    return subset(ring1400, list(range(n_big)) + list(range(n_big, ring1400.n_components, 8)))


_shapes = {}


def shape(p, name):
    """One-slot problems with a few free nodes at the local indices `spread` picks:
    "1100": the smallest natural component of at least 1100 nodes, 300 free nodes;
    "2000" / "4096" / "16383" / "16384": natural components merged to exactly that many nodes, with 200 /
    40 / 300 / 40 free nodes.  "4096" has 80 unknowns: only its node count keeps it from the warp tiers."""
    if name not in _shapes:
        sizes = sizes_of(p)
        n_free = {"1100": 300, "2000": 200, "4096": 40, "16383": 300, "16384": 40}[name]
        if name == "1100":
            q = subset(p, [int(np.nonzero(sizes >= 1100)[0][-1])])
        else:
            slots = slots_summing_to(p, int(name))
            assert slots is not None and len(slots) >= 2
            q = merge(p, slots)
        nc = int(q.comp_ptr[1])
        place = spread(nc, n_free, seed=nc)
        _shapes[name] = (promote_to_roots(q, 0, n_free, place, seed=nc), place)
    return _shapes[name]


def oracle_solve(oracle, p, n_threads=1):
    t = time.perf_counter()
    pos, st = oracle.solve(p, oracle.default_options(n_threads=n_threads))
    return pos, st, time.perf_counter() - t


def assert_agree(p, pos_g, st_g, pos_o, st_o):
    """test_gpu_parity.py's acceptance on every component: positions within 1e-4 px, identical
    iteration counts and termination codes, costs to _compare's tolerances.  Returns the per-component
    max |dx|."""
    err = np.zeros(p.n_components)
    for c in range(p.n_components):
        nodes = slot_nodes(p, c)
        err[c] = np.abs(pos_g[nodes] - pos_o[nodes]).max() if nodes.size else 0.0
    bad = np.nonzero((err > TOL_UNITS) | (st_g["iterations"] != st_o["iterations"]) |
                     (st_g["termination"] != st_o["termination"]))[0]
    assert bad.size == 0, [(int(c), int(sizes_of(p)[c]), float(err[c]), int(st_g["iterations"][c]),
                            int(st_o["iterations"][c]), int(st_g["termination"][c]), int(st_o["termination"][c]))
                           for c in bad[:8]]
    np.testing.assert_allclose(st_g["initial_cost"], st_o["initial_cost"], rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(st_g["final_cost"], st_o["final_cost"], rtol=1e-8, atol=1e-14)
    assert st_g["n_solved"] == st_o["n_solved"] and st_g["total_iterations"] == st_o["total_iterations"]
    return err


def profiled_solve(b200, p):
    """The solve through a plan created with LFR_DBG_PROFILE: positions, stats, decoded records."""
    from lfr_b200 import capi
    plan = capi.Plan(b200, p, b200.default_options(debug_flags=capi.DBG_PROFILE))
    try:
        plan.solve()
        pos, st = plan.download()
        rec, _ = plan.profile()
    finally:
        plan.close()
    return pos, st, rec


def assert_bitwise(a, b, what):
    (pa, sa), (pb, sb) = a, b
    assert np.array_equal(pa, pb), (what, float(np.abs(pa - pb).max()))
    for k in ("iterations", "termination", "initial_cost", "final_cost"):
        assert np.array_equal(sa[k], sb[k]), (what, k)


# ---------------------------------------------------------------------------------------------------
# CPU: the helpers and the judge
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["1100", "2000", "4096", "16383", "16384"])
def test_constructed_problems_are_valid(ring1400, name):
    """comp_ptr monotone; comp, track and comp_nodes agree (a slot holds whole components and whole
    tracks, so every kept edge ends inside its slot); the free nodes are exactly the requested local
    indices and each has an out-edge inside its component."""
    p = ring1400
    q, place = shape(p, name)
    nc = int(q.comp_ptr[-1])
    assert q.n_components == 1 and np.all(np.diff(q.comp_ptr.astype(np.int64)) >= 0)
    assert nc == int(name) if name != "1100" else 1100 <= nc < 1200
    nodes = slot_nodes(q, 0)
    assert len(np.unique(nodes)) == nc
    assert np.array_equal(np.sort(nodes), np.sort(np.nonzero(q.comp == q.comp[nodes[0]])[0]))
    in_slot = np.zeros(q.graph.n_nodes, bool)
    in_slot[nodes] = True
    assert np.all(in_slot[np.isin(q.track, np.unique(q.track[nodes]))])
    free_local = np.nonzero(q.is_root[nodes] == 0)[0]
    assert np.array_equal(free_local, np.asarray(place))
    assert np.all(internal_out_degree(q, nodes[free_local], nodes) > 0)
    assert set(i for i in EDGE_INDICES if i < nc) | {nc - 1} <= set(free_local.tolist())
    # outside the slot nothing changed
    assert np.array_equal(q.is_root[~in_slot], p.is_root[~in_slot]) and np.array_equal(q.comp[~in_slot], p.comp[~in_slot])
    r = reverse_slot(q, 0)
    assert np.array_equal(np.nonzero(r.is_root[slot_nodes(r, 0)] == 0)[0], np.sort(nc - 1 - free_local))


def test_subset_and_natural_sizes(ring1400, natural):
    """The natural subset holds at least 25 components over 1024 nodes and 20 in size class 0."""
    p, q = ring1400, natural
    sizes, nfree = sizes_of(q), non_roots(q)
    assert (sizes > ROWS_CACHED).sum() >= 25 and (nfree > CLASS_MAX_FREE[1]).sum() >= 20
    assert sizes.max() == sizes_of(p).max() > 1300
    assert len(np.unique(q.comp_nodes)) == len(q.comp_nodes)
    for k, s in enumerate(q.comp_order.tolist()):
        nodes = slot_nodes(q, k)
        assert np.all(p.comp[nodes] == s) and len(nodes) == int((p.comp == s).sum())


@pytest.mark.parametrize("name,reverse", [("1100", False), ("1100", True), ("16383", False)])
def test_numpy_cost_matches_oracle_on_constructed_shapes(oracle, ring1400, name, reverse):
    """The oracle's initial and final costs equal a numpy restatement of the cost over the kept edges
    to 1e-12: the oracle treats promoted roots, merged components and node order as intended."""
    q, _ = shape(ring1400, name)
    if reverse:
        q = reverse_slot(q, 0)
    pos, st, dt = oracle_solve(oracle, q)
    assert st["n_solved"] == 1 and st["iterations"][0] > 0
    zero = np.zeros((q.graph.n_nodes, 2))
    c0, c1 = numpy_cost(q, 0, zero), numpy_cost(q, 0, pos)
    assert abs(c0 - st["initial_cost"][0]) <= 1e-12 * max(1.0, c0), (c0, st["initial_cost"][0])
    assert abs(c1 - st["final_cost"][0]) <= 1e-12 * max(1.0, c1), (c1, st["final_cost"][0])
    # roots stay where they started
    nodes = slot_nodes(q, 0)
    assert np.all(pos[nodes[q.is_root[nodes] != 0]] == 0.0)
    print("%s%s: oracle %.1f s, %d iterations" % (name, " reversed" if reverse else "", dt, st["iterations"][0]))


# ---------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_natural_components_over_1024_nodes_match_oracle(b200, oracle, natural):
    """Every natural component over 1024 nodes (uncached block rows) and every 8th of the others, with
    at least 20 in size class 0 (more than 1008 free nodes, `<256, 2>`): all agree with the oracle."""
    q = natural
    sizes, nfree = sizes_of(q), non_roots(q)
    n_big, n_cls0 = int((sizes > ROWS_CACHED).sum()), int((nfree > CLASS_MAX_FREE[1]).sum())
    assert n_big >= 25 and n_cls0 >= 20
    t = time.perf_counter()
    pos_g, st_g = b200.solve(q)
    t_gpu = time.perf_counter() - t
    pos_o, st_o, t_orc = oracle_solve(oracle, q, n_threads=os.cpu_count() or 8)
    err = assert_agree(q, pos_g, st_g, pos_o, st_o)
    print("natural: %d components (%d over 1024 nodes, %d over 1008 free nodes, largest %d nodes / %d free), "
          "max |dx| %.2e units, %d LM iterations; gpu %.2f s, oracle %.1f s on %d threads" % (
              q.n_components, n_big, n_cls0, sizes.max(), nfree.max(), err.max(), st_g["total_iterations"],
              t_gpu, t_orc, os.cpu_count() or 8))


@pytest.mark.gpu
def test_natural_components_take_the_cta_tier(b200, natural):
    """Proof of route: a profiled solve of the same subset records tier 4 (CTA) with CG iterations for
    every component of more than 96 unknowns, and its positions are bitwise those of the plain solve;
    size class 0 is populated."""
    q = natural
    nfree = non_roots(q)
    assert sum(class_of(int(n)) == 0 for n in nfree) >= 20
    plain = b200.solve(q)
    pos_p, st_p, rec = profiled_solve(b200, q)
    assert_bitwise(plain, (pos_p, st_p), "profiled")
    cta = 2 * nfree > 96
    assert cta.sum() >= 25
    assert np.all(rec["tier"][cta] == TIER_CTA), np.unique(rec["tier"][cta])
    assert np.all(rec["counter"][cta] > 0)
    print("profile: %d components on tier 4, CG iterations %d..%d; tiers of the others %s" % (
        int(cta.sum()), int(rec["counter"][cta].min()), int(rec["counter"][cta].max()),
        sorted(set(rec["tier"][~cta].tolist()))))


@pytest.mark.gpu
@pytest.mark.parametrize("var,value", [("LFR_CTA_SMEM_VECS", "0,0,0,0"), ("LFR_CTA_SMEM_VECS", "5,5,5,5"),
                                       ("LFR_CTA_SMEM_VECS", "3,3,3,3"), ("LFR_CTA_MINB", "4,4,4,4"),
                                       ("LFR_CTA_MINB", "2,2,2,2")])
def test_cg_vector_placement_and_minb_are_bitwise_neutral(b200, natural, monkeypatch, var, value):
    """prepare_large's tuning hooks, read on every call: CG vectors all in HBM (0), all but the
    preconditioner in shared memory (5: the layout of a component with more than 1969 free nodes, whose
    13 doubles per free node exceed 200 KB), p, w, r only (3); every size class through `<256, 4>` or
    `<256, 2>`.  Same operations at other addresses / register budgets: bitwise the default solve, on
    ring60 and on the ring1400 subset.  Unset again, the default solve is reproduced."""
    from conftest import get_problem
    monkeypatch.delenv("LFR_CTA_SMEM_VECS", raising=False)
    monkeypatch.delenv("LFR_CTA_MINB", raising=False)
    problems = {"ring60": get_problem("ring60")[1], "ring1400": natural}
    # by default every CG vector of these components is on chip, so each setting moves some to HBM
    assert 13 * non_roots(natural).max() <= SMEM_VEC_DOUBLES
    default = {k: b200.solve(p) for k, p in problems.items()}
    monkeypatch.setenv(var, value)
    for k, p in problems.items():
        assert_bitwise(default[k], b200.solve(p), "%s=%s %s" % (var, value, k))
    monkeypatch.delenv(var)
    for k, p in problems.items():
        assert_bitwise(default[k], b200.solve(p), "%s unset again, %s" % (var, k))


@pytest.mark.gpu
@pytest.mark.parametrize("reverse", [False, True], ids=["order", "reversed"])
@pytest.mark.parametrize("name", ["1100", "2000", "4096"])
def test_free_nodes_beyond_the_cached_rows_match_oracle(b200, oracle, ring1400, name, reverse):
    """Components of 1100, 2000 and 4096 nodes, all roots but 300 / 200 / 40 nodes placed at local
    indices 0, 1023, 1024, 1025, 4095, Nc - 1 and random others, in the given order and reversed: the
    free nodes beyond row 1024 are walked by the uncached row loop.  All take the CTA tier; the 4096-node
    one (80 unknowns, few edges) only because of its node count."""
    q, place = shape(ring1400, name)
    if reverse:
        q = reverse_slot(q, 0)
    nodes = slot_nodes(q, 0)
    free_local = np.nonzero(q.is_root[nodes] == 0)[0]
    assert (free_local >= ROWS_CACHED).sum() >= 3
    if name == "4096":
        rp = q.graph.row_ptr.astype(np.int64)
        assert 2 * len(free_local) <= 96 and int((rp[nodes + 1] - rp[nodes]).sum()) <= 65535 and len(nodes) > 4095
    pos_g, st_g = b200.solve(q)
    pos_o, st_o, dt = oracle_solve(oracle, q)
    err = assert_agree(q, pos_g, st_g, pos_o, st_o)
    pos_p, st_p, rec = profiled_solve(b200, q)
    assert_bitwise((pos_g, st_g), (pos_p, st_p), "profiled")
    assert rec["tier"][0] == TIER_CTA and rec["counter"][0] > 0
    print("%s nodes%s: %d free (%d beyond row 1024), |dx| %.2e units, %d iterations, %d CG iterations, oracle %.1f s"
          % (name, " reversed" if reverse else "", len(free_local), int((free_local >= ROWS_CACHED).sum()), err[0],
             st_g["iterations"][0], int(rec["counter"][0]), dt))


@pytest.mark.gpu
def test_14_bit_node_limit(b200, oracle, ring1400):
    """A merged component of exactly 16 383 nodes, with free nodes at local indices 0, 1024, 4096, 8191,
    8192 and 16 382 among 300, agrees with the oracle, costs included (every kept edge of the free nodes
    is evaluated).  One of 16 384 nodes is refused on the host with LFR_EUNSUPPORTED, and the library
    still solves ring60 correctly afterwards."""
    from conftest import get_problem
    q, _ = shape(ring1400, "16383")
    assert int(q.comp_ptr[1]) == MAX_CTA_NODES
    nodes = slot_nodes(q, 0)
    assert all(q.is_root[nodes[i]] == 0 for i in (0, 1024, 4096, 8191, 8192, MAX_CTA_NODES - 1))
    pos_g, st_g = b200.solve(q)
    pos_o, st_o, dt = oracle_solve(oracle, q)
    err = assert_agree(q, pos_g, st_g, pos_o, st_o)
    assert st_g["iterations"][0] > 0 and st_o["initial_cost"][0] > 0
    _, _, rec = profiled_solve(b200, q)
    assert rec["tier"][0] == TIER_CTA and rec["counter"][0] > 0
    print("16383 nodes: 300 free, |dx| %.2e units, %d iterations, oracle %.1f s" % (err[0], st_g["iterations"][0], dt))

    big, _ = shape(ring1400, "16384")
    assert int(big.comp_ptr[1]) == MAX_CTA_NODES + 1
    with pytest.raises(RuntimeError, match=r"\(%d\).*16383 nodes" % LFR_EUNSUPPORTED):
        b200.solve(big)
    _, p = get_problem("ring60")
    pos_g, st_g = b200.solve(p)
    pos_o, st_o, _ = oracle_solve(oracle, p, n_threads=os.cpu_count() or 8)
    assert_agree(p, pos_g, st_g, pos_o, st_o)
