"""Every solve tier's first Levenberg-Marquardt step against an extended-precision solve of the same
damped system (tests/lm_step_ref.py).

Whole solves against the oracle cannot see a slightly wrong step: LM corrects it in the next iteration.
So these tests stop every component after its first step.  liblfr_b200_lmstep.so is the product built
with -DLFR_DBG_LM_STEP (csrc/build.py): lm_solve takes iteration 0 and one lm_step at the initial radius,
writes dl to the free nodes' positions and {cost, gmax, validity, model change, g . dl, |dl|_inf, tier
(its integer part; the fraction is the tier's counter x 2^-32: CG iterations on the CTA tier), n} to the
slot's LFR_DBG_PROFILE record, and returns.

Components are built directly as lfr_problem arrays: every register class edge of the warp2 tier (in
its per-bucket launches and in the queue kernel), the tile tier at 64 and 128 threads, the shared-memory
Cholesky tier and the CTA tier up to components past 1008 free nodes, 1024 nodes and 1969 free nodes
(CG vectors in HBM); duplicated directed edges, edges without a twin, roots between free nodes, root-root
and cross-component edges, rows of out-degree 1 to 31 and 40 in one 32-row slice, reversed node order;
radius 1e-8 to 1e16, the LM diagonal clamp, sims over twelve decades, a node whose every edge is a Tukey
outlier, clusters held to the roots by links of sim 2e-11 to 1.5e-8 only (kappa 8e9 to 2e11, as high
as a meaningful bound allows at their sizes), flows with I + grad flow nearly singular, start points at
zero, inside and beyond the box, both Tukey variants and non-default loss widths.  Each runs on the five
routes of test_gpu_tier_options.ROUTES.

Acceptance per component: valid; the tier the route sends it to; |dl - dl*| <= 8 n kappa 2^-53 |dl*|
(kappa = kappa_2 of the damped system), the model change and g . dl to the same relative bound; cost and
gmax to 1e-13; the Cholesky tier's normwise backward error |A y - b| / (|A| |y| + |b|) <= 8 n 2^-53 in
longdouble; roots bitwise at their start; and a component's dl bitwise the same in the queue kernel and
in its per-bucket launch.  No case is run whose bound 8 n kappa 2^-53 exceeds 1e-2: above that a step
of roughly the right size passes whatever its error (test_cases_are_meaningful checks the cases on the
CPU).  The module ends by printing, per tier, the largest |dl - dl*| / (n kappa 2^-53 |dl*|) and the
largest kappa checked.
"""
import ctypes as C
import os

import numpy as np
import pytest

import lm_step_ref as ref
from test_gpu_tier_options import ROUTES, TIER_WARP, expected_tier, options

LMSTEP_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "local-feature-refinement_b200",
                          "csrc", "liblfr_b200_lmstep.so")
U = 2.0 ** -53
MAX_BOUND = 1e-2   # a case whose 8 n kappa 2^-53 is not well below 1 could not fail: none is run
TIER_NAMES = {1: "warp2", 2: "tile", 3: "warp", 4: "cta"}


# ---------------------------------------------------------------------------------------------------
# constructed components (pure numpy)
# ---------------------------------------------------------------------------------------------------
HUB_DEGREE = 40


def component(rng, n_free, n_roots=1, extra=1.0, twins="all", dup=0, sims="plain", singular=0.0, hub=False,
              outlier_node=False):
    """One component: `n_free` free nodes and `n_roots` roots at random local indices, a random spanning
    tree plus `extra` x nodes random pairs; every pair gives two twin edges ("all"), one ("none") or two
    for half of the pairs ("mixed"); `dup` directed edges duplicated; tracks of three consecutive nodes
    (Cauchy inside a track, Tukey across).  `hub`: free local nodes 1..31 get out-degrees 1..31 and node 0
    out-degree 40, all in the first 32-row slice (the roots sit past it).
    `outlier_node`: one free node whose every edge is a Tukey outlier.  `singular`: the fraction of edges
    whose flow is -(1 - 1e-3) x (I + grad flow = 1e-3 I)."""
    nc = n_free + n_roots
    is_root = np.zeros(nc, np.uint8)
    is_root[rng.choice(np.arange(32 if hub else 0, nc), n_roots, replace=False)] = 1
    # a chain inside every track (Cauchy edges: no node's column vanishes when its Tukey edges are
    # outliers), a random spanning tree and random extra pairs
    pairs = [(v - 1, v) for v in range(1, nc) if v % 3]
    pairs += [(int(rng.integers(0, v)), v) for v in range(1, nc)]
    pairs += [tuple(int(t) for t in rng.choice(nc, 2, replace=False)) for _ in range(int(extra * nc))]
    if hub:
        targets = np.arange(32, nc)
        pairs = [(v - 1, v) for v in range(33, nc) if v % 3]
        pairs += [(l, int(k)) for l in range(1, 32) for k in rng.choice(targets, l, replace=False)]
        pairs += [(0, int(k)) for k in rng.choice(targets, HUB_DEGREE, replace=False)]
        pairs += [(int(rng.integers(32, v)), v) for v in range(33, nc)]
    # each unordered pair once: duplicates only where `dup` asks, so the components with clean twins are
    # "regular" and take the CTA tier's BCSR product
    seen = set()
    pairs = [q for q in pairs if frozenset(q) not in seen and not seen.add(frozenset(q))]
    src, dst = [], []
    for k, (u, v) in enumerate(pairs):
        both = twins == "all" or (twins == "mixed" and k % 2 == 0)
        src += [u, v] if both else [u]
        dst += [v, u] if both else [v]
    for k in rng.choice(len(src), dup, replace=False) if dup else []:
        src.append(src[k])
        dst.append(dst[k])
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    # |flow| <= 0.03: every residual is a Tukey inlier at a start of zero, so no sub-cluster floats free
    flow = rng.uniform(-0.03, 0.03, (len(src), 18)).astype(np.float32)
    if singular:
        t = np.array([-0.5, 0.0, 0.5])
        lin = np.zeros((3, 3, 2))
        lin[:, :, 0] = -(1 - 1e-3) * t[:, None]
        lin[:, :, 1] = -(1 - 1e-3) * t[None, :]
        pick = rng.random(len(src)) < singular
        flow[pick] = lin.reshape(18).astype(np.float32)
    if sims == "spread":
        sim = (10.0 ** rng.uniform(-6, 6, len(src))).astype(np.float32)
    else:
        sim = rng.uniform(0.5, 1.0, len(src)).astype(np.float32)
    track = np.arange(nc) // 3
    if outlier_node:
        v = int(np.nonzero(is_root == 0)[0][0])
        track = track + 1
        track[v] = 0                                         # alone on its track: Tukey edges only
        at = (src == v) | (dst == v)
        flow[at] = 0.5                                       # |r| ~ 0.7 >> tukey_a at a start near zero
    return dict(nc=nc, is_root=is_root, src=src, dst=dst, flow=flow, sim=sim, track=track)


def weak_cluster(rng, n_held, n_loose, link_sim, n_roots=2):
    """A component of two parts: `n_held` free nodes with the roots, and `n_loose` free nodes held to them
    (and to every root) only by four inlier edge pairs of sim `link_sim`."""
    a = component(rng, n_held, n_roots)
    b = component(rng, n_loose, 0)
    b["flow"][:] = b["flow"][:, :1]      # constant flows: a translation of the loose part costs nothing
    off = a["nc"]
    link_s = rng.choice(off, 4)
    link_d = off + rng.choice(b["nc"], 4)
    src = np.concatenate([a["src"], b["src"] + off, link_s, link_d])
    dst = np.concatenate([a["dst"], b["dst"] + off, link_d, link_s])
    flow = np.concatenate([a["flow"], b["flow"], np.full((8, 18), 0.01, np.float32)])
    sim = np.concatenate([a["sim"], b["sim"], np.full(8, link_sim, np.float32)])
    track = np.concatenate([a["track"], b["track"] + a["track"].max() + 1])
    return dict(nc=off + b["nc"], is_root=np.concatenate([a["is_root"], b["is_root"]]), src=src, dst=dst,
                flow=flow, sim=sim, track=track)


def problem(comps, reverse=(), cross=0, root_root=0, seed=0):
    """One lfr_problem of the components `comps` (dispatch slot k = comps[k], node lists reversed for the
    slots in `reverse`), plus `cross` edges between different components and `root_root` edges between
    two roots of one component (neither makes a residual block)."""
    from lfr_b200.graph import EDGE_DTYPE, MatchGraph, Problem
    rng = np.random.default_rng(seed)
    offs = np.concatenate([[0], np.cumsum([c["nc"] for c in comps])]).astype(np.int64)
    N = int(offs[-1])
    toffs = np.concatenate([[0], np.cumsum([c["track"].max() + 1 for c in comps])]).astype(np.int64)
    src = [c["src"] + o for c, o in zip(comps, offs)]
    dst = [c["dst"] + o for c, o in zip(comps, offs)]
    flow = [c["flow"] for c in comps]
    sim = [c["sim"] for c in comps]
    is_root = np.concatenate([c["is_root"] for c in comps])
    for _ in range(cross):
        i, j = rng.choice(len(comps), 2, replace=False)
        src.append(np.array([offs[i] + rng.integers(comps[i]["nc"])]))
        dst.append(np.array([offs[j] + rng.integers(comps[j]["nc"])]))
    for _ in range(root_root):
        roots = [k for k, c in enumerate(comps) if c["is_root"].sum() >= 2]
        k = roots[rng.integers(len(roots))]
        u, v = rng.choice(np.nonzero(comps[k]["is_root"])[0], 2, replace=False)
        src.append(np.array([offs[k] + u]))
        dst.append(np.array([offs[k] + v]))
    n_extra = len(src) - len(comps)
    flow += [rng.uniform(-0.3, 0.3, (n_extra, 18)).astype(np.float32)] if n_extra else []
    sim += [np.full(n_extra, 0.9, np.float32)] if n_extra else []
    src, dst = np.concatenate(src), np.concatenate(dst)
    order = np.argsort(src, kind="stable")
    edges = np.zeros(len(src), EDGE_DTYPE)
    edges["flow"] = np.concatenate(flow)[order]
    edges["sim"] = np.concatenate(sim)[order]
    edges["dst"] = dst[order]
    row_ptr = np.zeros(N + 1, np.uint32)
    np.cumsum(np.bincount(src, minlength=N), out=row_ptr[1:])
    g = MatchGraph(n_nodes=N, node_image=np.zeros(N, np.int64), node_feat=np.zeros(N, np.uint32),
                   und_sim=np.zeros(0), und_n1=np.zeros(0), und_n2=np.zeros(0), row_ptr=row_ptr, edges=edges,
                   image_names=[], image_fact={}, n_images=0)
    comp = np.repeat(np.arange(len(comps)), np.diff(offs)).astype(np.uint32)
    track = np.concatenate([c["track"] + t for c, t in zip(comps, toffs)]).astype(np.uint32)
    lists = [np.arange(offs[k], offs[k + 1])[::-1 if k in reverse else 1] for k in range(len(comps))]
    return Problem(graph=g, track=track, comp=comp, is_root=is_root, comp_ptr=offs.astype(np.uint32),
                   comp_nodes=np.concatenate(lists).astype(np.uint32),
                   comp_order=np.arange(len(comps), dtype=np.uint32))


def start_point(p, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "zero":
        return np.zeros((p.graph.n_nodes, 2))
    if kind == "inside":
        return rng.uniform(-0.9, 0.9, (p.graph.n_nodes, 2))
    return rng.uniform(-1.6, 1.6, (p.graph.n_nodes, 2))      # "beyond": free nodes projected to the box


# ---------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------
# unknowns at every class edge: warp2 8|10, 16|18, 24|26, 32 | tile 34, 48|50, 64|66, 80 | warp 82, 96 | CTA
SIZES = (2, 8, 10, 16, 18, 24, 26, 32, 34, 48, 50, 64, 66, 80, 82, 96, 98, 300)


def sizes_problem():
    rng = np.random.default_rng(1)
    return problem([component(rng, n // 2, n_roots=1 + (n // 2) % 3) for n in SIZES])


def large_problem():
    """CTA components past 1008 free nodes, past 1024 nodes (with roots in between) and past 1969 free
    nodes (whose CG vectors stay in HBM)."""
    rng = np.random.default_rng(2)
    return problem([component(rng, 1970, 3, extra=0.5), component(rng, 1010, 30, extra=0.5),
                    component(rng, 600, 430, extra=0.5)])


def structure_problem():
    rng = np.random.default_rng(3)
    comps = [component(rng, 12, 2, dup=6), component(rng, 40, 3, dup=10), component(rng, 70, 4, dup=12),
             component(rng, 8, 2, twins="none"), component(rng, 30, 2, twins="none"),
             component(rng, 150, 5, twins="none"), component(rng, 45, 3, twins="mixed"),
             component(rng, 160, 6, twins="mixed", dup=8), component(rng, 20, 12), component(rng, 130, 60),
             component(rng, 120, 4, hub=True), component(rng, 14, 2), component(rng, 36, 5),
             component(rng, 200, 10)]
    return problem(comps, reverse={11, 12, 13}, cross=40, root_root=30, seed=3)


CONDITIONING = {
    # name: (options, start kind, component keywords)
    "radius_1e-8": (dict(initial_trust_region_radius=1e-8), "inside", {}),
    "radius_1": (dict(initial_trust_region_radius=1.0), "inside", {}),
    "radius_1e16": (dict(initial_trust_region_radius=1e16), "zero", {}),
    "lm_diagonal_clamp": (dict(min_lm_diagonal=1e2, max_lm_diagonal=1e3), "inside", {}),
    "sims_12_decades": (dict(initial_trust_region_radius=1e16), "zero", dict(sims="spread")),
    "tukey_outlier_node": ({}, "zero", dict(outlier_node=True)),
    "near_singular_flow": (dict(initial_trust_region_radius=1e16), "zero", dict(singular=0.3)),
    "start_zero": ({}, "zero", {}),
    "start_beyond_box": ({}, "beyond", {}),
    "tukey_variant_2": (dict(tukey_variant=2), "inside", {}),
    "loss_widths": (dict(cauchy_a=0.1, tukey_a=0.2), "inside", {}),
}
# free nodes: 12 / 28 unknowns warp2, 48 / 72 tile (64 / 128 threads), 90 Cholesky warp, 250 CTA (default route)
COND_SIZES = (6, 14, 24, 36, 45, 125)


def conditioning_problem(name):
    rng = np.random.default_rng(10 + sorted(CONDITIONING).index(name))
    kw = CONDITIONING[name][2]
    return problem([component(rng, n, 2, **kw) for n in COND_SIZES])


# (held free nodes, loose free nodes, link sim): kappa as high as a bound 8 n kappa 2^-53 of a few 1e-3
# allows at 16, 60, 84, 92 and 420 unknowns (warp2, tile, tile, Cholesky warp, CTA under the default
# route).  Links of sim 1e-12 give kappa 4e12 to 1e14 here, where that bound reaches 0.06 to 46 and no
# longer tells a good step from a bad one.
WEAK = ((5, 3, 2e-11), (20, 10, 3e-10), (30, 12, 6e-10), (30, 16, 8e-10), (150, 60, 1.5e-8))


def weak_problem():
    rng = np.random.default_rng(4)
    return problem([weak_cluster(rng, h, l, sim) for h, l, sim in WEAK])


# ---------------------------------------------------------------------------------------------------
# running the diagnostic build
# ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lmstep():
    from lfr_b200.capi import Library
    lib = Library(LMSTEP_LIB)
    f = lib.lib.lfr_debug_plan_cycles
    f.argtypes = [C.c_void_p, C.c_void_p]
    f.restype = C.c_int
    return lib


def counter_of(word):
    """The tier's counter carried by a record's tier word, tier + counter x 2^-32 (csrc/lfr_lm.cuh): the
    step's CG iterations on the CTA tier."""
    return int(round((word - int(word)) * 2.0 ** 32))


def first_steps(lib, p, route, start, **opts):
    """(positions [N, 2] with dl at the free nodes, records [C, 8] as doubles) of one launch."""
    from lfr_b200 import capi
    plan = capi.Plan(lib, p, options(lib, route, True, **opts), positions=start)
    try:
        plan.solve()
        pos, _ = plan.download()
        rec = np.zeros((p.n_components, 8), np.uint64)
        lib.check(lib.lib.lfr_debug_plan_cycles(plan.handle, rec.ctypes.data), "lfr_debug_plan_cycles")
    finally:
        plan.close()
    return pos, rec.view(np.float64)


_statements = {}


@pytest.fixture(scope="module")
def report(request):
    """Collects, per tier, the largest |dl - dl*| / (n kappa u |dl*|) and the largest kappa checked, and
    prints them at the end of the module to the terminal, past output capture (visible without -s)."""
    worst = {}
    yield worst
    tr = request.config.pluginmanager.getplugin("terminalreporter")
    cm = request.config.pluginmanager.getplugin("capturemanager")
    lines = ["first LM step, %-5s %4d components: largest |dl - dl*| / (n kappa u |dl*|) = %.3e, largest kappa "
             "%.2e" % (TIER_NAMES[t], m, r, k) for t, (r, k, m) in sorted(worst.items())]
    if tr is None or cm is None:
        print("\n".join(lines))
        return
    with cm.global_and_fixture_disabled():
        tr.write_line("")
        for line in lines:
            tr.write_line(line)


def statements(key, p, start, opts):
    if key not in _statements:
        from oracle_util import load_oracle
        o = load_oracle().default_options(**opts)
        _statements[key] = [ref.first_step(p, s, o, start) for s in range(p.n_components)]
    return _statements[key]


def check(lib, report, key, p, start, route, opts):
    """Runs one launch and holds every slot to the acceptance bar.  Returns the positions and records."""
    pos, rec = first_steps(lib, p, route, start, **opts)
    roots = p.is_root != 0
    assert np.array_equal(pos[roots], start[roots]), (key, route, "roots moved")
    for s, st in enumerate(statements(key, p, start, opts)):
        n, what = st.n, (key, route, s, st.n)
        cost, gmax, valid, mc, gd, dmax, tier, n_rec = rec[s]
        assert valid == 1.0 and int(n_rec) == n, (what, rec[s])
        assert int(tier) == expected_tier(n, route), (what, int(tier))
        dl = pos[st.free_nodes]
        dl_ref = st.dl.astype(np.float64)
        bound = ref.step_bound(n, st.kappa)
        assert bound <= MAX_BOUND, (what, "kappa too large for a meaningful bound", st.kappa, bound)
        norm = float(np.linalg.norm(st.dl.astype(np.float64)))
        err = float(np.sqrt((((dl.astype(ref.LD) - st.dl) ** 2).sum()).astype(np.float64)))
        assert err <= bound * norm, (what, "step", err / norm, bound, st.kappa)
        assert abs(mc - st.model_change) <= bound * abs(st.model_change), (what, "model change", mc, st.model_change)
        assert abs(gd - st.gd) <= bound * abs(st.gd), (what, "g . dl", gd, st.gd)
        assert abs(dmax - np.abs(dl_ref).max()) <= bound * norm, (what, "|dl|_inf")
        assert dmax == np.abs(dl).max(), what
        assert abs(cost - st.cost) <= 1e-13 * st.cost, (what, "cost", cost, st.cost)
        assert abs(gmax - st.gmax) <= 1e-13 * st.gmax, (what, "gmax", gmax, st.gmax)
        if int(tier) == TIER_WARP:   # dense Cholesky: backward stable
            y = -dl.reshape(-1).astype(ref.LD) / st.S
            a_norm = float(np.abs(st.A.dense()).sum(axis=1).max())
            res = float(np.abs(st.A.matvec(y) - st.b).max())
            eta = res / (a_norm * float(np.abs(y).max()) + float(np.abs(st.b).max()))
            assert eta <= 8 * n * U, (what, "backward error", eta)
        w = report.setdefault(int(tier), [0.0, 0.0, 0])
        w[0] = max(w[0], err / (n * st.kappa * U * norm) if norm else 0.0)
        w[1] = max(w[1], st.kappa)
        w[2] += 1
    return pos, rec


# ---------------------------------------------------------------------------------------------------
# the tests
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_every_class_edge(lmstep, report, route):
    p = sizes_problem()
    check(lmstep, report, "sizes", p, start_point(p, "inside", 1), route, {})


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_cta_past_1008_free_1024_nodes_and_shared_memory(lmstep, report, route):
    p = large_problem()
    check(lmstep, report, "large", p, start_point(p, "inside", 2), route, {})


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_structure(lmstep, report, route):
    """Duplicated edges, edges without twins and both kinds, roots between free nodes, root-root and
    cross-component edges (dropped), hubs of degree 1..40 in one slice, reversed node lists."""
    p = structure_problem()
    check(lmstep, report, "structure", p, start_point(p, "inside", 3), route, {})


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("name", list(CONDITIONING))
def test_conditioning(lmstep, report, name, route):
    opts, kind, _ = CONDITIONING[name]
    p = conditioning_problem(name)
    check(lmstep, report, name, p, start_point(p, kind, 4), route, opts)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_weak_cluster_at_radius_1e16(lmstep, report, route):
    """Free clusters held to the roots by links of sim 2e-11 to 1.5e-8 only (WEAK): kappa 8e9 to 2e11 at
    radius 1e16, each as high as a bound of ~3e-3 allows, on every tier the route reaches."""
    p = weak_problem()
    opts = dict(initial_trust_region_radius=1e16)
    check(lmstep, report, "weak", p, start_point(p, "zero"), route, opts)
    assert min(st.kappa for st in _statements["weak"]) >= 5e9


@pytest.mark.gpu
def test_queue_is_the_per_bucket_launch(lmstep):
    """Components of at most 16 unknowns run the per-bucket kernels alone and the queue kernel next to
    one of 18 unknowns: the same dl, bit for bit."""
    rng = np.random.default_rng(6)
    small = [component(rng, n // 2, 1) for n in (2, 4, 8, 10, 12, 16)]
    wide = component(rng, 9, 1)
    alone, with_wide = problem(small), problem(small + [wide])
    start = start_point(with_wide, "inside", 6)
    n_small = alone.graph.n_nodes
    pos_a, rec_a = first_steps(lmstep, alone, "default", start[:n_small])
    pos_q, rec_q = first_steps(lmstep, with_wide, "default", start)
    assert np.array_equal(pos_a, pos_q[:n_small])
    assert np.array_equal(rec_a.view(np.uint64), rec_q[:len(small)].view(np.uint64))


# ---------------------------------------------------------------------------------------------------
# CPU: the cases themselves
# ---------------------------------------------------------------------------------------------------
CASES = dict({"sizes": (sizes_problem, {}, "inside", 1), "large": (large_problem, {}, "inside", 2),
              "structure": (structure_problem, {}, "inside", 3),
              "weak": (weak_problem, dict(initial_trust_region_radius=1e16), "zero", 0)},
             **{k: ((lambda k=k: conditioning_problem(k)), v[0], v[1], 4) for k, v in CONDITIONING.items()})


def test_cases_are_meaningful():
    """Every checked slot has 8 n kappa 2^-53 <= MAX_BOUND; the hub rows of the first slice have out-degrees
    1..31 and 40; the conditioning sweep reaches warp2, both tile widths, the Cholesky warp and the CTA
    tier on the default route; the weak clusters reach kappa 5e9 and more on every tier."""
    worst = 0.0
    for key, (make, opts, kind, seed) in CASES.items():
        p = make()
        sts = statements(key, p, start_point(p, kind, seed), opts)
        for s, st in enumerate(sts):
            b = ref.step_bound(st.n, st.kappa)
            assert b <= MAX_BOUND, (key, s, st.n, st.kappa, b)
            worst = max(worst, b)
    p = structure_problem()
    hub = 10
    nodes = p.comp_nodes[p.comp_ptr[hub]:p.comp_ptr[hub + 1]].astype(np.int64)[:32]
    src = ref.kept_blocks(p, hub)[0]
    deg = np.bincount(src, minlength=p.graph.n_nodes)[nodes]     # kept out-edges (the ELL rows)
    assert sorted(deg.tolist()) == list(range(1, 32)) + [HUB_DEGREE] and not p.is_root[nodes].any()
    n2 = [2 * int((p_.is_root[p_.comp_nodes[p_.comp_ptr[s]:p_.comp_ptr[s + 1]]] == 0).sum())
          for p_ in [conditioning_problem("start_zero")] for s in range(p_.n_components)]
    assert [expected_tier(n, "default") for n in n2] == [1, 1, 2, 2, 3, 4]
    assert sorted({64 if n <= 64 else 128 for n in n2 if 32 < n <= 80}) == [64, 128]   # tile threads
    weak = [ref.step_bound(st.n, st.kappa) for st in _statements["weak"]]
    assert min(st.kappa for st in _statements["weak"]) >= 5e9 and max(weak) <= 5e-3
    print("largest bound 8 n kappa u over all slots: %.2e" % worst)
