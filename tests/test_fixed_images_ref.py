"""Fixed images against the REFERENCE's own create_and_solve_problem, on the CPU.

To the solve, a fixed image is a wider constant mask: every node of the image is held constant as a root
is.  The reference's create_and_solve_problem (solve.cc:79-160) takes that mask (`is_root`) and the start
point (`positions`) as arguments and calls SetParameterBlockConstant on every node whose mask entry is set,
so compiled unmodified against mini-Ceres (oracle/ref_solve_shim.cc -> oracle/_ref/libref_solve.so) it is
an independent statement of what fixing an image means.  This file holds the CPU checker
(oracle/liblfr_ref.so) to it on masks the reference's own roots never produce:

  * same-track (Cauchy) blocks with both ends constant, whole tracks held constant, constant non-roots at
    both ends of a Tukey block: blocks that must be dropped and counted in Ceres' fixed cost;
  * masks whose fixing moves components across every tier boundary of the GPU schedule, components left
    with one free node (2 unknowns), components made EMPTY next to ordinary ones, and a mask longer than
    the scene's image count;
  * starts joined from a SolutionFile with values outside the box, exactly on +-bound and +-0.5 (the flow
    grid's clamp edge), just past +-0.5, -0.0 and a float32 denormal, on constant and free nodes.

The mask cases and the start are shared with tests/test_gpu_fixed_tiers.py.  Each case is checked to hold
what its name claims.  Acceptance, component by component: positions within 1e-4 px, identical iteration
counts, termination codes and line-search step totals, and the checker's initial cost equal to
Summary::initial_cost - fixed_cost to 1e-11 relative (the C ABI reports the cost without the blocks
between two constant nodes).
"""
import numpy as np
import pytest

from lfr_b200 import synth, wire
from lfr_b200.graph import problem_from_stage
from refsrc_util import load_refsolve, ref_solve
from test_fixed_images import displacement, image, stage

TOL_UNITS = 1e-4 / 16.0   # 1e-4 px, 1 solver unit = 16 px
EMPTY = 7
# the scenes of tests/test_gpu_tier_options.py: together they reach every tier of the GPU schedule
SCENES = {"cfg1": 1.0, "cfg2": 0.05, "cfg4": 0.25, "ring60": 0.3}
# here cfg4 runs at 3 % (the same unknown counts, 12 % of the nodes): the reference function is generic
# mini-Ceres, and the file stays within the time of tests/test_ref_solve.py; the GPU file runs it at 25 %
CPU_SCALES = dict(SCENES, cfg4=0.03)
CASES = ("every_third", "tier_moves", "whole_track", "same_track_pair", "tukey_both_fixed", "one_free",
         "empty_mixed", "long_mask")
MOVES = ("cta_to_register", "tile_to_warp2", "nreg_class")
# start values planted on constant and free nodes (float32, as a SolutionFile holds them)
PLANTED = np.array([1.0, -1.0, 0.5, -0.5, np.nextafter(np.float32(0.5), np.float32(1)),
                    np.nextafter(np.float32(-0.5), np.float32(-1)), -0.0, np.float32(1e-40)], np.float32)


def cases_of(name):
    """The cases a scene can hold: cfg1's components are single tracks of at most 2 unknowns, so it has
    no Tukey block and no tier to move across."""
    return tuple(c for c in CASES if not (name == "cfg1" and c in ("tukey_both_fixed", "tier_moves")))


# ---------------------------------------------------------------------------------------------------
# scenes, masks and starts (shared with tests/test_gpu_fixed_tiers.py)
# ---------------------------------------------------------------------------------------------------
def edge_ends(g):
    rp = g["row_ptr"].astype(np.int64)
    src = np.repeat(np.arange(rp.shape[0] - 1), np.diff(rp))
    return src, g["edges"]["dst"].astype(np.int64)


def constant_of(g, fixed):
    """is_const [N] uint8: a root, or a node of an image with a non-zero `fixed` entry."""
    fixed = np.asarray(fixed, bool)
    return ((g["is_root"] != 0) | fixed[g["node_image"].astype(np.int64)]).astype(np.uint8)


def sizes_of(g):
    return np.diff(g["comp_ptr"].astype(np.int64))


def unknowns(g, const):
    """2 x the free nodes of every dispatch slot."""
    sizes = sizes_of(g)
    free = (np.asarray(const)[g["comp_nodes"].astype(np.int64)] == 0).astype(np.int64)
    out = np.zeros(sizes.shape[0], np.int64)
    nz = sizes > 0
    out[nz] = 2 * np.add.reduceat(free, g["comp_ptr"][:-1][nz].astype(np.int64))
    return out


def default_tier(n2):
    """The tier of the default route (tests/test_gpu_tier_options.expected_tier): 1 warp2 (n <= 32),
    2 tile (n <= 80), 3 shared-memory Cholesky warp (n <= 96), 4 CTA; 0 without unknowns."""
    n2 = np.asarray(n2)
    return np.where(n2 == 0, 0, np.where(n2 <= 32, 1, np.where(n2 <= 80, 2, np.where(n2 <= 96, 3, 4))))


def moves(g, const):
    """The tier moves of `const` against the reference's roots, by kind: slots that leave the CTA tier for
    a register tier (n <= 80), leave the tile tier for warp2, or change warp2 NREG class (8 / 16 / 24 / 32)."""
    before, after = unknowns(g, g["is_root"]), unknowns(g, const)
    tb, ta = default_tier(before), default_tier(after)
    solved = sizes_of(g) > 1
    return {"cta_to_register": np.nonzero(solved & (tb == 4) & ((ta == 1) | (ta == 2)))[0],
            "tile_to_warp2": np.nonzero(solved & (tb == 2) & (ta == 1))[0],
            "nreg_class": np.nonzero(solved & (tb == 1) & (ta == 1) & ((before + 7) // 8 != (after + 7) // 8))[0]}


def _tier_moves(g, n_images):
    """For each kind of move, the images of one slot's free nodes, fixed one at a time until that slot
    makes the move; the union over the kinds, kept only where it still makes every move found."""
    root = g["is_root"] != 0
    node_image = g["node_image"].astype(np.int64)
    comp_ptr, comp_nodes = g["comp_ptr"].astype(np.int64), g["comp_nodes"].astype(np.int64)
    tier0 = default_tier(unknowns(g, g["is_root"]))
    fixed = np.zeros(n_images, bool)
    have = set()
    for kind, t_from in (("cta_to_register", 4), ("tile_to_warp2", 2), ("nreg_class", 1)):
        for c in np.nonzero((tier0 == t_from) & (sizes_of(g) > 1))[0][::-1]:      # smallest first
            nodes = comp_nodes[comp_ptr[c]:comp_ptr[c + 1]]
            trial = fixed.copy()
            for k in node_image[nodes[~root[nodes]]]:
                trial[k] = True
                if c in moves(g, constant_of(g, trial))[kind]:
                    break
            got = {m for m, s in moves(g, constant_of(g, trial)).items() if s.size}
            if kind in got and got >= have and trial.sum() <= n_images // 2:
                fixed, have = trial, got
                break
    return fixed


def mask_cases(g, n_images):
    """{case: fixed-by-image-id bool array} of one scene's graph arrays (host stage or plan export)."""
    node_image, track = g["node_image"].astype(np.int64), g["track"].astype(np.int64)
    root = g["is_root"] != 0
    src, dst = edge_ends(g)
    same = track[src] == track[dst]
    tukey = ~same & (g["comp"][src] == g["comp"][dst])
    out = {}
    out["every_third"] = np.arange(n_images) % 3 == 0
    f = _tier_moves(g, n_images)
    if f.any():
        out["tier_moves"] = f
    # all images of a track of at least two nodes: the smallest whose slot keeps a free node, else the smallest
    tsize = np.bincount(track)
    f = None
    for t in np.argsort(tsize, kind="stable"):
        if tsize[t] < 2:
            continue
        trial = np.zeros(n_images, bool)
        trial[node_image[track == t]] = True
        if f is None:
            f = trial
        c = g["comp"][track == t][0]
        if (constant_of(g, trial)[g["comp"] == c] == 0).any():
            f = trial
            break
    out["whole_track"] = f
    # the image of a non-root node with a same-track edge to its track's root
    e = np.nonzero(same & root[src] & ~root[dst])[0][0]
    f = np.zeros(n_images, bool)
    f[node_image[dst[e]]] = True
    out["same_track_pair"] = f
    # the images of both ends of a Tukey edge between two non-roots (a scene without Tukey blocks has none)
    e = np.nonzero(tukey & ~root[src] & ~root[dst] & (node_image[src] != node_image[dst]))[0]
    if e.size:
        f = np.zeros(n_images, bool)
        f[[node_image[src[e[0]]], node_image[dst[e[0]]]]] = True
        out["tukey_both_fixed"] = f
    # a slot left with one free node: every image of its other free nodes, where none holds the one kept
    sizes, comp_ptr, comp_nodes = sizes_of(g), g["comp_ptr"].astype(np.int64), g["comp_nodes"].astype(np.int64)
    n2 = unknowns(g, g["is_root"])
    for c in np.argsort(n2, kind="stable"):
        nodes = comp_nodes[comp_ptr[c]:comp_ptr[c + 1]]
        free = nodes[~root[nodes]]
        if free.size < 2:
            continue
        keep = free[np.argmax(np.bincount(node_image[free]).take(node_image[free]) == 1)]
        others = node_image[free[free != keep]]
        if node_image[keep] in set(others.tolist()):
            continue
        f = np.zeros(n_images, bool)
        f[others] = True
        out["one_free"] = f
        break
    # up to three of the smallest slots with a free node made EMPTY, fixing at most half of the images
    f = np.zeros(n_images, bool)
    n_empty = 0
    for c in np.nonzero((sizes > 1) & (n2 > 0))[0][::-1]:
        nodes = comp_nodes[comp_ptr[c]:comp_ptr[c + 1]]
        trial = f.copy()
        trial[node_image[nodes[~root[nodes]]]] = True
        if trial.sum() > max(1, n_images // 2):
            continue
        f, n_empty = trial, n_empty + 1
        if n_empty == 3:
            break
    out["empty_mixed"] = f
    # longer than the image count; the entries past it name no image
    out["long_mask"] = np.concatenate([np.arange(n_images) % 3 == 1, np.ones(7, bool)])
    return out


def planted_solution(ms, g, seed):
    """A SolutionFile over the scene's nodes (90 % of them; the rest start at 0) with values from
    uniform(-1.5, 1.5) and, on 40 % of the entries, one or both coordinates planted from PLANTED."""
    rng = np.random.default_rng(seed)
    node_image, node_feat = g["node_image"].astype(np.int64), g["node_feat"]
    msgs = []
    for k, name in enumerate(ms.image_names):
        feats = node_feat[node_image == k]
        feats = feats[rng.random(feats.shape[0]) < 0.9]
        vals = rng.uniform(-1.5, 1.5, (feats.shape[0], 2)).astype(np.float32)
        plant = rng.random(feats.shape[0]) < 0.4
        which = rng.integers(0, 3, feats.shape[0])                     # 0: di, 1: dj, 2: both
        pick = PLANTED[rng.integers(0, PLANTED.shape[0], (feats.shape[0], 2))]
        vals[plant & (which != 1), 0] = pick[plant & (which != 1), 0]
        vals[plant & (which != 0), 1] = pick[plant & (which != 0), 1]
        msgs.append(image(name, [displacement(f, a, b) for f, (a, b) in zip(feats.tolist(), vals)]))
    return b"".join(msgs)


def joined_start(ms, g, data):
    """The start point the drop-in joins from SolutionFile bytes."""
    start, _ = wire.join_solution(data, ms.image_names, g["node_image"], g["node_feat"])
    return start


def starts(ms, g, seed):
    return {"zero": np.zeros((g["node_image"].shape[0], 2)), "joined": joined_start(ms, g, planted_solution(ms, g, seed))}


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


_cache = {}


def host_scene(name):
    """(MatchSet, host-stage graph arrays, Problem) of a scene at CPU_SCALES."""
    if name not in _cache:
        ms = synth.generate(name, scale=CPU_SCALES[name])
        skip, g, sz = stage(ms)
        _cache[name] = (ms, g, problem_from_stage(ms, skip, g, sz, "native"))
    return _cache[name]


def host_cases(name):
    """({case: fixed}, {start kind: start}) of host_scene(name)."""
    key = ("cases", name)
    if key not in _cache:
        ms, g, _ = host_scene(name)
        _cache[key] = (mask_cases(g, len(ms.image_names)), starts(ms, g, 17))
    return _cache[key]


def with_mask(p, const):
    import copy
    q = copy.copy(p)
    q.is_root = np.ascontiguousarray(const, np.uint8)
    return q


# ---------------------------------------------------------------------------------------------------
# the judge: the reference function against a solve's positions and statistics
# ---------------------------------------------------------------------------------------------------
def assert_matches_reference(p, got, ref, what, sel=None, cost_rtol=(1e-11, 1e-11), ls_steps=True):
    """Per slot (all, or those of `sel`): positions within 1e-4 px, identical iterations and termination
    codes, initial cost = Summary::initial_cost - fixed_cost and (where the solution is usable) final cost
    = Summary::final_cost - fixed_cost to `cost_rtol`; line-search step totals equal."""
    pos, st = got
    pos_r, st_r = ref
    sizes = np.diff(p.comp_ptr.astype(np.int64))
    sel = np.ones(p.n_components, bool) if sel is None else sel
    err = np.zeros(p.n_components)
    nz = sizes > 0
    err[nz] = np.maximum.reduceat(np.abs(pos - pos_r).max(axis=1)[p.comp_nodes.astype(np.int64)],
                                  p.comp_ptr[:-1][nz].astype(np.int64))
    bad = np.nonzero(sel & ((err > TOL_UNITS) | (st["iterations"] != st_r["iterations"]) |
                            (st["termination"] != st_r["termination"])))[0]
    assert bad.size == 0, (what, [(int(c), int(sizes[c]), float(err[c]), int(st["iterations"][c]), int(st_r["iterations"][c]),
                                   int(st["termination"][c]), int(st_r["termination"][c])) for c in bad[:8]])
    assert np.all(st_r["termination"][sel & (sizes > 1)] > 0), what        # every summary mapped to a code
    np.testing.assert_allclose(st["initial_cost"][sel], (st_r["initial_cost"] - st_r["fixed_cost"])[sel],
                               rtol=cost_rtol[0], atol=1e-14, err_msg=str(what))
    usable = sel & (sizes > 1) & (st_r["termination"] != 6)
    np.testing.assert_allclose(st["final_cost"][usable], (st_r["final_cost"] - st_r["fixed_cost"])[usable],
                               rtol=cost_rtol[1], atol=1e-14, err_msg=str(what))
    if ls_steps:
        assert st["total_line_search_steps"] == st_r["total_line_search_steps"], what
    return float(err[sel].max(initial=0.0))


# ---------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------
def test_reference_solve_library_is_built():
    """The reference's create_and_solve_problem as a library: built with the package, never skipped."""
    assert load_refsolve() is not None


@pytest.mark.parametrize("name", list(SCENES))
def test_mask_cases_hold_what_they_claim(name):
    ms, g, p = host_scene(name)
    n_images = len(ms.image_names)
    node_image, track = g["node_image"].astype(np.int64), g["track"].astype(np.int64)
    root = g["is_root"] != 0
    src, dst = edge_ends(g)
    same = track[src] == track[dst]
    tukey = ~same & (g["comp"][src] == g["comp"][dst])
    sizes = sizes_of(g)
    n2_0 = unknowns(g, g["is_root"])
    cases = host_cases(name)[0]
    assert set(cases) == set(cases_of(name))
    if name == "cfg1":
        assert not tukey.any() and n2_0.max() <= 8      # one track per component, one NREG class
    for case, fixed in cases.items():
        const = constant_of(g, fixed).astype(bool)
        assert fixed[:n_images].any() and not fixed[:n_images].all(), case
        n2 = unknowns(g, const)
        assert (n2[sizes > 1] > 0).sum() >= (sizes > 1).sum() // 3, (case, "most slots keep free nodes")
        # same-track blocks with both ends constant: one end a node that is not its track's root
        assert (same & const[src] & const[dst] & ~(root[src] & root[dst])).any(), case
        if case == "whole_track":
            tsize = np.bincount(track)
            whole = np.nonzero((tsize >= 2) & (np.bincount(track, weights=const) == tsize))[0]
            comp_of_t = np.zeros(tsize.shape[0], np.int64)
            comp_of_t[track] = g["comp"]
            # a whole constant track inside a slot that is still solved
            alive = set(np.asarray(g["comp"])[g["comp_nodes"][g["comp_ptr"][:-1][(sizes > 1) & (n2 > 0)].astype(np.int64)]].tolist())
            assert any(not root[track == t].all() for t in whole), case
            assert any(int(comp_of_t[t]) in alive for t in whole) or name == "cfg1", case
        if case == "same_track_pair":
            assert (same & root[src] & const[dst] & ~root[dst]).any(), case
        if case == "tukey_both_fixed":
            assert (tukey & const[src] & const[dst] & ~root[src] & ~root[dst]).any(), case
        if case == "one_free":
            assert ((n2 == 2) & (n2_0 > 2) & (sizes > 1)).any(), case
        if case == "empty_mixed":
            made_empty = (sizes > 1) & (n2 == 0) & (n2_0 > 0)
            assert made_empty.sum() >= 1 and ((sizes > 1) & (n2 > 0)).sum() >= (sizes > 1).sum() // 2, case
        if case == "long_mask":
            assert fixed.shape[0] > n_images and fixed[n_images:].all()
            assert np.array_equal(const, constant_of(g, fixed[:n_images]).astype(bool))
        if case == "tier_moves":
            got = {m for m, s in moves(g, const).items() if s.size}
            want = {"cfg1": set(), "cfg2": {"nreg_class"}, "cfg4": {"tile_to_warp2", "nreg_class"},
                    "ring60": set(MOVES)}[name]
            assert got >= want, (case, got)


@pytest.mark.parametrize("name", list(SCENES))
def test_planted_starts_reach_constant_and_free_nodes(name):
    """Every planted value sits on a constant and on a free node of a solved slot under every case; the
    joined start holds values outside the box, and nodes without an entry start at +0.0."""
    ms, g, p = host_scene(name)
    cases, x = host_cases(name)
    x0 = x["joined"]
    assert np.abs(x0).max() > 1.0 and (bits(x0) == 0).any()
    in_solved = np.zeros(x0.shape[0], bool)
    in_solved[p.comp_nodes[np.repeat(sizes_of(g) > 1, sizes_of(g))].astype(np.int64)] = True
    for case, fixed in cases.items():
        const = constant_of(g, fixed).astype(bool)
        for v in PLANTED.astype(np.float64):
            hit = (bits(x0) == bits(np.array([v]))[0]).any(axis=1) & in_solved
            assert (hit & const).any() and (hit & ~const).any(), (case, v)


@pytest.mark.parametrize("name,case", [(n, c) for n in SCENES for c in cases_of(n)])
def test_reference_function_equals_the_checker(oracle, name, case):
    """create_and_solve_problem on the mask and start against the CPU checker's lfr_solve on the same
    arrays, from zeros and from the joined start: the same iterations, terminations, line-search steps
    and costs, positions to 1e-4 px (in practice to ~1e-15), constant nodes at their start bits."""
    ms, g, p = host_scene(name)
    cases, x = host_cases(name)
    const = constant_of(g, cases[case])
    q = with_mask(p, const)
    for kind, x0 in x.items():
        ref = ref_solve(p, const, x0)
        pos, st = oracle.solve(q, oracle.default_options(n_threads=8), positions=x0)
        err = assert_matches_reference(q, (pos, st), ref, (name, case, kind))
        assert err <= 1e-12, (name, case, kind, err)
        c = const.astype(bool)
        assert np.array_equal(bits(pos[c]), bits(x0[c])) and np.array_equal(bits(ref[0][c]), bits(x0[c]))
        assert ref[1]["n_solved"] == int((sizes_of(g) > 1).sum()) == st["n_solved"]
        if case == "empty_mixed":
            assert (ref[1]["termination"] == EMPTY).sum() >= 1 and (st["termination"] == EMPTY).sum() >= 1
