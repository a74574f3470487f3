"""Every solve tier's line-search trial, its slope, the accepted and the rejected step's bookkeeping and
the second LM step against an extended-precision statement (tests/lm_step_ref.py: probe, step_at).

Whole solves against the oracle cannot see a slightly wrong phi' or trial cost: the interpolated step
moves a little inside [1e-3, 0.6] alpha, Armijo still accepts it and the solve converges to the same
point.  liblfr_b200_lsprobe.so is the product built with -DLFR_DBG_LS_PROBE (csrc/build.py): every
component takes its first LM step at the initial radius, then calls the driver's members in a fixed
order.  The mode and alpha are passed as line_search_sufficient_function_decrease, which only the Armijo
test reads and which this build never reaches:
  mode A (0 < value <= 1 = alpha): trial(alpha), step_norm(), trial_slope(alpha), slope(), accept(),
    assemble(false); dl goes to the free nodes' positions and {cost by trial, cost by trial_slope, phi'
    by trial_slope, phi' by slope(), |x - xc|, |xc|, gmax at xc, tier} to the slot's LFR_DBG_PROFILE
    record;
  mode B (value = -alpha): the same, then a second lm_step from xc with iteration 0's Jacobi scaling;
    dl2 and the record of the LFR_DBG_LM_STEP build;
  mode C (value > 1): trial(1), slope(), reject() and lm_step at half the radius from the unchanged x,
    the driver's path after a rejected step; dl2 and the same record.

alpha is 1, 2^-1, 2^-10 (about Ceres' 1e-3 contraction) or 2^-30: a power of two, so x + alpha dl rounds
once, FMA or not, and xc = clip(fl(x + alpha dl), +-bound) is known on the host bit for bit.  Every value
is held to a bound derived from the kernels' arithmetic at that point (lm_step_ref.PROBE_BOUNDS), not to
a tolerance fitted to their output:
  * the cost from trial and from trial_slope within the cost bound, and bitwise equal to each other;
  * phi' from trial_slope and from slope() within the phi' bound; phi' is the full gradient at xc dotted
    with dl, so the coordinates the box clips count too;
  * |x - xc| and |xc| within gamma_{n+1} / 2 + u relative; gmax at xc within the largest per-coordinate
    gradient bound;
  * dl bitwise the same at every alpha, and bitwise liblfr_b200_lmstep.so's step; mode B's cost and gmax at xc bitwise those of mode A at alpha 1 (the same first step);
  * modes B and C: the criteria of test_gpu_lm_step.check for dl2 against step_at(xc, S0) and against
    first_step at half the radius, kappa of that damped system, with the gradient's evaluation error at
    the point added to the solve's bound (second_step_bound);
  * roots untouched; the queue kernel's record and positions bitwise those of the per-bucket launch.
Cases: the components of test_gpu_lm_step (every class edge, the CTA past 1008 free nodes / 1024 nodes /
1969 free nodes, the structure problem, the conditioning set, the weak clusters) and two more: "box",
starts with |x| in [0.9, 1] at radius 1e16, so the projection binds at alpha = 1, and "bound_0.05".  Each
runs on the five routes of test_gpu_tier_options.ROUTES.  The module ends by printing, per tier and per
quantity, the largest error / bound ratio.
"""
import os

import numpy as np
import pytest

import lm_step_ref as ref
from test_gpu_lm_step import (COND_SIZES, CONDITIONING, MAX_BOUND, TIER_NAMES, component, conditioning_problem,
                              first_steps, large_problem, problem, sizes_problem, start_point, structure_problem,
                              weak_problem)
from test_gpu_tier_options import ROUTES, TIER_WARP, expected_tier

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "local-feature-refinement_b200", "csrc")
LSPROBE_LIB = os.path.join(CSRC, "liblfr_b200_lsprobe.so")
LMSTEP_LIB = os.path.join(CSRC, "liblfr_b200_lmstep.so")
U = 2.0 ** -53
ALPHAS = (1.0, 2.0 ** -1, 2.0 ** -10, 2.0 ** -30)


# ---------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------
def box_problem():
    rng = np.random.default_rng(20)
    return problem([component(rng, n, 2) for n in COND_SIZES + (8, 30)])


def box_start(p, seed=20):
    """|x| in [0.9, 1], one sign per component and axis (so that the residuals stay Tukey inliers), the
    roots on the bound: the first step at radius 1e16 spreads the free nodes around the roots, out of the
    box."""
    rng = np.random.default_rng(seed)
    sign = rng.choice([-1.0, 1.0], (p.n_components, 2))[p.comp.astype(np.int64)]
    x = rng.uniform(0.9, 1.0, (p.graph.n_nodes, 2))
    x[p.is_root != 0] = 1.0
    return x * sign


def bound_problem():
    rng = np.random.default_rng(21)
    return problem([component(rng, n, 2) for n in COND_SIZES])


# key: (problem, options, start)
CASES = dict({"sizes": (sizes_problem, {}, lambda p: start_point(p, "inside", 1)),
              "large": (large_problem, {}, lambda p: start_point(p, "inside", 2)),
              "structure": (structure_problem, {}, lambda p: start_point(p, "inside", 3)),
              "weak": (weak_problem, dict(initial_trust_region_radius=1e16), lambda p: start_point(p, "zero")),
              "box": (box_problem, dict(initial_trust_region_radius=1e16, tukey_a=0.5), box_start),
              "bound_0.05": (bound_problem, dict(bound=0.05), lambda p: start_point(p, "inside", 21))},
             **{k: ((lambda k=k: conditioning_problem(k)), v[0], (lambda p, kind=v[1]: start_point(p, kind, 4)))
                for k, v in CONDITIONING.items()})

_made = {}


def case(key):
    """(problem, options dict, start, lfr_options of the oracle library, first steps of the statement)."""
    if key not in _made:
        from oracle_util import load_oracle
        make, opts, start = CASES[key]
        p = make()
        x0 = start(p)
        o = load_oracle().default_options(**opts)
        firsts = [ref.first_step(p, s, o, x0, want_kappa=False) for s in range(p.n_components)]
        _made[key] = (p, opts, x0, o, firsts)
    return _made[key]


# ---------------------------------------------------------------------------------------------------
# running the diagnostic build
# ---------------------------------------------------------------------------------------------------
def _library(path):
    import ctypes as C
    from lfr_b200.capi import Library
    lib = Library(path)
    f = lib.lib.lfr_debug_plan_cycles
    f.argtypes = [C.c_void_p, C.c_void_p]
    f.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def lsprobe():
    return _library(LSPROBE_LIB)


@pytest.fixture(scope="module")
def lmstep():
    return _library(LMSTEP_LIB)


def run(lib, p, route, start, alpha, opts, mode="A"):
    """(positions [N, 2], records [C, 8]) of one probe launch: mode A or B at alpha, or mode C."""
    suff = {"A": alpha, "B": -alpha, "C": 2.0}[mode]
    return first_steps(lib, p, route, start, line_search_sufficient_function_decrease=suff, **opts)


QUANTITIES = ("cost", "phi' trial_slope", "phi' slope", "|x - xc|", "|xc|", "gmax", "step 2", "rejected")


@pytest.fixture(scope="module")
def report(request):
    """Per tier and quantity the largest error / bound ratio; printed at the end of the module past output
    capture."""
    worst = {}
    yield worst
    tr = request.config.pluginmanager.getplugin("terminalreporter")
    cm = request.config.pluginmanager.getplugin("capturemanager")
    lines = []
    for t in sorted(k for k in worst if isinstance(k, int)):
        w = worst[t]
        lines.append("line-search probe, %-5s %5d probes: " % (TIER_NAMES[t], w["n"]) +
                     ", ".join("%s %.3e" % (q, w.get(q, 0.0)) for q in QUANTITIES) +
                     "; dl bitwise the lmstep build's in %d components" % w["same"])
    if tr is None or cm is None:
        print("\n".join(lines))
        return
    with cm.global_and_fixture_disabled():
        tr.write_line("")
        for line in lines:
            tr.write_line(line)


def _note(report, tier, q, ratio):
    w = report.setdefault(tier, {"n": 0, "same": 0})
    w[q] = max(w.get(q, 0.0), ratio)


def check_mode_a(lib, report, key, route, alpha, dl_seen):
    p, opts, x0, o, firsts = case(key)
    pos, rec = run(lib, p, route, x0, alpha, opts)
    roots = p.is_root != 0
    assert np.array_equal(pos[roots], x0[roots]), (key, route, alpha, "roots moved")
    for s, st in enumerate(firsts):
        what = (key, route, alpha, s, st.n)
        cost_t, cost_s, dphi_t, dphi_s, dn, xn, gmax, tier = rec[s]
        tier = int(tier)
        assert tier == expected_tier(st.n, route), (what, tier)
        dl = pos[st.free_nodes]
        if s in dl_seen:
            assert np.array_equal(dl, dl_seen[s]), (what, "dl differs between launches")
        dl_seen[s] = dl
        pr = ref.probe(p, s, o, x0, dl, alpha)
        assert cost_t == cost_s, (what, "trial and trial_slope costs differ", cost_t, cost_s)
        assert abs(cost_t - pr.cost) <= pr.cost_bound, (what, "cost", cost_t, pr.cost, pr.cost_bound)
        assert abs(dphi_t - pr.dphi) <= pr.dphi_bound, (what, "phi' trial_slope", dphi_t, pr.dphi, pr.dphi_bound)
        assert abs(dphi_s - pr.dphi) <= pr.dphi_bound, (what, "phi' slope", dphi_s, pr.dphi, pr.dphi_bound)
        assert abs(dn - pr.dn) <= pr.norm_bound * pr.dn, (what, "|x - xc|", dn, pr.dn)
        assert abs(xn - pr.xn) <= pr.norm_bound * pr.xn, (what, "|xc|", xn, pr.xn)
        assert abs(gmax - pr.gmax) <= pr.gmax_bound, (what, "gmax", gmax, pr.gmax, pr.gmax_bound)
        _note(report, tier, "cost", abs(cost_t - pr.cost) / pr.cost_bound)
        _note(report, tier, "phi' trial_slope", abs(dphi_t - pr.dphi) / pr.dphi_bound)
        _note(report, tier, "phi' slope", abs(dphi_s - pr.dphi) / pr.dphi_bound)
        _note(report, tier, "|x - xc|", abs(dn - pr.dn) / (pr.norm_bound * pr.dn) if pr.dn else 0.0)
        _note(report, tier, "|xc|", abs(xn - pr.xn) / (pr.norm_bound * pr.xn) if pr.xn else 0.0)
        _note(report, tier, "gmax", abs(gmax - pr.gmax) / pr.gmax_bound if pr.gmax_bound else 0.0)
        report[tier]["n"] += 1
    return pos, rec


def second_step_bound(st2, pr):
    """(8 n kappa u, eta, |dy|, max A_ii) of the second step st2 at the probe's xc.  The kernels' g at xc
    carries evaluation errors up to pr.g_bound (PROBE_BOUNDS (5)); near the optimum they are not small
    against |g|.  They move y = A^-1 S g by at most |dy| = |A^-1|_2 |S gb|_2, |A^-1|_2 <= kappa / max A_ii,
    and dl = -S y by eta = max S |dy|, on top of the solve's 8 n kappa u."""
    a_max = float(st2.A.vals[st2.A.rows == st2.A.cols].max())
    ey = st2.kappa / a_max * float(np.linalg.norm(st2.S.astype(np.float64) * pr.g_bound.astype(np.float64)))
    return ref.step_bound(st2.n, st2.kappa), float(np.abs(st2.S).max()) * ey, ey, a_max


def judge_step(report, what, rec_row, dl, st2, pr, quantity):
    """One slot's second step (mode B or C) against the statement st2 at the probe's point: the criteria
    of test_gpu_lm_step.check, with the gradient's evaluation error at that point added to the solve's
    bound (second_step_bound).  A slot whose bound exceeds MAX_BOUND could not fail and is skipped
    (test_ls_probe_ref.test_cases_are_meaningful counts them)."""
    cost, gmax, valid, mc, gd, dmax, tier, n_rec = rec_row
    n = st2.n
    assert valid == 1.0 and int(n_rec) == n, (what, rec_row)
    bound, eta, ey, a_max = second_step_bound(st2, pr)
    norm = float(np.linalg.norm(st2.dl.astype(np.float64)))
    assert abs(cost - st2.cost) <= pr.cost_bound, (what, "cost", cost, st2.cost)
    assert abs(gmax - st2.gmax) <= pr.gmax_bound, (what, "gmax", gmax, st2.gmax)
    if bound * norm + eta > MAX_BOUND * norm:
        return
    gb = pr.g_bound.astype(np.float64)
    g2 = np.abs(st2.b / st2.S).astype(np.float64)
    err = float(np.sqrt((((dl.astype(ref.LD) - st2.dl) ** 2).sum()).astype(np.float64)))
    assert err <= bound * norm + eta, (what, "step", err / norm, bound, eta / norm, st2.kappa)
    adl = np.abs(dl.reshape(-1))
    tol_gd = bound * abs(st2.gd) + float((gb * adl).sum()) + eta * float(np.linalg.norm(g2))
    # model change 1/2 y . (S g + D^2 y)
    tol_mc = bound * abs(st2.model_change) + 0.5 * float((gb * adl).sum()) + 0.5 * ey * (
        float(np.linalg.norm(st2.b.astype(np.float64))) + 2 * a_max * float(np.linalg.norm(st2.y.astype(np.float64))))
    assert abs(mc - st2.model_change) <= tol_mc, (what, "model change", mc, st2.model_change, tol_mc)
    assert abs(gd - st2.gd) <= tol_gd, (what, "g . dl", gd, st2.gd, tol_gd)
    assert abs(dmax - np.abs(st2.dl.astype(np.float64)).max()) <= bound * norm + eta, (what, "|dl|_inf")
    assert dmax == np.abs(dl).max(), what
    if int(tier) == TIER_WARP:   # dense Cholesky: backward stable
        y = -dl.reshape(-1).astype(ref.LD) / st2.S
        a_norm = float(np.abs(st2.A.dense()).sum(axis=1).max())
        res = float(np.abs(st2.A.matvec(y) - st2.b).max())
        bwd = res / (a_norm * float(np.abs(y).max()) + float(np.abs(st2.b).max()))
        assert bwd <= 8 * n * U, (what, "backward error", bwd)
    _note(report, int(tier), quantity, err / (bound * norm + eta) if norm else 0.0)


def check_mode_b(lib, report, key, route, rec_a, dl_a):
    """Mode B at alpha = 1 against step_at(xc, S0), xc from mode A's dl (the same first step: its cost and
    gmax at xc must be mode A's bit for bit)."""
    p, opts, x0, o, firsts = case(key)
    pos, rec = run(lib, p, route, x0, 1.0, opts, mode="B")
    roots = p.is_root != 0
    assert np.array_equal(pos[roots], x0[roots]), (key, route, "roots moved")
    for s, st in enumerate(firsts):
        what = (key, route, "mode B", s, st.n)
        assert int(rec[s, 6]) == expected_tier(st.n, route), (what, rec[s, 6])
        assert rec[s, 0] == rec_a[s, 0] and rec[s, 1] == rec_a[s, 6], (what, "not mode A's first step")
        pr = ref.probe(p, s, o, x0, dl_a[s], 1.0)
        judge_step(report, what, rec[s], pos[st.free_nodes], ref.step_at(p, s, o, pr.xc, S=st.S), pr, "step 2")


def check_mode_c(lib, report, key, route):
    """Mode C: the step after a rejected one, from the unchanged x at half the initial radius, against
    first_step at that radius (the gradient at x, not at the trial point slope() evaluated)."""
    p, opts, x0, o, firsts = case(key)
    pos, rec = run(lib, p, route, x0, 1.0, opts, mode="C")
    roots = p.is_root != 0
    assert np.array_equal(pos[roots], x0[roots]), (key, route, "roots moved")
    radius = 0.5 * o.initial_trust_region_radius
    for s, st in enumerate(firsts):
        what = (key, route, "mode C", s, st.n)
        assert int(rec[s, 6]) == expected_tier(st.n, route), (what, rec[s, 6])
        pr = ref.probe(p, s, o, x0, np.zeros((len(st.free_nodes), 2)), 1.0)
        judge_step(report, what, rec[s], pos[st.free_nodes], ref.first_step(p, s, o, x0, radius=radius), pr,
                   "rejected")


def check_case(lsprobe, lmstep, report, key, route):
    p, opts, x0, _, firsts = case(key)
    dl_seen = {}
    recs = {}
    for alpha in ALPHAS:
        pos, recs[alpha] = check_mode_a(lsprobe, report, key, route, alpha, dl_seen)
    check_mode_b(lsprobe, report, key, route, recs[1.0], dl_seen)
    check_mode_c(lsprobe, report, key, route)
    pos_l, _ = first_steps(lmstep, p, route, x0, **opts)
    for s, st in enumerate(firsts):
        assert np.array_equal(pos_l[st.free_nodes], dl_seen[s]), (key, route, s, "not the lmstep build's dl")
        report[int(recs[1.0][s, 7])]["same"] += 1


# ---------------------------------------------------------------------------------------------------
# the tests
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("key", list(CASES))
def test_probe(lsprobe, lmstep, report, key, route):
    check_case(lsprobe, lmstep, report, key, route)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["A", "B", "C"])
def test_queue_is_the_per_bucket_launch(lsprobe, mode):
    """Components of at most 16 unknowns run the per-bucket kernels alone and the queue kernel next to
    one of 18 unknowns: the same positions and records, bit for bit."""
    rng = np.random.default_rng(6)
    small = [component(rng, n // 2, 1) for n in (2, 4, 8, 10, 12, 16)]
    wide = component(rng, 9, 1)
    alone, with_wide = problem(small), problem(small + [wide])
    start = start_point(with_wide, "inside", 6)
    n_small = alone.graph.n_nodes
    pos_a, rec_a = run(lsprobe, alone, "default", start[:n_small], 2.0 ** -1, {}, mode)
    pos_q, rec_q = run(lsprobe, with_wide, "default", start, 2.0 ** -1, {}, mode)
    assert np.array_equal(pos_a, pos_q[:n_small])
    assert np.array_equal(rec_a.view(np.uint64), rec_q[:len(small)].view(np.uint64))
