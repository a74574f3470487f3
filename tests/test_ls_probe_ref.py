"""The line-search probe of the extended-precision statement (tests/lm_step_ref.py: probe, step_at) on the
CPU.

Five ties keep the statement honest before it judges the GPU tiers (tests/test_gpu_ls_probe.py):
  1. phi'* = grad f(xc) . dl against a central difference of f(xc + t dl) in mpmath at 40 digits, where
     no coordinate is clamped and no Tukey edge or grid clamp is crossed within the stencil;
  2. on a hand-built case with clamped coordinates: phi'* is the full gradient's dot product (the
     derivative of f(xc + t dl)), and that differs from the derivative of the projected path
     f(P(x + (alpha + t) dl)) by the clamped coordinates' share;
  3. the trial cost and phi'* against the oracle's harvested line-search states (Ceres'
     LineSearchFunction) on single components whose first full step fails the Armijo test;
  4. the second step against the oracle's second iteration, with iteration 0's Jacobi scaling kept, and
     a recomputed scaling shown to miss;
  5. the bounds have teeth: none looser than 1e-9 of its magnitude sum, and on every tier some case
     where a clamped coordinate's, a duplicated edge's or an M / M^T confusion's share of phi' exceeds
     the phi' bound; the box cases clamp; some sources cross the +-0.5 grid clamp.
"""
import types

import numpy as np
import pytest

import lm_step_ref as ref
import test_gpu_ls_probe as gp
from test_gpu_lm_step import MAX_BOUND, component, problem, sizes_problem, start_point
from test_gpu_tier_options import ROUTES, expected_tier

U = 2.0 ** -53


# ---------------------------------------------------------------------------------------------------
# an independent evaluation of f in mpmath
# ---------------------------------------------------------------------------------------------------
def mp_cost(mpmath, p, slot, ov, x):
    """1/2 sum sim rho over the kept edges of `slot` at positions x (a dict node -> (mpf, mpf))."""
    src, dst, eidx, kind = ref.kept_blocks(p, slot)
    e = p.graph.edges[eidx]
    half, one = mpmath.mpf(1) / 2, mpmath.mpf(1)
    total = mpmath.mpf(0)
    for k in range(len(src)):
        xs, xd = x[int(src[k])], x[int(dst[k])]
        D = e["flow"][k].astype(np.float64).reshape(3, 3, 2)
        c = [min(max(v, -half), half) for v in xs]
        lag = [[2 * t * (t - half), -4 * (t - half) * (t + half), 2 * t * (t + half)] for t in c]
        r = [xd[q] - xs[q] - sum(lag[0][i] * lag[1][j] * mpmath.mpf(float(D[i, j, q]))
                                  for i in range(3) for j in range(3)) for q in range(2)]
        s = r[0] ** 2 + r[1] ** 2
        sim = mpmath.mpf(float(np.float64(e["sim"][k])))
        if kind[k] == ref.CAUCHY:
            b = mpmath.mpf(ov["cauchy_a"]) ** 2
            rho = b * mpmath.log(one + s / b)
        else:
            a2 = mpmath.mpf(ov["tukey_a"]) ** 2
            w = 3 if int(ov["tukey_variant"]) == 2 else 6
            rho = a2 / w * (one - (one - min(s, a2) / a2) ** 3)
        total += sim * rho
    return total / 2


def mp_slope(mpmath, p, slot, ov, base, dl, free_nodes, h, project=None):
    """Central difference along t of f(base + t dl) at t = 0 (or of f(P(base + t dl)) with `project`
    the bound), mpmath at 40 digits."""
    mpmath.mp.dps = 40
    nodes = p.comp_nodes[p.comp_ptr[slot]:p.comp_ptr[slot + 1]].astype(np.int64)
    fi = {int(v): k for k, v in enumerate(free_nodes)}

    def f(t):
        x = {}
        for v in nodes:
            v = int(v)
            pt = [mpmath.mpf(float(base[v, q])) for q in range(2)]
            if v in fi:
                pt = [pt[q] + t * mpmath.mpf(float(dl[fi[v], q])) for q in range(2)]
                if project is not None:
                    pt = [min(max(c, -mpmath.mpf(project)), mpmath.mpf(project)) for c in pt]
            x[v] = pt
        return mp_cost(mpmath, p, slot, ov, x)

    h = mpmath.mpf(h)
    return float((f(h) - f(-h)) / (2 * h)), float(f(0))


# ---------------------------------------------------------------------------------------------------
# 1. phi'* against mpmath
# ---------------------------------------------------------------------------------------------------
def test_slope_matches_mpmath(oracle):
    """Slots of up to 34 unknowns of the class-edge problem at alpha = 1/2 from an inside start: phi'* and
    the cost within 1e-17 of their magnitude sums of mpmath's central difference (h = 1e-12) and value."""
    mpmath = pytest.importorskip("mpmath")
    p = sizes_problem()
    x0 = start_point(p, "inside", 1)
    o = oracle.default_options()
    ov = ref.option_values(o)
    a2 = ov["tukey_a"] ** 2
    checked = 0
    for s in range(p.n_components):
        st = ref.first_step(p, s, o, x0, want_kappa=False)
        if st.n > 34:
            continue
        dl = st.dl.astype(np.float64)
        pr = ref.probe(p, s, o, x0, dl, 0.5)
        src, dst, _, _ = ref.kept_blocks(p, s)
        r, _ = ref.edge_terms(p.graph.edges["flow"][ref.kept_blocks(p, s)[2]], pr.xc[src], pr.xc[dst])
        sq = (r * r).sum(axis=1).astype(np.float64)
        # the stencil moves a coordinate by at most 1e-12: no clamp, no Tukey threshold, no grid edge
        assert not pr.clamped.any()
        assert np.all(np.abs(sq - a2) > 1e-9) and np.all(np.abs(np.abs(pr.xc[src]) - 0.5) > 1e-9)
        d, f0 = mp_slope(mpmath, p, s, ov, pr.xc, dl, st.free_nodes, 1e-12)
        assert abs(pr.dphi - d) <= 1e-17 * pr.dphi_mag, (s, pr.dphi, d)
        assert abs(pr.cost - f0) <= 1e-17 * pr.cost_mag, (s, pr.cost, f0)
        checked += 1
    assert checked >= 8


# ---------------------------------------------------------------------------------------------------
# 2. clamped coordinates
# ---------------------------------------------------------------------------------------------------
def test_clamped_coordinates_count_in_the_slope(oracle):
    """Three free nodes near the bound and a step that pushes four of their six coordinates out of the
    box: phi'* is the derivative of f(xc + t dl) (the full gradient at xc dotted with dl), which differs
    from the derivative of the projected path f(P(x + (1 + t) dl)) by exactly the clamped share."""
    mpmath = pytest.importorskip("mpmath")
    rng = np.random.default_rng(7)
    p = problem([component(rng, 3, 1)])
    o = oracle.default_options()
    ov = ref.option_values(o)
    nodes = p.comp_nodes.astype(np.int64)
    free = nodes[p.is_root[nodes] == 0]
    x0 = np.full((p.graph.n_nodes, 2), 0.3)
    x0[free] = [[0.95, -0.9], [0.92, 0.97], [-0.96, 0.1]]
    dl = np.array([[0.2, -0.25], [-0.1, 0.125], [-0.15, 0.05]])
    pr = ref.probe(p, 0, o, x0, dl, 1.0)
    assert pr.clamped.sum() == 4
    full, _ = mp_slope(mpmath, p, 0, ov, pr.xc, dl, free, 1e-12)
    x = x0.copy()
    x[free] = np.clip(x0[free], -1, 1)
    x[free] += dl                                   # P(x + (1 + t) dl) = P(x + dl + t dl)
    projected, _ = mp_slope(mpmath, p, 0, ov, x, dl, free, 1e-12, project=1.0)
    assert abs(pr.dphi - full) <= 1e-17 * pr.dphi_mag
    share = float((pr.g * dl.reshape(-1))[pr.clamped.reshape(-1)].sum())
    assert abs((pr.dphi - projected) - share) <= 1e-15 * pr.dphi_mag    # (a difference taken in double)
    assert abs(pr.dphi - projected) == pytest.approx(pr.clamped_share, rel=1e-12)
    assert pr.clamped_share > 1e6 * pr.dphi_bound


# ---------------------------------------------------------------------------------------------------
# 3. the trial cost and phi'* against the oracle's line search
# ---------------------------------------------------------------------------------------------------
def _harvest(oracle, q, o, x0):
    oracle.lib.lfr_ref_harvest(1)
    try:
        oracle.solve(q, o, positions=x0)
        n = int(oracle.lib.lfr_ref_harvest_take(None, 0))
        states = np.zeros((n, 11))
        if n:
            oracle.lib.lfr_ref_harvest_take(states.ctypes.data, n)
    finally:
        oracle.lib.lfr_ref_harvest(0)
    return states


def _unbounded(o):
    """The statement's option values with the box removed (for gradients on both sides of a bound)."""
    ov = ref.option_values(o)
    ov["bound"] = 1e300
    return types.SimpleNamespace(**ov)


def hessian_norm(q, slot, o, xc, free_nodes, h=1e-6):
    """|grad^2 f(xc)|_2 by central differences of the longdouble gradient (truncation ~h^2)."""
    ou = _unbounded(o)
    n = 2 * len(free_nodes)
    zero = np.zeros((len(free_nodes), 2))
    H = np.zeros((n, n))
    for i in range(n):
        xp, xm = xc.copy(), xc.copy()
        xp[free_nodes[i // 2], i % 2] += h
        xm[free_nodes[i // 2], i % 2] -= h
        H[:, i] = ((ref.probe(q, slot, ou, xp, zero, 1.0).g - ref.probe(q, slot, ou, xm, zero, 1.0).g)
                   / (2 * h)).astype(np.float64)
    return float(np.linalg.norm((H + H.T) / 2, 2))


def test_trial_matches_the_oracles_line_search(oracle):
    """Components of the line-search fixture, from zero and from a start spread over the box, whose
    first full step (max_num_iterations = 1) fails the Armijo test: the oracle's (f_1, phi'_1) at step 1
    equal probe(dl*, 1) within the evaluation bounds plus what |dl - dl*| <= 8 n kappa u |dl*| can move
    them: |grad f| |dl - dl*| for f, (|grad f| + |grad^2 f| |dl|) |dl - dl*| for phi'."""
    import os
    from lfr_b200 import build_problem, wire
    from test_gpu_cta_limits import subset
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "linesearch_matches.pb")
    with open(path, "rb") as fh:
        p = build_problem(wire.decode_matching_file(fh.read()))
    sizes = np.diff(p.comp_ptr.astype(np.int64))
    compared = clamped = 0
    for s in np.nonzero(sizes >= 2)[0]:
        q = subset(p, [int(s)])
        for kind in ("zero", "box"):
            x0 = np.zeros((q.graph.n_nodes, 2)) if kind == "zero" else \
                np.random.default_rng(int(s)).uniform(-1, 1, (q.graph.n_nodes, 2))
            o = oracle.default_options(n_threads=1, max_num_iterations=1)
            states = _harvest(oracle, q, o, x0)
            if not len(states):
                continue
            assert states[0, 2] == 1.0                        # the first contraction, from the full step
            st = ref.first_step(q, 0, o, x0)
            assert st.kappa <= 1e4
            dl = st.dl.astype(np.float64)
            pr = ref.probe(q, 0, o, x0, dl, 1.0)
            e = ref.step_bound(st.n, st.kappa) * float(np.linalg.norm(dl))
            gn = float(np.linalg.norm(pr.g.astype(np.float64)))
            hn = hessian_norm(q, 0, o, pr.xc, st.free_nodes)
            tol_f = pr.cost_bound + e * gn
            tol_g = pr.dphi_bound + e * (gn + hn * float(np.linalg.norm(dl)))
            assert abs(states[0, 3] - pr.cost) <= tol_f, (s, kind, states[0, 3], pr.cost, tol_f)
            assert abs(states[0, 4] - pr.dphi) <= tol_g, (s, kind, states[0, 4], pr.dphi, tol_g)
            compared += 1
            clamped += int(pr.clamped.any())
    assert compared >= 4 and clamped >= 1, (compared, clamped)


# ---------------------------------------------------------------------------------------------------
# 4. the second step against the oracle
# ---------------------------------------------------------------------------------------------------
def two_full_steps(oracle, opts):
    """(q, x0, x1, x2, options, S0, radius1) of the small components on which the oracle takes two full
    steps (no line-search step, both accepted, x2 strictly inside the box) and whose first step's
    statement has rho >= 0.95, so that the radius after it is exactly 3x the initial one."""
    from test_lm_step_ref import small_components
    out = []
    for q, slot in small_components():
        N = q.graph.n_nodes
        for x0 in (np.zeros((N, 2)), np.random.default_rng(int(q.comp_nodes[0])).uniform(-0.6, 0.6, (N, 2))):
            o1 = oracle.default_options(n_threads=1, max_num_iterations=1, **opts)
            o2 = oracle.default_options(n_threads=1, max_num_iterations=2, **opts)
            x1, s1 = oracle.solve(q, o1, positions=x0)
            x2, s2 = oracle.solve(q, o2, positions=x0)
            st = ref.first_step(q, slot, o1, x0, want_kappa=False)
            f = st.free_nodes
            if s1["total_line_search_steps"] or s2["total_line_search_steps"] or s2["iterations"][0] != 2 \
                    or s2["termination"][0] != 5 or np.array_equal(x1[f], x0[f]) or np.array_equal(x2[f], x1[f]) \
                    or np.abs(x2[f]).max() >= 1.0:
                continue
            cost1 = ref.probe(q, slot, o1, x1, np.zeros((len(f), 2)), 1.0).cost
            rho = (st.cost - cost1) / st.model_change
            if rho < 0.95:
                continue
            # TrustRegionMinimizer: radius / max(1/3, 1 - (2 rho - 1)^3), in double as the oracle has it
            radius1 = min(o1.initial_trust_region_radius / (1.0 / 3.0), o1.max_trust_region_radius)
            out.append((q, slot, x0, x1, x2, o2, st.S, radius1))
    return out


@pytest.mark.parametrize("opts", [{}, dict(min_lm_diagonal=1e2, max_lm_diagonal=1e3)],
                         ids=["defaults", "lm_diagonal_clamp"])
def test_second_step_is_the_oracles_second_iteration(oracle, opts):
    """max_num_iterations = 2: x2 - x1 = step_at(x1, S0, 3 radius0).dl within 8 n kappa u |dl2*| plus the
    move the oracle's own gradient error can make (test_gpu_ls_probe.second_step_bound) and the rounding
    of x1 + dl2.  With the LM diagonal clamp binding, a Jacobi scaling recomputed at x1 misses that
    bound on at least one component: Ceres fixes it in iteration 0."""
    cases = two_full_steps(oracle, opts)
    assert len(cases) >= 4, len(cases)
    missed = 0
    for q, slot, x0, x1, x2, o, S0, radius1 in cases:
        f = ref.first_step(q, slot, o, x0, want_kappa=False).free_nodes
        pr = ref.probe(q, slot, o, x1, np.zeros((len(f), 2)), 1.0)
        st2 = ref.step_at(q, slot, o, x1, S=S0, radius=radius1)
        bound, eta, _, _ = gp.second_step_bound(st2, pr)
        dl2 = st2.dl.astype(np.float64)
        norm = float(np.linalg.norm(dl2))
        tol = bound * norm + eta + 2 * U * float(np.linalg.norm(x2[f])) * np.sqrt(st2.n)
        err = float(np.linalg.norm((x2[f] - x1[f]) - dl2))
        assert err <= tol, (st2.n, st2.kappa, err, tol)
        rec = ref.step_at(q, slot, o, x1, S=None, radius=radius1, want_kappa=False).dl.astype(np.float64)
        missed += int(np.linalg.norm((x2[f] - x1[f]) - rec) > tol)
    if opts:
        assert missed >= 1
    print("%s: %d components, %d miss with a recomputed scaling" % (opts, len(cases), missed))


# ---------------------------------------------------------------------------------------------------
# 5. the cases have teeth
# ---------------------------------------------------------------------------------------------------
def test_cases_are_meaningful():
    """Over every case of test_gpu_ls_probe at every alpha (with the statement's step): no cost or phi'
    bound looser than 1e-9 of its magnitude sum; on every tier some probe where the clamped
    coordinates' share, one duplicated edge's share and the M / M^T difference of phi' each exceed the
    phi' bound; the box cases clamp at least 10 % of the free coordinates of every slot at alpha = 1;
    sources cross the +-0.5 grid clamp between x and xc.  Mode B skips a slot whose bound (8 n kappa u plus
    the move the gradient's evaluation error can make) exceeds MAX_BOUND: only the eight where kappa of
    the second system is 8e9 or more (the five weak clusters, two Tukey-outlier-node and one loss-width
    component, where Tukey edges turned outliers at xc leave clusters loosely held)."""
    teeth = {}
    crossed = skipped = 0
    for key in gp.CASES:
        p, _, x0, o, firsts = gp.case(key)
        for s, st in enumerate(firsts):
            tiers = {expected_tier(st.n, r) for r in ROUTES}
            dl = st.dl.astype(np.float64)
            for alpha in gp.ALPHAS:
                pr = ref.probe(p, s, o, x0, dl, alpha)
                assert pr.cost_bound <= 1e-9 * pr.cost_mag and pr.dphi_bound <= 1e-9 * pr.dphi_mag, (key, s, alpha)
                for t in tiers:
                    w = teeth.setdefault(t, set())
                    w |= {q for q, v in (("clamped", pr.clamped_share), ("duplicate", pr.dup_share),
                                         ("M^T", pr.mt_diff)) if v > pr.dphi_bound}
                crossed += pr.grid_cross
                if alpha == 1.0 and key == "box":
                    assert pr.clamped.mean() >= 0.1, (s, pr.clamped.mean())
                if alpha == 1.0:
                    st2 = ref.step_at(p, s, o, pr.xc, S=st.S)
                    bound, eta, _, _ = gp.second_step_bound(st2, pr)
                    if bound + eta / float(np.linalg.norm(st2.dl.astype(np.float64))) > MAX_BOUND:
                        assert st2.kappa >= 8e9, (key, s, st2.kappa)
                        skipped += 1
    assert all(teeth.get(t) == {"clamped", "duplicate", "M^T"} for t in (1, 2, 3, 4)), teeth
    assert crossed > 0
    assert skipped <= 8, skipped
    print("mode B slots skipped: %d; grid crossings: %d" % (skipped, crossed))
