"""The extended-precision statement of the first LM step (tests/lm_step_ref.py) on the CPU.

Three ties keep the statement honest before it judges the GPU tiers (tests/test_gpu_lm_step.py):
  1. its solve (float64 factorisation + longdouble refinement) against mpmath at 40 digits, on systems of
     up to 64 unknowns up to kappa 1e12: agreement to kappa 1e-18;
  2. its residuals and Jacobians against the oracle's edge evaluation (bitwise the reference's cost.cc,
     tests/test_ref_cost.py) within 4 ulp of the evaluation's term scale, and its loss terms against the
     oracle's;
  3. its step against the oracle's first iteration (max_num_iterations = 1) on components where Ceres
     takes the full step (no line-search step, no bound reached): x1 - x0 = dl within the step bound.
"""
import copy
import ctypes as C

import numpy as np
import pytest

import lm_step_ref as ref
from refsrc_util import cost_cases

U = 2.0 ** -53


# ---------------------------------------------------------------------------------------------------
# 1. the solve against mpmath
# ---------------------------------------------------------------------------------------------------
def spd(n, kappa, seed):
    """A float64 symmetric positive definite matrix of condition ~kappa with a random eigenbasis."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = np.logspace(0, -np.log10(kappa), n)
    a = (q * lam) @ q.T
    return (a + a.T) / 2


def to_mp(mpmath, v):
    """longdouble values as mpmath numbers, exactly (each the sum of two doubles)."""
    v = np.asarray(v, ref.LD)
    hi = v.astype(np.float64)
    lo = (v - hi.astype(ref.LD)).astype(np.float64)
    return [mpmath.mpf(float(h)) + mpmath.mpf(float(l)) for h, l in zip(hi.reshape(-1), lo.reshape(-1))]


def rel_err_mp(mpmath, A, b, y):
    """|y - A^-1 b| / |A^-1 b| with A^-1 b solved by mpmath at 40 digits."""
    n = len(b)
    mpmath.mp.dps = 40
    Am = mpmath.matrix(n, n)
    for k, v in enumerate(to_mp(mpmath, A)):
        Am[k // n, k % n] = v
    ya = mpmath.lu_solve(Am, mpmath.matrix(to_mp(mpmath, b)))
    ym = to_mp(mpmath, y)
    err = mpmath.sqrt(sum((ym[i] - ya[i]) ** 2 for i in range(n)))
    return float(err / mpmath.sqrt(sum(ya[i] ** 2 for i in range(n))))


@pytest.mark.parametrize("n", [2, 8, 33, 64])
@pytest.mark.parametrize("kappa", [1e2, 1e8, 1e12])
def test_refined_solve_matches_mpmath(n, kappa):
    mpmath = pytest.importorskip("mpmath")
    a = spd(n, kappa, seed=n)
    b = np.random.default_rng(n + 1).standard_normal(n)
    y, steps = ref.solve_refined(a.astype(ref.LD), b.astype(ref.LD))
    err = rel_err_mp(mpmath, a, b, y)
    k2 = np.linalg.cond(a)
    assert err <= k2 * 1e-18, (n, kappa, k2, err, steps)
    print("n %d kappa %.1e: relative error %.1e (kappa 1e-18 = %.1e), %d refinement steps"
          % (n, k2, err, k2 * 1e-18, steps))


def test_statement_system_matches_mpmath(oracle):
    """A component's own damped system at radius 1e16 (the least damping the default options allow)."""
    mpmath = pytest.importorskip("mpmath")
    p, slot = small_components()[-1]
    o = oracle.default_options(initial_trust_region_radius=1e16)
    st = ref.first_step(p, slot, o, np.zeros((p.graph.n_nodes, 2)))
    assert 8 <= st.n <= 64
    err = rel_err_mp(mpmath, st.A.dense(), st.b, st.y)
    assert err <= st.kappa * 1e-18, (err, st.kappa)
    print("n %d kappa %.1e: relative error %.1e" % (st.n, st.kappa, err))


# ---------------------------------------------------------------------------------------------------
# 2. residuals, Jacobians and losses against the oracle's edge evaluation
# ---------------------------------------------------------------------------------------------------
def _edges(grids32, sim):
    from lfr_b200.graph import EDGE_DTYPE
    e = np.zeros(grids32.shape[0], dtype=EDGE_DTYPE)
    e["flow"] = grids32
    e["sim"] = sim
    e["dst"] = 1
    return e


def test_edge_terms_match_oracle_edge_eval(oracle):
    """200 000 random, clamped and boundary inputs (refsrc_util.cost_cases): the oracle's double residuals
    and Jacobians are within 4 ulp of the longdouble statement, an ulp taken at the evaluation's own
    scale: the sum of the magnitudes of its terms (|x_dst| + |x_src| + sum |L_i L_j D_ij| for a residual,
    1 + sum |L_i' L_j D_ij| for a Jacobian entry).  Nine products summed in double may be off by a few
    units of that scale; where the terms cancel, an ulp of the result itself would be far too fine."""
    grids, x1, x2 = cost_cases(200000, seed=11)
    n = grids.shape[0]
    r_o, jac_o, _ = oracle.edge_eval(_edges(grids, 0.9), np.ones(n, np.uint8), x1, x2)
    r, J = ref.edge_terms(grids, x1, x2)
    D = np.abs(grids.astype(np.float64).reshape(-1, 3, 3, 2))
    c = np.clip(x1, -0.5, 0.5).astype(ref.LD)
    L0, L1 = (np.abs(ref._lag(c[:, k]).astype(np.float64)) for k in (0, 1))
    d0, d1 = (np.abs(ref._dlag(c[:, k]).astype(np.float64)) for k in (0, 1))
    sum_f = np.einsum("ei,ej,eijk->ek", L0, L1, D)
    sum_d0 = np.einsum("ei,ej,eijk->ek", d0, L1, D)
    sum_d1 = np.einsum("ei,ej,eijk->ek", L0, d1, D)
    scale_r = np.abs(x1) + np.abs(x2) + sum_f
    scale_j = np.stack([1 + sum_d0[:, 0], sum_d1[:, 0], sum_d0[:, 1], 1 + sum_d1[:, 1]], axis=1)
    for got, want, scale, what in ((r, r_o, scale_r, "residual"), (J.reshape(n, 4), jac_o, scale_j, "jacobian")):
        u = np.abs((got - want.astype(ref.LD)).astype(np.float64)) / np.spacing(scale)
        assert u.max() <= 4.0, (what, float(u.max()))
        print("%s: max %.2f ulp of the term scale" % (what, float(u.max())))
    # clamped coordinates have zero flow derivative, as in cost.cc
    out = np.abs(x1[:, 0]) > 0.5
    assert out.sum() > 1000 and np.all(J[out, :, 0] == np.array([-1.0, 0.0]))


@pytest.mark.parametrize("opts", [{}, dict(tukey_variant=2), dict(cauchy_a=0.1, tukey_a=0.2)])
def test_loss_terms_match_oracle(oracle, opts):
    """sim rho and sim rho' of both kinds, inside and outside the Tukey width, within 4 ulp of their
    scales: sim a^2 + rho for rho (Ceres' log(1 + s / b) and 1 - (1 - s / a^2)^3 cancel for small s), sim for
    rho'.  Zero rho' exactly where the oracle has it (Tukey outliers)."""
    rng = np.random.default_rng(3)
    n = 20000
    kind = rng.integers(1, 3, n).astype(np.uint8)
    sim = rng.uniform(1e-3, 1.0, n).astype(np.float32)
    s = np.exp(rng.uniform(np.log(1e-8), np.log(1.0), n))
    o = oracle.default_options(**opts)
    rho_o = np.zeros((n, 3))
    for i in range(n):
        oracle.lib.lfr_ref_loss(int(kind[i]), float(sim[i]), float(s[i]), C.byref(o), rho_o[i].ctypes.data)
    rho, d1 = ref.loss_terms(kind, sim, s, ref.option_values(o))
    width2 = np.where(kind == ref.CAUCHY, o.cauchy_a, o.tukey_a) ** 2
    sim64 = sim.astype(np.float64)
    u_rho = np.abs((rho - rho_o[:, 0]).astype(np.float64)) / np.spacing(sim64 * width2 + rho_o[:, 0])
    u_d1 = np.abs((d1 - rho_o[:, 1]).astype(np.float64)) / np.spacing(sim64)
    print("rho %.2f ulp, rho' %.2f ulp" % (u_rho.max(), u_d1.max()))
    assert u_rho.max() <= 4 and u_d1.max() <= 4
    assert np.array_equal(rho_o[:, 1] == 0, d1 == 0)
    assert ((kind == ref.TUKEY) & (rho_o[:, 1] == 0)).sum() > 100   # outliers reached


# ---------------------------------------------------------------------------------------------------
# 3. the step against the oracle's first iteration
# ---------------------------------------------------------------------------------------------------
_small = []


def small_components():
    """One-slot problems of cfg2 (x 0.05): twelve components of 8 to 64 unknowns."""
    if not _small:
        from lfr_b200 import build_problem, synth
        from test_gpu_cta_limits import subset
        p = build_problem(synth.generate("cfg2", scale=0.05))
        nodes = p.comp_nodes.astype(np.int64)
        free = np.add.reduceat((p.is_root[nodes] == 0).astype(np.int64), p.comp_ptr[:-1].astype(np.int64))
        sizes = np.diff(p.comp_ptr.astype(np.int64))
        n2 = np.where(sizes > 0, 2 * free, 0)
        picks = [int(s) for s in np.nonzero((n2 >= 8) & (n2 <= 64) & (sizes > 1))[0]]
        picks = sorted(picks, key=lambda s: n2[s])
        step = max(1, len(picks) // 12)
        for s in picks[::step][:12]:
            _small.append((subset(p, [s]), 0))
    return _small


@pytest.mark.parametrize("start_kind", ["zero", "random"])
@pytest.mark.parametrize("opts", [{}, dict(initial_trust_region_radius=1.0), dict(tukey_variant=2),
                                  dict(cauchy_a=0.1, tukey_a=0.2)], ids=["defaults", "radius_1", "tukey_2", "widths"])
def test_statement_is_the_oracles_first_iteration(oracle, opts, start_kind):
    """max_num_iterations = 1 from the start: where the oracle accepts the full step (NO_CONVERGENCE after
    one iteration, no line-search step, the free nodes moved, no coordinate at the bound), x1 - x0 equals
    the statement's dl within 8 n kappa 2^-53 |dl| (plus the rounding of x0 + dl), and its initial cost
    equals the statement's to 1e-13."""
    compared = 0
    worst = 0.0
    for q, slot in small_components():
        N = q.graph.n_nodes
        rng = np.random.default_rng(q.comp_nodes[0])
        start = np.zeros((N, 2)) if start_kind == "zero" else rng.uniform(-0.6, 0.6, (N, 2))
        o = oracle.default_options(n_threads=1, max_num_iterations=1, **opts)
        pos, st = oracle.solve(q, o, positions=start)
        step = ref.first_step(q, slot, o, start)
        assert abs(st["initial_cost"][0] - step.cost) <= 1e-13 * step.cost
        x0 = np.clip(start[step.free_nodes], -1.0, 1.0)
        x1 = pos[step.free_nodes]
        full = (st["iterations"][0] == 1 and st["termination"][0] == 5 and st["total_line_search_steps"] == 0
                and not np.array_equal(x1, x0) and np.all(np.abs(x0 + step.dl.astype(np.float64)) < 1.0))
        if not full:
            continue
        dl = step.dl.astype(np.float64)
        err = np.linalg.norm((x1 - x0) - dl)
        tol = ref.step_bound(step.n, step.kappa) * np.linalg.norm(dl) + 2 * U * np.linalg.norm(x1) * np.sqrt(step.n)
        assert err <= tol, (step.n, step.kappa, err, tol)
        worst = max(worst, err / (ref.step_bound(step.n, step.kappa) * np.linalg.norm(dl)))
        compared += 1
    assert compared >= 6, compared
    print("%s %s: %d components, largest |x1 - x0 - dl| / bound %.2e" % (opts, start_kind, compared, worst))


def test_dropped_blocks(oracle):
    """Root-root edges and edges to another component are not blocks; edges to roots are: the statement's
    cost equals the oracle's initial cost on a component whose every other node is made a root."""
    q, slot = small_components()[-1]
    q = copy.copy(q)
    nodes = q.comp_nodes.astype(np.int64)
    q.is_root = q.is_root.copy()
    q.is_root[nodes[::2]] = 1
    src, dst, _, _ = ref.kept_blocks(q, slot)
    assert not np.any((q.is_root[src] != 0) & (q.is_root[dst] != 0))
    assert np.any((q.is_root[src] != 0) | (q.is_root[dst] != 0))
    start = np.random.default_rng(1).uniform(-0.4, 0.4, (q.graph.n_nodes, 2))
    o = oracle.default_options(n_threads=1, max_num_iterations=0)
    _, st = oracle.solve(q, o, positions=start)
    step = ref.first_step(q, slot, o, start, want_kappa=False)
    assert abs(st["initial_cost"][0] - step.cost) <= 1e-13 * step.cost
