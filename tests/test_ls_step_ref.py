"""The exact statement of the line search's step selection (tests/ls_step_ref.py), checked without a GPU:

- it encodes Ceres' rule: the oracle's literal polynomial.cc restatement meets its criterion wherever
  Ceres' own fit keeps full rank;
- it confirms K: a float64 model of the kernel's formulation (the interpolant of
  test_gpu_root_polish._quintic_der, its cubic twin and the candidate scan of hermite_minimizer, with
  exact roots) meets the criterion at K / 2 on every population (K itself is the a-priori bound derived
  in ls_step_ref; the model's measured worst ratio is far below it);
- the oracle's fast formulation, which the CPU oracle solves with, meets it on every population,
  ill-conditioned states included;
- the reference itself: closed-form minimisers, exact reproduction of the data, Lambda by hand."""
from fractions import Fraction as Fr
import math

import numpy as np
import pytest

import ls_step_ref as R
from ls_step_ref import harvested_populations, population_exacts
from oracle_util import minimize_interpolating, well_conditioned
from test_linesearch_modes import _random_states

# the model's worst ratio must stay below K / 2 (the calibration margin of ls_step_ref.K)
MODEL_MARGIN = 0.5


def _horner(c, t):
    v = 0.0
    for a in c:
        v = v * t + a
    return v


def model_step(s):
    """hermite_minimizer's formulation in float64 (no FMA), with the exact roots of its computed
    derivative in [tlo, thi] rounded to double."""
    f0, g0, x1, f1, g1, three, x2, f2, g2, lo, hi = [float(v) for v in s]
    three = three != 0.0
    h = max(x1, x2) if three else x1
    ih = 1.0 / h
    g0h = g0 * h
    if not three:
        u, v = f1 - f0 - g0h, (g1 - g0) * h
        c = [v - 2.0 * u, 3.0 * u - v, g0h, f0]
    else:
        ta, tb = x1 * ih, x2 * ih
        ita, itb, iw = 1.0 / ta, 1.0 / tb, 1.0 / (tb - ta)
        Sa = (f1 - f0 - g0h * ta) * (ita * ita)
        Sb = (f2 - f0 - g0h * tb) * (itb * itb)
        Da = ((g1 - g0) * h - 2.0 * ta * Sa) * (ita * ita)
        Db = ((g2 - g0) * h - 2.0 * tb * Sb) * (itb * itb)
        m = (Sb - Sa) * iw
        e2 = (m - Da) * iw
        e3 = ((Db - m) - (m - Da)) * iw * iw
        c = [e3, e2 - e3 * (2.0 * ta + tb), Da + ta * (e3 * (ta + 2.0 * tb) - 2.0 * e2),
             Sa + ta * (ta * (e2 - e3 * tb) - Da), g0h, f0]
    tlo, thi = lo * ih, hi * ih
    while len(c) > 1 and c[0] == 0.0:
        c = c[1:]
    ox = (lo + hi) / 2.0
    ov = _horner(c, ox * ih)
    for t, x in ((tlo, lo), (thi, hi)):
        v = _horner(c, t)
        if v < ov:
            ov, ox = v, x
    n = len(c) - 1
    der = [Fr((n - i) * a) for i, a in enumerate(c[:-1])]
    if len(der) >= 2 and tlo < thi:
        for r, _ in R.real_roots(list(reversed(der)), Fr(tlo), Fr(thi)):
            t = float(r)
            v = _horner(c, t)
            if v < ov:
                ov, ox = v, t * h
    for x in ([0.0, x1, x2] if three else [0.0, x1]):
        if lo <= x <= hi:
            v = _horner(c, x * ih)
            if v < ov:
                ov, ox = v, x
    return ox


def _all_populations(oracle):
    pops = dict(R.constructed_populations())
    pops["thi_root"] = R.thi_root_states()
    pops.update({"harvest_" + k: v for k, v in harvested_populations(oracle).items()})
    return pops


def _report(name, states, xs, exacts, k=R.K):
    fails, decided, worst, _ = R.judge_all(states, xs, k, exacts)
    return fails, decided, worst


# ---- the reference itself ---------------------------------------------------------------------------
def test_interpolant_reproduces_the_data_exactly():
    pops = R.constructed_populations()
    rows = np.concatenate([pops["tiny_steps"], pops["value_scale"], pops["low_degree"][:10]])
    for s in rows:
        ex = R.Exact(s)
        for (x, f, g) in ex.nodes:
            assert R.peval(ex.P, x) == f and R.peval(ex.dP, x) == g
        assert len(ex.P) == (6 if s[5] else 4)


def test_dyadic_polynomials_with_known_minimisers():
    # P(x) = (x - 1/4)^2 sampled at 0 and 1 (a cubic route that is really a quadratic): m* at 1/4
    P = lambda x: (x - 0.25) ** 2
    s = [P(0), -0.5, 1.0, P(1), 1.5, 0.0, 0.0, 0.0, 0.0, 1e-3, 0.6]
    ex = R.Exact(s)
    assert ex.crit == [0.25] and ex.m_star == 0 and ex.judge(0.25) is None
    assert ex.judge(0.25 + 2.0 ** -20) is not None and ex.judge(0.6 * (1 + 2.0 ** -29)) is not None
    # P(x) = x^4/4 - x^3/2 (P' = x^2 (x - 3/2)): the minimum at 3/2 on [0, 2], the double root 0 is no minimum
    P = lambda x: x ** 4 / 4 - x ** 3 / 2
    dP = lambda x: x ** 3 - 1.5 * x ** 2
    s = [P(0), dP(0), 1.0, P(1), dP(1), 1.0, 2.0, P(2), dP(2), 0.0, 2.0]
    ex = R.Exact(s)
    assert [float(r) for r in ex.crit] == [0.0, 1.5]
    assert ex.m_star == Fr(P(1.5)) and ex.judge(1.5) is None and ex.judge(0.0) is not None
    # a tie: P = (x^2 - 1/4)^2 on [-1, 1] has equal minima at +-1/2
    roots = R.real_roots([Fr(1, 16), Fr(0), Fr(-1, 2), Fr(0), Fr(1)], Fr(-1), Fr(1))
    assert [(float(r), m) for r, m in roots] == [(-0.5, 2), (0.5, 2)]


def test_lambda_of_a_two_sample_cubic_by_hand():
    # nodes 0 and 1: B_g,0(t) = t (1 - t)^2, increasing on [0, 1/3]; with g0 = 1 and all else 0,
    # Lambda on [0, 1/4] is B_g,0(1/4) = 9/64
    ex = R.Exact([0.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.25])
    assert ex.lam == 9.0 / 64.0
    # f0 = f1 = 1, g = 0: B_f,0 + B_f,1 = 1 everywhere
    ex = R.Exact([1.0, 0.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    assert abs(ex.lam - 1.0) <= 4 * R.U
    # the same scaled to h = 2^-10 and slopes 2^10: Lambda does not depend on the step's unit
    ex = R.Exact([0.0, 1024.0, 2.0 ** -10, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 2.0 ** -12])
    assert ex.lam == 9.0 / 64.0


def test_quartic_roots_reference():
    # (t - 1/4)^2 (t - 1/2) (t + 1): a double root, a simple one inside, one outside
    q = np.poly([0.25, 0.25, 0.5, -1.0])
    got = R.quartic_real_roots(q, 0.0, 1.0)
    assert [(r, m) for r, m, _ in got] == [(0.25, 2), (0.5, 1)]
    assert got[0][2] == 0.0 and abs(got[1][2] - 0.25) < 1e-15


# ---- Ceres' rule -----------------------------------------------------------------------------------
def test_literal_ceres_meets_the_criterion_where_its_fit_has_full_rank(oracle):
    states = _random_states(np.random.default_rng(5), 600, smallest=0.02)
    harvest = np.concatenate([v for v in harvested_populations(oracle).values()])
    harvest = harvest[well_conditioned(harvest)]
    for name, st in (("random", states), ("harvest", harvest)):
        assert well_conditioned(st).all() and st.shape[0] > 300, (name, st.shape)
        xs = minimize_interpolating(oracle, st, fast=False)
        fails, decided, worst, _ = R.judge_all(st, xs)
        assert not fails, (name, len(fails), fails[:3])
        assert decided > 0.9 * st.shape[0], (name, decided, st.shape[0])


# ---- calibration of K, and the oracle's fast formulation --------------------------------------------
def test_kernel_model_calibrates_k(oracle):
    """The float64 model of the kernel's formulation needs at most K / 2 on every population."""
    for name, st in _all_populations(oracle).items():
        exacts = population_exacts(name, st)
        xs = np.array([model_step(s) for s in st])
        fails, decided, worst = _report(name, st, xs, exacts, k=R.K * MODEL_MARGIN)
        assert not fails, (name, len(fails), fails[:3])
        assert decided >= min(0.5 * st.shape[0], 20), (name, decided, st.shape[0])
        print("model %-32s states %5d decided %5d worst %.3g" % (name, st.shape[0], decided, worst))


def test_oracle_fast_formulation_meets_the_criterion(oracle):
    for name, st in _all_populations(oracle).items():
        exacts = population_exacts(name, st)
        xs = minimize_interpolating(oracle, st, fast=True)
        fails, decided, worst = _report(name, st, xs, exacts)
        assert not fails, (name, len(fails), fails[:3])
        print("oracle fast %-26s states %5d decided %5d worst %.3g" % (name, st.shape[0], decided, worst))


def test_oracle_root_finder_meets_the_exact_root_check(oracle):
    """The root check of test_gpu_ls_step_exact.py on the oracle's derivative recursion
    (lfr_ref_polynomial_roots), which polishes its roots the way the kernel's recursion does."""
    from test_gpu_parity import _quartic_cases
    c1, l1 = _quartic_cases(np.random.default_rng(99), 600)
    c2, l2 = R.constructed_quartics()
    c3, l3 = R.last_ulp_quartics()
    out = np.zeros(8)
    bad = []
    for q, (lo, hi) in zip(np.concatenate([c1, c2, c3]), np.concatenate([l1, l2, l3])):
        q = np.ascontiguousarray(q)
        n = oracle.lib.lfr_ref_polynomial_roots(q.ctypes.data, 5, float(lo), float(hi), out.ctypes.data)
        msg = R.check_roots(q, float(lo), float(hi), list(out[:n]))
        if msg:
            bad.append(msg)
    assert not bad, (len(bad), bad[:3])
