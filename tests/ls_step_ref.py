"""An exact statement of the Armijo line search's step selection (Ceres' MinimizeInterpolatingPolynomial,
SURVEY A.6), and the states it is judged on.

Written from the rule alone, independently of the oracle's code and of the kernel's formulation
(csrc/lfr_math.cuh :: hermite_minimizer):

  * A state is the 11 doubles {f0, g0, x1, f1, g1, three, x2, f2, g2, lo, hi} of lfr_debug_ls_minimizer.
    Every double is taken as the exact rational it is.
  * The interpolant P(x), in the raw step x, is the Hermite interpolant of {value, slope} at 0 and x1
    (a cubic) and also at x2 when `three` is set (a quintic), built with fractions.Fraction from Newton's
    divided differences on the doubled nodes.
  * m* = min P over [lo, hi]: over lo, hi and every real root of P' inside the interval.  The roots are
    isolated exactly (sympy's real-root isolation of the rational P') and refined to 90 digits inside
    their isolating intervals (bisection-safeguarded Newton on the square-free part, mpmath at 300 bits).
    The critical points that lie in the interval also give max P, hence the range of P there.
  * Lambda = max over [lo, hi] of sum_i |d_i| |B_i(x)|: d_i are the data (values and slopes), B_i the
    Hermite cardinal functions in closed form, B_f,j = (1 - 2 l_j'(z_j)(x - z_j)) l_j(x)^2 and
    B_g,j = (x - z_j) l_j(x)^2 with l_j the Lagrange basis of the distinct nodes z_j.  It bounds how far
    the interpolant's values move under relative perturbations of the data of size 1: u Lambda is the
    value error that rounding the data alone can cause.  It is an ESTIMATE: the maximum is taken in
    float64 over a fixed grid of 513 points plus the critical points of P, not over the whole interval.

The criterion for a returned step x (`judge`):
  * lo <= x <= hi (1 + 2^-30): the margin lm_solve's skip rule allows for the rounding of t -> x of a
    root found in the normalised variable t = x / h;
  * P(x) - m* <= K u Lambda + |P'(x)| 4 ulp(x), u = 2^-53.  The second term is what four roundings of
    the abscissa itself may cost (t = x / h, the root in t, t h).

K = 64 is an a-priori bound; the CPU tests (tests/test_ls_step_ref.py) confirm it with a float64 model
of the kernel's formulation with exact roots rather than fit it.  Derivation: the selection compares the float64 values of the interpolant
at the candidates, so it can lose twice the worst value error of the computed interpolant.  That error
has three parts, each a small multiple of u Lambda: rounding the normalised abscissae (x1 / h, x2 / h,
lo / h, hi / h: a node moved by one ulp moves P by about u Lambda), the coefficient formulas (each of
the divided differences takes a handful of roundings, and the expansion to monomials a few more, all
relative to the data, so some 10 u Lambda), and Horner's evaluation (10 roundings of terms each at most
Lambda in size near the interval, so 10 u Lambda).  2 x (1 + 10 + 10) ~ 42, rounded up to the next
power of two: K = 64.  The model must meet the criterion at K / 2 on every population.  Its measured worst
ratio is about 1.1e-6 (a near-double pair beside the minimiser; 0 to 2e-12 elsewhere), so K has a
headroom of some 7 orders of magnitude: the value criterion is loose at an interior minimum, where a
misplaced abscissa costs only P'' d^2 / 2, and sharp where candidates compete (tied minima to 1e-12,
a lost root, a wrong end).

A state is DECIDED when K u Lambda is below 1e-3 (max P - min P) on [lo, hi]: there the criterion
actually discriminates between candidates.  Every population must contain a stated number of decided
states, so a test cannot pass on hopeless states alone.

`quartic_real_roots` states the exact real roots of a quartic on [lo, hi] with their multiplicities and
their separation from the nearest other root, real or complex, for the root-finder tests.
"""
from fractions import Fraction as Fr
import math

import mpmath
import numpy as np
import sympy

U = 2.0 ** -53
K = 64
STEP_MARGIN = 2.0 ** -30
DECIDED_FRACTION = 1e-3
_PREC = 300
_X = sympy.Symbol("x")
_GRID = np.linspace(0.0, 1.0, 513)


# ---- exact polynomials (Fractions, lowest degree first) --------------------------------------------
def peval(c, x):
    v = Fr(0)
    for a in reversed(c):
        v = v * x + a
    return v


def pder(c):
    return [k * c[k] for k in range(1, len(c))]


def hermite(nodes):
    """Exact Hermite interpolant through [(x, f, g), ...] (Fractions), monomial coefficients lowest first."""
    z, fv = [], []
    for (x, f, g) in nodes:
        z += [x, x]
        fv += [(f, g), (f, g)]
    n = len(z)
    col = [fv[i][0] for i in range(n)]
    coefs = [col[0]]
    for k in range(1, n):
        nxt = []
        for i in range(n - k):
            if z[i + k] == z[i]:          # k == 1 on a doubled node: the slope
                nxt.append(fv[i][1])
            else:
                nxt.append((col[i + 1] - col[i]) / (z[i + k] - z[i]))
        col = nxt
        coefs.append(col[0])
    # Newton form -> monomials
    poly = [Fr(0)] * n
    basis = [Fr(1)]
    for k in range(n):
        for i, b in enumerate(basis):
            poly[i] += coefs[k] * b
        basis = [Fr(0)] + basis                        # * x
        for i in range(len(basis) - 1):
            basis[i] -= z[k] * basis[i + 1]            # - z_k * previous
    return poly


def _mp(v):
    if isinstance(v, Fr):
        return mpmath.mpf(v.numerator) / v.denominator
    return mpmath.mpf(v)


def real_roots(c, lo, hi):
    """Real roots of the exact polynomial c (lowest first) in [lo, hi], as [(mpf root, multiplicity)],
    ascending.  Exact isolation, then 90-digit refinement."""
    while c and c[-1] == 0:
        c = c[:-1]
    if len(c) <= 1:
        return []
    P = sympy.Poly(list(reversed([sympy.Rational(a.numerator, a.denominator) for a in c])), _X, domain=sympy.QQ)
    ivs = P.intervals(inf=sympy.Rational(lo.numerator, lo.denominator),
                      sup=sympy.Rational(hi.numerator, hi.denominator))
    if not ivs:
        return []
    sqf = P.sqf_part()
    qc = [_mp(Fr(int(a.p), int(a.q))) for a in sqf.all_coeffs()]   # highest first
    dq = [qc[i] * (len(qc) - 1 - i) for i in range(len(qc) - 1)]
    out = []
    with mpmath.workprec(_PREC):
        qc = [+a for a in qc]
        for (a, b), mult in ivs:
            A, B = _mp(Fr(int(a.p), int(a.q))), _mp(Fr(int(b.p), int(b.q)))
            if A == B:
                out.append((A, mult))
                continue
            # an end of a non-degenerate isolating interval may be another (simple) root: the sign
            # just inside it is then the opposite of the other end's
            fa, fb = mpmath.polyval(qc, A), mpmath.polyval(qc, B)
            assert fa != 0 or fb != 0
            if fa == 0:
                fa = -fb
            x = (A + B) / 2
            tol = mpmath.mpf(2) ** (-_PREC + 20) * max(abs(A), abs(B))
            for _ in range(400):
                fx = mpmath.polyval(qc, x)
                if fx == 0:
                    break
                if (fx < 0) == (fa < 0):
                    A, fa = x, fx
                else:
                    B = x
                d = mpmath.polyval(dq, x)
                xn = x - fx / d if d != 0 else (A + B) / 2
                if not (min(A, B) < xn < max(A, B)):
                    xn = (A + B) / 2
                if abs(xn - x) <= tol or abs(B - A) <= tol:
                    x = xn
                    break
                x = xn
            out.append((x, mult))
    return out


# ---- the interpolant of a state ----------------------------------------------------------------
class Exact:
    """The exact interpolant of one state and everything the criterion needs."""

    def __init__(self, s):
        s = [float(v) for v in s]
        f0, g0, x1, f1, g1, three, x2, f2, g2, lo, hi = s
        self.state = s
        self.three = three != 0.0
        nodes = [(Fr(0), Fr(f0), Fr(g0)), (Fr(x1), Fr(f1), Fr(g1))]
        if self.three:
            nodes.append((Fr(x2), Fr(f2), Fr(g2)))
        self.nodes = nodes
        self.lo, self.hi = Fr(lo), Fr(hi)
        self.P = hermite(nodes)
        self.dP = pder(self.P)
        self.crit = [r for r, _ in real_roots(self.dP, self.lo, self.hi)]
        with mpmath.workprec(_PREC):
            Pm = [_mp(a) for a in reversed(self.P)]
            vals = [_mp(peval(self.P, self.lo)), _mp(peval(self.P, self.hi))]
            vals += [mpmath.polyval(Pm, r) for r in self.crit]
            self.m_star = min(vals)
            self.m_max = max(vals)
        self.range = float(self.m_max - self.m_star)
        self.lam = self._lambda()

    def _lambda(self):
        """Lambda, in float64 on the normalised abscissa t = x / h."""
        xs = [float(n[0]) for n in self.nodes]
        h = max(xs)
        z = np.array(xs) / h
        fs = np.array([abs(float(n[1])) for n in self.nodes])
        gs = np.array([abs(float(n[2])) * h for n in self.nodes])
        tlo, thi = float(self.lo) / h, float(self.hi) / h
        t = np.concatenate([tlo + (thi - tlo) * _GRID, [float(r) / h for r in self.crit]])
        tot = np.zeros_like(t)
        for j in range(len(z)):
            l = np.ones_like(t)
            dl = 0.0
            for k in range(len(z)):
                if k != j:
                    l = l * (t - z[k]) / (z[j] - z[k])
                    dl += 1.0 / (z[j] - z[k])
            l2 = l * l
            tot += fs[j] * np.abs((1.0 - 2.0 * dl * (t - z[j])) * l2) + gs[j] * np.abs((t - z[j]) * l2)
        return float(tot.max())

    def excess(self, x):
        """P(x) - m* (float) at the double x."""
        with mpmath.workprec(_PREC):
            return float(_mp(peval(self.P, Fr(float(x)))) - self.m_star)

    def slope_term(self, x):
        return abs(float(peval(self.dP, Fr(float(x))))) * 4.0 * math.ulp(float(x))

    def tolerance(self, x, k=K):
        return k * U * self.lam + self.slope_term(x)

    def decided(self, k=K):
        return k * U * self.lam < DECIDED_FRACTION * self.range

    def ratio(self, x):
        """(P(x) - m* - |P'(x)| 4 ulp(x)) / (u Lambda): the K the step x needs."""
        return (self.excess(x) - self.slope_term(x)) / (U * self.lam) if self.lam > 0 else 0.0

    def judge(self, x, k=K):
        """None if x satisfies the criterion, else a description of the failure."""
        x = float(x)
        lo, hi = float(self.lo), float(self.hi)
        if not (lo <= x <= hi * (1.0 + STEP_MARGIN)):
            return "step %r outside [%r, %r (1 + 2^-30)]" % (x, lo, hi)
        e, tol = self.excess(x), self.tolerance(x, k)
        if not e <= tol:
            return "P(x) - m* = %.3e > tol %.3e (ratio %.3g, x %r, m* at %s)" % (
                e, tol, self.ratio(x), x, [float(r) for r in self.crit])
        return None


def judge_all(states, xs, k=K, exacts=None):
    """(failures [(index, message)], decided count, worst ratio, Exact objects)."""
    fails, decided, worst = [], 0, 0.0
    out = []
    for i, s in enumerate(states):
        ex = exacts[i] if exacts is not None else Exact(s)
        out.append(ex)
        msg = ex.judge(xs[i], k)
        if msg is not None:
            fails.append((i, msg))
        if ex.decided(k):
            decided += 1
        if ex.lam > 0:
            worst = max(worst, ex.ratio(xs[i]))
    return fails, decided, worst, out


# ---- exact quartic roots ---------------------------------------------------------------------------
def quartic_real_roots(q, lo, hi):
    """Exact real roots of the double quartic q (highest degree first) in [lo, hi]:
    [(root as float, multiplicity, separation from the nearest other root, real or complex)]."""
    c = [Fr(float(a)) for a in reversed(q)]
    rr = real_roots(c, Fr(float(lo)), Fr(float(hi)))
    if not rr:
        return []
    allr = all_roots(q)
    out = []
    for r, mult in rr:
        if mult > 1:
            out.append((float(r), mult, 0.0))
            continue
        d = sorted(abs(z - float(r)) for z in allr)
        out.append((float(r), mult, float(d[1]) if len(d) > 1 else math.inf))
    return out


def all_roots(q):
    """Every root of the double quartic q (highest degree first), complex ones included (mpmath)."""
    with mpmath.workprec(160):
        try:
            return [complex(z) for z in mpmath.polyroots([mpmath.mpf(float(a)) for a in q], maxsteps=200, extraprec=160)]
        except mpmath.libmp.NoConvergence:
            return [complex(z) for z in np.roots(q)]


def root_bound(q, z, c=16.0):
    """How far a root-finder working in double precision may place the root z of q: with
    eps = c u sum|q_i||z|^i (c = 16, as tests/test_gpu_root_polish.py; the Horner evaluation error of q
    near z), the smallest of (k! eps / |q^(k)(z)|)^(1/k), k = 1 .. 4: the simple-root bound eps / |q'| for
    an isolated root, the square-root bound for a double root or a pair closer than that, and so on.
    Plus 4 ulp."""
    q = [float(a) for a in q]
    a = abs(z)
    eps = c * U * float(np.polyval(np.abs(q), a))
    best = math.inf
    d = np.array(q)
    for k in range(1, len(q)):
        d = np.polyder(d)
        v = abs(np.polyval(d, z))
        if v > 0:
            best = min(best, (math.factorial(k) * eps / v) ** (1.0 / k))
    return best + 4.0 * math.ulp(max(a, 1e-300))


# ---- constructed states --------------------------------------------------------------------------
# Each is built from an exact polynomial P~(t) in the normalised variable t = x / h, then rounded to
# double data: f_j = P~(x_j / h), g_j = P~'(x_j / h) / h at double abscissae x_j, with lo = 1e-3 x1 and
# hi = 0.6 x1 as ls_next_step passes them (h = max(x1, x2)).
def poly_from_slope(a, real=(), pairs=(), f0=1.0):
    """P~ = f0 + integral_0^t a prod(s - r) prod((s - c)^2 + d^2) ds, exact (lowest first)."""
    d = [Fr(a)]
    for r in real:
        r = Fr(r)
        d = [Fr(0)] + d
        for i in range(len(d) - 1):
            d[i] -= r * d[i + 1]
    for c, w in pairs:
        c, w = Fr(c), Fr(w)
        q = [c * c + w * w, -2 * c, Fr(1)]
        nd = [Fr(0)] * (len(d) + 2)
        for i, u in enumerate(d):
            for j, v in enumerate(q):
                nd[i + j] += u * v
        d = nd
    return [Fr(f0)] + [d[k] / (k + 1) for k in range(len(d))]


def state_of(Pt, h, x1, x2=None, lo=None, hi=None):
    """The double state sampling P~ at 0, x1 [and x2] with step scale h."""
    H = Fr(float(h))
    dPt = pder(Pt)

    def data(x):
        t = Fr(float(x)) / H
        return float(peval(Pt, t)), float(peval(dPt, t) / H)

    f0, g0 = data(0.0)
    f1, g1 = data(x1)
    three = x2 is not None
    f2, g2 = data(x2) if three else (0.0, 0.0)
    lo = 1e-3 * x1 if lo is None else lo
    hi = 0.6 * x1 if hi is None else hi
    return [f0, g0, float(x1), f1, g1, 1.0 if three else 0.0, float(x2) if three else 0.0, f2, g2, lo, hi]


def kernel_interval(x1, h):
    """tlo, thi and the 32 grid points t_L of quartic_roots_grid for lo = 1e-3 x1, hi = 0.6 x1."""
    ih = 1.0 / h
    tlo, thi = (1e-3 * x1) * ih, (0.6 * x1) * ih
    w = (thi - tlo) * (1.0 / 31.0)
    return tlo, thi, [thi if L == 31 else float(Fr(w) * L + Fr(tlo)) for L in range(32)]


def _ulps(t, k):
    return float(Fr(t) + k * Fr(math.ulp(t)))


def _generic(rng, tlo, thi):
    """A quintic with one real critical point inside [tlo, thi] and three others of varied kind."""
    span = thi - tlo
    r1 = tlo + span * rng.uniform(0.05, 0.95)
    r2 = tlo + span * rng.uniform(-1.0, 2.0)
    c, d = tlo + span * rng.uniform(0.0, 1.0), span * 10.0 ** rng.uniform(-2, 0.5)
    a = rng.choice([-1.0, 1.0]) * 10.0 ** rng.uniform(-1, 1) / span ** 3
    if rng.uniform() < 0.5:
        return poly_from_slope(a, real=(r1, r2), pairs=((c, d),))
    return poly_from_slope(a, real=(r1, r2, c - d, c + d))


def constructed_populations():
    """{name: [state, ...]}: the adversarial states, deterministic."""
    rng = np.random.default_rng(20261018)
    pops = {}

    # a critical point on each grid point t_L (t_0 = tlo, t_31 = thi), offset by 0, +-1, +-2^10 ulps
    rows = []
    for ta in (0.5, 0.3):
        h, x1 = 1.0, ta
        tlo, thi, ts = kernel_interval(x1, h)
        for L in range(32):
            for off in (0, 1, -1, 1024, -1024):
                r = _ulps(ts[L], off)
                for a in (1.0, -1.0):
                    Pt = poly_from_slope(a / thi ** 3, real=(r, 1.5 * thi), pairs=((0.5 * thi, 0.3 * thi),))
                    rows.append(state_of(Pt, h, x1, 1.0))
    pops["grid_points"] = rows

    # two (kind-2 cells) and three (two extrema of P' in one cell: the recursion fallback) critical
    # points in one grid cell
    rows = []
    tlo, thi, ts = kernel_interval(0.5, 1.0)
    w = ts[1] - ts[0]
    for L in range(0, 31, 3):
        for a in (1.0, -1.0):
            two = (ts[L] + 0.3 * w, ts[L] + 0.7 * w)
            rows.append(state_of(poly_from_slope(a / thi ** 3, real=two + (-0.2, 2.0 * thi)), 1.0, 0.5, 1.0))
            three = (ts[L] + 0.2 * w, ts[L] + 0.5 * w, ts[L] + 0.8 * w)
            rows.append(state_of(poly_from_slope(a / thi ** 3, real=three + (2.0 * thi,)), 1.0, 0.5, 1.0))
    pops["cell_pairs"] = rows

    # a near-double critical pair (real or complex, separation 1e-4 .. 1e-10) beside the minimiser
    rows = []
    for ta in (0.5, 0.05):
        tlo, thi, _ = kernel_interval(ta, 1.0)
        m = tlo + 0.4 * (thi - tlo)
        for e in range(4, 11):
            sep = 10.0 ** -e * thi
            for c in (m + 0.1 * (thi - tlo), m + 10.0 * sep):
                rows.append(state_of(poly_from_slope(1.0 / thi ** 3, real=(m, c - sep / 2, c + sep / 2, -0.3 * thi)),
                                     1.0, ta, 1.0))
                rows.append(state_of(poly_from_slope(1.0 / thi ** 3, real=(m, -0.3 * thi), pairs=((c, sep / 2),)),
                                     1.0, ta, 1.0))
    pops["near_double"] = rows

    # two local minima r1 < r3 whose values tie exactly, to 1 ulp of f and to 1e-12 (max r2 between)
    rows = []
    for ta in (0.5, 0.1):
        tlo, thi, _ = kernel_interval(ta, 1.0)
        sp = thi - tlo
        for (u1, u3) in ((0.1, 0.9), (0.2, 0.6), (0.05, 0.3), (0.7, 0.95)):
            r1, r3, s = Fr(tlo + u1 * sp), Fr(tlo + u3 * sp), Fr(-0.5 * thi)
            a = 1.0 / thi ** 4
            g = poly_from_slope(1.0, real=(r1, r3, s), f0=0.0)[1:]    # g = (t - r1)(t - r3)(t - s), lowest first
            G0 = sum(g[k] * (r3 ** (k + 1) - r1 ** (k + 1)) / (k + 1) for k in range(len(g)))
            G1 = sum(g[k] * (r3 ** (k + 2) - r1 ** (k + 2)) / (k + 2) for k in range(len(g)))
            for delta in (0.0, 2.0 ** -52, -2.0 ** -52, 1e-12, -1e-12):
                # P(r3) - P(r1) = a (G1 - r2 G0) = delta
                r2 = (G1 - Fr(delta) / Fr(a)) / G0
                assert r1 < r2 < r3
                rows.append(state_of(poly_from_slope(a, real=(r1, r2, r3, s)), 1.0, ta, 1.0))
    pops["tied_minima"] = rows

    # the minimum at a sample abscissa inside [lo, hi]
    rows = []
    for xs in (0.3, 0.45, 0.6, 1e-3):
        for off in (0, 1, -1):
            r = _ulps(xs, off)
            Pt = poly_from_slope(1.0, real=(r, -0.4), pairs=((0.8, 0.5),))
            rows.append(state_of(Pt, 1.0, 1.0, xs, lo=1e-3, hi=0.6))
    for lo, hi in ((0.5, 2.0), (0.25, 1.0), (1.0, 1.5)):   # two samples, x1 = 1 inside [lo, hi]
        for off in (0, 1, -1):
            Pt = poly_from_slope(1.0, real=(_ulps(1.0, off), -2.0))
            rows.append(state_of(Pt, 1.0, 1.0, lo=lo, hi=hi))
    pops["sample_minimum"] = rows

    # a vanishing leading coefficient: exact dyadic quadratics and cubics, two and three samples
    rows = []
    for k in range(80):
        three = k % 2 == 1
        x2 = 2.0 ** -int(rng.integers(0, 6))
        x1 = x2 * (0.5 if three else 1.0)
        deg = 2 if k % 4 < 2 else 3
        co = [Fr(int(v)) for v in rng.integers(-4, 5, size=deg + 1)]   # lowest first
        if co[1] >= 0:
            co[1] = Fr(-1)
        if co[-1] == 0:
            co[-1] = Fr(1)
        # P(x) = sum co_i x^i, so P~(t) = sum co_i h^i t^i with h = x2
        rows.append(state_of([c * Fr(x2) ** i for i, c in enumerate(co)], x2, x1, x2 if three else None))
    pops["low_degree"] = rows

    # the two-sample cubic with its derivative's discriminant exactly zero, tiny positive and negative
    rows = []
    for r in (0.25, 0.125, 0.375, 0.5):
        for eps in (0.0, 2.0 ** -40, -2.0 ** -40, 2.0 ** -50, -2.0 ** -50):
            for a in (1.0, -1.0):
                for h in (1.0, 2.0 ** -20):
                    Pt = [Fr(1), Fr(a) * (3 * Fr(r) ** 2 + Fr(eps)), Fr(a) * -3 * Fr(r), Fr(a)]
                    rows.append(state_of(Pt, h, h))
    pops["cubic_discriminant"] = rows

    # x1 from 1 down to 1e-12 (the failing contractions), at varied x1 / x2
    rows = []
    for e in range(13):
        for _ in range(5):
            x1 = 10.0 ** -e * rng.uniform(0.5, 1.0)
            ratio = 10.0 ** rng.uniform(-3, np.log10(0.6))
            x2 = x1 / ratio
            tlo, thi, _ = kernel_interval(x1, x2)
            rows.append(state_of(_generic(rng, tlo, thi), x2, x1, x2))
    pops["tiny_steps"] = rows

    # |f| from 1e-8 to 1e8, with and without an offset as large as the variation
    rows = []
    for e in range(-8, 9):
        for off in (0.0, 1.0):
            for _ in range(2):
                x2 = rng.uniform(0.2, 1.0)
                x1 = x2 * rng.uniform(0.1, 0.6)
                tlo, thi, _ = kernel_interval(x1, x2)
                Pt = _generic(rng, tlo, thi)
                base = sum(abs(c) for c in Pt[1:])
                scale = Fr(10.0 ** e) / base
                rows.append(state_of([Fr(10.0 ** e) * off] + [c * scale for c in Pt[1:]], x2, x1, x2))
    pops["value_scale"] = rows

    # x1 / x2 from 1e-3 to 0.6
    rows = []
    for ratio in np.geomspace(1e-3, 0.6, 12):
        for _ in range(4):
            x2 = rng.uniform(0.05, 1.0)
            x1 = x2 * float(ratio)
            tlo, thi, _ = kernel_interval(x1, x2)
            rows.append(state_of(_generic(rng, tlo, thi), x2, x1, x2))
    pops["step_ratio"] = rows

    # two samples, g0 > 0: an interior local minimum at the larger critical point wins over both ends
    rows = []
    for r1 in (0.05, 0.1, 0.15):
        for r2 in (0.3, 0.4, 0.5):
            for h in (1.0, 2.0 ** -20, 3e-7):
                Pt = poly_from_slope(3.0, real=(r1, r2), f0=0.0)
                lo, hi = Fr(1e-3), Fr(0.6)
                if peval(Pt, Fr(r2)) < min(peval(Pt, lo), peval(Pt, hi)):
                    rows.append(state_of(Pt, h, h))
    assert len(rows) >= 12
    pops["cubic_larger_root"] = rows
    return {k: np.ascontiguousarray(v, dtype=np.float64) for k, v in pops.items()}


def thi_root_states():
    """States whose winning critical point lies 0 .. 4 ulps below thi, at step scales h that are not
    powers of two (so t -> x rounds): the returned step may exceed hi only by lm_solve's margin."""
    rng = np.random.default_rng(7)
    rows = []
    for _ in range(24):
        x2 = rng.uniform(0.05, 1.0)
        x1 = x2 * rng.uniform(0.1, 0.6)
        tlo, thi, _ = kernel_interval(x1, x2)
        for k in range(5):
            r = _ulps(thi, -k)
            # P decreasing on [tlo, r], minimum at r, a maximum just past hi
            Pt = poly_from_slope(1.0 / thi ** 4, real=(r, -thi), pairs=((0.5 * thi, 0.4 * thi),))
            rows.append(state_of(Pt, x2, x1, x2))
            _, thi1, _ = kernel_interval(x1, x1)                                # the same in two samples
            Pt = poly_from_slope(1.0, real=(_ulps(thi1, -k), -thi1))
            rows.append(state_of(Pt, x1, x1))
    return np.ascontiguousarray(rows, dtype=np.float64)


def last_ulp_quartics():
    """Quartics on [2^-10, thi] whose only root in the interval lies strictly between the last two doubles
    below thi, where the grid point t_31 = fma(w, 31, lo) falls one ulp short of thi: coef [n, 5], lohi
    [n, 2].  q(t) = (t - thi) s(t) + eps with s of small dyadic coefficients and eps > 0 one or a few
    ulps of the constant term, so that Horner's evaluation at thi is exact (q(thi) = eps) and q changes
    sign on [t_30, thi] without rounding doubt: a bracketing root finder must return that root."""
    tlo = 2.0 ** -10
    coef, lohi = [], []
    for k in range(17, 64):
        thi = k / 64.0
        w = (thi - tlo) * (1.0 / 31.0)
        t31 = float(Fr(w) * 31 + Fr(tlo))
        if t31 >= thi:
            continue
        for roots in ((1, 2, 3), (1, 2, 4), (0.5, 3, 5), (2, 2, 2)):
            sc = poly_from_slope(1.0, real=[-r for r in roots], f0=0.0)[1:]   # s, lowest first
            q = [Fr(0)] + sc                                                 # t s(t)
            for i in range(len(sc)):
                q[i] -= Fr(thi) * sc[i]                                      # - thi s(t)
            for j in range(1, 64):
                eps = j * Fr(math.ulp(float(q[0])))
                qq = [q[0] + eps] + q[1:]
                if peval(qq, Fr(t31)) >= 0:                                  # the root left the last ulp
                    break
                hf = [float(c) for c in reversed(qq)]
                if not all(Fr(a) == b for a, b in zip(hf, reversed(qq))):
                    continue
                coef.append(hf)
                lohi.append([tlo, thi])
    return np.ascontiguousarray(coef, dtype=np.float64), np.ascontiguousarray(lohi, dtype=np.float64)


# ---- quartics for the root finders ------------------------------------------------------------------
def constructed_quartics():
    """The derivative, in t = x / h, of the exact interpolant of every constructed three-sample state,
    rounded to double, on [lo / h, hi / h]: coef [n, 5] (highest degree first), lohi [n, 2]."""
    coef, lohi = [], []
    for rows in list(constructed_populations().values()) + [thi_root_states()]:
        for s in rows:
            if s[5] == 0.0:
                continue
            ex = Exact(s)
            h = Fr(max(s[2], s[6]))
            d = [c * h ** (k + 1) for k, c in enumerate(ex.dP)]      # d/dt P(t h), lowest first
            q = [float(c) for c in reversed(d)]
            lo, hi = float(ex.lo / h), float(ex.hi / h)
            if q[0] != 0.0 and lo < hi:
                coef.append(q)
                lohi.append([lo, hi])
    return np.ascontiguousarray(coef, dtype=np.float64), np.ascontiguousarray(lohi, dtype=np.float64)


def check_roots(q, lo, hi, got):
    """None if the roots `got` a finder returned for the quartic q on [lo, hi] agree with its exact
    roots, else why:
      * every returned value lies in [lo, hi] and within root_bound of some root of q (a complex one
        whose bound reaches the real axis included);
      * every simple real root inside [lo, hi], farther than twice its bound from any other root and
        than its bound from the ends, is returned within its bound;
      * the count differs from those only by roots that are not so separated (clusters, multiple
        roots, roots within their bound of an end, complex pairs within their bound of the axis)."""
    zs = all_roots(q)
    bounds = [root_bound(q, z) for z in zs]
    for r in got:
        if not lo <= r <= hi:
            return "returned %r outside [%r, %r]" % (r, lo, hi)
        if not any(abs(r - z) <= b for z, b in zip(zs, bounds)):
            return "returned %r is no root: roots %s" % (r, zs)
    required = optional = inside = 0
    for r, mult, sep in quartic_real_roots(q, lo, hi):
        inside += mult
        b = root_bound(q, r)
        if mult == 1 and sep > 2.0 * b and lo + b < r < hi - b:
            required += 1
            if not any(abs(g - r) <= b for g in got):
                return "exact root %r (bound %.3g, separation %.3g) not returned: %s" % (r, b, sep, got)
        else:
            optional += mult
    # roots within their bound of the interval and of the real axis, beyond the exact ones inside
    near = sum(1 for z, b in zip(zs, bounds) if abs(z.imag) <= b and lo - b <= z.real <= hi + b)
    optional += max(near - inside, 0)
    if not required <= len(got) <= required + optional:
        return "%d roots returned, %d required, %d optional" % (len(got), required, optional)
    return None


# ---- harvested states --------------------------------------------------------------------------------
# harvested states above this many are subsampled (deterministically); every state whose smallest
# sample step is below 0.02 is kept
HARVEST_CAP = 1500
SMALL_STEP = 0.02
RESTORED_FULL_STEP = dict(line_search_sufficient_function_decrease=0.9, max_num_line_search_step_size_iterations=3)


def _keep(states, cap=HARVEST_CAP, seed=0):
    three = states[:, 5] != 0.0
    smallest = np.where(three, np.minimum(states[:, 2], states[:, 6]), states[:, 2])
    small = smallest < SMALL_STEP
    rest = np.nonzero(~small)[0]
    room = max(cap - int(small.sum()), 0)
    if rest.size > room:
        rest = np.sort(np.random.default_rng(seed).choice(rest, room, replace=False))
    return np.ascontiguousarray(states[np.sort(np.concatenate([np.nonzero(small)[0], rest]))])


def _harvest(oracle, p, opt, positions=None):
    """Every interpolation state of one oracle solve (oracle_util.harvest_line_search_states, with a start)."""
    oracle.lib.lfr_ref_harvest(1)
    try:
        oracle.solve(p, opt, positions=positions)
        n = int(oracle.lib.lfr_ref_harvest_take(None, 0))
        st = np.zeros((n, 11))
        if n:
            oracle.lib.lfr_ref_harvest_take(st.ctypes.data, n)
    finally:
        oracle.lib.lfr_ref_harvest(0)
    return st


_harvest_cache = {}


def harvested_populations(oracle):
    """{name: states}: every line-search state of the oracle's solves (its harvest keeps the failing
    contractions too) of cfg2, cfg4 at 0.5, ring60, the line-search fixture, and of cfg1 and cfg2 at
    5 % under the restored-full-step options from a zero and a random start (the scenes and starts of
    test_gpu_restored_full_step.py); subsampled above HARVEST_CAP with every small-step state kept."""
    if not _harvest_cache:
        import os
        from conftest import get_problem
        from lfr_b200 import build_problem, wire
        out = {}
        for name, scale in (("cfg2", 1.0), ("cfg4", 0.5), ("ring60", 1.0)):
            out[name] = _harvest(oracle, get_problem(name, scale=scale)[1], oracle.default_options(n_threads=8))
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "linesearch_matches.pb")
        with open(path, "rb") as fh:
            p = build_problem(wire.decode_matching_file(fh.read()))
        out["linesearch_fixture"] = _harvest(oracle, p, oracle.default_options(n_threads=1))
        for name, scale in (("cfg1", 1.0), ("cfg2", 0.05)):
            p = get_problem(name, scale=scale)[1]
            opt = oracle.default_options(n_threads=8, **RESTORED_FULL_STEP)
            # test_gpu_tier_options.start_of: zeros, and uniform(-1.5, 1.5) seeded by the scene's name
            starts = [np.zeros((p.graph.n_nodes, 2)),
                      np.random.default_rng(7 + sum(map(ord, name))).uniform(-1.5, 1.5, size=(p.graph.n_nodes, 2))]
            out[name + "_restored_full_step"] = np.concatenate([_harvest(oracle, p, opt, s) for s in starts])
        _harvest_cache.update({k: _keep(v) for k, v in out.items()})
    return _harvest_cache


_exact_cache = {}


def population_exacts(name, states):
    """The Exact objects of a population's states, computed once per session."""
    key = (name, states.shape[0], hash(states.tobytes()))
    if key not in _exact_cache:
        _exact_cache[key] = [Exact(s) for s in states]
    return _exact_cache[key]
