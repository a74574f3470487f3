"""The grid route's root polish (csrc/lfr_math.cuh :: quartic_roots_grid, cell_root_n): each root
of a one-root cell starts from one Halley step on the Taylor expansion the grid point holds, and
Newton with a double-precision quotient finishes it.

- on the GPU, the roots it returns are those of an extended-precision Newton to a few ulps,
  beyond what the root's conditioning allows in double precision;
- on the CPU, a model of the start and the safeguarded Newton on every quintic interpolant the
  line searches of cfg2 go through takes at most two Horner evaluations per root in the median."""
import ctypes as C

import numpy as np
import pytest

from conftest import get_problem
from test_gpu_parity import _quartic_cases
from test_grid_roots_model import classify, taylor

EPS = np.finfo(np.float64).eps


def _refine_ld(q, r):
    """Newton in np.longdouble from r on the quartic q (highest degree first)."""
    ql = [np.longdouble(c) for c in q]
    x = np.longdouble(r)
    for _ in range(8):
        f, df = ql[0], np.longdouble(0)
        for c in ql[1:]:
            df = df * x + f
            f = f * x + c
        if df == 0:
            break
        x = x - f / df
    return x


@pytest.mark.gpu
def test_grid_roots_are_correctly_rounded_to_a_few_ulps(b200, oracle):
    rng = np.random.default_rng(99)
    n = 6000
    coef, lohi = _quartic_cases(rng, n)
    f = b200.lib.lfr_debug_quartic_roots
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
    roots = np.zeros((n, 4))
    cnt = np.zeros(n, dtype=np.int32)
    assert f(coef.ctypes.data, lohi.ctypes.data, n, 1, roots.ctypes.data, cnt.ctypes.data) == 0
    ro = np.zeros(8)
    checked = 0
    for k in range(n):
        no = oracle.lib.lfr_ref_polynomial_roots(coef[k].ctypes.data, 5, float(lohi[k, 0]), float(lohi[k, 1]),
                                                 ro.ctypes.data)
        if no != cnt[k] or no == 0:
            continue
        ref = ro[:no].copy()
        allr = np.roots(coef[k])
        for i in range(no):
            # well separated: no other root of q (real or complex) within 1e-3
            others = np.abs(allr - ref[i])
            if np.sort(others)[1] < 1e-3:
                continue
            x = _refine_ld(coef[k], ref[i])
            q = coef[k]
            dq = np.polyval(np.polyder(q), ref[i])
            # the accuracy double-precision evaluation of q allows at this root (its condition)
            cond = 8 * EPS * np.polyval(np.abs(q), abs(ref[i])) / abs(dq)
            err = abs(np.longdouble(roots[k, i]) - x)
            assert err <= 4 * np.spacing(abs(float(x))) + cond, (k, i, roots[k, i], float(x), float(err))
            checked += 1
    assert checked > 3000, checked


def _quintic_der(s):
    """The derivative of the kernel's quintic interpolant (normalised t) and [tlo, thi], or None."""
    f0, g0, x1, f1, g1, three, x2, f2, g2, lo, hi = s
    if three == 0.0:
        return None
    h = max(x1, x2)
    ih = 1.0 / h
    g0h = g0 * h
    ta, tb = x1 * ih, x2 * ih
    ita, itb, iw = 1.0 / ta, 1.0 / tb, 1.0 / (tb - ta)
    Sa = (f1 - f0 - g0h * ta) * ita * ita
    Sb = (f2 - f0 - g0h * tb) * itb * itb
    Da = ((g1 - g0) * h - 2.0 * ta * Sa) * ita * ita
    Db = ((g2 - g0) * h - 2.0 * tb * Sb) * itb * itb
    m = (Sb - Sa) * iw
    e2 = (m - Da) * iw
    e3 = ((Db - m) - (m - Da)) * iw * iw
    c = [e3, e2 - e3 * (2.0 * ta + tb), Da + ta * (e3 * (ta + 2.0 * tb) - 2.0 * e2),
         Sa + ta * (ta * (e2 - e3 * tb) - Da), g0h]
    if c[0] == 0.0:
        return None
    return [5.0 * c[0], 4.0 * c[1], 3.0 * c[2], 2.0 * c[3], c[4]], lo * ih, hi * ih


def _polish_count(q, x0, a, b, fa, fb):
    """Horner evaluations of cell_root_n's safeguarded Newton from x0 (exact quotient)."""
    xl, xh = (a, b) if fa < 0.0 else (b, a)
    x = x0
    if not (min(a, b) < x < max(a, b)):
        x = a - fa * (b - a) / (fb - fa)
        if not (min(a, b) < x < max(a, b)):
            x = 0.5 * (a + b)
    for nh in range(1, 101):
        f, df = q[0], 0.0
        for c in q[1:]:
            df = df * x + f
            f = f * x + c
        if f == 0.0:
            return nh
        if f < 0.0:
            xl = x
        else:
            xh = x
        dx = f / df if df != 0.0 else np.inf
        xn = x - dx
        if xn == x:
            return nh
        if not (min(xl, xh) <= xn <= max(xl, xh)):
            xn = 0.5 * (xl + xh)
            dx = x - xn
        if xn == x:
            return nh
        x = xn
        if abs(dx) <= 1e-8 * abs(x):
            return nh
    return 100


def test_halley_start_takes_two_horner_evaluations_per_root(oracle):
    from oracle_util import harvest_line_search_states
    _, p = get_problem("cfg2")
    _, _, states = harvest_line_search_states(oracle, p, oracle.default_options(n_threads=8))
    counts = []
    for s in states:
        d = _quintic_der(s)
        if d is None:
            continue
        q, tlo, thi = d
        kinds, ts = classify(q, tlo, thi)
        if kinds is None:
            continue
        for L, kind in enumerate(kinds):
            if kind != 1:
                continue
            a4, a3, a2, _, _ = taylor(q, ts[L])
            fb = np.polyval(q, ts[L + 1])
            den = a3 * a3 - a2 * a4
            x0 = ts[L] - a4 * a3 / den if den != 0.0 else ts[L]
            counts.append(_polish_count(q, x0, ts[L], ts[L + 1], a4, fb))
    assert len(counts) > 20, len(counts)
    assert np.median(counts) <= 2, np.bincount(counts)
