"""The line search's step selection on the GPU (csrc/lfr_math.cuh :: hermite_minimizer through
lfr_debug_ls_minimizer, quartic_roots_grid and the derivative recursion through lfr_debug_quartic_roots)
against the exact statement of tests/ls_step_ref.py: the step must reach the exact minimum of the
interpolant over [lo, hi] to within K u Lambda, on every state the oracle's line searches go through
and on states built where the formulation and the 31-cell root grid are fragile.  No conditioning
filter: the states with tiny steps, where Ceres' own Vandermonde fit loses rank, are judged too."""
import ctypes as C

import numpy as np
import pytest

import ls_step_ref as R
from ls_step_ref import harvested_populations, population_exacts


def _gpu_steps(b200, states):
    f = b200.lib.lfr_debug_ls_minimizer
    f.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    states = np.ascontiguousarray(states, dtype=np.float64)
    xs = np.zeros(states.shape[0])
    assert f(states.ctypes.data, states.shape[0], xs.ctypes.data) == 0
    return xs


def _judge_population(b200, name, states, min_decided):
    xs = _gpu_steps(b200, states)
    fails, decided, worst, _ = R.judge_all(states, xs, R.K, population_exacts(name, states))
    print("gpu %-28s states %5d decided %5d worst %.3g" % (name, states.shape[0], decided, worst))
    assert not fails, (name, len(fails), fails[:3])
    assert decided >= min_decided, (name, decided, states.shape[0])


# every harvested population holds this many decided states at least (cfg2's slowest component's
# failing searches included: its population is the smallest)
HARVEST_MIN_DECIDED = 100


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2", "cfg4", "ring60", "linesearch_fixture", "cfg1_restored_full_step",
                                  "cfg2_restored_full_step"])
def test_harvested_states_reach_the_exact_minimum(b200, oracle, name):
    states = harvested_populations(oracle)[name]
    _judge_population(b200, "harvest_" + name, states, HARVEST_MIN_DECIDED)


# each constructed population: at least this fraction of its states decided
CONSTRUCTED_MIN_DECIDED = 0.9


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(R.constructed_populations().keys()))
def test_constructed_states_reach_the_exact_minimum(b200, name):
    states = R.constructed_populations()[name]
    _judge_population(b200, name, states, int(CONSTRUCTED_MIN_DECIDED * states.shape[0]))


@pytest.mark.gpu
def test_step_never_exceeds_hi_by_more_than_the_skip_rules_margin(b200):
    """lm_solve skips a contraction whose longest step (hi (1 + 2^-30)) is below the minimum step size:
    that is only right if no selected step exceeds hi by more.  The winning root sits 0 .. 4 ulps below
    thi = hi / h at step scales that round t -> x."""
    states = R.thi_root_states()
    xs = _gpu_steps(b200, states)
    hi = states[:, 10]
    assert np.all(xs <= hi * (1.0 + R.STEP_MARGIN)), np.max(xs / hi - 1.0)
    assert np.all(xs >= states[:, 9])
    # the root does win: the steps land within a few ulps of hi, on both sides
    assert np.all(np.abs(xs - hi) <= 8 * np.spacing(hi)), np.max(np.abs(xs - hi) / np.spacing(hi))
    _judge_population(b200, "thi_root", states, int(CONSTRUCTED_MIN_DECIDED * states.shape[0]))


def _scalable(states, k_max=40):
    """States whose scaled copies stay clear of overflow and subnormals for |k| <= k_max."""
    a = np.abs(states[:, [1, 2, 4, 6, 8, 9, 10]])
    nz = np.where(a > 0, a, 1.0)
    lim = 2.0 ** (k_max + 60)
    return np.all((nz > np.finfo(np.float64).tiny * lim) & (nz < np.finfo(np.float64).max / lim), axis=1)


@pytest.mark.gpu
def test_power_of_two_rescaling_scales_the_step_exactly(b200, oracle):
    """x1, x2, lo, hi times 2^k and g0, g1, g2 times 2^-k leave every quantity of hermite_minimizer in
    the normalised variable bit for bit the same (h, 1 / h and every product with them scale exactly),
    so the step must be exactly 2^k times the original, k = -40 .. 40."""
    pops = dict(R.constructed_populations())
    pops["thi_root"] = R.thi_root_states()
    pops.update(harvested_populations(oracle))
    states = np.concatenate(list(pops.values()))
    states = states[_scalable(states)]
    assert states.shape[0] > 5000, states.shape
    base = _gpu_steps(b200, states)
    ks = np.arange(-40, 41)
    big = np.repeat(states[None], ks.size, axis=0)
    sc = np.ldexp(1.0, ks)[:, None]
    for col in (2, 6, 9, 10):
        big[:, :, col] *= sc
    for col in (1, 4, 8):
        big[:, :, col] /= sc
    xs = _gpu_steps(b200, big.reshape(-1, 11)).reshape(ks.size, -1)
    want = base[None] * sc
    bad = np.argwhere(xs != want)
    assert bad.size == 0, (bad.shape[0], [(int(ks[i]), states[j].tolist(), xs[i, j], want[i, j]) for i, j in bad[:3]])


# ---- the quartic root finders against exact roots -------------------------------------------------
def _quartic_roots(b200, coef, lohi, use_grid):
    n = coef.shape[0]
    f = b200.lib.lfr_debug_quartic_roots
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
    roots = np.zeros((n, 4))
    cnt = np.zeros(n, dtype=np.int32)
    coef, lohi = np.ascontiguousarray(coef), np.ascontiguousarray(lohi)
    assert f(coef.ctypes.data, lohi.ctypes.data, n, use_grid, roots.ctypes.data, cnt.ctypes.data) == 0
    return roots, cnt


@pytest.mark.gpu
@pytest.mark.parametrize("use_grid", [1, 0], ids=["grid", "recursion"])
def test_quartic_roots_match_exact_roots(b200, use_grid):
    from test_gpu_parity import _quartic_cases
    c1, l1 = _quartic_cases(np.random.default_rng(99), 2000)
    c2, l2 = R.constructed_quartics()
    coef, lohi = np.concatenate([c1, c2]), np.concatenate([l1, l2])
    roots, cnt = _quartic_roots(b200, coef, lohi, use_grid)
    bad = []
    for k in range(coef.shape[0]):
        msg = R.check_roots(coef[k], float(lohi[k, 0]), float(lohi[k, 1]), list(roots[k, :cnt[k]]))
        if msg:
            bad.append((k, msg))
    assert not bad, (len(bad), bad[:3])
    assert (cnt >= 3).sum() > 100 and c2.shape[0] > 1000


@pytest.mark.gpu
@pytest.mark.parametrize("use_grid", [1, 0], ids=["grid", "recursion"])
def test_root_in_the_last_ulp_below_hi_is_found(b200, use_grid):
    """A root strictly between the last two doubles below hi, where fma(w, 31, lo) falls one ulp short of
    hi: q(hi) evaluates exactly, so a bracketing finder must return exactly that one root (the grid's
    last point is hi itself, not fma(w, 31, lo))."""
    coef, lohi = R.last_ulp_quartics()
    assert coef.shape[0] >= 20
    roots, cnt = _quartic_roots(b200, coef, lohi, use_grid)
    assert np.all(cnt == 1), np.nonzero(cnt != 1)[0]
    hi = lohi[:, 1]
    assert np.all((roots[:, 0] >= hi - 4 * np.spacing(hi)) & (roots[:, 0] <= hi)), roots[:, 0] - hi
