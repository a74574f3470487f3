"""An extended-precision statement of the first Levenberg-Marquardt step of one component.

Ceres' TrustRegionMinimizer (LEVENBERG_MARQUARDT, SPARSE_NORMAL_CHOLESKY) takes its first step from
IterationZero at the initial radius.  Written here from the `lfr_problem` arrays, the options and the
start point alone, in np.longdouble (64-bit mantissa), independently of the CPU oracle's code:

  * IterationZero: free start values are projected onto [-bound, bound]; roots are constant as given.
  * Residual blocks (solve.cc:98-143): an out-edge v -> w is a Cauchy block when v and w share a track, a
    Tukey block when they only share a component, and no block otherwise; a block whose two ends are
    both roots is constant and dropped.  Every kept directed edge is its own block.
  * r = x_w - x_v - flow(clamp(x_v)), J_v = -(I + grad flow), J_w = I (cost.cc's biquadratic
    interpolation; a clamped coordinate has zero derivative).
  * Loss: a = sim rho'(|r|^2); r and J are scaled by sqrt(a) (Ceres' Corrector where rho'' <= 0, which
    holds for Cauchy and both Tukey variants).
  * S = 1 / (1 + sqrt(diag H)), H = J^T J, g = J^T r;  D^2 = clamp(diag(S H S), min_lm_diagonal,
    max_lm_diagonal) / radius;  A = S H S + D^2, b = S g;  A y = b, dl = -S y.
  * The solve: a float64 factorisation, then iterative refinement with the residual in longdouble until
    the correction stalls.
  * Derived values: Ceres' model cost change -(J dl)^T (r + J dl / 2), g . dl, |dl|_inf, the cost
    1/2 sum sim rho and gmax = |x - P(x - g)|_inf, and kappa_2(A) of the float64 A.
  * step_at: the same step at any accepted point with iteration 0's Jacobi scaling kept (Ceres fixes it
    in iteration 0 only); first_step is step_at at the start.

The line search and an accepted step (probe): at xc = P(x + alpha dl), alpha a power of two and dl the
device's own step, the cost, phi' = grad f(xc) . dl over EVERY free coordinate (Ceres'
LineSearchFunction dots the full gradient at the projected point, clamped coordinates included), |x - xc|,
|xc| and gmax at xc.  xc is known bit for bit, so each value comes with a bound on the error of a float64
evaluation of the kernels' operations at that very point.

PROBE_BOUNDS: standard forward error analysis, u = 2^-53, gamma_k = k u / (1 - k u); each rounding of a
product or sum of computed values is (1 + delta), |delta| <= u, and errors of inputs are carried to first
order with their computed magnitudes inflated by their own bounds (so second-order terms are covered).
  (1) r_e = x_d - x_s - sum_ij Lr_i Lc_j D_ij.  Each Lagrange weight takes up to 3 roundings, each of the
      two nested three-term sums 3, the two subtractions 2: |dr_k| <= gamma_14 m_k with the magnitude sum
      m_k = |x_d| + |x_s| + sum_ij |Lr_i Lc_j D_ijk|.  M = I + grad flow: |dM_kj| <= gamma_11 (delta_kj +
      sum |dL L D|).  (The flow grid is float32, exact in double; the clamp of x_s to +-0.5 is exact.)
  (2) s = |r|^2: |ds| <= sum_k (2 |r_k| |dr_k| + |dr_k|^2) + gamma_3 sum_k (|r_k| + |dr_k|)^2.
  (3) Losses.  Cauchy: sum = 1 + s c (c = 1 / b and b = a^2 are rounded on the host), log to one ulp
      (2 u relative), 1/2 sim b log in three roundings; a = sim / sum in two.  So
        |d log| <= d sum / (sum - d sum) + 2 u |log|,   d sum = (ds / b + gamma_4 s / b + u sum)(1 + u),
        |d(1/2 sim rho)| <= 1/2 sim b (|d log| + gamma_4 (|log| + |d log|)),
        |da| <= a (d sum / (sum - d sum) + gamma_3) (x 1.01 for the second order).
      Tukey: v = 1 - s / a^2 to dv = (ds / a^2 + gamma_4 s / a^2 + u (1 + s / a^2))(1 + u), V = max(v, 0)
      + dv bounds |v| on whichever branch the kernel takes (rho is C^1 at the threshold, so a branch
      taken on the other side of it costs at most the terms in V), then
        |d(1/2 sim rho)| <= 1/2 sim rho0 (3 V^2 dv + gamma_2 V^3 + u (1 + V^3) + gamma_5 (1 + V^3)),
        |da| <= sim rho1 (2 V dv + dv^2 + gamma_3 V^2);
      an edge with s - ds > a^2 is an outlier on both sides: a = 0 exactly, rho within gamma_3.
  (4) cost = sum_e 1/2 sim rho_e in any order: sum_e |d(1/2 sim rho_e)| + gamma_{E-1} sum_e (|1/2 sim rho_e|
      + its bound).
  (5) phi' = sum_e a_e r_e^T (dl_d - M_e dl_s) = a sum of products a r_k M_kj dl_j and a r_k dl_k.  Every
      tier and route (the fused edge pass, the per-node gradient lists, the twin tuples, the serial
      path) forms each product and adds it along a chain of at most 2 E + n + 16 roundings (at most 6
      inside one edge's term or gradient contribution, E accumulations into one node or one thread, n
      over the nodes, 9 in the warp and CTA reductions).  With W_k = |dl_d,k| + sum_j (|M_kj| + |dM_kj|)
      |dl_s,j| and R_k = |r_k| + |dr_k|:
        |d phi'| <= sum_e (|da| R.W + a |dr|.W + a sum_k R_k sum_j |dM_kj| |dl_s,j|)
                    + gamma_{2E+n+16} sum_e (a + |da|) R.W.
      Each gradient coordinate g_i gets the same bound over the edges that touch node i.
  (6) gmax = |xc - P(xc - g)|_inf: P is 1-Lipschitz and the two subtractions round once each, so
      |d gmax| <= max_i |dg_i| + 2 u max_i (|xc_i| + |g_i| + |dg_i|).
  (7) |x - xc| and |xc|: xc is exact, so each term rounds at most twice, the sum of n terms n - 1 times and
      the square root once: relative gamma_{n+1} / 2 + u.
The longdouble statement itself is exact to about 2^-64 of the same magnitude sums, 2^-11 of the bounds.
Nothing here is fitted to any kernel's output.
"""
from dataclasses import dataclass

import numpy as np
import scipy.linalg
import scipy.sparse
import scipy.sparse.linalg

LD = np.longdouble
DBL_MIN = np.finfo(np.float64).tiny
CAUCHY, TUKEY = 1, 2          # LFR_EDGE_* (include/lfr.h)
DENSE_MAX = 1600              # unknowns up to which A is factorised and its kappa taken densely


def option_values(o):
    """The option fields the step reads, from an lfr_options struct (or anything with those attributes)."""
    return {k: float(getattr(o, k)) for k in ("bound", "cauchy_a", "tukey_a", "tukey_variant", "min_lm_diagonal",
                                               "max_lm_diagonal", "initial_trust_region_radius")}


# ---------------------------------------------------------------------------------------------------
# one residual block
# ---------------------------------------------------------------------------------------------------
def _lag(t):
    return np.stack([LD(2) * t * (t - LD(0.5)), LD(-4) * (t - LD(0.5)) * (t + LD(0.5)), LD(2) * t * (t + LD(0.5))],
                    axis=-1)


def _dlag(t):
    return np.stack([LD(4) * t - LD(1), LD(-8) * t, LD(4) * t + LD(1)], axis=-1)


def edge_terms(flow, xs, xd):
    """Residual r [E, 2] and d r / d x_src [E, 2, 2] (rows: residual channel, columns: coordinate) of edges
    with flow grids `flow` [E, 18] at source / destination positions xs, xd [E, 2], in longdouble."""
    D = np.asarray(flow).astype(np.float64).astype(LD).reshape(-1, 3, 3, 2)
    xs = np.asarray(xs).astype(LD)
    xd = np.asarray(xd).astype(LD)
    c = np.clip(xs, LD(-0.5), LD(0.5))
    free = (c == xs)
    L0, L1 = _lag(c[:, 0]), _lag(c[:, 1])
    f = np.einsum("ei,ej,eijk->ek", L0, L1, D)
    d0 = np.einsum("ei,ej,eijk->ek", _dlag(c[:, 0]), L1, D) * free[:, :1]
    d1 = np.einsum("ei,ej,eijk->ek", L0, _dlag(c[:, 1]), D) * free[:, 1:]
    r = xd - xs - f
    J = np.empty((len(r), 2, 2), LD)
    J[:, :, 0] = -d0
    J[:, :, 1] = -d1
    J[:, 0, 0] -= 1
    J[:, 1, 1] -= 1
    return r, J


def loss_terms(kind, sim, s, ov):
    """sim * rho(s) and sim * rho'(s) of Cauchy (kind 1) / Tukey (kind 2) blocks, in longdouble."""
    s = np.asarray(s, LD)
    sim = np.asarray(sim).astype(np.float64).astype(LD)
    b = LD(ov["cauchy_a"]) ** 2
    rho_c = b * np.log1p(s / b)
    d1_c = np.maximum(LD(DBL_MIN), LD(1) / (LD(1) + s / b))
    a2 = LD(ov["tukey_a"]) ** 2
    v = LD(1) - np.minimum(s, a2) / a2
    if int(ov["tukey_variant"]) == 2:
        rho_t, d1_t = a2 / 3 * (1 - v ** 3), v * v
    else:
        rho_t, d1_t = a2 / 6 * (1 - v ** 3), v * v / 2
    inside = s <= a2
    rho_t = np.where(inside, rho_t, a2 / (3 if int(ov["tukey_variant"]) == 2 else 6))
    d1_t = np.where(inside, d1_t, LD(0))
    cauchy = np.asarray(kind) == CAUCHY
    return sim * np.where(cauchy, rho_c, rho_t), sim * np.where(cauchy, d1_c, d1_t)


# ---------------------------------------------------------------------------------------------------
# the linear solve
# ---------------------------------------------------------------------------------------------------
class SymSparse:
    """A symmetric matrix as COO triplets (duplicates summed) in longdouble, with a float64 copy."""

    def __init__(self, n, rows, cols, vals):
        self.n = n
        key = rows.astype(np.int64) * n + cols
        uniq, inv = np.unique(key, return_inverse=True)
        v = np.zeros(len(uniq), LD)
        np.add.at(v, inv, vals)
        self.rows, self.cols, self.vals = (uniq // n).astype(np.int64), (uniq % n).astype(np.int64), v

    def matvec(self, y):
        out = np.zeros(self.n, LD)
        np.add.at(out, self.rows, self.vals * np.asarray(y, LD)[self.cols])
        return out

    def float64(self):
        return scipy.sparse.csc_matrix((self.vals.astype(np.float64), (self.rows, self.cols)), shape=(self.n, self.n))

    def dense(self):
        d = np.zeros((self.n, self.n), LD)
        d[self.rows, self.cols] = self.vals
        return d


def solve_refined(A, b, max_steps=40):
    """y with A y = b: a float64 factorisation of A (dense Cholesky, or sparse LU for large n), then
    iterative refinement with residuals b - A y in longdouble until the correction stops shrinking.
    `A` is a SymSparse or a dense longdouble array.  Returns (y in longdouble, refinement steps)."""
    b = np.asarray(b, LD)
    if isinstance(A, SymSparse):
        n, mv = A.n, A.matvec
        if n <= DENSE_MAX:
            A64 = A.float64().toarray()
        else:
            A64 = A.float64()
    else:
        n = A.shape[0]
        A = np.asarray(A, LD)
        mv = lambda y: A @ y  # noqa: E731
        A64 = A.astype(np.float64)
    if scipy.sparse.issparse(A64):
        lu = scipy.sparse.linalg.splu(A64)
        fsolve = lu.solve
    else:
        try:
            cf = scipy.linalg.cho_factor(A64)
            fsolve = lambda v: scipy.linalg.cho_solve(cf, v)  # noqa: E731
        except np.linalg.LinAlgError:
            lu = scipy.linalg.lu_factor(A64)
            fsolve = lambda v: scipy.linalg.lu_solve(lu, v)  # noqa: E731
    y = fsolve(b.astype(np.float64)).astype(LD)
    prev = np.inf
    for k in range(max_steps):
        res = b - mv(y)
        d = fsolve(res.astype(np.float64)).astype(LD)
        nd = float(np.abs(d).max()) if n else 0.0
        y = y + d
        if nd == 0.0 or nd >= 0.5 * prev or nd <= 1e-21 * float(np.abs(y).max()):
            return y, k + 1
        prev = nd
    return y, max_steps


def kappa2(A):
    """kappa_2 of the float64 A (symmetric positive definite): the ratio of its extreme eigenvalues."""
    if A.n <= DENSE_MAX:
        return float(np.linalg.cond(A.float64().toarray()))
    A64 = A.float64()
    hi = scipy.sparse.linalg.eigsh(A64, k=1, which="LA", return_eigenvectors=False)[0]
    lo = scipy.sparse.linalg.eigsh(A64, k=1, sigma=0.0, which="LM", return_eigenvectors=False)[0]
    return float(hi / lo)


# ---------------------------------------------------------------------------------------------------
# the component's step
# ---------------------------------------------------------------------------------------------------
@dataclass
class Step:
    free_nodes: np.ndarray   # [nf] node ids of the free nodes (comp_nodes order): unknowns 2 f, 2 f + 1
    dl: np.ndarray           # [nf, 2] longdouble
    y: np.ndarray            # [2 nf] longdouble
    A: SymSparse
    b: np.ndarray            # [2 nf] longdouble
    S: np.ndarray            # [2 nf] longdouble Jacobi scaling
    kappa: float
    cost: float
    gmax: float
    model_change: float
    gd: float
    dmax: float
    n_blocks: int
    refine_steps: int

    @property
    def n(self):
        return 2 * len(self.free_nodes)


def kept_blocks(p, slot):
    """(src, dst, edge index, kind) of the kept directed edges of dispatch slot `slot`, in out-edge order."""
    g = p.graph
    nodes = p.comp_nodes[p.comp_ptr[slot]:p.comp_ptr[slot + 1]].astype(np.int64)
    rp = g.row_ptr.astype(np.int64)
    deg = rp[nodes + 1] - rp[nodes]
    src = np.repeat(nodes, deg)
    eidx = np.concatenate([np.arange(rp[v], rp[v + 1]) for v in nodes]) if len(nodes) else np.zeros(0, np.int64)
    dst = g.edges["dst"][eidx].astype(np.int64)
    cauchy = p.track[src] == p.track[dst]
    tukey = ~cauchy & (p.comp[src] == p.comp[dst])
    keep = (cauchy | tukey) & ~((p.is_root[src] != 0) & (p.is_root[dst] != 0))
    kind = np.where(cauchy, CAUCHY, TUKEY)
    return src[keep], dst[keep], eidx[keep], kind[keep]


def step_at(p, slot, options, x, S=None, radius=None, want_kappa=True):
    """The LM step of dispatch slot `slot` at positions `x` [N, 2] under lfr_options `options` (at `radius`,
    default the options' initial radius).  S=None is iteration 0: the free values of x are projected onto
    the box and the Jacobi scaling is fixed from H at x.  A given S [2 nf] is that scaling, kept: Ceres
    fixes it in iteration 0 only, and x (an accepted point, inside the box) is taken as it is."""
    ov = option_values(options)
    radius = LD(ov["initial_trust_region_radius"] if radius is None else radius)
    g = p.graph
    nodes = p.comp_nodes[p.comp_ptr[slot]:p.comp_ptr[slot + 1]].astype(np.int64)
    free_nodes = nodes[p.is_root[nodes] == 0]
    nf = len(free_nodes)
    n = 2 * nf
    fidx = np.full(g.n_nodes, -1, np.int64)
    fidx[free_nodes] = np.arange(nf)
    x = np.asarray(x, np.float64).astype(LD).copy()
    bound = LD(ov["bound"])
    if S is None:
        x[free_nodes] = np.clip(x[free_nodes], -bound, bound)

    src, dst, eidx, kind = kept_blocks(p, slot)
    e = g.edges[eidx]
    r, Js = edge_terms(e["flow"], x[src], x[dst])
    srho, a = loss_terms(kind, e["sim"], (r * r).sum(axis=1), ov)
    cost = LD(0.5) * srho.sum()

    # H = sum a J^T J and g = sum a J^T r, block by block (J_dst = I)
    fs, fd = fidx[src], fidx[dst]
    rows, cols, vals = [], [], []
    gvec = np.zeros(n, LD)
    JtJ = np.einsum("eki,ekj->eij", Js, Js)
    Jtr = np.einsum("eki,ek->ei", Js, r)
    for i in range(2):
        m = fs >= 0
        np.add.at(gvec, 2 * fs[m] + i, a[m] * Jtr[m, i])
        m = fd >= 0
        np.add.at(gvec, 2 * fd[m] + i, a[m] * r[m, i])
        for j in range(2):
            m = fs >= 0
            rows.append(2 * fs[m] + i); cols.append(2 * fs[m] + j); vals.append(a[m] * JtJ[m, i, j])
            m = fd >= 0
            if i == j:
                rows.append(2 * fd[m] + i); cols.append(2 * fd[m] + j); vals.append(a[m])
            m = (fs >= 0) & (fd >= 0)
            # (src, dst) block = a J_src^T, (dst, src) block = a J_src
            rows.append(2 * fs[m] + i); cols.append(2 * fd[m] + j); vals.append(a[m] * Js[m, j, i])
            rows.append(2 * fd[m] + i); cols.append(2 * fs[m] + j); vals.append(a[m] * Js[m, i, j])
    rows = np.concatenate(rows + [np.arange(n)])
    cols = np.concatenate(cols + [np.arange(n)])
    vals = np.concatenate(vals + [np.zeros(n, LD)])   # every diagonal entry present
    H = SymSparse(n, rows, cols, vals)
    diag = np.zeros(n, LD)
    on = H.rows == H.cols
    diag[H.rows[on]] = H.vals[on]
    S = LD(1) / (LD(1) + np.sqrt(diag)) if S is None else np.asarray(S, LD)
    d2 = np.clip(diag * S * S, LD(ov["min_lm_diagonal"]), LD(ov["max_lm_diagonal"])) / radius
    avals = H.vals * S[H.rows] * S[H.cols] + np.where(on, d2[H.rows], LD(0))
    A = SymSparse(n, H.rows, H.cols, avals)
    b = S * gvec
    y, steps = solve_refined(A, b)
    dl = -S * y

    # Ceres' model cost change: -(J dl)^T (r + J dl / 2), with the corrected J and r
    dls = np.zeros((len(src), 2), LD)
    dld = np.zeros((len(src), 2), LD)
    dls[fs >= 0] = dl.reshape(-1, 2)[fs[fs >= 0]]
    dld[fd >= 0] = dl.reshape(-1, 2)[fd[fd >= 0]]
    Jdl = np.einsum("eij,ej->ei", Js, dls) + dld
    model_change = -(a[:, None] * Jdl * (r + Jdl / 2)).sum()
    xf = x[free_nodes].reshape(-1)
    gmax = np.abs(xf - np.clip(xf - gvec, -bound, bound)).max() if n else LD(0)
    return Step(free_nodes=free_nodes, dl=dl.reshape(-1, 2), y=y, A=A, b=b, S=S,
                kappa=kappa2(A) if (want_kappa and n) else float("nan"), cost=float(cost), gmax=float(gmax),
                model_change=float(model_change), gd=float((gvec * dl).sum()),
                dmax=float(np.abs(dl).max()) if n else 0.0, n_blocks=len(src), refine_steps=steps)


def first_step(p, slot, options, start, radius=None, want_kappa=True):
    """The first LM step of dispatch slot `slot` from `start` [N, 2] under lfr_options `options` (at
    `radius`, default the options' initial radius)."""
    return step_at(p, slot, options, start, radius=radius, want_kappa=want_kappa)


def step_bound(n, kappa):
    """The relative error a backward-stable solve of an n-unknown system of condition kappa may have:
    8 n kappa 2^-53."""
    return 8.0 * n * kappa * 2.0 ** -53


# ---------------------------------------------------------------------------------------------------
# the line search's trial point, its slope and the accepted point's bookkeeping
# ---------------------------------------------------------------------------------------------------
U = 2.0 ** -53


def gamma(k):
    """gamma_k = k u / (1 - k u): the relative error bound of k roundings."""
    return k * U / (1.0 - k * U)


@dataclass
class Probe:
    """The probe of one component at xc = P(x + alpha dl); each value with its derived bound (PROBE_BOUNDS)."""
    free_nodes: np.ndarray
    xc: np.ndarray          # [N, 2] float64: x + alpha dl rounded once, clipped to the box
    clamped: np.ndarray     # [nf, 2] bool: free coordinates the box clips at xc
    cost: float
    cost_bound: float
    cost_mag: float         # sum of |1/2 sim rho| over the kept edges
    dphi: float             # grad f(xc) . dl over every free coordinate, clamped ones included
    dphi_bound: float
    dphi_mag: float         # sum of the magnitudes of the products a r_k M_kj dl_j and a r_k dl_k
    dn: float               # |x - xc| over the free coordinates
    xn: float               # |xc| over the free coordinates
    norm_bound: float       # relative bound of dn and xn
    gmax: float             # |xc - P(xc - g)|_inf
    gmax_bound: float
    g: np.ndarray           # [2 nf] longdouble gradient at xc
    g_bound: np.ndarray     # [2 nf] its per-coordinate bound
    clamped_share: float    # |sum of g_i dl_i over the clamped coordinates|
    dup_share: float        # largest |a r^T (dl_d - M dl_s)| of an edge whose (src, dst) is kept twice or more
    mt_diff: float          # |phi' with M^T in place of M - phi'|
    grid_cross: int         # free coordinates on the source side of an edge that cross +-0.5 between x and xc


def _edge_eval_bounds(flow, xs, xd, kind, sim, ov):
    """The longdouble evaluation of every kept edge and the bounds of a float64 evaluation by the kernels'
    operations (PROBE_BOUNDS, (1) - (3)): r, M, a, 1/2 sim rho with their error bounds."""
    D = np.asarray(flow).astype(np.float64).astype(LD).reshape(-1, 3, 3, 2)
    xs = np.asarray(xs).astype(LD)
    xd = np.asarray(xd).astype(LD)
    r, J = edge_terms(flow, xs, xd)
    M = -J
    c = np.clip(xs, LD(-0.5), LD(0.5))
    free = (c == xs)
    aD = np.abs(D)
    L0, L1 = np.abs(_lag(c[:, 0])), np.abs(_lag(c[:, 1]))
    mf = np.einsum("ei,ej,eijk->ek", L0, L1, aD)
    md0 = np.einsum("ei,ej,eijk->ek", np.abs(_dlag(c[:, 0])), L1, aD) * free[:, :1]
    md1 = np.einsum("ei,ej,eijk->ek", L0, np.abs(_dlag(c[:, 1])), aD) * free[:, 1:]
    # (1) r: the Lagrange weights carry 3 roundings, each of the two nested three-term sums 3 more, the
    # two subtractions 2: 14 roundings against |x_d| + |x_s| + sum |L L D|
    er = gamma(14) * (np.abs(xd) + np.abs(xs) + mf)
    # M = I + grad flow: the derivative weights carry 1 rounding, 1 + . one more: 11
    eM = np.empty_like(M)
    eM[:, :, 0] = gamma(11) * md0
    eM[:, :, 1] = gamma(11) * md1
    eM[:, 0, 0] += gamma(11)
    eM[:, 1, 1] += gamma(11)
    # (2) s = r0^2 + r1^2
    s = (r * r).sum(axis=1)
    R = np.abs(r) + er
    es = (2 * np.abs(r) * er + er * er).sum(axis=1) + gamma(3) * (R * R).sum(axis=1)
    sim = np.asarray(sim).astype(np.float64).astype(LD)
    srho, a = loss_terms(kind, sim, s, ov)
    hr = srho / 2
    cauchy = np.asarray(kind) == CAUCHY
    # Cauchy: sum = 1 + s c with c = 1 / b, b = a_c^2 (2 roundings each), log to 1 ulp (2 u), then b log and
    # 1/2 sim b log (3 roundings); a = sim / sum (2)
    b = LD(ov["cauchy_a"]) ** 2
    sm = 1 + s / b
    esum = (es / b + gamma(4) * s / b + U * sm) * (1 + gamma(1))
    lg = np.log(sm)
    elog = esum / (sm - esum) + 2 * U * np.abs(lg)
    ehr_c = sim * b / 2 * (elog + gamma(4) * (np.abs(lg) + elog))
    ea_c = (a * (esum / (sm - esum) + gamma(3))) * 1.01
    # Tukey: v = 1 - s / a_t^2 (inverse 2 roundings, product 1, difference 1), v^3 (2), 1 - v^3 (1), rho0
    # (2), two products (2); a = sim rho1 v^2.  V bounds |v| at the device's branch, whichever it takes
    a2 = LD(ov["tukey_a"]) ** 2
    rho0 = a2 / (3 if int(ov["tukey_variant"]) == 2 else 6)
    rho1 = LD(1) if int(ov["tukey_variant"]) == 2 else LD(0.5)
    ev = (es / a2 + gamma(4) * s / a2 + U * (1 + s / a2)) * (1 + gamma(1))
    V = np.maximum(LD(1) - s / a2, LD(0)) + ev
    outlier = s - es > a2          # both branches certainly the outlier's: rho' = 0, rho constant
    ehr_t = sim * rho0 / 2 * (3 * V * V * ev + gamma(2) * V ** 3 + U * (1 + V ** 3) + gamma(5) * (1 + V ** 3))
    ea_t = sim * rho1 * (2 * V * ev + ev * ev + gamma(3) * V * V)
    ehr_t = np.where(outlier, gamma(3) * sim * rho0 / 2, ehr_t)
    ea_t = np.where(outlier, LD(0), ea_t)
    ehr = np.where(cauchy, ehr_c, ehr_t)
    ea = np.where(cauchy, ea_c, ea_t)
    return r, M, a, hr, er, eM, ea, ehr


def probe(p, slot, options, x0, dl, alpha):
    """The values the line search and an accepted step read at xc = P(x + alpha dl), from the start x0
    (projected as in iteration 0) and the device's own step dl [nf, 2] (float64), in longdouble, with the
    bound a float64 evaluation by the kernels' operations must meet (PROBE_BOUNDS).  alpha is a power of
    two, so x + alpha dl rounds once whether or not it is contracted to an FMA."""
    ov = option_values(options)
    g = p.graph
    nodes = p.comp_nodes[p.comp_ptr[slot]:p.comp_ptr[slot + 1]].astype(np.int64)
    free_nodes = nodes[p.is_root[nodes] == 0]
    nf = len(free_nodes)
    n = 2 * nf
    fidx = np.full(g.n_nodes, -1, np.int64)
    fidx[free_nodes] = np.arange(nf)
    bound = float(ov["bound"])
    x = np.asarray(x0, np.float64).copy()
    x[free_nodes] = np.clip(x[free_nodes], -bound, bound)
    dl = np.asarray(dl, np.float64).reshape(nf, 2)
    assert np.frexp(alpha)[0] == 0.5, alpha
    raw = x[free_nodes] + alpha * dl
    xc = x.copy()
    xc[free_nodes] = np.clip(raw, -bound, bound)
    clamped = raw != xc[free_nodes]

    src, dst, eidx, kind = kept_blocks(p, slot)
    e = g.edges[eidx]
    E = len(src)
    r, M, a, hr, er, eM, ea, ehr = _edge_eval_bounds(e["flow"], xc[src], xc[dst], kind, e["sim"], ov)
    cost = hr.sum()
    cost_mag = np.abs(hr).sum()
    # (4) the cost: a sum of E terms in any order
    cost_bound = ehr.sum() + gamma(max(E - 1, 1)) * (cost_mag + ehr.sum())

    fs, fd = fidx[src], fidx[dst]
    dlL = dl.astype(LD)
    ds = np.zeros((E, 2), LD)
    dd = np.zeros((E, 2), LD)
    ds[fs >= 0] = dlL[fs[fs >= 0]]
    dd[fd >= 0] = dlL[fd[fd >= 0]]
    w = dd - np.einsum("ekj,ej->ek", M, ds)
    term = a * (r * w).sum(axis=1)
    # gradient: g_src -= a M^T r, g_dst += a r
    gv = np.zeros(n, LD)
    gsrc = -a[:, None] * np.einsum("ekj,ek->ej", M, r)
    for i in range(2):
        np.add.at(gv, 2 * fs[fs >= 0] + i, gsrc[fs >= 0, i])
        np.add.at(gv, 2 * fd[fd >= 0] + i, (a[:, None] * r)[fd >= 0, i])
    dphi = (gv * dlL.reshape(-1)).sum()
    # (5) phi' = sum_e a r^T (dl_d - M dl_s): per edge, the errors of a, r and M carried through, and every
    # product a r_k M_kj dl_j / a r_k dl_k rounded along a chain of at most 2 E + n + 16 operations
    R = np.abs(r) + er
    AM = np.abs(M) + eM
    Aa = a + ea
    W = np.abs(dd) + np.einsum("ekj,ej->ek", AM, np.abs(ds))
    mag_e = Aa * (R * W).sum(axis=1)
    err_e = ea * (R * W).sum(axis=1) + a * (er * W).sum(axis=1) + \
        a * (R * np.einsum("ekj,ej->ek", eM, np.abs(ds))).sum(axis=1)
    h = gamma(2 * E + n + 16)
    dphi_mag = mag_e.sum()
    dphi_bound = err_e.sum() + h * dphi_mag
    # the same for every gradient coordinate
    gb = np.zeros(n, LD)
    gm = np.zeros(n, LD)
    src_err = ea[:, None] * np.einsum("ekj,ek->ej", AM, R) + a[:, None] * (
        np.einsum("ekj,ek->ej", AM, er) + np.einsum("ekj,ek->ej", eM, R))
    src_mag = Aa[:, None] * np.einsum("ekj,ek->ej", AM, R)
    dst_err = ea[:, None] * R + a[:, None] * er
    dst_mag = Aa[:, None] * R
    for i in range(2):
        np.add.at(gb, 2 * fs[fs >= 0] + i, src_err[fs >= 0, i])
        np.add.at(gm, 2 * fs[fs >= 0] + i, src_mag[fs >= 0, i])
        np.add.at(gb, 2 * fd[fd >= 0] + i, dst_err[fd >= 0, i])
        np.add.at(gm, 2 * fd[fd >= 0] + i, dst_mag[fd >= 0, i])
    gb = gb + h * gm
    xf = xc[free_nodes].reshape(-1).astype(LD)
    gmax = np.abs(xf - np.clip(xf - gv, LD(-bound), LD(bound))).max() if n else LD(0)
    # (6) gmax: P is 1-Lipschitz; x - g and x - P(.) round once each
    gmax_bound = (gb.max() + 2 * U * (np.abs(xf) + np.abs(gv) + gb).max()) if n else 0.0

    x_f = x[free_nodes].astype(LD)
    xc_f = xc[free_nodes].astype(LD)
    dn = np.sqrt(((x_f - xc_f) ** 2).sum())
    xn = np.sqrt((xc_f ** 2).sum())
    cm = clamped.reshape(-1)
    pair = src * g.n_nodes + dst
    _, inv, cnt = np.unique(pair, return_inverse=True, return_counts=True)
    dup = cnt[inv] > 1
    wt = dd - np.einsum("ekj,ej->ek", np.swapaxes(M, 1, 2), ds)
    mt = a * (r * wt).sum(axis=1)
    xs0, xs1 = x[src], xc[src]
    cross = ((np.abs(xs0) > 0.5) != (np.abs(xs1) > 0.5)) & (fs >= 0)[:, None]
    return Probe(free_nodes=free_nodes, xc=xc, clamped=clamped, cost=float(cost), cost_bound=float(cost_bound),
                 cost_mag=float(cost_mag), dphi=float(dphi), dphi_bound=float(dphi_bound),
                 dphi_mag=float(dphi_mag), dn=float(dn), xn=float(xn),
                 norm_bound=float(gamma(n + 1) / 2 + U), gmax=float(gmax), gmax_bound=float(gmax_bound),
                 g=gv, g_bound=gb,
                 clamped_share=float(abs((gv * dlL.reshape(-1))[cm].sum())),
                 dup_share=float(np.abs(term[dup]).max()) if dup.any() else 0.0,
                 mt_diff=float(abs((mt - term).sum())),
                 grid_cross=int(len(np.unique((src[:, None] * 2 + np.arange(2))[cross])))
                 )
