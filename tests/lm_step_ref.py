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


def first_step(p, slot, options, start, radius=None, want_kappa=True):
    """The first LM step of dispatch slot `slot` from `start` [N, 2] under lfr_options `options` (at
    `radius`, default the options' initial radius)."""
    ov = option_values(options)
    radius = LD(ov["initial_trust_region_radius"] if radius is None else radius)
    g = p.graph
    nodes = p.comp_nodes[p.comp_ptr[slot]:p.comp_ptr[slot + 1]].astype(np.int64)
    free_nodes = nodes[p.is_root[nodes] == 0]
    nf = len(free_nodes)
    n = 2 * nf
    fidx = np.full(g.n_nodes, -1, np.int64)
    fidx[free_nodes] = np.arange(nf)
    x = np.asarray(start, np.float64).astype(LD).copy()
    bound = LD(ov["bound"])
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
    S = LD(1) / (LD(1) + np.sqrt(diag))
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


def step_bound(n, kappa):
    """The relative error a backward-stable solve of an n-unknown system of condition kappa may have:
    8 n kappa 2^-53."""
    return 8.0 * n * kappa * 2.0 ** -53
