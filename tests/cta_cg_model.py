"""A float64 numpy restatement of the CTA tier's linear solve (cta_lm_step, csrc/lfr_solve_cta.cuh).

The kernel solves the damped system A y = b of one component, A = S H S + D^2 and b = S g (the statement
of lm_step_ref.step_at), by conjugate gradients preconditioned with the inverse of A's 2x2 diagonal blocks
(block-Jacobi):
  * y = 0, r = b, z = P^-1 r, p = z; the recurrence stops once r . r <= 1e-28 b . b;
  * then the true residual r = b - A y is formed; when r . r <= 4e-30 b . b (or r . P^-1 r <= 0) the
    solve ends, else CG restarts from it (z = P^-1 r, p = z), at most twice;
  * the iterations of the first pass and both restarts share one budget of 8 n + 100 (n unknowns): a
    solve that reaches it ends there and returns what it has.
This model takes the same decisions in the same order on a float64 A and b rounded from the statement.
Its sums are not the kernel's, so its iteration counts are a prediction of the kernel's, not a bit-exact
copy: they tell how long CG runs on a component and whether the cap is near.
"""
from dataclasses import dataclass

import numpy as np
import scipy.sparse

TOL2 = 1e-28          # recurrence: |r|^2 <= 1e-28 |b|^2
TRUE_TOL2 = 4e-30     # true residual: |b - A y|^2 <= 4e-30 |b|^2
MAX_RESTARTS = 2


def cg_cap(n):
    """The kernel's iteration budget for n unknowns, shared by the first pass and the restarts."""
    return 8 * n + 100


@dataclass
class CgRun:
    iterations: int       # CG iterations over the first pass and the restarts (the kernel's counter)
    restarts: int         # restarts taken from the true residual
    capped: bool          # the budget ran out before the recurrence residual met its tolerance
    y: np.ndarray         # the solution
    true_residual: float  # |b - A y| / |b| at the end


def block_jacobi_inverse(A):
    """The inverse of A's 2x2 diagonal blocks as (i00, i01, i11) per block, formed as the kernel forms it
    (adjugate over the determinant)."""
    d = A.diagonal()
    off = A.diagonal(1)[0::2]
    p00, p11 = d[0::2], d[1::2]
    inv_det = 1.0 / (p00 * p11 - off * off)
    return p11 * inv_det, -off * inv_det, p00 * inv_det


def _apply(pinv, r):
    i00, i01, i11 = pinv
    z = np.empty_like(r)
    z[0::2] = i00 * r[0::2] + i01 * r[1::2]
    z[1::2] = i01 * r[0::2] + i11 * r[1::2]
    return z


def pcg(A, b, max_restarts=MAX_RESTARTS):
    """cta_lm_step's iteration on A y = b (A a scipy sparse float64 matrix, b float64); max_restarts
    other than the kernel's 2 shows what the restarts contribute."""
    A = scipy.sparse.csr_matrix(A)
    b = np.asarray(b, np.float64)
    n = len(b)
    pinv = block_jacobi_inverse(A)
    y = np.zeros(n)
    r = b.copy()
    z = _apply(pinv, r)
    p = z.copy()
    bb = float(b @ b)
    rz = float(r @ z)
    max_it = cg_cap(n)
    it = restarts = 0
    capped = False
    while bb > 0.0:
        converged = False
        while it < max_it:
            w = A @ p
            pw = float(p @ w)
            if not (pw > 0.0 and np.isfinite(pw)):
                raise ArithmeticError("A is not positive definite in float64")
            alpha = rz / pw
            y += alpha * p
            r -= alpha * w
            z = _apply(pinv, r)
            rr, rz_new = float(r @ r), float(r @ z)
            it += 1
            if rr <= TOL2 * bb:
                converged = True
                break
            p = z + (rz_new / rz) * p
            rz = rz_new
        if it >= max_it:      # the kernel leaves without a true residual, converged on the last one or not
            capped = not converged
            break
        if restarts >= max_restarts:
            break
        r = b - A @ y
        z = _apply(pinv, r)
        rt, rzt = float(r @ r), float(r @ z)
        if rt <= TRUE_TOL2 * bb or not rzt > 0.0:
            break
        p = z.copy()
        rz = rzt
        restarts += 1
    res = float(np.linalg.norm(b - A @ y) / np.sqrt(bb)) if bb > 0.0 else 0.0
    return CgRun(iterations=it, restarts=restarts, capped=capped, y=y, true_residual=res)


def model_of(step):
    """The model's run on the damped system of an lm_step_ref.Step."""
    return pcg(step.A.float64(), step.b.astype(np.float64))
