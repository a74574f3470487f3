"""Test-side access to oracle/_ref/libref_cost.so — the REFERENCE's own cost.cc compiled against
the shim headers (oracle/build_ref.py).  Test infrastructure only."""
import ctypes as C
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def _build_mod():
    spec = importlib.util.spec_from_file_location("lfr_build_ref", os.path.join(ROOT, "oracle", "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_refsrc():
    """Returns the ctypes library, or None when it is neither built nor buildable here."""
    global _lib
    if _lib is None:
        try:
            path = _build_mod().build_cost()
        except Exception:
            return None
        L = C.CDLL(path)
        for name, n in (("lfr_refsrc_interpolate", 6), ("lfr_refsrc_cost", 7), ("lfr_refsrc_residual", 5)):
            getattr(L, name).argtypes = [C.c_uint64] + [C.c_void_p] * (n - 1)
            getattr(L, name).restype = None
        _lib = L
    return _lib


_solve_lib = None


def load_refsolve():
    """oracle/_ref/libref_solve.so: the reference's create_and_solve_problem (oracle/ref_solve_shim.cc).
    Raises when it is neither built nor buildable: the tests that use it fail rather than skip."""
    global _solve_lib
    if _solve_lib is None:
        path = _build_mod().build_solve_lib()
        L = C.CDLL(path)
        L.lfr_refsrc_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
        L.lfr_refsrc_solve.restype = C.c_int
        _solve_lib = L
    return _solve_lib


def ref_solve(p, is_const, start, n_threads=None):
    """create_and_solve_problem on every slot of `p` (more than one node) with is_root = `is_const`
    [n_nodes] and positions = `start` [n_nodes, 2].  Returns (positions, stats): stats holds the oracle's
    per-slot names (iterations, termination, initial_cost, final_cost) plus ls_steps and fixed_cost per
    slot, and the totals; initial_cost and final_cost are the Summary's, fixed cost included."""
    from lfr_b200.capi import Library
    L = load_refsolve()
    s, keep = Library.marshal(p)
    n, C_ = p.graph.n_nodes, p.n_components
    mask = np.ascontiguousarray(is_const, np.uint8).reshape(n)
    x0 = np.ascontiguousarray(start, np.float64).reshape(n, 2)
    pos = np.zeros((n, 2))
    st = dict(iterations=np.zeros(C_, np.int32), termination=np.zeros(C_, np.int32), ls_steps=np.zeros(C_, np.int32),
              initial_cost=np.zeros(C_), final_cost=np.zeros(C_), fixed_cost=np.zeros(C_))
    rc = L.lfr_refsrc_solve(C.addressof(s), mask.ctypes.data, x0.ctypes.data, int(n_threads or os.cpu_count() or 8),
                            pos.ctypes.data, *[st[k].ctypes.data for k in ("iterations", "termination", "ls_steps",
                                                                           "initial_cost", "final_cost", "fixed_cost")])
    del keep
    assert rc >= 0, "lfr_refsrc_solve could not match a summary to its component"
    st["n_solved"] = rc
    st["total_iterations"] = int(st["iterations"].sum())
    st["total_line_search_steps"] = int(st["ls_steps"].sum())
    return pos, st


def ref_interpolate(L, grids, rc):
    n = grids.shape[0]
    grids = np.ascontiguousarray(grids, np.float64)
    rc = np.ascontiguousarray(rc, np.float64)
    f = np.zeros((n, 2)); dr = np.zeros((n, 2)); dc = np.zeros((n, 2))
    L.lfr_refsrc_interpolate(n, grids.ctypes.data, rc.ctypes.data, f.ctypes.data, dr.ctypes.data, dc.ctypes.data)
    return f, dr, dc


def ref_cost(L, grids, x1, x2):
    n = grids.shape[0]
    grids = np.ascontiguousarray(grids, np.float64)
    x1 = np.ascontiguousarray(x1, np.float64)
    x2 = np.ascontiguousarray(x2, np.float64)
    r = np.zeros((n, 2)); j1 = np.zeros((n, 4)); j2 = np.zeros((n, 4))
    L.lfr_refsrc_cost(n, grids.ctypes.data, x1.ctypes.data, x2.ctypes.data, r.ctypes.data, j1.ctypes.data, j2.ctypes.data)
    return r, j1, j2


def cost_cases(n, seed=0):
    """Random, clamped and boundary inputs (grids are fp32 values widened, as solve.cc:460-472 does)."""
    rng = np.random.default_rng(seed)
    grids = rng.uniform(-0.6, 0.6, (n, 18)).astype(np.float32)
    x1 = rng.uniform(-1.0, 1.0, (n, 2))
    k = max(n // 20, 1)
    x1[0 * k:1 * k, 0] = 0.5
    x1[1 * k:2 * k, 1] = -0.5
    x1[2 * k:3 * k] = 0.0
    x1[3 * k:4 * k, 0] = np.nextafter(0.5, 1.0)
    x1[4 * k:5 * k] = [0.5, -0.5]
    x1[5 * k:6 * k, 1] = np.nextafter(-0.5, -1.0)
    x1[6 * k:7 * k] = rng.uniform(-0.5, 0.5, (k, 2))
    x2 = rng.uniform(-1.0, 1.0, (n, 2))
    return grids, x1, x2
